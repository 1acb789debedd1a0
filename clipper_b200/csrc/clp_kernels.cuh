// clp_kernels.cuh -- sm_90a device code of the CLIPPER hot path.
//
//   K1  score_tile_kernel     scorePairwiseConsistency + invariants   (ref clipper.cpp:21-65,
//                             euclidean_distance.cpp:13-31, pointnormal_distance.cpp:13-35)
//   K2  matvec_*              penalised mat-vec  Mhat v, Chat v       (ref clipper.cpp:194-271)
//                             other sweeps of the same matrix: clp_dense2.cuh (column stripes, upper triangle
//                             two-sided), clp_sparse.cuh (compact sliced-ELL copy: the default when sparse)
//   K3-K5 solver_kernel       whole findDenseClique() as ONE persistent cooperative kernel:
//                             step/projection, objective, backtracking line search, penalty
//                             ramp, all decided on the device            (ref clipper.cpp:172-283)
//                             -- the segmented solver (any m, dense sweeps).  The default for m <= 27648 is
//                             solver_resident_kernel in clp_resident.cuh (whole trial vector in shared memory, one
//                             device-wide synchronisation per evaluation); clp_batch.cuh runs that solver body with
//                             one CTA per problem for batches of small problems
//   K7  encode/decode kernels  get/setMatrixData                        (ref clipper.cpp:131-166)
//
// Data layout in HBM.  The affinity matrix is DENSE and symmetric, row-major with a leading
// dimension ld (multiple of 128 elements) and the row count padded to a multiple of 32.  One
// stored element s carries BOTH matrices of the reference:
//        M_ij = |s|            C_ij = (sign bit of s clear)
// so "inconsistent" (M=0,C=0) is -0.0, "consistent" is +score, "no affinity but no penalty"
// (M=0,C=1, legal through setMatrixData) is +0.0.  The diagonal is stored as -0.0 and the
// identity is applied analytically exactly like the reference does (clipper.cpp:58,194,238).
// Storage type T is float (default; 4 B/entry is the only O(m^2) traffic) or double.
// Every O(m) vector, every accumulator and every scalar decision is fp64.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

#include "clp_score_tile.cuh"

namespace clp {

constexpr int kSegMax = 4096;          // max columns of v staged in shared memory per pass
constexpr int kMaxSeg = 64;            // max number of column segments (m <= 262144)
constexpr int kRedVals = 8;            // doubles per CTA in the partial-reduction table

enum StageMode : int { STAGE_RAW = 0, STAGE_DIV = 1, STAGE_STEP = 2 };

// ------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ double2 ldg_stream(const double2* p) {
  double2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.f64 {%0,%1}, [%2];"
               : "=d"(r.x), "=d"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------------------------------
// device-wide barrier for the persistent kernel (all CTAs co-resident: cooperative launch).
// Two-level arrival tree (nleaf counters on separate L2 lines, then one root) so that the ~300
// arrival atomics do not serialise on one address; monotonic round numbers, no reset inside a
// launch; the LAST CTA to arrive is told so (it performs the global reduction before releasing
// the others).  Every spin is bounded: a lost CTA / peer can never hang the GPU.
// ------------------------------------------------------------------------------------------
struct SyncBlock {  // zeroed by the host before every launch
  unsigned long long leaf[32][16]; // arrival counters, one 128-byte line each
  unsigned long long root[16];
  unsigned long long gen[16];      // generation published by the last arriver
  double bcast[2][kRedVals];       // globally reduced scalars of the current exchange
  int error;                       // 1: barrier / peer time-out, 2: bad association index
  int flags;                       // input-contract violations found by the encode kernels
  unsigned long long counts[2];
  unsigned int scale_bits;         // scoring: float bits of max |position coordinate| (gather_endpoints_kernel)
  unsigned int expo[2];            // compact build: largest kept fp32 exponent, 255 - smallest (atomicMax, see pack_window)
  unsigned int score_next;         // scoring: next work unit of score_tile_kernel_runs (ScoreArgs::next_unit)
};

struct TreeBar {
  SyncBlock* sb;
  int nleaf;     // <= 32 arrival counters; CTA b arrives at leaf b % nleaf
  int G;         // CTAs in the grid (leaves differ in size by at most one)
};

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// all threads call; returns true (to every thread) on the CTA that completed round `round`
__device__ __forceinline__ bool bar_arrive(const TreeBar& b, unsigned long long round, int* smem_flag) {
  __syncthreads();
  if (threadIdx.x == 0) {
    int last = 0;
    __threadfence();
    const int leaf = blockIdx.x % b.nleaf;
    const int leafsize = b.G / b.nleaf + (leaf < b.G % b.nleaf ? 1 : 0);
    unsigned long long old = atomicAdd(&b.sb->leaf[leaf][0], 1ULL);
    if (old + 1ULL == round * (unsigned long long)leafsize) {
      __threadfence();
      old = atomicAdd(&b.sb->root[0], 1ULL);
      if (old + 1ULL == round * (unsigned long long)b.nleaf) { last = 1; __threadfence(); }
    }
    *smem_flag = last;
  }
  __syncthreads();
  return *smem_flag != 0;
}
__device__ __forceinline__ void bar_release(const TreeBar& b, unsigned long long round) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    st_release_u64(&b.sb->gen[0], round);
  }
}
__device__ __forceinline__ void bar_wait(const TreeBar& b, unsigned long long round) {
  if (threadIdx.x == 0) {
    const long long t0 = clock64();
    while (ld_acquire_u64(&b.sb->gen[0]) < round) {
      __nanosleep(20);
      if (clock64() - t0 > 4000000000LL) { atomicExch(&b.sb->error, 1); break; }  // ~2 s
    }
    __threadfence();
  }
  __syncthreads();
}
__device__ __forceinline__ void grid_barrier(const TreeBar& b, unsigned long long round, int* smem_flag) {
  if (bar_arrive(b, round, smem_flag)) bar_release(b, round);
  else bar_wait(b, round);
  __syncthreads();
}

// ------------------------------------------------------------------------------------------
// "LL" cells for everything that crosses NVLink: a double travels as one 16-byte store
// {lo32, tag, hi32, tag}.  The reader spins until both tags equal the expected sequence number,
// so the datum validates itself -- no system-scope fence, no separate flag, write order free.
// (8-byte halves are written atomically; the tag is unique per exchange step.)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void ll_store(uint4* p, double v, unsigned tag) {
  const unsigned lo = (unsigned)__double2loint(v), hi = (unsigned)__double2hiint(v);
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(lo), "r"(tag), "r"(hi), "r"(tag) : "memory");
}
__device__ __forceinline__ double ll_load(const uint4* p, unsigned tag, int* error) {
  unsigned lo, t1, hi, t2;
  long long t0 = 0;
  for (;;) {
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(t1), "=r"(hi), "=r"(t2) : "l"(p) : "memory");
    if (t1 == tag && t2 == tag) break;
    if (t0 == 0) t0 = clock64();
    else if (clock64() - t0 > 4000000000LL) { atomicExch(error, 1); break; }
  }
  return __hiloint2double((int)hi, (int)lo);
}

// ------------------------------------------------------------------------------------------
// K1: scoring
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float sqrt_approx(float x) {  // MUFU.SQRT, relative error <= 2^-22
  float r;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// Threshold of the fp32 screen (score_tile_kernel_runs, batch scoring): a pair is dropped iff |l1_32 - l2_32| >= thr.
// R = largest |position coordinate| after conversion to fp32, u = 2^-24.  Converting the inputs (u R per coordinate),
// the subtraction (2 u R more), the three-term sum of squares (3 u relative) and sqrt.approx (2^-22 relative) put the
// fp32 length within 7 u R + 10 u l <= 42 u R of the exact one (d <= 3, l <= 2 sqrt(3) R) as long as no square
// overflows or rounds to an fp32 subnormal; the final subtraction adds at most 4 u R: |c32 - c| < 90 u R, and 1024 u R
// is used.  The two scale limits keep that analysis true:
//   R <= 2^62:  a sum of squares is at most 3 (2R)^2 (1 + u)^3 < 2^128, so nothing overflows.  (Above, an infinite
//               l_32 next to a finite one would satisfy inf >= thr and drop a pair the exact test may keep.)
//   R >= 2^-58: each square and fma may lose up to 2^-150 absolutely to subnormal rounding (inputs and differences
//               are exact or within u R there), i.e. 3 * 2^-150 on the sum, at most sqrt(3 * 2^-150) < 2^-74 on a
//               length and 2^-73 = 2^-15 * 2^-58 <= 512 u R on c32: 90 u R + 512 u R < 1024 u R.
// Outside [2^-58, 2^62], and for R = Inf / NaN (a non-finite coordinate), thr is NaN: `c32 >= NaN` is false, every
// pair takes the exact fp64 path.  Inside, the threshold is the one of the unguarded screen, bit for bit.
__device__ __forceinline__ float screen_threshold(double eps, float R) {
  if (!(R >= 0x1p-58f && R <= 0x1p62f)) return __int_as_float(0x7fffffff);
  return __double2float_ru((eps + 1024.0 * 5.9604644775390625e-08 * (double)R) * (1.0 + 9.5367431640625e-07));
}


// ------------------------------------------------------------------------------------------
// K1, screened: fp32 storage and Euclidean d = 2, 3 or PointNormal.  The kernel is bound by fp64 arithmetic
// (two square roots and an exp per pair), yet only ~15 % of the pairs pass the consistency test |l1 - l2| < epsilon.
// Every pair is first screened in fp32 against epsilon + a rigorous error margin (a pair is dropped only when the
// exact test must fail too, so every stored value is still produced by the exact fp64 path, bit for bit); the
// survivors of a warp's 4 x 128 block are compacted into a shared-memory queue and scored 32 at a time with all lanes
// busy, the results pass through a shared-memory copy of the block so that the stores stay row-wise float4.
//
// Persistent: one wave of CTAs draws work units from a device-wide counter.  A unit is a run of up to kRunTiles
// consecutive 32 x 128 tiles of one row block, aligned to kRunTiles tiles (MIRROR: only tiles touching the upper
// triangle).  A count-segment width W is only a multiple of 128 (mode 3 cuts round_up(ceil(m / NSEG), 128)), so a
// run may cross a segment boundary: the row counts are flushed whenever the next tile lies in another segment.  Units are numbered row block by row block, left to right: the CTAs
// of a wave work on neighbouring row blocks, and the last units handed out are the short rows at the bottom.
//   * the row side (fp64 endpoints, association pair, fp32 positions of 32 rows) is loaded once per unit;
//   * per-row kept counts are added up along the run and flushed once per (row block, column segment), the 16-column
//     window bits once per 32-bit word, the exponent range once per CTA;
//   * the column side of the next tile (fp64 endpoints, fp32 positions, association pairs) is copied into the other
//     half of a double buffer with cp.async while the current tile is screened, scored and stored; columns at or past
//     m are zero-filled by the copy itself.
// The stores, the elements written and every stored bit are those of one tile of the unscreened kernel.
// ------------------------------------------------------------------------------------------
template <int DD>
struct ScoreRunSmem {
  static constexpr int kES = 2 * DD + 1;  // E1 then E2 of one endpoint; odd stride against bank conflicts
  double colE[2][128][kES];               // double-buffered column endpoints
  double rowE[kRowTile][kES];
  float4 rowF[2][kRowTile];               // fp32 positions and association pair of the rows: read as broadcasts
  int2 rowA[kRowTile];
  float4 colF[2][2][128];                // [buffer][F1, F2][slot]: column c at slot (c & 3) * 32 + (c >> 2)
  int colA[2][2][128];                    // [buffer][A0, A1][slot], same slots
  float tile[kRowTile][132];              // row stride 132: the transposed reads of the mirror stores hit 8 banks, not 1
  unsigned short queue[kWarps][kRowsPerWarp * 128];
  unsigned int expo[2];
  unsigned int unit[2];                   // the CTA's current and next work unit, alternating slots
};

template <int N>
__device__ __forceinline__ void cp_async_zfill(void* dst, const void* src, bool ok) {  // N bytes, or N zero bytes
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;"
               ::"r"((unsigned int)__cvta_generic_to_shared(dst)), "l"(src), "n"(N), "r"(ok ? N : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

constexpr int kRunTiles = 8;  // tiles per work unit of score_tile_kernel_runs (a power of two <= kSegMax / 128)

// work units of row blocks 0 .. rb-1 (nruns = runs of a full row; MIRROR: row block rb starts at tile rb / 4, i.e. in
// run rb / (4 kRunTiles))
template <bool MIRROR>
__host__ __device__ __forceinline__ long long score_units_before(int rb, int nruns) {
  if (!MIRROR) return (long long)rb * nruns;
  constexpr long long P = 4 * kRunTiles;
  const long long q = rb / P, s = rb % P;
  return (long long)rb * nruns - (P * q * (q - 1) / 2 + s * q);  // minus sum over r < rb of r / P
}

// unit u -> row block rb and its tiles [tb, tend)
template <bool MIRROR>
__device__ __forceinline__ void score_unit(unsigned int u, int nrb, int nt, int& rb, int& tb, int& tend) {
  const int nruns = (nt + kRunTiles - 1) / kRunTiles;
  int lo = 0;
  for (int hi = nrb; hi - lo > 1;) {
    const int mid = (lo + hi) >> 1;
    if (score_units_before<MIRROR>(mid, nruns) <= (long long)u) lo = mid; else hi = mid;
  }
  rb = lo;
  const int tb0 = MIRROR ? (rb >> 2) : 0;
  const int run = tb0 / kRunTiles + (int)((long long)u - score_units_before<MIRROR>(rb, nruns));
  tb = max(run * kRunTiles, tb0);
  tend = min(run * kRunTiles + kRunTiles, nt);
}

template <int DD>
__device__ __forceinline__ void score_fetch_columns(const ScoreArgs& a, ScoreRunSmem<DD>& s, int buf, int tb) {
  const int j0 = tb * 128;
  for (int idx = threadIdx.x; idx < 128 * DD; idx += kThreads) {
    const int c = idx / DD, t = idx - c * DD, j = j0 + c;
    const bool ok = j < a.m;
    const size_t g = ok ? (size_t)j * DD + t : 0;
    cp_async_zfill<8>(&s.colE[buf][c][t], a.E1 + g, ok);
    cp_async_zfill<8>(&s.colE[buf][c][DD + t], a.E2 + g, ok);
  }
  const int c = threadIdx.x & 127, side = threadIdx.x >> 7, j = j0 + c, slot = (c & 3) * 32 + (c >> 2);
  const bool ok = j < a.m;
  cp_async_zfill<16>(&s.colF[buf][side][slot], (side ? a.F2 : a.F1) + (ok ? j : 0), ok);
  cp_async_zfill<4>(&s.colA[buf][side][slot], (side ? a.A1 : a.A0) + (ok ? j : 0), ok);
}

template <int KIND, int D, bool MIRROR>
__global__ void __launch_bounds__(kThreads, 4) score_tile_kernel_runs(ScoreArgs a) {
  constexpr int DD = (KIND == 1) ? 6 : D;
  static_assert(DD > 0, "the screened kernel needs a compile-time dimension");
  extern __shared__ __align__(16) unsigned char score_smem[];
  ScoreRunSmem<DD>& s = *reinterpret_cast<ScoreRunSmem<DD>*>(score_smem);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nt = (int)(a.ld / 128), nrb = a.rows_pad / kRowTile;
  const long long total = score_units_before<MIRROR>(nrb, (nt + kRunTiles - 1) / kRunTiles);
  float* Mbase = reinterpret_cast<float*>(a.M);

  if (threadIdx.x == 0) s.unit[0] = atomicAdd(a.next_unit, 1u);
  if (threadIdx.x < 2) s.expo[threadIdx.x] = 0u;
  __syncthreads();
  if ((long long)s.unit[0] >= total) return;
  int rb, tb, tend;
  score_unit<MIRROR>(s.unit[0], nrb, nt, rb, tb, tend);
  score_fetch_columns<DD>(a, s, 0, tb);
  cp_async_commit();

  // Screening threshold (screen_threshold: the error analysis and the scales where the screen is off).  A NaN
  // length or threshold makes the comparison below false, i.e. the pair goes to the exact path.
  const float thr = screen_threshold(a.p1, __uint_as_float(*a.scale_bits));  // epsilon (Euclidean) / epsp (PointNormal)
  unsigned int rowc = 0u, roww = 0u, ehi = 0u, elo = 0u;  // run accumulators (rowc, roww: lane q < 4 for row q)
  int rb_loaded = -1;
  unsigned int seq = 0, unext = 0;  // units taken so far; the unit after the current one
  bool unit_start = true;

  for (int n = 0;; ++n) {
    const int buf = n & 1;
    // the next unit is drawn while the current one starts; slot (seq + 1) & 1 was last read before the previous
    // unit's first barrier, which thread 0 has passed
    if (unit_start && threadIdx.x == 0) s.unit[(seq + 1) & 1] = atomicAdd(a.next_unit, 1u);

    const int lr0 = rb * kRowTile + warp * kRowsPerWarp;  // local row of the warp's first row
    if (rb != rb_loaded) {  // the row side of a new row block
      __syncthreads();      // every warp is done with the previous block's rowE
      for (int idx = threadIdx.x; idx < kRowTile * DD; idx += kThreads) {
        const int r = idx / DD, t = idx - r * DD, li = rb * kRowTile + r;
        s.rowE[r][t] = (li < a.rows) ? __ldg(a.E1 + (size_t)(a.row0 + li) * DD + t) : 0.0;
        s.rowE[r][DD + t] = (li < a.rows) ? __ldg(a.E2 + (size_t)(a.row0 + li) * DD + t) : 0.0;
      }
      if (threadIdx.x < kRowTile) {
        const int li = rb * kRowTile + threadIdx.x;
        int2 ai = make_int2(-1, -1);
        float4 f1 = make_float4(0.f, 0.f, 0.f, 0.f), f2 = f1;
        if (li < a.rows) {
          const int i = a.row0 + li;
          ai = make_int2(__ldg(a.A0 + i), __ldg(a.A1 + i)); f1 = __ldg(a.F1 + i); f2 = __ldg(a.F2 + i);
        }
        s.rowA[threadIdx.x] = ai; s.rowF[0][threadIdx.x] = f1; s.rowF[1][threadIdx.x] = f2;
      }
      rb_loaded = rb;
    }
    cp_async_wait_all();
    // this tile's columns and the row side are visible; every warp is done with the previous tile, so its column
    // buffer and the shared block may be refilled
    __syncthreads();
    if (unit_start) unext = s.unit[(seq + 1) & 1];
    int nrb_ = rb, ntb = tb + 1, ntend = tend;  // the next tile
    const bool more = ntb < tend || (long long)unext < total;
    if (ntb >= tend && more) score_unit<MIRROR>(unext, nrb, nt, nrb_, ntb, ntend);
    if (more) {
      score_fetch_columns<DD>(a, s, buf ^ 1, ntb);
      cp_async_commit();
    }

    const int c0 = tb * 128 + lane * 4;
    float out[kRowsPerWarp][4];
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q) {
#pragma unroll
      for (int e = 0; e < 4; ++e) out[q][e] = -0.0f;
      Quad<float>::store(&s.tile[warp * kRowsPerWarp + q][lane * 4], out[q]);
    }
    unsigned int cnt = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = c0 + e;
      const bool jok = (j < a.m) && !(MIRROR && j <= a.row0 + lr0);
      const int slot = e * 32 + lane;
      const int aj0 = s.colA[buf][0][slot], aj1 = s.colA[buf][1][slot];
      const float4 f1j = s.colF[buf][0][slot], f2j = s.colF[buf][1][slot];
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q) {
        const int li = lr0 + q;
        const int i = a.row0 + li;
        const float4 f1i = s.rowF[0][warp * kRowsPerWarp + q], f2i = s.rowF[1][warp * kRowsPerWarp + q];
        const int2 ai = s.rowA[warp * kRowsPerWarp + q];
        const float x1 = f1i.x - f1j.x, y1 = f1i.y - f1j.y, z1 = f1i.z - f1j.z;
        const float x2 = f2i.x - f2j.x, y2 = f2i.y - f2j.y, z2 = f2i.z - f2j.z;
        const float l1 = sqrt_approx(fmaf(z1, z1, fmaf(y1, y1, x1 * x1)));
        const float l2 = sqrt_approx(fmaf(z2, z2, fmaf(y2, y2, x2 * x2)));
        // distinctness (ref clipper.cpp:35-38); "certainly inconsistent" last: a NaN keeps the pair
        const bool cand = jok && li < a.rows && i != j && !(MIRROR && j < i) && ai.x != aj0 && ai.y != aj1 &&
                          !(fabsf(l1 - l2) >= thr);
        const unsigned int vote = __ballot_sync(0xffffffffu, cand);
        if (cand) s.queue[warp][cnt + __popc(vote & ((1u << lane) - 1u))] = (unsigned short)((q << 7) | (e << 5) | lane);
        cnt += __popc(vote);
      }
    }
    __syncwarp();
    for (unsigned int k = lane; k < cnt; k += 32) {
      const unsigned int code = s.queue[warp][k];
      const int q = code >> 7, e = (code >> 5) & 3, l = code & 31;
      const int r = warp * kRowsPerWarp + q, c = l * 4 + e;
      double e1i[DD], e2i[DD], e1j[DD], e2j[DD];
#pragma unroll
      for (int t = 0; t < DD; ++t) {
        e1i[t] = s.rowE[r][t]; e2i[t] = s.rowE[r][DD + t];
        e1j[t] = s.colE[buf][c][t]; e2j[t] = s.colE[buf][c][DD + t];
      }
      double scr;
      if (KIND == 0) {
        const double l1 = point_dist<DD>(e1i, e1j, 0), l2 = point_dist<DD>(e2i, e2j, 0);
        scr = euclid_score(l1, l2, a.p0, a.p1, a.p2);
      } else {
        const double l1 = point_dist<3>(e1i, e1j, 0), l2 = point_dist<3>(e2i, e2j, 0);
        const double dot1 = __dadd_rn(__dadd_rn(__dmul_rn(e1i[3], e1j[3]), __dmul_rn(e1i[4], e1j[4])), __dmul_rn(e1i[5], e1j[5]));
        const double dot2 = __dadd_rn(__dadd_rn(__dmul_rn(e2i[3], e2j[3]), __dmul_rn(e2i[4], e2j[4])), __dmul_rn(e2i[5], e2j[5]));
        scr = pointnormal_score(l1, l2, dot1, dot2, a.p0, a.p1, a.p2, a.p3);
      }
      if (keep_score(scr, a.affinityeps)) s.tile[r][c] = encode<float>(scr, true);
    }
    __syncwarp();
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q)
#pragma unroll
      for (int e = 0; e < 4; ++e) out[q][e] = s.tile[warp * kRowsPerWarp + q][lane * 4 + e];

    if (a.cnt) {  // kept entries of the warp's four rows in this tile, added to the run's counts
      const int seg = (tb * 128) / a.W;
      const bool flush = !more || nrb_ != rb || (ntb * 128) / a.W != seg;
      unsigned int packed = 0;  // four 8-bit fields, <= 128 each after the warp sum
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q)
#pragma unroll
        for (int e = 0; e < 4; ++e) packed += (is_neutral<float>(out[q][e]) ? 0u : 1u) << (8 * q);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) packed += __shfl_xor_sync(0xffffffffu, packed, o);
      if (lane < kRowsPerWarp) rowc += (packed >> (8 * lane)) & 0xffu;
      if (flush) {
        if (lane < kRowsPerWarp && rowc) atomicAdd(a.cnt + (size_t)seg * (a.rows_pad + 1) + lr0 + lane, rowc);
        rowc = 0u;
      }
      if (a.win) {  // packed layout: occupied 16-column windows (lanes 4w..4w+3 = window w of the tile), exponent range
#pragma unroll
        for (int q = 0; q < kRowsPerWarp; ++q) {
          bool any = false;
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if (is_neutral<float>(out[q][e])) continue;
            any = true;
            const unsigned int x = (__float_as_uint(out[q][e]) >> 23) & 0xffu;
            ehi = max(ehi, x); elo = max(elo, 255u - x);
          }
          const unsigned int v = __ballot_sync(0xffffffffu, any);
          unsigned int wm = 0u;
#pragma unroll
          for (int w = 0; w < 8; ++w) wm |= ((v >> (4 * w)) & 0xfu) ? (1u << w) : 0u;
          if (lane == q) roww |= wm << (8 * (tb & 3));
        }
        // one word holds the windows of 4 tiles
        if (flush || (ntb >> 2) != (tb >> 2)) {
          if (lane < kRowsPerWarp && roww) atomicOr(a.win + (size_t)(lr0 + lane) * a.wwords + (tb >> 2), roww);
          roww = 0u;
        }
      }
    }

    if (!MIRROR) {
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q) {
        const int li = lr0 + q;
        if (li < a.rows_pad && c0 < a.ld) Quad<float>::store(Mbase + (size_t)li * a.ld + c0, out[q]);
      }
    } else {
      // MIRROR: row0 == 0 and rows == m.  Row-wise stores of the part right of the diagonal (and the diagonal itself) ...
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q) {
        const int i = lr0 + q;
        if (i >= a.rows_pad || c0 >= a.ld) continue;
        if (c0 > i) Quad<float>::store(Mbase + (size_t)i * a.ld + c0, out[q]);
        else {
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (c0 + e >= i) Mbase[(size_t)i * a.ld + c0 + e] = out[q][e];
        }
      }
      // ... and the mirror image through the shared-memory block: column cc of the block is 32 consecutive
      // elements (one 128-byte line) of row j = column index, stored by one warp instruction.  The counts of the 16
      // columns of a warp are kept one per lane and added with one warp-wide atomic each.
      __syncthreads();
      const int i = rb * kRowTile + lane;
      unsigned int myvote = 0u;
#pragma unroll 4
      for (int k = 0; k < 128 / kWarps; ++k) {
        const int cc = warp + k * kWarps, j = tb * 128 + cc;
        const bool st = j < a.rows_pad && i < j && i < a.ld;
        const float v = s.tile[lane][cc];
        if (st) Mbase[(size_t)j * a.ld + i] = v;
        const unsigned int vote = __ballot_sync(0xffffffffu, st && !is_neutral<float>(v));
        if (lane == k) myvote = vote;
      }
      if (a.cnt && lane < 128 / kWarps && myvote) {  // the column's entries are a piece of row j in the segment of rb
        const int j = tb * 128 + warp + lane * kWarps;
        atomicAdd(a.cnt + (size_t)((rb * kRowTile) / a.W) * (a.rows_pad + 1) + j, (unsigned int)__popc(myvote));
        if (a.win) {  // the two 16-column windows of row j covered by this block's rows
          const unsigned int wm = ((myvote & 0xffffu) ? 1u : 0u) | ((myvote >> 16) ? 2u : 0u);
          atomicOr(a.win + (size_t)j * a.wwords + (rb * kRowTile) / 512, wm << (((rb * kRowTile) / 16) & 31u));
        }
      }
    }
    if (!more) break;
    unit_start = tb + 1 >= tend;
    if (unit_start) ++seq;
    rb = nrb_; tb = ntb; tend = ntend;
  }
  if (a.win) {  // the exponent range of every tile this CTA scored
    ehi = __reduce_max_sync(0xffffffffu, ehi); elo = __reduce_max_sync(0xffffffffu, elo);
    if (lane == 0 && (ehi | elo)) { atomicMax(&s.expo[0], ehi); atomicMax(&s.expo[1], elo); }
    __syncthreads();
    if (threadIdx.x == 0 && (s.expo[0] | s.expo[1])) { atomicMax(a.expo, s.expo[0]); atomicMax(a.expo + 1, s.expo[1]); }
  }
}

// utils::createAllToAll (ref utils.h:61-71) on the device: association r = (r / n2, r % n2), column-major m x 2,
// so the all-to-all hypothesis never crosses PCIe (SURVEY 8f rank 2)
__global__ void all_to_all_kernel(long long n1, long long n2, int* A) {
  const long long m = n1 * n2;
  for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < m; r += (long long)gridDim.x * blockDim.x) {
    A[r] = (int)(r / n2);
    A[m + r] = (int)(r % n2);
  }
}

// E1[i][:] = D1[:, A(i,0)], E2[i][:] = D2[:, A(i,1)]; flags out-of-range association indices
__global__ void gather_endpoints_kernel(const double* D1, const double* D2, const int* A0, const int* A1,
                                        int m, int d, long long n1, long long n2, double* E1, double* E2,
                                        float4* F1, float4* F2, unsigned int* scale_bits, int* error) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float big = 0.f;
  if (i < m) {
    const int a0 = A0[i], a1 = A1[i];
    if (a0 < 0 || a0 >= n1 || a1 < 0 || a1 >= n2) { atomicExch(error, 2); }
    else {
      float f1[3] = {0.f, 0.f, 0.f}, f2[3] = {0.f, 0.f, 0.f};
      for (int q = 0; q < d; ++q) {
        const double x1 = D1[(size_t)a0 * d + q], x2 = D2[(size_t)a1 * d + q];
        E1[(size_t)i * d + q] = x1;
        E2[(size_t)i * d + q] = x2;
        if (q < 3) {  // positions (point-normal data: normals follow)
          f1[q] = (float)x1; f2[q] = (float)x2;
          // NaN must not be lost in the maximum: it becomes +Inf (screen_threshold is then NaN: every pair takes
          // the exact path)
          const float m1 = fabsf(f1[q]), m2 = fabsf(f2[q]);
          big = fmaxf(big, (m1 == m1) ? m1 : __int_as_float(0x7f800000));
          big = fmaxf(big, (m2 == m2) ? m2 : __int_as_float(0x7f800000));
        }
      }
      F1[i] = make_float4(f1[0], f1[1], f1[2], 0.f);
      F2[i] = make_float4(f2[0], f2[1], f2[2], 0.f);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) big = fmaxf(big, __shfl_xor_sync(0xffffffffu, big, o));
  if ((threadIdx.x & 31) == 0 && big > 0.f) atomicMax(scale_bits, __float_as_uint(big));  // non-negative floats order like their bits
}

// ------------------------------------------------------------------------------------------
// K2: the penalised mat-vec (device functions shared by the stand-alone and persistent kernels)
// ------------------------------------------------------------------------------------------
struct MatView {
  const void* M;   // T [rows_pad][ld], local row block
  long long ld;
  int m;           // number of columns == global problem size
  int row0;        // first global row stored locally
  int rows;        // real local rows
  int rows_pad;
};

struct Plan {
  int G;     // CTAs in the grid
  int SG;    // column-segment groups (CTA b works on segments b%SG, b%SG+SG, ...)
  int RG;    // row groups = G / SG (CTA b works on row tiles b/SG, b/SG+RG, ...)
  int NSEG;  // number of column segments
  int W;     // segment width (multiple of 128, <= kSegMax)
  int NRT;   // number of local row tiles (rows_pad / kRowTile)
};

// shared-memory position of column offset c (within a segment).  For 4-byte storage a lane owns
// 4 consecutive columns; the two 16-byte halves of its 4 doubles are stored 64 doubles apart so
// that both LDS.128 of a warp are bank-conflict free.
template <typename T> __device__ __forceinline__ int vs_pos(int c);
template <> __device__ __forceinline__ int vs_pos<float>(int c) {
  const int q = c >> 7, r = c & 127, l = r >> 2, e = r & 3;
  return (q << 7) + ((e >> 1) << 6) + (l << 1) + (e & 1);
}
template <> __device__ __forceinline__ int vs_pos<double>(int c) { return c; }

struct StageArgs {
  int mode;            // StageMode
  const double* srcA;  // RAW: the vector; STEP: u
  const uint4* llA;    // DIV: the un-normalised vector, LL cells
  const uint4* llB;    // STEP: gradF, LL cells
  unsigned tag;        // expected tag of the LL cells
  int* error;          // time-out flag for LL reads
  double alpha;        // STEP
  double z;            // DIV/STEP: squared norm of the un-normalised vector
  double* dst;         // where the segment owner writes the staged (normalised) vector, or null
  double* segsum;      // [NSEG] sum of the staged vector over each segment (written by owner)
};

// v_j for one column, exactly the reference's statement order:
//   STEP: unew = (u + alpha*gradF).cwiseMax(0); unew.normalize()   (clipper.cpp:235-237)
//   DIV : u /= u.norm()                                            (clipper.cpp:198)
__device__ __forceinline__ double staged_value(const StageArgs& s, int j, double nrm) {
  if (s.mode == STAGE_RAW) return s.srcA[j];
  if (s.mode == STAGE_DIV) return ll_load(s.llA + j, s.tag, s.error) / nrm;
  double w = __dadd_rn(s.srcA[j], __dmul_rn(s.alpha, ll_load(s.llB + j, s.tag, s.error)));
  w = (w < 0.0) ? 0.0 : w;
  return (s.z > 0.0 && w != 0.0) ? w / nrm : w;  // 0 / nrm == 0: skip the division's special-case path
}

// Stage columns [seg*W, seg*W+W) of v into shared memory (zero beyond m).  If `owner`, also
// publish the vector and its segment sum.  All threads of the CTA must call.
template <typename T>
__device__ void stage_segment(const StageArgs& s, const Plan& p, int m, int seg, bool owner,
                              double* vs, double* red_smem) {
  const double nrm = sqrt(s.z);
  const int cbeg = seg * p.W;
  double part = 0.0;
  // four columns per thread and trip: the LL cells (and u) of all four are requested before the first tag is
  // looked at -- one L2 round trip per trip instead of one per column (the spin loop of ll_load would otherwise
  // serialise them); a cell whose tag is not there yet falls back to ll_load.
  constexpr int kBatch = 4;
  for (int c = threadIdx.x; c < p.W; c += kBatch * kThreads) {
    double v[kBatch];
    if (s.mode == STAGE_RAW) {
#pragma unroll
      for (int b = 0; b < kBatch; ++b) {
        const int cc = c + b * kThreads, j = cbeg + cc;
        v[b] = (cc < p.W && j < m) ? s.srcA[j] : 0.0;
      }
    } else {
      const uint4* cells = (s.mode == STAGE_DIV) ? s.llA : s.llB;
      unsigned lo[kBatch], t1[kBatch], hi[kBatch], t2[kBatch];
      double ua[kBatch];
#pragma unroll
      for (int b = 0; b < kBatch; ++b) {
        const int cc = c + b * kThreads, j = cbeg + cc;
        lo[b] = hi[b] = 0u; t1[b] = t2[b] = s.tag; ua[b] = 0.0;
        if (cc < p.W && j < m) {
          asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                       : "=r"(lo[b]), "=r"(t1[b]), "=r"(hi[b]), "=r"(t2[b]) : "l"(cells + j) : "memory");
          if (s.mode == STAGE_STEP) ua[b] = s.srcA[j];
        }
      }
#pragma unroll
      for (int b = 0; b < kBatch; ++b) {
        const int cc = c + b * kThreads, j = cbeg + cc;
        v[b] = 0.0;
        if (cc < p.W && j < m) {
          const double x = (t1[b] == s.tag && t2[b] == s.tag) ? __hiloint2double((int)hi[b], (int)lo[b])
                                                              : ll_load(cells + j, s.tag, s.error);
          if (s.mode == STAGE_DIV) v[b] = x / nrm;
          else {
            double w = __dadd_rn(ua[b], __dmul_rn(s.alpha, x));
            w = (w < 0.0) ? 0.0 : w;
            v[b] = (s.z > 0.0 && w != 0.0) ? w / nrm : w;  // most entries are exactly 0: skip the division's slow special-case path
          }
        }
      }
    }
#pragma unroll
    for (int b = 0; b < kBatch; ++b) {
      const int cc = c + b * kThreads, j = cbeg + cc;
      if (cc < p.W) {
        if (owner && s.dst && j < m) s.dst[j] = v[b];
        vs[vs_pos<T>(cc)] = v[b];
        part += v[b];
      }
    }
  }
  if (owner) {  // deterministic block sum: warp butterflies, then warp 0 adds the 8 partials in order
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) red_smem[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += red_smem[w];
      s.segsum[seg] = t;
    }
  }
  __syncthreads();
}

// One warp: rows [lr, lr+4) x the staged segment.  accM += |s| v, accC += (C bit) v.
template <typename T> struct RowSweep;

template <> struct RowSweep<float> {
  static __device__ __forceinline__ void run(const MatView& mv, int lr, int cbeg, int W, const double* vs,
                                             double (&accM)[kRowsPerWarp], double (&accC)[kRowsPerWarp]) {
    const int lane = threadIdx.x & 31;
    const float* base = reinterpret_cast<const float*>(mv.M) + (size_t)lr * mv.ld + cbeg + lane * 4;
    const int nsteps = W >> 7;
    int s = 0;
    for (; s + 2 <= nsteps; s += 2) {
      float4 a0[kRowsPerWarp], a1[kRowsPerWarp];
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        a0[r] = ldg_stream(reinterpret_cast<const float4*>(base + (size_t)r * mv.ld + (s << 7)));
        a1[r] = ldg_stream(reinterpret_cast<const float4*>(base + (size_t)r * mv.ld + ((s + 1) << 7)));
      }
      const double2 v00 = *reinterpret_cast<const double2*>(vs + (s << 7) + lane * 2);
      const double2 v01 = *reinterpret_cast<const double2*>(vs + (s << 7) + 64 + lane * 2);
      const double2 v10 = *reinterpret_cast<const double2*>(vs + ((s + 1) << 7) + lane * 2);
      const double2 v11 = *reinterpret_cast<const double2*>(vs + ((s + 1) << 7) + 64 + lane * 2);
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        acc(a0[r].x, v00.x, accM[r], accC[r]); acc(a0[r].y, v00.y, accM[r], accC[r]);
        acc(a0[r].z, v01.x, accM[r], accC[r]); acc(a0[r].w, v01.y, accM[r], accC[r]);
        acc(a1[r].x, v10.x, accM[r], accC[r]); acc(a1[r].y, v10.y, accM[r], accC[r]);
        acc(a1[r].z, v11.x, accM[r], accC[r]); acc(a1[r].w, v11.y, accM[r], accC[r]);
      }
    }
    for (; s < nsteps; ++s) {
      float4 a0[kRowsPerWarp];
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r)
        a0[r] = ldg_stream(reinterpret_cast<const float4*>(base + (size_t)r * mv.ld + (s << 7)));
      const double2 v00 = *reinterpret_cast<const double2*>(vs + (s << 7) + lane * 2);
      const double2 v01 = *reinterpret_cast<const double2*>(vs + (s << 7) + 64 + lane * 2);
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        acc(a0[r].x, v00.x, accM[r], accC[r]); acc(a0[r].y, v00.y, accM[r], accC[r]);
        acc(a0[r].z, v01.x, accM[r], accC[r]); acc(a0[r].w, v01.y, accM[r], accC[r]);
      }
    }
  }
  static __device__ __forceinline__ void acc(float x, double v, double& aM, double& aC) {
    aM = fma((double)fabsf(x), v, aM);
    if (__float_as_int(x) >= 0) aC += v;
  }
};

template <> struct RowSweep<double> {
  static __device__ __forceinline__ void run(const MatView& mv, int lr, int cbeg, int W, const double* vs,
                                             double (&accM)[kRowsPerWarp], double (&accC)[kRowsPerWarp]) {
    const int lane = threadIdx.x & 31;
    const double* base = reinterpret_cast<const double*>(mv.M) + (size_t)lr * mv.ld + cbeg + lane * 2;
    const int nsteps = W >> 6;
    int s = 0;
    for (; s + 2 <= nsteps; s += 2) {
      double2 a0[kRowsPerWarp], a1[kRowsPerWarp];
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        a0[r] = ldg_stream(reinterpret_cast<const double2*>(base + (size_t)r * mv.ld + (s << 6)));
        a1[r] = ldg_stream(reinterpret_cast<const double2*>(base + (size_t)r * mv.ld + ((s + 1) << 6)));
      }
      const double2 v0 = *reinterpret_cast<const double2*>(vs + (s << 6) + lane * 2);
      const double2 v1 = *reinterpret_cast<const double2*>(vs + ((s + 1) << 6) + lane * 2);
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        acc(a0[r].x, v0.x, accM[r], accC[r]); acc(a0[r].y, v0.y, accM[r], accC[r]);
        acc(a1[r].x, v1.x, accM[r], accC[r]); acc(a1[r].y, v1.y, accM[r], accC[r]);
      }
    }
    for (; s < nsteps; ++s) {
      double2 a0[kRowsPerWarp];
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r)
        a0[r] = ldg_stream(reinterpret_cast<const double2*>(base + (size_t)r * mv.ld + (s << 6)));
      const double2 v0 = *reinterpret_cast<const double2*>(vs + (s << 6) + lane * 2);
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        acc(a0[r].x, v0.x, accM[r], accC[r]); acc(a0[r].y, v0.y, accM[r], accC[r]);
      }
    }
  }
  static __device__ __forceinline__ void acc(double x, double v, double& aM, double& aC) {
    aM = fma(fabs(x), v, aM);
    if (__double2hiint(x) >= 0) aC += v;
  }
};

// Whole mat-vec phase of one CTA: for each of its segments stage v, then sweep its row tiles and
// write the per-segment partial products  partM[seg][lrow], partC[seg][lrow].
template <typename T>
__device__ void matvec_phase(const MatView& mv, const Plan& p, const StageArgs& st, double* partM,
                             double* partC, double* vs, double* red_smem) {
  const int sg = blockIdx.x % p.SG, rg = blockIdx.x / p.SG;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int seg = sg; seg < p.NSEG; seg += p.SG) {
    // the last segment is ragged: never sweep past the leading dimension (ld = round_up(m,128))
    const long long rem = mv.ld - (long long)seg * p.W;
    const int wseg = rem < (long long)p.W ? (rem > 0 ? (int)rem : 0) : p.W;
    stage_segment<T>(st, p, mv.m, seg, rg == 0, vs, red_smem);
    for (int rt = rg; rt < p.NRT; rt += p.RG) {
      const int lr = rt * kRowTile + warp * kRowsPerWarp;
      double accM[kRowsPerWarp], accC[kRowsPerWarp];
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) { accM[r] = 0.0; accC[r] = 0.0; }
      RowSweep<T>::run(mv, lr, seg * p.W, wseg, vs, accM, accC);
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) { accM[r] = warp_sum(accM[r]); accC[r] = warp_sum(accC[r]); }
      if (lane == 0) {
#pragma unroll
        for (int r = 0; r < kRowsPerWarp; ++r) {
          partM[(size_t)seg * mv.rows_pad + lr + r] = accM[r];
          partC[(size_t)seg * mv.rows_pad + lr + r] = accC[r];
        }
      }
    }
    __syncthreads();  // vs is re-staged by the next segment pass
  }
}

// sum of the per-segment partials of local row lr, fixed order
__device__ __forceinline__ void gather_partials(const double* partM, const double* partC, int nseg,
                                                int rows_pad, int lr, double& Mv, double& Cv) {
  double a = 0.0, c = 0.0;
  for (int s = 0; s < nseg; ++s) {
    a += partM[(size_t)s * rows_pad + lr];
    c += partC[(size_t)s * rows_pad + lr];
  }
  Mv = a; Cv = c;
}

// gradF_i exactly as the reference builds it (clipper.cpp:219 / :238-241):
//   (1 + d) * u - d * ones * u.sum() + Mhat*u + Chat*u * d      evaluated left to right
__device__ __forceinline__ double grad_entry(double ui, double sumu, double Mv, double Cv, double d) {
  const double t1 = __dmul_rn(__dadd_rn(1.0, d), ui);
  const double t2 = __dmul_rn(__dmul_rn(d, 1.0), sumu);
  return __dadd_rn(__dadd_rn(__dsub_rn(t1, t2), Mv), __dmul_rn(Cv, d));
}

}  // namespace clp
#include "clp_dense2.cuh"
#include "clp_sparse.cuh"
namespace clp {

// ------------------------------------------------------------------------------------------
// stand-alone mat-vec kernels (clp_matvec / the c5 sweep): partials, then combine
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
matvec_partials_kernel(MatView mv, Plan p, StageArgs st, double* partM, double* partC) {
  __shared__ __align__(16) double vs[kSegMax];
  __shared__ double red_smem[kWarps];
  matvec_phase<T>(mv, p, st, partM, partC, vs, red_smem);
}

__global__ void matvec_combine_kernel(MatView mv, Plan p, const double* partM, const double* partC,
                                      const double* segsum, const double* v, double d, double* y,
                                      double* Mv_out, double* Cv_out) {
  const int lr = blockIdx.x * blockDim.x + threadIdx.x;
  if (lr >= mv.rows) return;
  double sumv = 0.0;
  for (int s = 0; s < p.NSEG; ++s) sumv += segsum[s];
  double Mv, Cv;
  gather_partials(partM, partC, p.NSEG, mv.rows_pad, lr, Mv, Cv);
  const int i = mv.row0 + lr;
  if (Mv_out) Mv_out[i] = Mv;
  if (Cv_out) Cv_out[i] = Cv;
  if (y) y[i] = grad_entry(v[i], sumv, Mv, Cv, d);
}

// sparse sweep (clp_sparse.cuh); the combine step is matvec_combine_kernel
template <typename T>
__global__ void __launch_bounds__(kThreads, 3)
matvec_sparse_partials_kernel(MatView mv, Plan p, StageArgs st, SparseView sp, double* partM, double* partC) {
  __shared__ __align__(16) double vs[kSegMax + 2];
  __shared__ double red_smem[kWarps];
  sparse_phase<T>(mv, p, st, sp, partM, partC, vs, red_smem);
}

// the same two steps for the stripe decomposition (clp_dense2.cuh)
template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
matvec2_partials_kernel(MatView mv, Plan2 p, StageArgs st, Dense2Buffers buf) {
  __shared__ __align__(16) double smem[2 * 8 * 32 * 2 + 2 * 32];
  dense2_phase<T>(mv, p, st, buf, smem);
}

__global__ void matvec2_combine_kernel(MatView mv, Plan2 p, Dense2Buffers buf, const double* v, double d, double* y,
                                       double* Mv_out, double* Cv_out) {
  __shared__ double smem[kWarps];
  const double sumv = block_sum_ordered(buf.sumpart, p.G, smem);
  const int lr = blockIdx.x * blockDim.x + threadIdx.x;
  if (lr >= mv.rows) return;
  double Mv, Cv;
  dense2_gather(mv, p, buf, lr, Mv, Cv);
  const int i = mv.row0 + lr;
  if (Mv_out) Mv_out[i] = Mv;
  if (Cv_out) Cv_out[i] = Cv;
  if (y) y[i] = grad_entry(v[i], sumv, Mv, Cv, d);
}

// ------------------------------------------------------------------------------------------
// K3-K5: the persistent solver (single GPU, or one rank of a row-block-sharded multi-GPU solve)
//
// Multi-GPU (SURVEY 8e): rank r owns rows [row0,row0+rows) of M and runs this same kernel.  All
// O(m) vectors are replicated.  One exchange step per objective evaluation, done INSIDE the
// kernel over NVLink peer memory (no host, no NCCL launch in the loop):
//   * the gradient entries of the local rows are stored straight into every peer's copy of the
//     vector (P2P st.global), while the candidate u is re-derived locally by every rank;
//   * each rank's partial sums (F, |du|^2, trial norms, ramp statistics) go to every peer's
//     CommBlock, followed by a release flag; every rank adds the per-rank partials in rank order,
//     so all ranks take bit-identical decisions with no broadcast and no rank-0 control.
// ------------------------------------------------------------------------------------------
constexpr int kMaxPeers = 8;

struct CommBlock {  // lives in each rank's HBM, mapped into every peer (CUDA IPC)
  uint4 xred[2][kMaxPeers][kRedVals];  // LL cells: per-rank partial sums, double-buffered
};

struct SolverParams {  // clipper::Params, ref clipper.h:27-60
  double tol_u, tol_F, beta, eps;
  int maxiniters, maxoliters, maxlsiters, rescale_u0;
};

struct SolverOut {  // written by CTA 0 at the end
  double F, d;
  int ifinal, cur, status;
  long long n_evals, n_inner, n_matvec;
  unsigned long long seq_end;
  unsigned long long ns_matvec, ns_combine, ns_exchange;  // CTA 0's view (globaltimer)
};

enum VecSlot : int { V_U0 = 0, V_U1 = 1, V_MV0 = 2, V_MV1 = 3, V_CV0 = 4, V_CV1 = 5, V_SLOTS = 6 };
enum LLSlot : int { L_X = 0, L_G0 = 1, L_G1 = 2, L_SLOTS = 3 };

struct SolverArgs {
  MatView mv;
  Plan plan;
  SolverParams prm;
  TreeBar bar;
  const double* u0;  // [m]
  double* vecs;      // V_SLOTS plain vectors, each mpad long (local only)
  uint4* ll;         // L_SLOTS vectors of LL cells, each mpad long (replicated on every rank)
  long long mpad;
  double* partM;     // [NSEG][rows_pad]
  double* partC;
  double* segsum;    // [NSEG]
  double* red;       // [2][G][kRedVals]  per-CTA partial sums, double-buffered
  Plan2 plan2;       // stripe decomposition (MODE 2)
  Dense2Buffers d2;
  SparseView sp;     // compact rows (MODE 3)
  double* u_final;   // [m] copy of the final iterate
  SolverOut* out;
  // row-block sharding
  int rank, world;
  uint4* peer_ll[kMaxPeers];        // every rank's LL block (peer_ll[rank] == ll)
  CommBlock* comm;                  // local
  CommBlock* peer_comm[kMaxPeers];  // every rank's CommBlock (peer_comm[rank] == comm)
  unsigned long long seq0;          // exchange sequence number before this launch
};

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// store one vector entry into the local AND every peer's replica (self-validating LL cell)
__device__ __forceinline__ void store_replicated(const SolverArgs& a, int slot, int i, double v, unsigned tag) {
  const size_t off = (size_t)slot * a.mpad + i;
  ll_store(a.ll + off, v, tag);
  for (int r = 0; r < a.world; ++r)
    if (r != a.rank) ll_store(a.peer_ll[r] + off, v, tag);
}

// one CTA reduces the per-CTA partial table in a fixed order
__device__ void reduce_table(const double* red, int G, double (&vals)[kRedVals], double* smem /*[kWarps*kRedVals]*/) {
  double loc[kRedVals];
#pragma unroll
  for (int q = 0; q < kRedVals; ++q) loc[q] = 0.0;
  for (int b = threadIdx.x; b < G; b += kThreads) {
#pragma unroll
    for (int q = 0; q < kRedVals; ++q) loc[q] += __ldcg(red + (size_t)b * kRedVals + q);
  }
#pragma unroll
  for (int q = 0; q < kRedVals; ++q) loc[q] = warp_sum(loc[q]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < kRedVals; ++q) smem[warp * kRedVals + q] = loc[q];
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < kRedVals; ++q) {
    double t = 0.0;
    for (int w = 0; w < kWarps; ++w) t += smem[w * kRedVals + q];
    vals[q] = t;
  }
  __syncthreads();
}

// CTA-level deterministic sum of per-thread partials into red[blockIdx.x][*]
__device__ void publish_partials(const double (&loc)[kRedVals], double* red, double* smem) {
  double t[kRedVals];
#pragma unroll
  for (int q = 0; q < kRedVals; ++q) t[q] = warp_sum(loc[q]);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < kRedVals; ++q) smem[warp * kRedVals + q] = t[q];
  }
  __syncthreads();
  if (threadIdx.x < kRedVals) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += smem[w * kRedVals + threadIdx.x];
    red[(size_t)blockIdx.x * kRedVals + threadIdx.x] = s;
  }
}

// Global sum of the per-thread partials `loc` over every CTA of every rank; result in `vals`,
// bit-identical on all CTAs of all ranks.  The last CTA to reach the barrier reduces the local
// table, (multi-GPU) trades the rank totals with the peers through LL cells and adds them in rank
// order, publishes the 8 scalars and only then releases the other CTAs.
// Returns false on a barrier / peer time-out.
__device__ bool exchange_sums(const SolverArgs& a, const double (&loc)[kRedVals], double (&vals)[kRedVals],
                              int& red_par, unsigned long long& round, unsigned long long& seq,
                              double* red_smem, int* smem_flag) {
  const int G = a.plan.G;
  SyncBlock* sb = a.bar.sb;
  double* table = a.red + (size_t)red_par * G * kRedVals;
  publish_partials(loc, table, red_smem);
  ++round;
  ++seq;
  if (bar_arrive(a.bar, round, smem_flag)) {
    reduce_table(table, G, vals, red_smem);
    if (a.world > 1) {
      const unsigned tag = (unsigned)seq;
      if (threadIdx.x == 0) {
#pragma unroll
        for (int q = 0; q < kRedVals; ++q) red_smem[q] = vals[q];
      }
      __syncthreads();
      if ((int)threadIdx.x < a.world * kRedVals) {  // thread (r,q): send total q to rank r, then fetch rank r's total q
        const int r = threadIdx.x / kRedVals, q = threadIdx.x % kRedVals;
        ll_store(&a.peer_comm[r]->xred[red_par][a.rank][q], red_smem[q], tag);
        red_smem[kRedVals + threadIdx.x] = ll_load(&a.comm->xred[red_par][r][q], tag, &sb->error);
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < kRedVals; ++q) {
        double t = 0.0;
        for (int r = 0; r < a.world; ++r) t += red_smem[kRedVals + r * kRedVals + q];
        vals[q] = t;
      }
      __syncthreads();
    }
    if (threadIdx.x == 0) {
#pragma unroll
      for (int q = 0; q < kRedVals; ++q) sb->bcast[red_par][q] = vals[q];
    }
    bar_release(a.bar, round);
  } else {
    bar_wait(a.bar, round);
#pragma unroll
    for (int q = 0; q < kRedVals; ++q) vals[q] = __ldcg(&sb->bcast[red_par][q]);
  }
  __syncthreads();
  red_par ^= 1;
  return *reinterpret_cast<volatile int*>(&sb->error) == 0;
}

// MODE 0: column-segment decomposition (matvec_phase); 2: stripes, upper triangle read once and applied
// two-sidedly (single GPU); 3: compact rows (clp_sparse.cuh) in the MODE-0 decomposition
template <typename T, int MODE>
__global__ void __launch_bounds__(kThreads, MODE == 3 ? 3 : 2) solver_kernel(SolverArgs a) {
  __shared__ __align__(16) double vs[kSegMax + 2];
  __shared__ double red_smem[kWarps * kRedVals + kMaxPeers * kRedVals];
  __shared__ int smem_flag;
  const MatView& mv = a.mv;
  const Plan& p = a.plan;
  const SolverParams& P = a.prm;
  const int gtid = blockIdx.x * kThreads + threadIdx.x;
  const int gthreads = p.G * kThreads;
  double vals[kRedVals];
  double loc[kRedVals];
  struct Vecs {  // U[c], MV[c], CV[c], GL[c] by arithmetic (no dynamically indexed local arrays)
    double* v; const uint4* l; long long mp;
    __device__ __forceinline__ double* U(int c) const { return v + (size_t)(V_U0 + c) * mp; }
    __device__ __forceinline__ double* MV(int c) const { return v + (size_t)(V_MV0 + c) * mp; }
    __device__ __forceinline__ double* CV(int c) const { return v + (size_t)(V_CV0 + c) * mp; }
    __device__ __forceinline__ const uint4* GL(int c) const { return l + (size_t)(L_G0 + c) * mp; }
  };
  const Vecs X{a.vecs, a.ll, a.mpad};
  int* const errp = &a.bar.sb->error;

  long long n_evals = 0, n_inner = 0, n_matvec = 0;
  int cur = 0;  // X.U(cur), G[cur], X.MV(cur), X.CV(cur) describe the current iterate
  double d = 0.0, F = 0.0, sum_cur = 0.0, z = 0.0;
  int i_outer = 0;
  int status = 0;
  // The partial-sum tables are double-buffered: a CTA may publish round r+1 while a slower CTA
  // (or rank) still reads round r.
  int red_par = 0;
  unsigned long long round = 0;     // barrier rounds of this launch
  unsigned long long seq = a.seq0;  // exchange steps since the shards were connected (LL tags)
  unsigned tagG0 = 0u, tagG1 = 0u;  // tag under which G[0] / G[1] were last written
  unsigned long long ns_mv = 0, ns_cb = 0, ns_ex = 0, tmark = global_ns();
#define CLP_LAP(acc) { const unsigned long long t_ = global_ns(); acc += t_ - tmark; tmark = t_; }

#define CLP_ZERO_LOC()            \
  _Pragma("unroll") for (int q_ = 0; q_ < kRedVals; ++q_) loc[q_] = 0.0;
  // rows are dealt to the CTAs in chunks of 32 consecutive rows, round-robin (chunk c -> CTA c % G):
  // coalesced inside a warp, and every CTA gets rows from all parts of the matrix (the gather cost of a
  // row grows with its stripe index in MODE 2)
#define CLP_FOR_ROWS(lr)                                                                    \
  for (int lr = (blockIdx.x + p.G * (threadIdx.x >> 5)) * 32 + (threadIdx.x & 31); lr < mv.rows; lr += p.G * kWarps * 32)
#define CLP_DENSE_PASS()                                                                    \
  if constexpr (MODE == 0) matvec_phase<T>(mv, p, st, a.partM, a.partC, vs, red_smem);      \
  else if constexpr (MODE == 3) sparse_phase<T>(mv, p, st, a.sp, a.partM, a.partC, vs, red_smem); \
  else dense2_phase<T>(mv, a.plan2, st, a.d2, vs);
#define CLP_GATHER()                                                                        \
  if constexpr (MODE == 0 || MODE == 3) gather_partials(a.partM, a.partC, p.NSEG, mv.rows_pad, lr, Mv, Cv); \
  else dense2_gather(mv, a.plan2, a.d2, lr, Mv, Cv);
#define CLP_SUMV(out)                                                                       \
  if constexpr (MODE == 0 || MODE == 3) { out = 0.0; for (int s_ = 0; s_ < p.NSEG; ++s_) out += __ldcg(a.segsum + s_); } \
  else out = block_sum_ordered(a.d2.sumpart, a.plan2.G, red_smem);
#define CLP_EXCHANGE()                                                                      \
  CLP_LAP(ns_cb);                                                                           \
  if (!exchange_sums(a, loc, vals, red_par, round, seq, red_smem, &smem_flag)) { status = 5; goto finish; } \
  CLP_LAP(ns_ex);
#define CLP_BAR_CHECK()                                               \
  ++round;                                                            \
  grid_barrier(a.bar, round, &smem_flag);                             \
  if (*reinterpret_cast<volatile int*>(errp) != 0) { status = 5; goto finish; } \
  CLP_LAP(ns_mv);

  // ---- initialisation: one power step (clipper.cpp:193-198) ------------------------------
  {
    StageArgs st;
    st.llA = nullptr; st.llB = nullptr; st.tag = 0; st.error = errp; st.alpha = 0.0; st.segsum = a.segsum;
    if (P.rescale_u0) {
      st.mode = STAGE_RAW; st.srcA = a.u0; st.z = 1.0; st.dst = nullptr;
      CLP_DENSE_PASS(); ++n_matvec;
      CLP_BAR_CHECK();
    }
    CLP_ZERO_LOC();
    const unsigned tagX = (unsigned)(seq + 1);
    CLP_FOR_ROWS(lr) {
      const int i = mv.row0 + lr;
      double t = a.u0[i];
      if (P.rescale_u0) {
        double Mv, Cv;
        CLP_GATHER();
        t = __dadd_rn(Mv, t);  // M*u0 + u0
      }
      store_replicated(a, L_X, i, t, tagX);
      loc[0] += t * t;
    }
    CLP_EXCHANGE();
    // u /= u.norm(), then Mhat u, Chat u for the initial d
    st.mode = STAGE_DIV; st.srcA = nullptr; st.llA = a.ll + (size_t)L_X * a.mpad; st.tag = tagX;
    st.z = vals[0]; st.dst = X.U(1);
    CLP_DENSE_PASS(); ++n_matvec;
    cur = 1;
    CLP_BAR_CHECK();
  }

  // ---- combine for the initial iterate + initial d (clipper.cpp:201-209) ------------------
  {
    double sumu;
    CLP_SUMV(sumu);
    sum_cur = sumu;
    CLP_ZERO_LOC();
    CLP_FOR_ROWS(lr) {
      const int i = mv.row0 + lr;
      double Mv, Cv;
      CLP_GATHER();
      X.MV(cur)[i] = Mv; X.CV(cur)[i] = Cv;
      const double ui = X.U(cur)[i];
      const double cbu = __dsub_rn(__dsub_rn(__dmul_rn(1.0, sumu), Cv), ui);
      if (cbu > P.eps && ui > P.eps) { loc[0] += 1.0; loc[1] += __dadd_rn(Mv, ui) / cbu; }
    }
    CLP_EXCHANGE();
    if (vals[0] > 0.0) d = vals[1] / vals[0];
  }

  // ---- graduated projected gradient ascent (clipper.cpp:218-281) --------------------------
  for (i_outer = 0; i_outer < P.maxoliters; ++i_outer) {
    // gradF and F for the current u under the current d (clipper.cpp:219-220), plus the squared
    // norm of the first trial point max(u + gradF, 0)
    CLP_ZERO_LOC();
    { const unsigned t_ = (unsigned)(seq + 1); if (cur) tagG1 = t_; else tagG0 = t_; }
    CLP_FOR_ROWS(lr) {
      const int i = mv.row0 + lr;
      const double ui = X.U(cur)[i];
      const double g = grad_entry(ui, sum_cur, X.MV(cur)[i], X.CV(cur)[i], d);
      store_replicated(a, L_G0 + cur, i, g, (cur ? tagG1 : tagG0));
      loc[0] += ui * g;
      double w = __dadd_rn(ui, __dmul_rn(1.0, g)); w = (w < 0.0) ? 0.0 : w;
      loc[1] += w * w;
    }
    CLP_EXCHANGE();
    F = vals[0];
    z = vals[1];

    for (int j = 0; j < P.maxiniters; ++j) {
      double alpha = 1.0;
      double Fnew = 0.0, deltaF = 0.0, du2 = 0.0, zB = 0.0, sum_trial = sum_cur;
      const int nxt = cur ^ 1;
      for (int k = 0; k < P.maxlsiters; ++k) {
        // Phase A: candidate point + dense pass over the local rows of M
        StageArgs st;
        st.mode = STAGE_STEP; st.srcA = X.U(cur); st.llA = nullptr; st.llB = X.GL(cur); st.tag = (cur ? tagG1 : tagG0);
        st.error = errp; st.alpha = alpha; st.z = z; st.dst = X.U(nxt); st.segsum = a.segsum;
        CLP_DENSE_PASS(); ++n_matvec; ++n_evals;
        CLP_BAR_CHECK();
        // Phase B: gradFnew, Fnew, |unew-u|^2 and the squared norms of both possible next trials
        double sumv;
        CLP_SUMV(sumv);
        const double alpha_rej = __dmul_rn(alpha, P.beta);
        CLP_ZERO_LOC();
        { const unsigned t_ = (unsigned)(seq + 1); if (nxt) tagG1 = t_; else tagG0 = t_; }
        CLP_FOR_ROWS(lr) {
          const int i = mv.row0 + lr;
          double Mv, Cv;
          CLP_GATHER();
          X.MV(nxt)[i] = Mv; X.CV(nxt)[i] = Cv;
          const double un = X.U(nxt)[i];
          const double g = grad_entry(un, sumv, Mv, Cv, d);
          store_replicated(a, L_G0 + nxt, i, g, (nxt ? tagG1 : tagG0));
          const double uo = X.U(cur)[i], go = ll_load(X.GL(cur) + i, (cur ? tagG1 : tagG0), errp);
          loc[0] += un * g;
          const double du = __dsub_rn(un, uo);
          loc[1] += du * du;
          double wa = __dadd_rn(uo, __dmul_rn(alpha_rej, go)); wa = (wa < 0.0) ? 0.0 : wa;
          loc[2] += wa * wa;
          double wb = __dadd_rn(un, __dmul_rn(1.0, g)); wb = (wb < 0.0) ? 0.0 : wb;
          loc[3] += wb * wb;
        }
        CLP_EXCHANGE();
        // Phase C: the line-search decision (clipper.cpp:242-251), identical on every CTA / rank
        Fnew = vals[0]; du2 = vals[1]; zB = vals[3];
        deltaF = Fnew - F;
        sum_trial = sumv;
        if (deltaF < -P.eps) {
          alpha = alpha_rej;
          if (k + 1 < P.maxlsiters) { z = vals[2]; continue; }
        }
        break;
      }
      // accept (also when the line search ran out, clipper.cpp:256-258)
      const double deltau = sqrt(du2);
      F = Fnew;
      cur = nxt;
      sum_cur = sum_trial;
      z = zB;
      ++n_inner;
      if (deltau < P.tol_u || fabs(deltaF) < P.tol_F) break;
    }

    // penalty ramp (clipper.cpp:268-280); MV/CV/sum_cur belong to the accepted u
    CLP_ZERO_LOC();
    CLP_FOR_ROWS(lr) {
      const int i = mv.row0 + lr;
      const double ui = X.U(cur)[i];
      const double cbu = __dsub_rn(__dsub_rn(__dmul_rn(1.0, sum_cur), X.CV(cur)[i]), ui);
      if (cbu > P.eps && ui > P.eps) { loc[0] += 1.0; loc[1] += fabs(__dadd_rn(X.MV(cur)[i], ui) / cbu); }
    }
    CLP_EXCHANGE();
    if (vals[0] > 0.0) d += vals[1] / vals[0];
    else break;
  }

  // every rank holds the complete iterate; copy it out, then (multi-GPU) one last rendez-vous so
  // that no rank starts overwriting a peer's replicas while that peer is still inside this launch
  for (int i = gtid; i < mv.m; i += gthreads) a.u_final[i] = X.U(cur)[i];
  if (a.world > 1) {
    CLP_ZERO_LOC();
    CLP_EXCHANGE();
  }

finish:
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.out->F = F; a.out->d = d; a.out->ifinal = i_outer; a.out->cur = cur; a.out->status = status;
    a.out->n_evals = n_evals; a.out->n_inner = n_inner; a.out->n_matvec = n_matvec; a.out->seq_end = seq;
    a.out->ns_matvec = ns_mv; a.out->ns_combine = ns_cb; a.out->ns_exchange = ns_ex;
  }
#undef CLP_LAP
#undef CLP_FOR_ROWS
#undef CLP_DENSE_PASS
#undef CLP_GATHER
#undef CLP_SUMV
#undef CLP_ZERO_LOC
#undef CLP_EXCHANGE
#undef CLP_BAR_CHECK
}

// ------------------------------------------------------------------------------------------
// K7: encode / decode between the reference's dense column-major fp64 M, C and the HBM layout
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void fill_neutral_kernel(T* M, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) M[i] = encode<T>(0.0, false);
}

// The storage rule of a dense entry (i, j), i < j, of caller-given M and C (fp64 or fp32 input; an fp32 x is stored as
// the fp64 (double)x would be): the element stored at (i, j) and (j, i).  bad |= 1 for a negative affinity, 2 for a
// constraint value outside {0, 1} (NaN included).  Every dense load stores through it: the host panels
// (encode_dense_panel_kernel), device tensors (load_dense_dev_kernel) and the batch (batch_dense_solve_kernel).
template <typename T, typename In>
__device__ __forceinline__ T dense_entry(In mv, In cv, unsigned int& bad) {
  const double mval = (double)mv, cval = (double)cv;
  if (mval < 0.0) bad |= 1u;
  if (cval != 0.0 && cval != 1.0) bad |= 2u;
  return encode<T>(mval, cval != 0.0);
}

// Panel of columns [j0, j1) of the column-major inputs (panel-local pointers). Only the strict
// upper triangle (i<j) is read (clipper.cpp:149-158); both (i,j) and (j,i) are written.
// flags: bit0 = negative affinity seen, bit1 = constraint value outside {0,1}
template <typename T>
__global__ void encode_dense_panel_kernel(const double* Mp, const double* Cp, int m, int j0, int j1,
                                          T* M, long long ld, int row0, int rows, int* flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = j0 + blockIdx.y;
  if (j >= j1 || i >= j) return;
  unsigned int bad = 0;
  const T e = dense_entry<T>(Mp[(size_t)(j - j0) * m + i], Cp[(size_t)(j - j0) * m + i], bad);
  if (bad) atomicOr(flags, (int)bad);
  if (i >= row0 && i < row0 + rows) M[(size_t)(i - row0) * ld + j] = e;
  if (j >= row0 && j < row0 + rows) M[(size_t)(j - row0) * ld + i] = e;
}

// 32 x 32 tile [i0, i0 + 32) x [j0, j0 + 32) of caller-given M and C (entry (i, j) at base[i * rs + j * cs], one of
// rs, cs is 1) into sh[i - i0][j - j0] through dense_entry, by 256 threads.  Entries outside i < j < m are neutral and
// are not read.  The reads are coalesced along the unit-stride dimension.
template <typename T, typename In>
__device__ __forceinline__ void dense_tile_load(const In* Mg, const In* Cg, long long rs, long long cs, int m, int i0, int j0,
                                                T (*sh)[33], unsigned int& bad) {
  const int lane = threadIdx.x & 31, k0 = threadIdx.x >> 5;
  const bool rowmajor = cs == 1;
  In mv[4], cv[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k = k0 + 8 * q;
    const int i = i0 + (rowmajor ? k : lane), j = j0 + (rowmajor ? lane : k);
    const bool in = i < j && j < m;
    const long long o = in ? (long long)i * rs + (long long)j * cs : 0;
    mv[q] = in ? Mg[o] : In(0);
    cv[q] = in ? Cg[o] : In(0);
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k = k0 + 8 * q;
    const int r = rowmajor ? k : lane, c = rowmajor ? lane : k;
    sh[r][c] = (i0 + r < j0 + c && j0 + c < m) ? dense_entry<T>(mv[q], cv[q], bad) : encode<T>(0.0, false);
  }
}

// clp_set_dense_dev: one CTA of 256 threads per tile pair (blockIdx.y <= blockIdx.x) of the strict upper triangle of
// device-resident M and C; the tile and its mirror are stored row by row (coalesced along the store's rows).  The store
// was filled with the neutral element before (begin_load), so only the entries i < j < m are written.
template <typename T, typename In>
__global__ void __launch_bounds__(256) load_dense_dev_kernel(const In* Mg, const In* Cg, int m, long long rs, long long cs,
                                                             T* M, long long ld, int* flags) {
  __shared__ T sh[32][33];
  if (blockIdx.y > blockIdx.x) return;
  const int i0 = blockIdx.y * 32, j0 = blockIdx.x * 32;
  unsigned int bad = 0;
  dense_tile_load<T, In>(Mg, Cg, rs, cs, m, i0, j0, sh, bad);
  __syncthreads();
  const int lane = threadIdx.x & 31, k0 = threadIdx.x >> 5;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int k = k0 + 8 * q;
    if (i0 + k < j0 + lane && j0 + lane < m) M[(size_t)(i0 + k) * ld + j0 + lane] = sh[k][lane];  // (i, j)
    if (i0 + lane < j0 + k && j0 + k < m) M[(size_t)(j0 + k) * ld + i0 + lane] = sh[lane][k];  // (j, i)
  }
  if (bad) atomicOr(flags, (int)bad);
}

// strictly-upper CSC -> HBM layout.  pass 0: M values (sign cleared => C=1 provisional is wrong),
// so the host runs: fill neutral; pass A writes |M| with C=0 (negative sign); pass B sets C bits.
// The per-entry bodies are shared with the batched matrix path (clp_batch_matrix.cuh): the storage rule of a CSC
// entry (i, j) lives here only.
template <typename T>
__device__ __forceinline__ void scatter_csc_M_entry(int i, int j, const double* vq, T* M, long long ld, int row0, int rows, int* flags) {
  if (i < 0 || i >= j) { atomicOr(flags, 4); return; }
  const double v = *vq;
  if (v < 0.0) atomicOr(flags, 1);
  const T e = encode<T>(v, false);
  if (i >= row0 && i < row0 + rows) M[(size_t)(i - row0) * ld + j] = e;
  if (j >= row0 && j < row0 + rows) M[(size_t)(j - row0) * ld + i] = e;
}
template <typename T>
__device__ __forceinline__ void scatter_csc_C_entry(int i, int j, const double* vq, T* M, long long ld, int row0, int rows, int* flags) {
  if (i < 0 || i >= j) { atomicOr(flags, 4); return; }
  const double v = *vq;
  if (v == 0.0) return;
  if (v != 1.0) atomicOr(flags, 2);
  if (i >= row0 && i < row0 + rows) { T* p = M + (size_t)(i - row0) * ld + j; double a; bool c; decode(*p, a, c); *p = encode<T>(a, true); }
  if (j >= row0 && j < row0 + rows) { T* p = M + (size_t)(j - row0) * ld + i; double a; bool c; decode(*p, a, c); *p = encode<T>(a, true); }
}
template <typename T>
__global__ void scatter_csc_M_kernel(const long long* colptr, const int* rowidx, const double* val, int m,
                                     T* M, long long ld, int row0, int rows, int* flags) {
  const int j = blockIdx.x;
  for (long long q = colptr[j] + threadIdx.x; q < colptr[j + 1]; q += blockDim.x)
    scatter_csc_M_entry<T>(rowidx[q], j, val + q, M, ld, row0, rows, flags);
}
template <typename T>
__global__ void scatter_csc_C_kernel(const long long* colptr, const int* rowidx, const double* val, int m,
                                     T* M, long long ld, int row0, int rows, int* flags) {
  const int j = blockIdx.x;
  for (long long q = colptr[j] + threadIdx.x; q < colptr[j + 1]; q += blockDim.x)
    scatter_csc_C_entry<T>(rowidx[q], j, val + q, M, ld, row0, rows, flags);
}

// columns [j0,j1) of getAffinityMatrix()/getConstraintMatrix(): out[(j-j0)*m + i], sym + I.
// By symmetry column j equals row j of the store, so reads are coalesced along i.
template <typename T>
__global__ void decode_dense_panel_kernel(const T* M, long long ld, int m, int j0, int j1, int which,
                                          double* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = j0 + blockIdx.y;
  if (j >= j1 || i >= m) return;
  double v;
  if (i == j) v = 1.0;
  else {
    double a; bool c;
    decode(M[(size_t)j * ld + i], a, c);
    v = which ? (c ? 1.0 : 0.0) : a;
  }
  out[(size_t)(j - j0) * m + i] = v;
}

// count stored affinities / constraints in the strict upper triangle
template <typename T>
__global__ void count_upper_kernel(const T* M, long long ld, int m, int row0, int rows,
                                   unsigned long long* counts) {
  unsigned long long nM = 0, nC = 0;
  const size_t total = (size_t)rows * (size_t)m;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int lr = (int)(t / m), j = (int)(t % m);
    const int i = row0 + lr;
    if (i >= j) continue;
    double a; bool c;
    decode(M[(size_t)lr * ld + j], a, c);
    nM += (a != 0.0); nC += c;
  }
  for (int o = 16; o > 0; o >>= 1) { nM += __shfl_xor_sync(0xffffffffu, nM, o); nC += __shfl_xor_sync(0xffffffffu, nC, o); }
  if ((threadIdx.x & 31) == 0) { atomicAdd(counts, nM); atomicAdd(counts + 1, nC); }
}

// k x k sub-block of M induced by the index set S (for Rounding::DSD): out column-major doubles
template <typename T>
__global__ void gather_subblock_kernel(const T* M, long long ld, const int* S, int k, double* out) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (a >= k || b >= k) return;
  double v = 0.0;
  if (a != b) { bool c; decode(M[(size_t)S[b] * ld + S[a]], v, c); }
  out[(size_t)b * k + a] = v;
}

}  // namespace clp
#include "clp_resident.cuh"
#include "clp_batch.cuh"
