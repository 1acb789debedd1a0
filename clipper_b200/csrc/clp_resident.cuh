// clp_resident.cuh -- the "resident vector" solver: findDenseClique() (ref clipper.cpp:172-283) with ONE device-wide
// synchronisation per objective evaluation.
//
// Why.  The segmented solver (solver_kernel in clp_kernels.cuh) cuts the columns into segments of <= 4096 so that a
// CTA's piece of the trial vector fits a small shared-memory buffer; a row's product is then spread over several CTAs,
// which costs a partial table in HBM, a device-wide barrier between the sweep and the combine step and a second one
// for the scalar sums: a fixed cost per evaluation that caps multi-GPU scaling and makes small problems
// latency-bound.  Here, for every problem whose
// WHOLE trial vector fits the 227 KB of shared memory of an SM (m <= 27 000 in fp64), one fat CTA per SM keeps the vector
// resident, every row is owned by exactly one CTA, and the combine step (gradient entry, objective and step-norm
// partial sums, BOTH candidate next trial points) runs in the tail of the sweep.  Per evaluation:
//     stage the candidate w (L2 -> shared, 8 B per column, as it is: eight cp.async.bulk copies with mbarrier completion
//     when unsharded, LL cells when sharded) -> sweep the CTA's rows -> per-row epilogue (unew = w / |w| is linear, so
//     the exact division by the norm is applied to the row's M w, C w and to sum(w) instead of to every entry of the
//     vector in every CTA) -> publish 8 partial sums -> one arrival counter -> every CTA adds the G x 8 table in the
//     same fixed order.
// No partial table in HBM, no last-arriver serial reduction, no release hop.
//
// Layout: the compact sliced-ELL copy of clp_sparse.cuh with ONE segment = the whole row (16-bit column INDEX per
// entry instead of a byte offset; padding entries point at column m, where the staged vector holds 0.0), or -- for a
// plain fp32 matrix on one GPU -- its packed variant: one 4-byte word per entry whose column is the running sum of
// 5-bit deltas (res_apply_packed: a segmented scan over the 8 lanes of a member, a carry from round to round).  Rows are
// sorted by length and grouped four at a time (an item, chunk-interleaved).  A CTA owns a contiguous, byte-balanced
// range of items (sparse_partition_kernel); inside the CTA the warps split the CTA's chunk STREAM evenly, regardless
// of item boundaries: a warp adds up the part of an item it covers (a "piece") and the per-row epilogue adds the
// pieces in stream order -- perfect balance inside the SM with one __syncthreads per sweep, and bit-reproducible.
//
// Loads: software-pipelined ld.global.nc rounds in registers (D rounds of U chunks per lane in flight); ResShape holds
// the one (threads, U, D) of each handle type.
//
// The same kernel body serves three callers: the single-GPU solve (grid = one CTA per SM), one rank of a row-sharded
// multi-GPU solve (candidate vectors and rank totals cross NVLink as self-validating LL cells) and, with G = 1 and
// no device-wide synchronisation at all, every problem of a batch of small problems (clp_batch.cuh).
#pragma once

namespace clp {

constexpr int kResThreads = 768;                  // widest resident instance (24 warps): sizes the fit test of compact_shape
constexpr int kResWarps = kResThreads / 32;
constexpr int kResMaxM = 27648;                   // largest m whose fp64 trial vector (+ scratch) fits 227 KB
constexpr int kPieceVals = 8;                     // a piece: 4 members x (|M| v, C v)

// Load pipeline of the resident kernels per handle type (storage T, sharded or not): NT threads, D rounds of U chunks
// per lane in flight.  On one H100 (sm_90a) the 512-thread fp32 pipeline gets 128 registers and spills less than a
// 768-thread one, which is capped at 80; it was the fastest with both layouts (DESIGN.md section 6).  Shards keep
// 768 threads (not measured on several H100s).  fp64 entries: one light 2 x 2 pipeline.
template <int NT_, int U_, int D_> struct ResPipe { static constexpr int NT = NT_, U = U_, D = D_; };
template <typename T, bool SHARDED> struct ResShapeOf { using type = ResPipe<512, 2, 2>; };
template <> struct ResShapeOf<float, false> { using type = ResPipe<512, 2, 4>; };
template <> struct ResShapeOf<float, true> { using type = ResPipe<768, 2, 3>; };
template <typename T, bool SHARDED> using ResShape = typename ResShapeOf<T, SHARDED>::type;

enum ResVec : int { R_U0 = 0, R_U1, R_G0, R_G1, R_MV0, R_MV1, R_CV0, R_CV1, R_SLOTS };
enum ResStage : int { RS_RAW = 0, RS_DIV = 1, RS_STEP = 2 };

// line-search evaluations by sweep kind and what the restricted sweeps read, over one solve
struct ResSweeps {
  long long full, rebuild, restricted;
  unsigned long long entries, padding;  // restricted sweeps: entries read, padding entries read
  long long fallback;                   // full sweeps after the first rebuild (the support grew past m / kSupportDiv)
};

struct ResArgs {
  SparseView sp;           // full-row compact copy: off16 holds column indices, itemptr [NI + 1], rowid [rows_pad]
  int m, row0, rows, rows_pad, NI;
  int G;                   // CTAs working on this problem (== gridDim.x of the solver launch)
  SolverParams prm;
  const double* u0;        // [m]
  double* vecs;            // R_SLOTS plain vectors x mpad (only the entries of the local rows are ever touched)
  double* cand;            // world == 1: candidate trial points, [2 parities][2: accept, reject][mpad] doubles
  uint4* ll;               // world  > 1: the same as LL cells + one more vector (final iterate): [5][mpad], replicated
  long long mpad;
  double* pieces;          // [(NI + G * warps)][8]
  SyncBlock* sb;
  double* u_final;         // [m]
  SolverOut* out;
  int rank, world;
  uint4* peer_ll[kMaxPeers];
  CommBlock* comm;
  CommBlock* peer_comm[kMaxPeers];
  unsigned long long seq0;
  long long spin_limit;    // clock64 ticks a wait may last before it raises the time-out flag
  unsigned int pieces_cap, state_cap;  // on-chip piece table (entries) / row state (rows) per CTA, 0: keep them in HBM
  uint4* redll;            // [2][G][8] per-CTA partial sums as self-validating LL cells (zeroed before the launch)
  double* prof_cta;        // nullable: [G][8] per-CTA phase times in ns (sweeps, epilogues, exchanges, staging), items, chunks,
                           //   restricted entries swept (rebuild and restricted evaluations), the split's largest overshoot (res_prof_split)
  int prof_laps;           // thread 0 of every CTA reads %globaltimer four times per evaluation (phase split in clp_solution)
  const int* wcol;         // packed layout: [G][warps][4] column of each member's last entry before the warp's stream (-1: none)
  // packed layout on one GPU: the restricted copy (res_restrict_build; null rval: every sweep reads the whole copy)
  float* rval;             // entries of every row whose column lies in S', in column order, padded to a multiple of 4
  unsigned short* rcol;    //   with (0, column m); row slot of member s of item it: roff[it] + s * (roff[it + 1] - roff[it]) / 4
  const unsigned int* roff;  // [NI + 1]
  unsigned int* rlen;      // [rows_pad] entries of every row slot (stream position 4 it + s), without the padding
  unsigned int* rbits;     // [G][ceil(m / 32)] S' as a column bitmap, one copy per CTA
  uint4* rprod;            // [rows_pad][2] M w, C w of every row slot from the last restricted sweep as LL cells tagged
                           //   with the evaluation's round (zeroed before the launch)
  ResSweeps* sweeps;       // counters of the last solve (written by CTA 0)
};

// S' is rebuilt when the candidate's support holds at most m / kSupportDiv columns
constexpr int kSupportDiv = 4;
// entries a row slot must hold: the row's stored entries, at most one per support column, rounded up to whole chunks
__host__ __device__ inline unsigned int res_restrict_cap(unsigned int row_entries, int m) {
  const unsigned int t = ((unsigned int)(m / kSupportDiv) + 3u) & ~3u;
  return row_entries < t ? row_entries : t;
}
// fixed charge of a row slot, in chunks, in the split of the restricted sweeps (res_restrict_split): the row's
// reduction, shuffles and store, and the rest of its last, partly filled round (32 was faster than 8 and 64 at c2,
// DESIGN.md section 6)
constexpr unsigned int kRowCost = 32;
static_assert(kRowCost >= 1, "every slot must cost something: the last range then ends at the last slot");

// ---------------------------------------------------------------------------------------------------------------
// mbarrier / bulk-copy primitives (SASS: SYNCS.*, UBLKCP)
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(void* bar, unsigned int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(void* bar, unsigned int bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned int bytes, void* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(void* bar, unsigned int parity) {
  unsigned int ok;
  asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
// bounded wait: a bulk copy that never lands raises the error flag instead of hanging the GPU
__device__ __forceinline__ void mbar_wait(void* bar, unsigned int parity, int* error) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 2000000000LL) { atomicExch(error, 1); break; }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// shared-memory plan of a resident CTA (dynamic shared memory; the host uses the same function)
// ---------------------------------------------------------------------------------------------------------------
constexpr unsigned int kStageBlocks = 8;  // sub-blocks (one mbarrier each) of a bulk-copied trial vector
struct ResSmem {
  unsigned int off_red, off_fin, off_wb, off_misc, off_sbar, total;
  // optional on-chip tables behind the plan's minimum (capacities chosen by the host, a few KB: the more shared
  // memory a CTA takes, the less L1 is left for the streaming loads): the CTA's piece table, and per row the solver
  // state (8 doubles) and a descriptor (global row, first / last warp of its pieces).  A CTA whose items / rows
  // exceed the capacities uses the HBM copies instead.
  unsigned int off_pieces, pieces_cap, off_state, state_cap, off_desc, total_ext;
};
__host__ __device__ inline ResSmem res_smem_plan(int m, int NW, unsigned int pieces_cap = 0, unsigned int state_cap = 0) {
  ResSmem s;
  unsigned int o = (unsigned int)(((m + 1 + 1) & ~1) * 8);        // vs[0..m], vs[m] = 0
  s.off_red = o; o += (unsigned int)(NW * kRedVals * 8);
  s.off_fin = o; o += (unsigned int)((2 + kMaxPeers) * kRedVals * 8);
  s.off_wb = o; o += (unsigned int)((NW + 1) * 4);
  o = (o + 7u) & ~7u;
  s.off_misc = o; o += (unsigned int)NW * 8;  // per warp: start of its stream (item, end)
  s.off_sbar = o; o += kStageBlocks * 8u;  // mbarriers of the bulk-copy staging (res_stage_bulk)
  s.total = o;
  o = (o + 15u) & ~15u;
  s.pieces_cap = pieces_cap; s.state_cap = state_cap;
  s.off_pieces = o; o += pieces_cap * kPieceVals * 8u;
  s.off_state = o; o += state_cap * R_SLOTS * 8u;
  s.off_desc = o; o += state_cap * 8u;
  s.total_ext = o;
  return s;
}

// x / y for a divisor shared by many dividends: r = RN(1/y); two residual corrections with FMA.  The last step is
// Markstein's correction applied to a quotient that is already within an ulp, which rounds like the IEEE division
// (as the reference's normalize() does) at a third of its instruction count.  Tiny, huge and non-finite operands take
// the true division.
__device__ __forceinline__ double div_by_invariant(double x, double y, double r) {
  // callers guarantee 0 < y < inf.  Most entries of a projected iterate are exactly 0: answer them at once -- the
  // IEEE division's special-case path for a zero dividend is a long subroutine, and with 95 % zeros it made staging
  // the trial vector a large share of every evaluation
  if (x == 0.0) return x;
  const double q0 = x * r;
  if (!(fabs(q0) > 1e-290 && fabs(q0) < 1e290)) return x / y;  // also 0, NaN, Inf
  const double e0 = fma(-q0, y, x);
  const double q1 = fma(e0, r, q0);
  const double e1 = fma(-q1, y, x);
  return fma(e1, r, q1);
}

// ---------------------------------------------------------------------------------------------------------------
// deterministic block reductions (identical result on every CTA given identical inputs)
// ---------------------------------------------------------------------------------------------------------------
template <int NT>
__device__ __forceinline__ double res_block_sum(double x, double* red_s, double* fin) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  x = warp_sum(x);
  __syncthreads();
  if (lane == 0) red_s[warp] = x;
  __syncthreads();
  if (warp == 0) {
    double t = (lane < NT / 32) ? red_s[lane] : 0.0;
    t = warp_sum(t);
    if (lane == 0) fin[0] = t;
  }
  __syncthreads();
  return fin[0];
}

// per-thread partials loc[8] -> red_row[8] (one CTA's row of the table)
template <int NT>
__device__ __forceinline__ void res_publish(const double (&loc)[kRedVals], double* red_row, double* red_s) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double t[kRedVals];
#pragma unroll
  for (int q = 0; q < kRedVals; ++q) t[q] = warp_sum(loc[q]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < kRedVals; ++q) red_s[warp * kRedVals + q] = t[q];
  }
  __syncthreads();
  if (threadIdx.x < kRedVals) {
    double s = 0.0;
    for (int w = 0; w < NT / 32; ++w) s += red_s[w * kRedVals + threadIdx.x];
    red_row[threadIdx.x] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// staging: the whole trial vector into shared memory; returns sum(v) (bit-identical on every CTA)
//   RS_RAW : v = src                                   (power step on u0, stand-alone mat-vec)
//   RS_DIV : v = w / |w|                               (u /= u.norm(), clipper.cpp:198 -- no zero guard)
//   RS_STEP: v = w / |w| if |w|^2 > 0 else w           (unew.normalize(), clipper.cpp:237), w = a candidate point
// ---------------------------------------------------------------------------------------------------------------
// LL cell load.  The cells live in LOCAL memory (peers store into it over NVLink, the home L2 is the point of
// coherence for every writer), so a gpu-scope relaxed load observes them; GPU_SCOPE = false uses the system-scope
// (volatile) load of the classic LL protocol.
template <bool GPU_SCOPE>
__device__ __forceinline__ void ll_ld4(const uint4* p, unsigned int& lo, unsigned int& t1, unsigned int& hi, unsigned int& t2) {
  if constexpr (GPU_SCOPE)
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(t1), "=r"(hi), "=r"(t2) : "l"(p) : "memory");
  else
    asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(t1), "=r"(hi), "=r"(t2) : "l"(p) : "memory");
}

template <int NT, bool SHARDED>
__device__ double res_stage(int mode, int m, const double* src, const uint4* cells, unsigned int tag, double z,
                            double* vs, double* red_s, double* fin, int* errp, long long spin_limit, int rot = 0,
                            bool raw = false) {
  // raw: the vector is staged as it is and nothing is summed (returns 0) -- the caller applies 1/|w| to the row results
  // Every CTA of the grid reads the SAME m values at the same moment.  With all CTAs walking the vector in the same
  // order, four 8-byte loads in flight per thread, this step took a fifth of the solver at m = 20 000 while the sweep
  // itself ran at the HBM peak.  So: 16-byte
  // loads, eight of them in flight per thread, and every CTA starts at a different place (rot) so that the SMs do not
  // queue on the same L2 lines; the sum is then taken in a CTA-independent order from shared memory.
  const double nrm = sqrt(z);
  const double rinv = 1.0 / nrm;
  const bool scale = !raw && ((mode == RS_DIV) || (mode == RS_STEP && z > 0.0));
  const int npair = (m + 1) >> 1;
  const int K = (npair + NT - 1) / NT;          // pair slots per thread
  const int span = K * NT;
  const int r0 = ((rot % span) + span) % span & ~31;  // whole warps stay contiguous
  auto finish = [&](int j, double w) {            // element j of the vector
    if (j < m) {
      double v = w;
      if (scale) v = (mode == RS_DIV) ? (w / nrm) : div_by_invariant(w, nrm, rinv);
      vs[j] = v;
    }
  };
  if (SHARDED && mode != RS_RAW) {
    constexpr int kB = 4;  // pairs (= 2 LL cells each) in flight per thread (7 made the sharded instance spill inside the
                           // sweep and did not shorten the staging)
    for (int k0 = 0; k0 < K; k0 += kB) {
      unsigned int lo[2 * kB], t1[2 * kB], hi[2 * kB], t2[2 * kB];
      int q[kB];
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        int pos = threadIdx.x + (k0 + b) * NT + r0; if (pos >= span) pos -= span;
        q[b] = (k0 + b < K && pos < npair) ? pos : -1;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          lo[2 * b + e] = hi[2 * b + e] = 0u; t1[2 * b + e] = t2[2 * b + e] = tag;
          if (q[b] >= 0 && 2 * q[b] + e < m)
            ll_ld4<true>(cells + 2 * q[b] + e, lo[2 * b + e], t1[2 * b + e], hi[2 * b + e], t2[2 * b + e]);
        }
      }
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        if (q[b] < 0) continue;
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int j = 2 * q[b] + e, c = 2 * b + e;
          if (j >= m) continue;
          if (!(t1[c] == tag && t2[c] == tag)) {  // not there yet: poll (bounded)
            long long t0 = 0;
            for (;;) {
              ll_ld4<false>(cells + j, lo[c], t1[c], hi[c], t2[c]);
              if (t1[c] == tag && t2[c] == tag) break;
              if (t0 == 0) t0 = clock64();
              else if (clock64() - t0 > spin_limit) { atomicExch(errp, 1); break; }
            }
          }
          finish(j, __hiloint2double((int)hi[c], (int)lo[c]));
        }
      }
    }
  } else {
    constexpr int kB = 8;  // 16-byte loads in flight per thread (14 = one round trip at m = 20 000 raised the kernel's stack frame
                           // to 336 bytes: spills; fetching only the non-zero entries through a flag byte per entry moved 1/6 of
                           // the bytes but added a dependent round trip and was slower)
    for (int k0 = 0; k0 < K; k0 += kB) {
      double2 w[kB];
      int q[kB];
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        int pos = threadIdx.x + (k0 + b) * NT + r0; if (pos >= span) pos -= span;
        q[b] = (k0 + b < K && pos < npair) ? pos : -1;
        w[b] = make_double2(0.0, 0.0);
        if (q[b] >= 0) {
          if (2 * q[b] + 1 < m) asm volatile("ld.global.cg.v2.f64 {%0,%1}, [%2];" : "=d"(w[b].x), "=d"(w[b].y) : "l"(src + 2 * q[b]) : "memory");
          else w[b].x = __ldcg(src + 2 * q[b]);   // odd m: never read past the caller's vector
        }
      }
#pragma unroll
      for (int b = 0; b < kB; ++b) {
        if (q[b] < 0) continue;
        finish(2 * q[b], w[b].x);
        finish(2 * q[b] + 1, w[b].y);
      }
    }
  }
  if (threadIdx.x == 0) vs[m] = 0.0;  // column of the padding entries
  __syncthreads();
  if (raw) return 0.0;
  double part = 0.0;                   // CTA-independent order: thread t adds entries t, t + NT, ...
  for (int j = threadIdx.x; j < m; j += NT) part += vs[j];
  return res_block_sum<NT>(part, red_s, fin);
}

// The same step with the copy engine: thread 0 issues the whole vector as kStageBlocks cp.async.bulk copies (SASS UBLKCP)
// straight from the L2-resident candidate array into vs, each completing its own mbarrier; the CTA then normalises the
// sub-blocks in place as they land.  No registers hold bytes in flight and the copies of all sub-blocks overlap the
// arithmetic of the first ones.  The candidate array was written by other CTAs with generic stores and acquired through
// the device-wide exchange: the issuing thread orders its async-proxy reads behind that with fence.proxy.async; every
// thread fences its in-place generic writes against the next call's async-proxy writes the same way.  Same values and
// the same CTA-independent summation order as res_stage (modes RS_DIV / RS_STEP, 16-byte aligned src).
template <int NT>
__device__ double res_stage_bulk(int mode, int m, const double* src, double z, double* vs, unsigned long long* bars,
                                 unsigned int& phase, double* red_s, double* fin, int* errp, int rot, bool raw = false) {
  // raw: the vector is staged as it is and nothing is summed (returns 0) -- the caller applies 1/|w| to the row results
  const double nrm = sqrt(z);
  const double rinv = 1.0 / nrm;
  const bool scale = !raw && ((mode == RS_DIV) || (mode == RS_STEP && z > 0.0));
  auto norm1 = [&](double w) { return (mode == RS_DIV) ? (w / nrm) : div_by_invariant(w, nrm, rinv); };
  const int m2 = m & ~1;                                                   // bulk part: a multiple of 16 bytes
  const int sb = (int)(((m2 + (int)kStageBlocks - 1) / (int)kStageBlocks + 1) & ~1);  // elements per sub-block (even)
  const int k0 = ((rot % (int)kStageBlocks) + (int)kStageBlocks) % (int)kStageBlocks;  // CTAs start at different sub-blocks
  __syncthreads();  // nobody still reads the previous trial vector
  if (threadIdx.x == 0) {
    asm volatile("fence.proxy.async;" ::: "memory");
#pragma unroll 1
    for (int t = 0; t < (int)kStageBlocks; ++t) {
      int k = k0 + t; if (k >= (int)kStageBlocks) k -= (int)kStageBlocks;
      const int lo = k * sb, hi = min(lo + sb, m2);
      const unsigned int bytes = hi > lo ? (unsigned int)(hi - lo) * 8u : 0u;
      mbar_expect_tx(&bars[k], bytes);  // 0 bytes: the arrival alone completes the phase
      if (bytes) bulk_g2s(vs + lo, src + lo, bytes, &bars[k]);
    }
    if (m & 1) { const double w = __ldcg(src + m - 1); vs[m - 1] = scale ? norm1(w) : w; }
    vs[m] = 0.0;  // column of the padding entries
  }
#pragma unroll 1
  for (int t = 0; t < (int)kStageBlocks; ++t) {
    int k = k0 + t; if (k >= (int)kStageBlocks) k -= (int)kStageBlocks;
    mbar_wait(&bars[k], phase & 1u, errp);
    if (!scale) continue;
    const int lo = k * sb, hi = min(lo + sb, m2);
    for (int j = lo + 2 * (int)threadIdx.x; j < hi; j += 2 * NT) {
      double2 w = *reinterpret_cast<double2*>(vs + j);
      w.x = norm1(w.x); w.y = norm1(w.y);
      *reinterpret_cast<double2*>(vs + j) = w;
    }
  }
  phase ^= 1u;
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  if (raw) return 0.0;
  double part = 0.0;                   // CTA-independent order: thread t adds entries t, t + NT, ...
  for (int j = threadIdx.x; j < m; j += NT) part += vs[j];
  return res_block_sum<NT>(part, red_s, fin);
}

// ---------------------------------------------------------------------------------------------------------------
// the sweep: this CTA's item range of the compact copy against the resident vector -> pieces
// ---------------------------------------------------------------------------------------------------------------
template <typename T, bool PLAIN>
__device__ __forceinline__ void res_apply_chunk(const Entry4<T>& E, const double* vs, double& aM, double& aC) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const double v = vs[off_of(E.k, q)];
    if (PLAIN) {
      aM = fma((double)E.get(q), v, aM);  // padding: -0.0 * 0.0
      aC += v;
    } else {
      double dM = 0.0, dC = 0.0;
      apply_elem<false>(E.get(q), v, 0.0, aM, aC, dM, dC);
    }
  }
}

// 4 packed entries of one row slice (clp_sparse.cuh, pack_word)
struct Packed4 {
  uint4 w;
  __device__ __forceinline__ void load(const unsigned int* val, unsigned long long at) {
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w) : "l"(val + at));
  }
  __device__ __forceinline__ void load_cg(const unsigned int* val, unsigned long long at) {
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(w.x), "=r"(w.y), "=r"(w.z), "=r"(w.w) : "l"(val + at));
  }
  __device__ __forceinline__ void neutral() { w = make_uint4(kPackPad, kPackPad, kPackPad, kPackPad); }
};
__device__ __forceinline__ unsigned int pack_delta(unsigned int w) { return ((w >> 27) + 1u) & 31u; }

// One round of U packed chunks (lane l holds chunks l, l + 32, ... of the round: member l & 3).  The columns are running
// sums of the deltas: inside a chunk in registers, over the 8 lanes of a member by ONE segmented scan for all U chunks
// (a 10-bit field per chunk: 8 x 4 x 31 < 1024; 3 shuffles + 1 for the member's total), and from round to round by the
// member's carry (column of its last entry).  Fillers and padding (code 0) add nothing to either sum.
template <int U>
__device__ __forceinline__ void res_apply_packed(const Packed4 (&E)[U], const double* vs, unsigned int ebias, int& carry,
                                                 double (&aM)[2], double (&aC)[2]) {
  static_assert(U <= 3, "three 10-bit fields per scan");
  const int lane = threadIdx.x & 31;
  unsigned int own = 0u;
#pragma unroll
  for (int u = 0; u < U; ++u)
    own += (pack_delta(E[u].w.x) + pack_delta(E[u].w.y) + pack_delta(E[u].w.z) + pack_delta(E[u].w.w)) << (10 * u);
  unsigned int inc = own;
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
  const unsigned int tot = __shfl_sync(0xffffffffu, inc, 28 + (lane & 3));
  const unsigned int exc = inc - own;
  int base = carry;
#pragma unroll
  for (int u = 0; u < U; ++u) {
    int col = base + (int)((exc >> (10 * u)) & 1023u);
    const unsigned int w4[4] = {E[u].w.x, E[u].w.y, E[u].w.z, E[u].w.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      col += (int)pack_delta(w4[q]);
      double v = 0.0;
      if (w4[q] & 0x07800000u) v = vs[col];
      aM[u & 1] = fma((double)__uint_as_float((w4[q] & 0x07ffffffu) + ebias), v, aM[u & 1]);
      aC[u & 1] += v;
    }
    base += (int)((tot >> (10 * u)) & 1023u);
  }
  carry = base;
}

// chunk range [s0, s1) of warp w out of NW over the CTA's stream [c_lo, c_hi): multiples of 4 chunks
__device__ __forceinline__ unsigned int res_warp_bound(unsigned int c_lo, unsigned int c_hi, int w, int NW) {
  if (w >= NW) return c_hi;
  const unsigned long long q = (unsigned long long)((c_hi - c_lo) >> 2);
  return c_lo + (unsigned int)(q * (unsigned long long)w / (unsigned long long)NW) * 4u;
}

// smallest index it in [lo, hi] with itemptr[it + 1] > c   (i.e. the non-empty item that holds chunk c)
__device__ __forceinline__ unsigned int res_item_of(const unsigned int* itemptr, unsigned int lo, unsigned int hi, unsigned int c) {
  while (lo < hi) {
    const unsigned int mid = lo + ((hi - lo) >> 1);
    if (itemptr[mid + 1] > c) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// COH: the compact copy was written earlier IN THIS LAUNCH (batched problems): no ld.global.nc, L2-coherent loads instead
// PACK: 4-byte packed entries (plain fp32 matrices): the columns come from the deltas, a warp whose stream starts inside
// an item takes its members' columns there from a.wcol; the carry restarts at -1 with every new item
template <typename T, int NT, int U, int D, bool COH = false, bool PACK = false>
__device__ void res_sweep(const ResArgs& a, const int bid, const double* vs, unsigned char* smem, const ResSmem& plan,
                          double* ptab, unsigned int isub) {
  constexpr int NW = NT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const SparseView& sp = a.sp;
  const unsigned int it0 = sp.cta_first[bid], it1 = sp.cta_first[bid + 1];
  if (it0 >= it1) return;
  const unsigned int* itemptr = sp.itemptr;
  const unsigned int c_lo = itemptr[it0], c_hi = itemptr[it1];
  const unsigned int s0 = res_warp_bound(c_lo, c_hi, warp, NW), s1 = res_warp_bound(c_lo, c_hi, warp + 1, NW);
  if (s0 >= s1) return;
  const T* val = reinterpret_cast<const T*>(sp.val);
  const unsigned short* idx = sp.off16;
  const unsigned int padk = (unsigned int)a.m | ((unsigned int)a.m << 16);  // column m holds 0.0
  double* pieces = ptab + (size_t)warp * kPieceVals;  // + (item - isub) * 8

  // ---- producer cursor (warp-uniform): the piece being loaded.  Where a warp's stream starts never changes during a
  // solve: found once (binary search over the item pointers = a chain of dependent L2 loads) and kept in shared memory
  uint2* wstart = reinterpret_cast<uint2*>(smem + plan.off_misc) + warp;
  unsigned int cit, ce;
  {
    const uint2 w = *wstart;
    if (w.y != 0u) { cit = w.x; ce = w.y; }
    else {
      cit = res_item_of(itemptr, it0, it1 - 1, s0);
      ce = min(itemptr[cit + 1], s1);
      __syncwarp();
      if (lane == 0) *wstart = make_uint2(cit, ce);   // ce > s0 >= 0: never 0
    }
  }
  unsigned int cj = s0;
  bool pdone = false;
  double aM[2] = {0.0, 0.0}, aC[2] = {0.0, 0.0};
  const unsigned int* pw = reinterpret_cast<const unsigned int*>(sp.val);
  int carry = -1;
  if constexpr (PACK) carry = a.wcol[((size_t)bid * NW + warp) * 4 + (lane & 3)];

  auto advance = [&](unsigned int& jbase, unsigned int& n, unsigned int& item, bool& last) {
    // describes the next round: first chunk, chunks in it, its item, whether it ends its piece; moves the cursor
    jbase = cj; item = cit;
    const unsigned int left = ce - cj;
    n = left < 32u * U ? left : 32u * U;
    last = (n == left);
    if (last) {
      cj = ce;
      if (cj >= s1) pdone = true;
      else {
        do { ++cit; } while (itemptr[cit + 1] <= cj);  // skip empty items
        ce = min(itemptr[cit + 1], s1);
      }
    } else cj += 32u * U;
  };
  auto flush = [&](unsigned int item) {
    double accM = aM[0] + aM[1], accC = aC[0] + aC[1];
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      accM += __shfl_xor_sync(0xffffffffu, accM, o);
      accC += __shfl_xor_sync(0xffffffffu, accC, o);
    }
    if (lane < 4) {
      double* p = pieces + (size_t)(item - isub) * kPieceVals;
      p[lane] = accM; p[4 + lane] = accC;
    }
    aM[0] = aM[1] = aC[0] = aC[1] = 0.0;
  };
  const bool plain = sp.plain != 0;

  // D rounds of U chunks per lane in registers; the refill of a round is issued right after it has been applied,
  // so D - 1 rounds are always in flight behind the one being consumed
  std::conditional_t<PACK, Packed4, Entry4<T>> E[D][U];
  unsigned int mitem[D];
  bool mlast[D], mvalid[D];
  auto produce = [&](int s) {
    mvalid[s] = !pdone;
    if (pdone) return;
    unsigned int jb, n;
    advance(jb, n, mitem[s], mlast[s]);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const unsigned int c = lane + 32u * u;
      if constexpr (PACK) {
        if (c < n) { if constexpr (COH) E[s][u].load_cg(pw, 4ull * (jb + c)); else E[s][u].load(pw, 4ull * (jb + c)); }
        else E[s][u].neutral();
      } else {
        if (c < n) { if constexpr (COH) E[s][u].load_cg(val, idx, 4ull * (jb + c)); else E[s][u].load(val, idx, 4ull * (jb + c)); }
        else E[s][u].neutral_at(padk);
      }
    }
  };
#pragma unroll
  for (int s = 0; s < D; ++s) produce(s);
  for (;;) {
    bool done = false;
#pragma unroll
    for (int s = 0; s < D; ++s) {
      if (!mvalid[s]) { done = true; break; }
      if constexpr (PACK) res_apply_packed<U>(E[s], vs, sp.ebias, carry, aM, aC);
      else {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (plain) res_apply_chunk<T, true>(E[s][u], vs, aM[u & 1], aC[u & 1]);
          else res_apply_chunk<T, false>(E[s][u], vs, aM[u & 1], aC[u & 1]);
        }
      }
      if (mlast[s]) { flush(mitem[s]); carry = -1; }
      produce(s);
    }
    if (done) break;
  }
}

// warps holding the first and the last chunk of item it (w0 > w1: the item is empty)
template <int NT>
__device__ __forceinline__ void res_piece_range(const ResArgs& a, const unsigned int* wb, unsigned int it, int& w0, int& w1) {
  constexpr int NW = NT / 32;
  const unsigned int b = a.sp.itemptr[it], e = a.sp.itemptr[it + 1];
  w0 = 1; w1 = 0;
  if (e > b) {
    w0 = 0;  // largest w with wb[w] <= chunk
#pragma unroll 1
    for (int w = 1; w < NW; ++w) { if (wb[w] <= b) w0 = w; if (wb[w] <= e - 1u) w1 = w; }
  }
}

// sum of the pieces of one row (item it of this CTA, member s) in stream order; wmask: warps that own chunks
__device__ __forceinline__ void res_gather_pieces(const double* ptab, unsigned int isub, bool ptab_shared, unsigned int wmask,
                                                  unsigned int it, int s, int w0, int w1, double& Mv, double& Cv) {
  double m_ = 0.0, c_ = 0.0;
  const double* p = ptab + ((size_t)w0 + (it - isub)) * kPieceVals;
  for (int w = w0; w <= w1; ++w, p += kPieceVals) {
    if (!((wmask >> w) & 1u)) continue;  // warp without chunks
    if (ptab_shared) { m_ += p[s]; c_ += p[4 + s]; }
    else { m_ += __ldcg(p + s); c_ += __ldcg(p + 4 + s); }
  }
  Mv = m_; Cv = c_;
}

// ---------------------------------------------------------------------------------------------------------------
// sweeps over the support of the trial vector (packed layout, one GPU)
// After the first penalty steps almost every entry of a projected candidate is an exact zero, and M_ij w_j with w_j = 0
// adds nothing to row i's sums.  So once the support of the staged candidate w holds at most m / kSupportDiv columns,
// every CTA copies those of its rows' entries whose column is in supp(w) -- S' -- into its own part of a restricted
// copy, and the following evaluations read only that copy as long as supp(w) stays inside S'.  A row is still summed by
// the CTA that owns it, from its own entries: only the terms multiplied by a zero of w are left out, so the sums are
// the same exact products with a different grouping of the terms.  Every CTA stages the same w and so takes the same
// decision without an exchange.
// ---------------------------------------------------------------------------------------------------------------
enum ResSweepKind : int { SW_FULL = 0, SW_REBUILD = 1, SW_RESTRICTED = 2 };

// The staged candidate w (vs, raw) against S' (the CTA's bitmap; have: the restricted copy is valid): restricted if
// supp(w) lies in S', else rebuild if |supp(w)| <= m / kSupportDiv, else full.  A rebuild stores supp(w) as the new S'.
template <int NT>
__device__ int res_support_kind(const ResArgs& a, int bid, const double* vs, bool have, double* red_s, double* fin) {
  constexpr int NW = NT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m = a.m, nwords = (m + 31) >> 5;
  unsigned int* bits = a.rbits + (size_t)bid * nwords;
  int nsup = 0;
  unsigned int outside = 0u;
  for (int g = warp * 32; g < nwords; g += NW * 32) {  // lane l holds word g + l of S'
    const unsigned int mine = (have && g + lane < nwords) ? bits[g + lane] : 0u;
    const int ng = min(32, nwords - g);
#pragma unroll 4
    for (int k = 0; k < ng; ++k) {
      const int j = (g + k) * 32 + lane;
      const unsigned int b = __ballot_sync(0xffffffffu, j < m && vs[j] != 0.0);
      nsup += __popc(b);
      outside |= b & ~__shfl_sync(0xffffffffu, mine, k);
    }
  }
  const double n = res_block_sum<NT>(lane == 0 ? (double)nsup : 0.0, red_s, fin);
  const bool out = __syncthreads_or(outside != 0u) != 0;
  if (have && !out) return SW_RESTRICTED;
  if (!((double)kSupportDiv * n <= (double)m)) return SW_FULL;
  for (int g = warp * 32; g < nwords; g += NW * 32) {
    unsigned int mine = 0u;
    const int ng = min(32, nwords - g);
    for (int k = 0; k < ng; ++k) {
      const int j = (g + k) * 32 + lane;
      const unsigned int b = __ballot_sync(0xffffffffu, j < m && vs[j] != 0.0);
      if (lane == k) mine = b;
    }
    if (g + lane < nwords) bits[g + lane] = mine;
  }
  return SW_REBUILD;
}

// Rebuild: one warp per item of the CTA reads the item's packed entries (columns from the deltas, as in
// res_apply_packed) and appends every entry whose column holds a non-zero of w to its row's slot, in column order; the
// slot is then padded to a whole chunk with (0, column m).  A slot holds at most min(row entries, m / kSupportDiv)
// entries, which res_restrict_cap rounds up to a chunk: it never overflows.
template <int NT>
__device__ void res_restrict_build(const ResArgs& a, int bid, const double* vs) {
  constexpr int NW = NT / 32, RB = 4;  // rounds of 32 chunks in flight per warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int it0 = a.sp.cta_first[bid], it1 = a.sp.cta_first[bid + 1];
  const unsigned int* pw = reinterpret_cast<const unsigned int*>(a.sp.val);
  for (unsigned int it = it0 + warp; it < it1; it += NW) {
    const unsigned int b = a.sp.itemptr[it], e = a.sp.itemptr[it + 1];
    const unsigned int r0 = a.roff[it], slot = r0 + (unsigned int)(lane & 3) * ((a.roff[it + 1] - r0) >> 2);
    int carry = -1;
    unsigned int cnt = 0u;  // entries of the member's row written so far (the same on its 8 lanes)
    for (unsigned int c0 = b; c0 < e; c0 += 32u * RB) {
      Packed4 E[RB];
#pragma unroll
      for (int u = 0; u < RB; ++u) {
        const unsigned int c = c0 + 32u * u + (unsigned int)lane;
        if (c < e) E[u].load(pw, 4ull * c); else E[u].neutral();
      }
#pragma unroll
      for (int u = 0; u < RB; ++u) {
        if (c0 + 32u * u >= e) break;  // warp-uniform
        const unsigned int w4[4] = {E[u].w.x, E[u].w.y, E[u].w.z, E[u].w.w};
        const unsigned int own = pack_delta(w4[0]) + pack_delta(w4[1]) + pack_delta(w4[2]) + pack_delta(w4[3]);
        unsigned int inc = own;
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        int col = carry + (int)(inc - own);
        carry += (int)__shfl_sync(0xffffffffu, inc, 28 + (lane & 3));
        unsigned int keep = 0u;
        int cols[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          col += (int)pack_delta(w4[q]);
          cols[q] = col;
          if ((w4[q] & 0x07800000u) && vs[col] != 0.0) keep |= 1u << q;
        }
        const unsigned int nk = (unsigned int)__popc(keep);
        unsigned int kin = nk;
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, kin, o); if (lane >= o) kin += y; }
        unsigned int at = slot + cnt + (kin - nk);
        cnt += __shfl_sync(0xffffffffu, kin, 28 + (lane & 3));
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (keep & (1u << q)) {
            a.rval[at] = __uint_as_float((w4[q] & 0x07ffffffu) + a.sp.ebias);
            a.rcol[at] = (unsigned short)cols[q];
            ++at;
          }
      }
    }
    if (lane < 4) {  // lane s: member s
      for (unsigned int k = cnt; k & 3u; ++k) { a.rval[slot + k] = 0.0f; a.rcol[slot + k] = (unsigned short)a.m; }
      a.rlen[4u * it + (unsigned int)lane] = cnt;
    }
  }
}

// The split of the restricted sweeps, chosen at the first restricted evaluation after a rebuild: the row slots are cut
// into G x NW contiguous ranges of equal cost, one per warp of the grid, a slot costing its chunks plus kRowCost; range
// k = b NW + w goes to warp w of CTA b and is [t_k, t_{k+1}), t_k = the first slot whose prefix cost reaches k / (G NW)
// of the total.  The rows' owners wrote rlen before the rebuild evaluation's exchange; every CTA reads all of it (L2
// loads: this SM's L1 may still hold an older S') and adds the same integers in the same order, so all CTAs agree on
// every bound without an exchange.  Thread t covers the items [t K, (t + 1) K), four slots each (one 16-byte load).
// Writes the bounds of the CTA's warps to bnd[0..NW].
template <int NT>
__device__ void res_restrict_split(const ResArgs& a, int bid, unsigned int* bnd, unsigned int* red_u) {
  constexpr int NW = NT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned int NI = (unsigned int)a.NI, K = (NI + NT - 1) / NT;
  const unsigned int s = min(NI, threadIdx.x * K), e = min(NI, s + K);
  const uint4* len4 = reinterpret_cast<const uint4*>(a.rlen);
  auto cost = [](unsigned int n) { return ((n + 3u) >> 2) + kRowCost; };
  unsigned int own = 0u;
#pragma unroll 4
  for (unsigned int it = s; it < e; ++it) { const uint4 n = __ldcg(len4 + it); own += cost(n.x) + cost(n.y) + cost(n.z) + cost(n.w); }
  unsigned int inc = own;  // inclusive scan over the warp, then over the warps' totals
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
  __syncthreads();
  if (lane == 31) red_u[warp] = inc;
  for (int k = threadIdx.x; k <= NW; k += NT) bnd[k] = (bid == 0 && k == 0) ? 0u : 4u * NI;  // t_0 = 0; no slot: past the end
  __syncthreads();
  unsigned int before = 0u;
  unsigned long long T = 0ull;
  for (int w = 0; w < NW; ++w) { const unsigned int x = red_u[w]; T += x; if (w < warp) before += x; }
  // slot t is t_k for every k >= 1 with Q(t - 1) GW < k T <= Q(t) GW, Q(t) = the cost of slots 0..t (all positive)
  const unsigned long long GW = (unsigned long long)a.G * NW, k0 = (unsigned long long)bid * NW;
  unsigned long long Q = before + inc - own;
  unsigned long long k = Q * GW / T + 1;  // the first target not reached before this thread's slots
#pragma unroll 4
  for (unsigned int it = s; it < e; ++it) {
    const uint4 n = __ldcg(len4 + it);
    const unsigned int n4[4] = {n.x, n.y, n.z, n.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      Q += cost(n4[q]);
      for (; k * T <= Q * GW; ++k)
        if (k >= k0 && k <= k0 + NW) bnd[k - k0] = 4u * it + (unsigned int)q + 1u;
    }
  }
  __syncthreads();
}

// profile: the entries of the row slots [lo, hi) (returned to thread 0)
template <int NT>
__device__ unsigned int res_prof_slots(const ResArgs& a, unsigned int lo, unsigned int hi, unsigned int* red_u) {
  constexpr int NW = NT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned int sum = 0u;
  for (unsigned int t = lo + threadIdx.x; t < hi; t += NT) sum += __ldcg(a.rlen + t);
  sum = __reduce_add_sync(0xffffffffu, sum);
  __syncthreads();
  if (lane == 0) red_u[warp] = sum;
  __syncthreads();
  unsigned int s = 0u;
  if (threadIdx.x == 0)
    for (int w = 0; w < NW; ++w) s += red_u[w];
  __syncthreads();
  return s;
}

// profile: what res_restrict_split balances, recomputed from rlen and the bounds it wrote.  The costliest range of this
// CTA's warps exceeds the share total / (G NW) by x times the costliest slot; the split keeps x < 1 (a range ends at
// the first slot whose prefix cost reaches the next target).  Raises the CTA's slot 7 to x.
template <int NT>
__device__ void res_prof_split(const ResArgs& a, int bid, const unsigned int* bnd, unsigned int* red_u) {
  constexpr int NW = NT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  auto cost = [&](unsigned int t) { return ((__ldcg(a.rlen + t) + 3u) >> 2) + kRowCost; };
  unsigned int tot = 0u, cmax = 0u, mine = 0u;
  for (unsigned int t = threadIdx.x; t < 4u * (unsigned int)a.NI; t += NT) { const unsigned int c = cost(t); tot += c; cmax = max(cmax, c); }
  for (unsigned int t = bnd[warp] + (unsigned int)lane; t < bnd[warp + 1]; t += 32u) mine += cost(t);  // the warp's range
  tot = __reduce_add_sync(0xffffffffu, tot);
  cmax = __reduce_max_sync(0xffffffffu, cmax);
  mine = __reduce_add_sync(0xffffffffu, mine);
  __syncthreads();
  if (lane == 0) { red_u[3 * warp] = tot; red_u[3 * warp + 1] = cmax; red_u[3 * warp + 2] = mine; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double T = 0.0, cm = 0.0, wm = 0.0;
    for (int w = 0; w < NW; ++w) { T += (double)red_u[3 * w]; cm = fmax(cm, (double)red_u[3 * w + 1]); wm = fmax(wm, (double)red_u[3 * w + 2]); }
    const double GW = (double)a.G * NW;
    a.prof_cta[(size_t)bid * 8 + 7] = fmax(a.prof_cta[(size_t)bid * 8 + 7], (wm * GW - T) / (cm * GW));
  }
  __syncthreads();
}

// The restricted sweep: the calling warp sums the row slots lo, lo + step, ... < hi into their LL cells in rprod, tagged
// ptag.  Lane l takes chunks l, l + 32, ... of a row; RD rounds of RU chunks per lane are in flight, carried on from one
// row to the next.  A row's sums depend on its slot alone, not on which CTA or warp sweeps it.  The slots may have been
// written by another CTA earlier in this launch: L2 loads (ld.global.cg), no ld.global.nc and no L1.
__device__ void res_sweep_restricted(const ResArgs& a, unsigned int lo, unsigned int hi, unsigned int step, const double* vs,
                                     unsigned int ptag) {
  constexpr int RU = 2, RD = 2;
  const int lane = threadIdx.x & 31;
  const int nrow = hi > lo ? (int)((hi - lo + step - 1) / step) : 0;
  for (int rb = 0; rb < nrow; rb += 32) {
    // lane i: slot and padded length of the warp's row rb + i
    const int nb = min(32, nrow - rb);
    unsigned int slot = 0u, len = 0u;
    if (lane < nb) {
      const unsigned int t = lo + step * (unsigned int)(rb + lane), it = t >> 2;
      const unsigned int r0 = a.roff[it];
      slot = r0 + (t & 3u) * ((a.roff[it + 1] - r0) >> 2);
      len = (__ldcg(a.rlen + t) + 3u) & ~3u;
    }
    int ci = 0;             // producer cursor: row of the batch, first entry of its next round
    unsigned int ck = 0u;
    float4 X[RD][RU];
    uint2 K[RD][RU];
    int srow[RD];
    bool slast[RD], sval[RD];
    auto produce = [&](int s) {
      sval[s] = ci < nb;
      if (!sval[s]) return;
      const unsigned int s0 = __shfl_sync(0xffffffffu, slot, ci), n0 = __shfl_sync(0xffffffffu, len, ci);
#pragma unroll
      for (int u = 0; u < RU; ++u) {
        const unsigned int k = ck + 4u * (unsigned int)lane + 128u * u;
        if (k < n0) {
          X[s][u] = __ldcg(reinterpret_cast<const float4*>(a.rval + s0 + k));
          K[s][u] = __ldcg(reinterpret_cast<const uint2*>(a.rcol + s0 + k));
        } else {
          X[s][u] = make_float4(0.f, 0.f, 0.f, 0.f);
          K[s][u] = make_uint2((unsigned int)a.m * 0x10001u, (unsigned int)a.m * 0x10001u);  // column m holds 0.0
        }
      }
      srow[s] = ci;
      slast[s] = ck + 128u * RU >= n0;
      if (slast[s]) { ++ci; ck = 0u; } else ck += 128u * RU;
    };
    double aM[2] = {0.0, 0.0}, aC[2] = {0.0, 0.0};
#pragma unroll
    for (int s = 0; s < RD; ++s) produce(s);
    for (;;) {
      bool done = false;
#pragma unroll
      for (int s = 0; s < RD; ++s) {
        if (!sval[s]) { done = true; break; }
#pragma unroll
        for (int u = 0; u < RU; ++u) {
          const float x4[4] = {X[s][u].x, X[s][u].y, X[s][u].z, X[s][u].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const double v = vs[off_of(K[s][u], q)];
            aM[u & 1] = fma((double)x4[q], v, aM[u & 1]);
            aC[u & 1] += v;
          }
        }
        if (slast[s]) {
          double accM = aM[0] + aM[1], accC = aC[0] + aC[1];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) {
            accM += __shfl_xor_sync(0xffffffffu, accM, o);
            accC += __shfl_xor_sync(0xffffffffu, accC, o);
          }
          if (lane < 2) ll_store(a.rprod + 2ull * (lo + step * (unsigned int)(rb + srow[s])) + lane, lane ? accC : accM, ptag);
          aM[0] = aM[1] = aC[0] = aC[1] = 0.0;
        }
        produce(s);
      }
      if (done) break;
    }
  }
}

// M w, C w of one row slot from its two LL cells (res_sweep_restricted): a cell whose tag is not ptag yet is re-polled;
// one that does not arrive within spin_limit raises the error flag
__device__ __forceinline__ void res_rprod_take(const uint4* p, unsigned int ptag, long long spin_limit, int* errp,
                                               double& Mv, double& Cv) {
  unsigned int lo[2], t1[2], hi[2], t2[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) ll_ld4<false>(p + e, lo[e], t1[e], hi[e], t2[e]);
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    long long t0 = 0;
    while (!(t1[e] == ptag && t2[e] == ptag)) {
      if (t0 == 0) t0 = clock64();
      else if (clock64() - t0 > spin_limit) { atomicExch(errp, 1); break; }
      ll_ld4<false>(p + e, lo[e], t1[e], hi[e], t2[e]);
    }
  }
  Mv = __hiloint2double((int)hi[0], (int)lo[0]);
  Cv = __hiloint2double((int)hi[1], (int)lo[1]);
}

// ---------------------------------------------------------------------------------------------------------------
// device-wide exchange of 8 partial sums: one arrival counter, every CTA reduces the table itself
// ---------------------------------------------------------------------------------------------------------------
template <int NT, bool SHARDED, bool SOLO>
__device__ bool res_exchange(const ResArgs& a, const int bid, const double (&loc)[kRedVals], double (&vals)[kRedVals], int& red_par,
                             unsigned long long& round, unsigned long long& seq, double* red_s, double* fin) {
  int* errp = &a.sb->error;
  ++round; ++seq;
  if constexpr (SOLO) {  // one CTA owns the whole problem: a block reduction is the exchange
    res_publish<NT>(loc, fin + kRedVals, red_s);
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kRedVals; ++q) vals[q] = fin[kRedVals + q];
    __syncthreads();
    return true;
  } else {
    // Every CTA publishes its 8 partial sums as self-validating LL cells {lo, tag, hi, tag} and arrives with one
    // acq_rel atomic; the last arriver releases a flag on another L2 line which the others poll (acquire, back-off).
    // Every CTA then reads the whole table -- a cell whose tag is not this round's is re-polled -- and adds the rows
    // in the same fixed order: no last-arriver serial reduction, no second release hop.
    const int G = a.G;
    uint4* table = a.redll + (size_t)red_par * G * kRedVals;
    const unsigned int rtag = (unsigned int)round;
    {
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
      double t[kRedVals];
#pragma unroll
      for (int q = 0; q < kRedVals; ++q) t[q] = warp_sum(loc[q]);
      __syncthreads();
      if (lane == 0) {
#pragma unroll
        for (int q = 0; q < kRedVals; ++q) red_s[warp * kRedVals + q] = t[q];
      }
      __syncthreads();
      if (threadIdx.x < kRedVals) {
        double sacc = 0.0;
        for (int w = 0; w < NT / 32; ++w) sacc += red_s[w * kRedVals + threadIdx.x];
        ll_store(table + (size_t)bid * kRedVals + threadIdx.x, sacc, rtag);
      }
      if (warp == 0) {
        __syncwarp();
        if (lane == 0) {
          // arrival: one returning relaxed atomic; the LAST arriver publishes the round number in a flag on another
          // L2 line, which the others poll with a back-off (polling the arrival counter itself makes every SM hammer
          // the address the atomics are queued on)
          // acq_rel / release / acquire at gpu scope: the epilogue's PLAIN stores (candidate points of the unsharded
          // solve, read by every CTA when it stages the next trial vector) are ordered before the arrival through the
          // __syncthreads above (causality order) and become visible to whoever observes the flag
          unsigned long long old;
          asm volatile("atom.acq_rel.gpu.global.add.u64 %0, [%1], %2;" : "=l"(old) : "l"(&a.sb->root[0]), "l"(1ULL) : "memory");
          if (old + 1ULL == round * (unsigned long long)G) {
            asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(&a.sb->gen[0]), "l"(round) : "memory");
          } else {
            const long long t0 = clock64();
            unsigned long long seen;
            for (;;) {
              asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(seen) : "l"(&a.sb->gen[0]) : "memory");
              if (seen >= round) break;
              __nanosleep(20);
              if (clock64() - t0 > a.spin_limit) { atomicExch(errp, 1); break; }
            }
          }
        }
      }
      __syncthreads();
    }
    {
      const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
      const int q = threadIdx.x & 7;
      double sacc = 0.0;
      for (int c = threadIdx.x >> 3; c < G; c += NT / 8) {
        const uint4* p = table + (size_t)c * kRedVals + q;
        unsigned lo, t1, hi, t2; long long t0 = 0;
        for (;;) {
          asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(t1), "=r"(hi), "=r"(t2) : "l"(p) : "memory");
          if (t1 == rtag && t2 == rtag) break;
          if (t0 == 0) t0 = clock64();
          else if (clock64() - t0 > a.spin_limit) { atomicExch(errp, 1); break; }
        }
        sacc += __hiloint2double((int)hi, (int)lo);
      }
      sacc += __shfl_xor_sync(0xffffffffu, sacc, 8);
      sacc += __shfl_xor_sync(0xffffffffu, sacc, 16);
      if (lane < kRedVals) red_s[warp * kRedVals + lane] = sacc;
      __syncthreads();
      if (threadIdx.x < kRedVals) {
        double tt = 0.0;
        for (int w = 0; w < NT / 32; ++w) tt += red_s[w * kRedVals + threadIdx.x];
        fin[threadIdx.x] = tt;
      }
      __syncthreads();
    }
    if constexpr (SHARDED) {
      const unsigned int tag = (unsigned int)seq;
      const int t = threadIdx.x;
      if (t < a.world * kRedVals) {
        const int r = t / kRedVals, q = t % kRedVals;
        if (bid == 0 && r != a.rank) ll_store(&a.peer_comm[r]->xred[red_par][a.rank][q], fin[q], tag);
        double x = fin[q];
        if (r != a.rank) {
          unsigned lo, t1, hi, t2; long long t0 = 0;
          const uint4* p = &a.comm->xred[red_par][r][q];
          for (;;) {
            asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(lo), "=r"(t1), "=r"(hi), "=r"(t2) : "l"(p) : "memory");
            if (t1 == tag && t2 == tag) break;
            if (t0 == 0) t0 = clock64();
            else if (clock64() - t0 > a.spin_limit) { atomicExch(errp, 1); break; }
          }
          x = __hiloint2double((int)hi, (int)lo);
        }
        fin[(2 + r) * kRedVals + q] = x;
      }
      __syncthreads();
      if (t < kRedVals) {
        double s = 0.0;
        for (int r = 0; r < a.world; ++r) s += fin[(2 + r) * kRedVals + t];
        fin[kRedVals + t] = s;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < kRedVals; ++q) vals[q] = fin[kRedVals + q];
    } else {
#pragma unroll
      for (int q = 0; q < kRedVals; ++q) vals[q] = fin[q];
    }
    __syncthreads();
    red_par ^= 1;
    return *reinterpret_cast<volatile int*>(errp) == 0;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// the solver body (shared by solver_resident_kernel and the batched kernel)
// ---------------------------------------------------------------------------------------------------------------
template <typename T, int NT, int U, int D, bool SHARDED, bool SOLO, bool COH = false, bool PACK = false, bool RESTRICT = false>
__device__ void res_solve_body(const ResArgs& a, unsigned char* smem) {
  constexpr int NW = NT / 32;
  const int bid = SOLO ? 0 : (int)blockIdx.x;  // CTA index within the problem (batched: one CTA per problem)
  const ResSmem plan = res_smem_plan(a.m, NW, a.pieces_cap, a.state_cap);
  double* vs = reinterpret_cast<double*>(smem);
  double* red_s = reinterpret_cast<double*>(smem + plan.off_red);
  double* fin = reinterpret_cast<double*>(smem + plan.off_fin);
  unsigned int* wb = reinterpret_cast<unsigned int*>(smem + plan.off_wb);
  const SolverParams& P = a.prm;
  int* const errp = &a.sb->error;
  const int m = a.m;
  const long long mp = a.mpad;

  // rows of this CTA: items [it0, it1), four member rows each; thread t serves rows t, t + NT, ... of that list
  const unsigned int it0 = a.sp.cta_first[bid], it1 = a.sp.cta_first[bid + 1];
  const int nrow = (int)(it1 - it0) * 4;
  if (threadIdx.x <= NW) {
    const unsigned int c_lo = a.sp.itemptr[it0], c_hi = a.sp.itemptr[it1];
    wb[threadIdx.x] = res_warp_bound(c_lo, c_hi, threadIdx.x, NW);
  }
  if (threadIdx.x < NW) reinterpret_cast<uint2*>(smem + plan.off_misc)[threadIdx.x] = make_uint2(0u, 0u);
  // bulk-copy staging of the candidate vector (one unsharded problem on the whole GPU only)
  unsigned long long* const sbars = reinterpret_cast<unsigned long long*>(smem + plan.off_sbar);
  unsigned int sphase = 0u;
  constexpr bool stage_bulk = !SHARDED && !SOLO;
  // candidate staged as it is, 1/|w| applied to the row results: whenever a CTA owns fewer rows than the vector has entries
  constexpr bool stage_raw = !SOLO;
  // sweeps over the support of the trial vector: packed copy, one GPU (res_support_kind)
  constexpr bool restrict_ok = RESTRICT && PACK && !SHARDED && !SOLO;
  if constexpr (!SHARDED && !SOLO) {
    if (threadIdx.x < kStageBlocks) mbar_init(&sbars[threadIdx.x], 1);
    fence_mbar_init();
  }
  // the row slots of this CTA's warps in the restricted sweeps, warp w: [rbnd[w], rbnd[w + 1]) (res_restrict_split), and
  // their entries (rbnd[NW + 1]): in the part of fin that only the sharded exchange uses
  static_assert(kMaxPeers * kRedVals * 2 >= kResWarps + 2, "fin holds the restricted split");
  unsigned int* const rbnd = reinterpret_cast<unsigned int*>(fin + 2 * kRedVals);
  if constexpr (restrict_ok)
    if (a.prof_cta && threadIdx.x == 0) { a.prof_cta[(size_t)bid * 8 + 6] = 0.0; a.prof_cta[(size_t)bid * 8 + 7] = -1.0; }
  __syncthreads();

  // piece table and per-row state (u, gradF, Mhat u, Chat u of the current and the next iterate): on chip when the
  // CTA's items / rows fit what the launch granted beyond the plan, else in HBM
  const bool ptab_sh = (it1 - it0) + (unsigned int)NW <= plan.pieces_cap;
  double* const ptab = ptab_sh ? reinterpret_cast<double*>(smem + plan.off_pieces) : a.pieces + (size_t)bid * NW * kPieceVals;
  const unsigned int isub = ptab_sh ? it0 : 0u;
  const bool st_sh = (unsigned int)nrow <= plan.state_cap;
  double* const st_sm = reinterpret_cast<double*>(smem + plan.off_state);
  const unsigned int st_cap = plan.state_cap;
  auto S = [&](int slot, int t_, int i) -> double& {
    return st_sh ? st_sm[(size_t)slot * st_cap + t_] : a.vecs[(size_t)slot * mp + i];
  };
  // per-row descriptors (global row, member, piece range): invariant over the solve, kept on chip with the state
  struct RowDesc { int i; unsigned char s, w0, w1, pad; };
  RowDesc* const desc = reinterpret_cast<RowDesc*>(smem + plan.off_desc);
  unsigned int wmask = 0u;
#pragma unroll 1
  for (int w = 0; w < NW; ++w) wmask |= (wb[w + 1] > wb[w] ? 1u : 0u) << w;
  auto row_of = [&](int t_, int& i, unsigned int& itx, int& sx, int& w0, int& w1) -> bool {
    itx = it0 + (unsigned int)(t_ >> 2);
    if (st_sh) {
      const RowDesc dsc = desc[t_];
      i = dsc.i; sx = dsc.s; w0 = dsc.w0; w1 = dsc.w1;
      return i >= 0;
    }
    sx = t_ & 3;
    const int lr = (int)a.sp.rowid[4u * itx + sx];
    i = a.row0 + lr;
    res_piece_range<NT>(a, wb, itx, w0, w1);
    return lr < a.rows;
  };
  if (st_sh) {
    for (int t_ = threadIdx.x; t_ < nrow; t_ += NT) {
      const unsigned int itx = it0 + (unsigned int)(t_ >> 2);
      const int sx = t_ & 3;
      const int lr = (int)a.sp.rowid[4u * itx + sx];
      int w0, w1;
      res_piece_range<NT>(a, wb, itx, w0, w1);
      RowDesc dsc; dsc.i = lr < a.rows ? a.row0 + lr : -1; dsc.s = (unsigned char)sx; dsc.w0 = (unsigned char)w0; dsc.w1 = (unsigned char)w1; dsc.pad = 0;
      desc[t_] = dsc;
    }
    __syncthreads();
  }
  // candidate trial points: parity par, kind 0 = "accept" (max(v + gradFnew, 0)), 1 = "reject" (max(u + alpha beta gradF, 0))
  auto cand_store = [&](int par, int kind, int i, double v, unsigned int tag) {
    const size_t off = (size_t)(par * 2 + kind) * mp + i;
    if constexpr (SHARDED) {
      ll_store(a.ll + off, v, tag);
      for (int r = 0; r < a.world; ++r)
        if (r != a.rank) ll_store(a.peer_ll[r] + off, v, tag);
    } else {
      a.cand[off] = v;
    }
  };

  double vals[kRedVals], loc[kRedVals];
  long long n_evals = 0, n_inner = 0, n_matvec = 0;
  long long n_sweep[3] = {0, 0, 0};  // line-search evaluations by ResSweepKind
  long long n_fallback = 0;
  double r_entries = 0.0, r_padding = 0.0;
  bool rhave = false;                // the restricted copy holds S'
  bool rsplit = false;               // rbnd holds the split of the current S'
  int skind = SW_FULL;               // sweep of the current evaluation
  int cur = 0, cpar = 0, red_par = 0, status = 0, i_outer = 0;
  double d = 0.0, F = 0.0, sum_cur = 0.0, z = 0.0, sw = 0.0;  // z, sw: |w|^2 and sum(w) of the candidate the next evaluation stages
  unsigned long long round = 0, seq = a.seq0;
  unsigned int ctag = 0u;  // tag under which the candidates of parity cpar were written
  unsigned long long ns_mv = 0, ns_cb = 0, ns_ex = 0, ns_st = 0, tmark = global_ns();
#define RES_LAP(acc) { if (a.prof_laps && threadIdx.x == 0) { const unsigned long long t_ = global_ns(); acc += t_ - tmark; tmark = t_; } }
#define RES_ZERO() _Pragma("unroll") for (int q_ = 0; q_ < kRedVals; ++q_) loc[q_] = 0.0;
#define RES_FOR_ROWS(i, itx, sx)                                                                    \
  for (int t_ = threadIdx.x, i = 0, sx = 0, w0_ = 0, w1_ = 0; t_ < nrow; t_ += NT)                  \
    if (unsigned int itx = 0u; row_of(t_, i, itx, sx, w0_, w1_))
#define RES_EXCHANGE()                                                                              \
  RES_LAP(ns_cb);                                                                                   \
  if (!res_exchange<NT, SHARDED, SOLO>(a, bid, loc, vals, red_par, round, seq, red_s, fin)) { status = 5; goto finish; } \
  RES_LAP(ns_ex);
#define RES_SWEEP()                                                                                 \
  res_sweep<T, NT, U, D, COH, PACK>(a, bid, vs, smem, plan, ptab, isub);                                             \
  ++n_matvec;                                                                                       \
  __syncthreads();                                                                                  \
  RES_LAP(ns_mv);

  // ---- phase 0: u = M u0 + u0 (or u0), squared norm (clipper.cpp:193-198) ---------------------
  {
    if (P.rescale_u0) {
      res_stage<NT, SHARDED>(RS_RAW, m, a.u0, nullptr, 0u, 1.0, vs, red_s, fin, errp, a.spin_limit, bid * 416);
      RES_LAP(ns_st);
      RES_SWEEP();
    }
    RES_ZERO();
    const unsigned int tag = (unsigned int)(seq + 1);
    RES_FOR_ROWS(i, itx, sx) {
      double t = a.u0[i];
      if (P.rescale_u0) {
        double Mv, Cv;
        res_gather_pieces(ptab, isub, ptab_sh, wmask, itx, sx, w0_, w1_, Mv, Cv);
        t = __dadd_rn(Mv, t);
      }
      cand_store(cpar ^ 1, 0, i, t, tag);
      loc[0] += t * t;
    }
    RES_EXCHANGE();
    cpar ^= 1; ctag = tag;
    z = vals[0];
  }
  // ---- phase 1: u /= |u|; Mhat u, Chat u; initial d (clipper.cpp:198-209) ----------------------
  {
    const double sumu = stage_bulk
        ? res_stage_bulk<NT>(RS_DIV, m, a.cand + (size_t)(cpar * 2) * mp, z, vs, sbars, sphase, red_s, fin, errp, bid)
        : res_stage<NT, SHARDED>(RS_DIV, m, a.cand + (size_t)(cpar * 2) * mp,
                                 SHARDED ? a.ll + (size_t)(cpar * 2) * mp : nullptr, ctag, z, vs, red_s, fin,
                                 errp, a.spin_limit, bid * 416);
    RES_LAP(ns_st);
    RES_SWEEP();
    cur = 1;
    sum_cur = sumu;
    RES_ZERO();
    RES_FOR_ROWS(i, itx, sx) {
      double Mv, Cv;
      res_gather_pieces(ptab, isub, ptab_sh, wmask, itx, sx, w0_, w1_, Mv, Cv);
      const double ui = vs[i];
      S(R_U0 + cur, t_, i) = ui; S(R_MV0 + cur, t_, i) = Mv; S(R_CV0 + cur, t_, i) = Cv;
      const double cbu = __dsub_rn(__dsub_rn(__dmul_rn(1.0, sumu), Cv), ui);
      if (cbu > P.eps && ui > P.eps) { loc[0] += 1.0; loc[1] += __dadd_rn(Mv, ui) / cbu; }
    }
    RES_EXCHANGE();
    if (vals[0] > 0.0) d = vals[1] / vals[0];
  }

  // ---- graduated projected gradient ascent (clipper.cpp:218-281) --------------------------------
  for (i_outer = 0; i_outer < P.maxoliters; ++i_outer) {
    // gradF and F of the current u under the current d (clipper.cpp:219-220) + the first trial point max(u + gradF, 0)
    {
      RES_ZERO();
      const unsigned int tag = (unsigned int)(seq + 1);
      RES_FOR_ROWS(i, itx, sx) {
        const double ui = S(R_U0 + cur, t_, i);
        const double g = grad_entry(ui, sum_cur, S(R_MV0 + cur, t_, i), S(R_CV0 + cur, t_, i), d);
        S(R_G0 + cur, t_, i) = g;
        loc[0] += ui * g;
        double w = __dadd_rn(ui, __dmul_rn(1.0, g)); w = (w < 0.0) ? 0.0 : w;
        loc[1] += w * w;
        loc[2] += w;
        cand_store(cpar ^ 1, 0, i, w, tag);
      }
      RES_EXCHANGE();
      cpar ^= 1; ctag = tag;
      F = vals[0]; z = vals[1]; sw = vals[2];
    }
    int ckind = 0;  // which candidate of parity cpar the next evaluation tries
    for (int j = 0; j < P.maxiniters; ++j) {
      double alpha = 1.0;
      double Fnew = 0.0, deltaF = 0.0, du2 = 0.0, zB = 0.0, swB = 0.0, sum_trial = sum_cur;
      const int nxt = cur ^ 1;
      for (int k = 0; k < P.maxlsiters; ++k) {
        // trial point into shared memory, sweep of the CTA's rows
        const size_t coff = (size_t)(cpar * 2 + ckind) * mp;
        // The candidate w is staged as it is (by the copy engine when unsharded); unew = w / |w| (clipper.cpp:237) is applied to
        // the row results instead -- M w, C w and sum(w) are linear in w -- i.e. to this CTA's ~m/G rows rather than to all
        // m entries in every CTA (the divisions were most of what this step cost when every CTA normalised every entry).
        const double nrm_l = sqrt(z), rinv_l = 1.0 / nrm_l;
        const bool lzs = stage_raw && z > 0.0;
        double sumv;
        if (stage_raw) {
          if (stage_bulk) res_stage_bulk<NT>(RS_STEP, m, a.cand + coff, z, vs, sbars, sphase, red_s, fin, errp, bid, true);
          else res_stage<NT, SHARDED>(RS_STEP, m, a.cand + coff, SHARDED ? a.ll + coff : nullptr, ctag, z, vs, red_s, fin, errp,
                                      a.spin_limit, bid * 416, true);
          sumv = lzs ? div_by_invariant(sw, nrm_l, rinv_l) : sw;
        } else {
          sumv = res_stage<NT, SHARDED>(RS_STEP, m, a.cand + coff, SHARDED ? a.ll + coff : nullptr, ctag, z,
                                        vs, red_s, fin, errp, a.spin_limit, bid * 416);
        }
        RES_LAP(ns_st);
        skind = SW_FULL;
        if constexpr (restrict_ok)
          if (a.rval) skind = res_support_kind<NT>(a, bid, vs, rhave, red_s, fin);
        if (skind == SW_FULL) {
          RES_SWEEP();
        } else {
          // a rebuild evaluation is swept by the rows' owners; the restricted evaluations that follow it by the split
          // of the new S', which the owners' rlen gives once the rebuild evaluation's exchange has published it
          unsigned int* const red_u = reinterpret_cast<unsigned int*>(red_s);
          const int warp = threadIdx.x >> 5;
          if (skind == SW_REBUILD) {
            res_restrict_build<NT>(a, bid, vs);
            rhave = true; rsplit = false;
            __syncthreads();
            if (a.prof_cta) {
              const unsigned int n = res_prof_slots<NT>(a, 4u * it0, 4u * it1, red_u);
              if (threadIdx.x == 0) a.prof_cta[(size_t)bid * 8 + 6] += (double)n;
            }
            res_sweep_restricted(a, 4u * it0 + (unsigned int)warp, 4u * it1, (unsigned int)NW, vs, (unsigned int)(round + 1));
          } else {
            if (!rsplit) {
              res_restrict_split<NT>(a, bid, rbnd, red_u);
              rsplit = true;
              if (a.prof_cta) {
                const unsigned int n = res_prof_slots<NT>(a, rbnd[0], rbnd[NW], red_u);
                if (threadIdx.x == 0) rbnd[NW + 1] = n;
                res_prof_split<NT>(a, bid, rbnd, red_u);
              }
            }
            if (a.prof_cta && threadIdx.x == 0) a.prof_cta[(size_t)bid * 8 + 6] += (double)rbnd[NW + 1];
            res_sweep_restricted(a, rbnd[warp], rbnd[warp + 1], 1u, vs, (unsigned int)(round + 1));
          }
          ++n_matvec;
          __syncthreads();
          RES_LAP(ns_mv);
        }
        ++n_sweep[skind];
        if (skind == SW_FULL && rhave) ++n_fallback;
        ++n_evals;
        // per-row epilogue: gradFnew, Fnew, |unew - u|^2 and BOTH possible next trial points
        const double alpha_rej = __dmul_rn(alpha, P.beta);
        RES_ZERO();
        const unsigned int tag = (unsigned int)(seq + 1);
        RES_FOR_ROWS(i, itx, sx) {
          double Mv, Cv;
          if (skind != SW_FULL) {
            // the row's sums, from whichever CTA swept its slot in this evaluation
            const unsigned int t = 4u * itx + (unsigned int)sx, n = a.rlen[t];
            res_rprod_take(a.rprod + 2ull * t, (unsigned int)(round + 1), a.spin_limit, errp, Mv, Cv);
            loc[6] += (double)n; loc[7] += (double)((0u - n) & 3u);
          } else {
            res_gather_pieces(ptab, isub, ptab_sh, wmask, itx, sx, w0_, w1_, Mv, Cv);
          }
          double un = vs[i];
          if (lzs) {
            un = div_by_invariant(un, nrm_l, rinv_l);
            Mv = div_by_invariant(Mv, nrm_l, rinv_l); Cv = div_by_invariant(Cv, nrm_l, rinv_l);
          }
          const double g = grad_entry(un, sumv, Mv, Cv, d);
          S(R_U0 + nxt, t_, i) = un; S(R_G0 + nxt, t_, i) = g; S(R_MV0 + nxt, t_, i) = Mv; S(R_CV0 + nxt, t_, i) = Cv;
          const double uo = S(R_U0 + cur, t_, i), go = S(R_G0 + cur, t_, i);
          loc[0] += un * g;
          const double du = __dsub_rn(un, uo);
          loc[1] += du * du;
          double wa = __dadd_rn(uo, __dmul_rn(alpha_rej, go)); wa = (wa < 0.0) ? 0.0 : wa;
          loc[2] += wa * wa;
          double wb_ = __dadd_rn(un, __dmul_rn(1.0, g)); wb_ = (wb_ < 0.0) ? 0.0 : wb_;
          loc[3] += wb_ * wb_;
          loc[4] += wb_; loc[5] += wa;
          cand_store(cpar ^ 1, 0, i, wb_, tag);
          cand_store(cpar ^ 1, 1, i, wa, tag);
        }
        RES_EXCHANGE();
        cpar ^= 1; ctag = tag;
        // the line-search decision (clipper.cpp:242-251), identical on every CTA / rank
        Fnew = vals[0]; du2 = vals[1]; zB = vals[3]; swB = vals[4];
        r_entries += vals[6]; r_padding += vals[7];
        deltaF = Fnew - F;
        sum_trial = sumv;
        if (deltaF < -P.eps) {
          alpha = alpha_rej;
          if (k + 1 < P.maxlsiters) { z = vals[2]; sw = vals[5]; ckind = 1; continue; }
        }
        break;
      }
      // accept (also when the line search ran out, clipper.cpp:256-258)
      const double deltau = sqrt(du2);
      F = Fnew; cur = nxt; sum_cur = sum_trial; z = zB; sw = swB; ckind = 0;
      ++n_inner;
      if (deltau < P.tol_u || fabs(deltaF) < P.tol_F) break;
    }
    // penalty ramp (clipper.cpp:268-280)
    RES_ZERO();
    RES_FOR_ROWS(i, itx, sx) {
      const double ui = S(R_U0 + cur, t_, i);
      const double cbu = __dsub_rn(__dsub_rn(__dmul_rn(1.0, sum_cur), S(R_CV0 + cur, t_, i)), ui);
      if (cbu > P.eps && ui > P.eps) { loc[0] += 1.0; loc[1] += fabs(__dadd_rn(S(R_MV0 + cur, t_, i), ui) / cbu); }
    }
    RES_EXCHANGE();
    if (vals[0] > 0.0) d += vals[1] / vals[0];
    else break;
  }

  // ---- the final iterate ---------------------------------------------------------------------
  if constexpr (SHARDED) {
    const unsigned int tag = (unsigned int)(seq + 1);
    const size_t off = (size_t)4 * mp;
    RES_FOR_ROWS(i, itx, sx) {
      const double ui = S(R_U0 + cur, t_, i);
      ll_store(a.ll + off + i, ui, tag);
      for (int r = 0; r < a.world; ++r)
        if (r != a.rank) ll_store(a.peer_ll[r] + off + i, ui, tag);
    }
    RES_ZERO();
    RES_EXCHANGE();  // also the last rendez-vous: no rank overwrites a peer's cells while it is still inside this launch
    for (int i = bid * NT + threadIdx.x; i < m; i += a.G * NT) a.u_final[i] = ll_load(a.ll + off + i, tag, errp);
  } else {
    RES_FOR_ROWS(i, itx, sx) { a.u_final[i] = S(R_U0 + cur, t_, i); }
  }

finish:
  if (a.prof_cta && threadIdx.x == 0) {
    a.prof_cta[(size_t)bid * 8 + 0] = (double)ns_mv; a.prof_cta[(size_t)bid * 8 + 1] = (double)ns_cb;
    a.prof_cta[(size_t)bid * 8 + 2] = (double)ns_ex; a.prof_cta[(size_t)bid * 8 + 3] = (double)ns_st;
    a.prof_cta[(size_t)bid * 8 + 4] = (double)(it1 - it0);
    a.prof_cta[(size_t)bid * 8 + 5] = (double)(a.sp.itemptr[it1] - a.sp.itemptr[it0]);
  }
  if (bid == 0 && threadIdx.x == 0) {
    if (*reinterpret_cast<volatile int*>(errp) != 0) status = 5;
    a.out->F = F; a.out->d = d; a.out->ifinal = i_outer; a.out->cur = cur; a.out->status = status;
    a.out->n_evals = n_evals; a.out->n_inner = n_inner; a.out->n_matvec = n_matvec; a.out->seq_end = seq;
    a.out->ns_matvec = ns_mv + ns_st; a.out->ns_combine = ns_cb; a.out->ns_exchange = ns_ex;
    if (restrict_ok && a.sweeps) {
      a.sweeps->full = n_sweep[SW_FULL]; a.sweeps->rebuild = n_sweep[SW_REBUILD]; a.sweeps->restricted = n_sweep[SW_RESTRICTED];
      a.sweeps->entries = (unsigned long long)r_entries; a.sweeps->padding = (unsigned long long)r_padding;
      a.sweeps->fallback = n_fallback;
    }
  }
#undef RES_LAP
#undef RES_ZERO
#undef RES_FOR_ROWS
#undef RES_EXCHANGE
#undef RES_SWEEP
}

// RESTRICT: the instance with sweeps over the support (packed copy on one GPU, larger than L2).  Its own instance
// because the new path costs the kernel registers (spills) that the solves without it should not pay.
template <typename T, bool SHARDED, bool PACK = false, bool RESTRICT = false>
__global__ void __launch_bounds__(ResShape<T, SHARDED>::NT, 1) solver_resident_kernel(ResArgs a) {
  extern __shared__ __align__(128) unsigned char clp_res_smem[];
  using S = ResShape<T, SHARDED>;
  res_solve_body<T, S::NT, S::U, S::D, SHARDED, false, false, PACK, RESTRICT>(a, clp_res_smem);
}

// stand-alone mat-vec on the resident layout: stage v, sweep, per-row epilogue -- one launch, no device-wide barrier.
// S: the ResShape of the handle's solver (the piece table and the warps' start columns are laid out for it)
template <typename T, typename S, bool PACK = false>
__global__ void __launch_bounds__(S::NT, 1) matvec_resident_kernel(ResArgs a, const double* v, double dpen, double* y,
                                                                   double* Mv_out, double* Cv_out) {
  extern __shared__ __align__(128) unsigned char clp_res_smem[];
  unsigned char* smem = clp_res_smem;
  constexpr int NT = S::NT, NW = NT / 32;
  const ResSmem plan = res_smem_plan(a.m, NW, a.pieces_cap, a.state_cap);
  double* vs = reinterpret_cast<double*>(smem);
  double* red_s = reinterpret_cast<double*>(smem + plan.off_red);
  double* fin = reinterpret_cast<double*>(smem + plan.off_fin);
  unsigned int* wb = reinterpret_cast<unsigned int*>(smem + plan.off_wb);
  const int bid = (int)blockIdx.x;
  const unsigned int it0 = a.sp.cta_first[bid], it1 = a.sp.cta_first[bid + 1];
  if (threadIdx.x <= NW) wb[threadIdx.x] = res_warp_bound(a.sp.itemptr[it0], a.sp.itemptr[it1], threadIdx.x, NW);
  if (threadIdx.x < NW) reinterpret_cast<uint2*>(smem + plan.off_misc)[threadIdx.x] = make_uint2(0u, 0u);
  __syncthreads();
  const double sumv = res_stage<NT, false>(RS_RAW, a.m, v, nullptr, 0u, 1.0, vs, red_s, fin, &a.sb->error, a.spin_limit, bid * 416);
  const bool ptab_sh = (it1 - it0) + (unsigned int)NW <= plan.pieces_cap;
  double* const ptab = ptab_sh ? reinterpret_cast<double*>(smem + plan.off_pieces) : a.pieces + (size_t)bid * NW * kPieceVals;
  const unsigned int isub = ptab_sh ? it0 : 0u;
  res_sweep<T, NT, S::U, S::D, false, PACK>(a, bid, vs, smem, plan, ptab, isub);
  __syncthreads();
  const int nrow = (int)(it1 - it0) * 4;
  unsigned int wmask = 0u;
#pragma unroll 1
  for (int w = 0; w < NW; ++w) wmask |= (wb[w + 1] > wb[w] ? 1u : 0u) << w;
  for (int t = threadIdx.x; t < nrow; t += NT) {
    const unsigned int itx = it0 + (unsigned int)(t >> 2);
    const int sx = t & 3;
    const int lr = (int)a.sp.rowid[4u * itx + sx];
    if (lr >= a.rows) continue;
    double Mv, Cv;
    int w0_, w1_;
    res_piece_range<NT>(a, wb, itx, w0_, w1_);
    res_gather_pieces(ptab, isub, ptab_sh, wmask, itx, sx, w0_, w1_, Mv, Cv);
    const int i = a.row0 + lr;
    if (Mv_out) Mv_out[i] = Mv;
    if (Cv_out) Cv_out[i] = Cv;
    if (y) y[i] = grad_entry(vs[i], sumv, Mv, Cv, dpen);
  }
}

// packed layout, once per build: a.wcol[(b * NW + w) * 4 + s] = column of member s's last entry in front of warp w's
// first chunk in CTA b (-1 when the warp starts at an item boundary).  One warp per (CTA, warp).
__global__ void res_warp_cols_kernel(SparseView sp, int G, int NW, int* wcol) {
  const long long gw = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (gw >= (long long)G * NW) return;
  const int b = (int)(gw / NW), w = (int)(gw - (long long)b * NW);
  const unsigned int it0 = sp.cta_first[b], it1 = sp.cta_first[b + 1];
  unsigned int sum = 0u;
  if (it0 < it1) {
    const unsigned int c_lo = sp.itemptr[it0], c_hi = sp.itemptr[it1];
    const unsigned int s0 = res_warp_bound(c_lo, c_hi, w, NW), s1 = res_warp_bound(c_lo, c_hi, w + 1, NW);
    if (s0 < s1) {
      const unsigned int cb = sp.itemptr[res_item_of(sp.itemptr, it0, it1 - 1, s0)];
      const unsigned int* pw = reinterpret_cast<const unsigned int*>(sp.val);
      for (unsigned int c = cb + lane; c < s0; c += 32u) {  // chunk c belongs to member (c - cb) & 3 = lane & 3
        const uint4 q = *reinterpret_cast<const uint4*>(pw + 4ull * c);
        sum += pack_delta(q.x) + pack_delta(q.y) + pack_delta(q.z) + pack_delta(q.w);
      }
    }
  }
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if (lane < 4) wcol[gw * 4 + lane] = (int)sum - 1;
}

// packed layout on one GPU, once per build: roff[it] = entries of item it's four row slots in the restricted copy
// (res_restrict_cap), roff[NI] = 0; the exclusive scan of clp_sparse.cuh then turns them into slot offsets
__global__ void res_restrict_caps_kernel(const unsigned int* itemptr, int NI, int m, unsigned int* roff) {
  const int it = blockIdx.x * blockDim.x + threadIdx.x;
  if (it < NI) roff[it] = 4u * res_restrict_cap(itemptr[it + 1] - itemptr[it], m);  // a member's entries = the item's chunks
  else if (it == NI) roff[it] = 0u;
}

}  // namespace clp
