// clp_score_tile.cuh -- the unscreened scoring kernel (K1), its batched form for caller's invariants, and what they
// depend on.
//
// This header has no includes: nvcc compiles it inside clp_kernels.cuh, and the library embeds its text and compiles it
// again with NVRTC at run time, followed by a caller's CUDA-source invariant (KIND 2: clp_score_custom, and
// batch_score_custom_kernel for clp_batch_*_custom).  Both compilers therefore see the same kernel text.
#pragma once

// KIND 2: the pairwise invariant a caller supplies as CUDA source (clp_score_custom), defined after this header in the
// NVRTC translation unit.  Called with i < j: ai, aj = D1 columns of associations i, j; bi, bj = D2 columns; d doubles
// each; prm = the caller's parameters in device memory.
__device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj, int d,
                                const double* prm);

namespace clp {

constexpr int kThreads = 256;          // threads per CTA everywhere
constexpr int kWarps = kThreads / 32;  // 8
constexpr int kRowsPerWarp = 4;        // register blocking of the mat-vec (rows per warp)
constexpr int kRowTile = kWarps * kRowsPerWarp;  // 32 rows per CTA item

// element -> (|s| as double, C bit)
__device__ __forceinline__ void decode(float s, double& a, bool& c) {
  a = (double)fabsf(s);
  c = __float_as_int(s) >= 0;
}
__device__ __forceinline__ void decode(double s, double& a, bool& c) {
  a = fabs(s);
  c = __double2hiint(s) >= 0;
}
template <typename T> __device__ __forceinline__ T encode(double mval, bool cbit);
template <> __device__ __forceinline__ float encode<float>(double mval, bool cbit) {
  const float a = fabsf((float)mval);
  return cbit ? a : -a;
}
template <> __device__ __forceinline__ double encode<double>(double mval, bool cbit) {
  const double a = fabs(mval);
  return cbit ? a : -a;
}
template <typename T> __device__ __forceinline__ bool is_neutral(T s);
template <> __device__ __forceinline__ bool is_neutral<float>(float s) { return __float_as_uint(s) == 0x80000000u; }
template <> __device__ __forceinline__ bool is_neutral<double>(double s) {
  return (unsigned long long)__double_as_longlong(s) == 0x8000000000000000ULL;
}

struct ScoreArgs {
  const double* E1;  // [m][d] endpoint in data set 1 of association i  (D1.col(A(i,0)))
  const double* E2;  // [m][d] endpoint in data set 2                   (D2.col(A(i,1)))
  const int* A0;     // A(:,0)
  const int* A1;     // A(:,1)
  void* M;           // T [rows_pad][ld]
  long long ld;
  int m;
  int row0;          // first global row stored here (row-block sharding)
  int rows;          // number of real local rows
  int rows_pad;
  int d;             // runtime dimension (generic path)
  double p0, p1, p2, p3;  // sigma,epsilon,mindist | sigp,epsp,sign,epsn
  double affinityeps;
  // fp32 screening (score_tile_kernel_runs): positions of both endpoints as float4 and the largest |coordinate|
  const float4* F1;  // [m] (x, y, z, 0) of E1
  const float4* F2;  // [m]
  const unsigned int* scale_bits;  // float bits of max |position coordinate| over E1 and E2 (written by the gather kernel)
  // optional by-product (score_tile_kernel_runs): kept entries per (column segment, local row), the first pass of the
  // compact-copy build (clp_sparse.cuh); zeroed by the host, += by the kernel
  unsigned int* cnt;  // [NSEG][rows_pad + 1] or null
  int W;              // segment width (multiple of 128)
  // optional with cnt (whole-row layout, packed candidate): per local row a bitmap of the aligned 16-column windows that
  // hold a kept entry ([rows_pad][wwords], zeroed by the host, |= by the kernel) and the kept exponent range (SyncBlock::expo)
  unsigned int* win;
  int wwords;
  unsigned int* expo;
  unsigned int* next_unit;  // screened kernel: work-unit counter, zeroed by the host (SyncBlock::score_next)
  const double* prm;        // KIND 2: the caller's parameters (device memory, up to 16 doubles); null for the built-ins
};

template <int D>
__device__ __forceinline__ double point_dist(const double* a, const double* b, int d_rt) {
  double s = 0.0;
  if (D > 0) {
#pragma unroll
    for (int q = 0; q < D; ++q) { const double t = __dsub_rn(a[q], b[q]); s = __dadd_rn(s, __dmul_rn(t, t)); }
  } else {
    for (int q = 0; q < d_rt; ++q) { const double t = __dsub_rn(a[q], b[q]); s = __dadd_rn(s, __dmul_rn(t, t)); }
  }
  return __dsqrt_rn(s);
}

// EuclideanDistance::operator()  (ref euclidean_distance.cpp:13-31), same operation order as
// the oracle, no FMA contraction in the distance / exponent argument.
__device__ __forceinline__ double euclid_score(double l1, double l2, double sigma, double epsilon,
                                               double mindist) {
  if (mindist > 0 && (l1 < mindist || l2 < mindist)) return 0.0;
  const double c = fabs(__dsub_rn(l1, l2));
  if (!(c < epsilon)) return 0.0;
  const double arg = __ddiv_rn(__dmul_rn(__dmul_rn(-0.5, c), c), __dmul_rn(sigma, sigma));
  return exp(arg);
}

// PointNormalDistance::operator()  (ref pointnormal_distance.cpp:13-35). acos is NOT clamped:
// |dot|>1 gives NaN, both comparisons are false, the score is 0.
__device__ __forceinline__ double pointnormal_score(double l1, double l2, double dot1, double dot2,
                                                    double sigp, double epsp, double sign, double epsn) {
  const double alpha1 = acos(dot1);
  const double alpha2 = acos(dot2);
  const double dp = fabs(__dsub_rn(l1, l2));
  const double dn = fabs(__dsub_rn(alpha1, alpha2));
  if (dp < epsp && dn < epsn) {
    const double sp = exp(__ddiv_rn(__dmul_rn(__dmul_rn(-0.5, dp), dp), __dmul_rn(sigp, sigp)));
    const double sn = exp(__ddiv_rn(__dmul_rn(__dmul_rn(-0.5, dn), dn), __dmul_rn(sign, sign)));
    return __dmul_rn(sp, sn);
  }
  return 0.0;
}

// A pair enters M and C iff its score exceeds affinityeps and is not 0: the reference writes scr > affinityeps into a
// dense M and takes M.sparseView() (exact zeros dropped) as M and its pattern as C (ref clipper.cpp:53-64), so a pair
// that scores exactly 0 is never in C, whatever the sign of affinityeps.  A positive score that fp32 storage rounds to
// +0.0 stays in C (M = 0, C = 1), as in the reference's fp64 M.
__device__ __forceinline__ bool keep_score(double scr, double affinityeps) {
  return scr > affinityeps && scr != 0.0;
}

template <typename T> struct Quad;
template <> struct Quad<float> {
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <> struct Quad<double> {
  static __device__ __forceinline__ void store(double* p, const double* v) {
    reinterpret_cast<double2*>(p)[0] = make_double2(v[0], v[1]);
    reinterpret_cast<double2*>(p)[1] = make_double2(v[2], v[3]);
  }
};

// One CTA = a 32-row x 128-column tile of the padded dense matrix; warp w owns 4 rows, lane l
// owns 4 consecutive columns -> every row is written as 512 B (float) of consecutive float4.
// KIND 0: EuclideanDistance with compile-time dimension D (D==0: runtime d). KIND 1: PointNormal.
// KIND 2: the caller's clp_invariant (dimension D, or runtime d when D == 0), always called with i < j: a pair (i, j)
// with j < i passes its arguments as (j, i), so the stored matrix is symmetric even when the function is not.
// MIRROR (unsharded handles): the score is symmetric in (i,j) bit for bit, so only tiles that touch the
// upper triangle are computed; every value s(i,j), i<j, is stored at [i][j] (row-wise float4) and mirrored
// to [j][i] (the lane's 4 rows of one column are 16 contiguous bytes of row j).  Halves the fp64 work.
// This is the unscreened kernel (fp64 storage, or a dimension without an fp32 screen); fp32 storage with
// d = 2, 3 or PointNormal runs score_tile_kernel_runs (clp_kernels.cuh).
template <typename T, int KIND, int D, bool MIRROR>
__global__ void __launch_bounds__(kThreads) score_tile_kernel(ScoreArgs a) {
  constexpr int DD = (KIND == 1) ? 6 : D;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = blockIdx.x * 128 + lane * 4;
  const int lr0 = blockIdx.y * kRowTile + warp * kRowsPerWarp;  // local row
  if (MIRROR && (int)(blockIdx.x * 128 + 127) < (int)(blockIdx.y * kRowTile)) return;  // tile entirely below the diagonal
  T* Mbase = reinterpret_cast<T*>(a.M);
  const int dd = (DD > 0) ? DD : a.d;

  T out[kRowsPerWarp][4];
#pragma unroll
  for (int q = 0; q < kRowsPerWarp; ++q)
#pragma unroll
    for (int e = 0; e < 4; ++e) out[q][e] = encode<T>(0.0, false);

  // row endpoints are warp-uniform: fetched through the read-only path as broadcasts
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int j = c0 + e;
    if (j >= a.m) continue;
    if (MIRROR && j <= a.row0 + lr0) continue;  // column not right of any of this thread's rows
    const int aj0 = __ldg(a.A0 + j), aj1 = __ldg(a.A1 + j);
    double e1j[DD > 0 ? DD : 1], e2j[DD > 0 ? DD : 1];
    if (DD > 0) {
#pragma unroll
      for (int q = 0; q < DD; ++q) { e1j[q] = __ldg(a.E1 + (size_t)j * DD + q); e2j[q] = __ldg(a.E2 + (size_t)j * DD + q); }
    }
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q) {
      const int li = lr0 + q;
      const int i = a.row0 + li;
      if (li >= a.rows || i == j) continue;
      if (MIRROR && j < i) continue;  // lower triangle: written as the mirror of (j,i)
      const int ai0 = __ldg(a.A0 + i), ai1 = __ldg(a.A1 + i);
      if (ai0 == aj0 || ai1 == aj1) continue;  // distinctness (ref clipper.cpp:35-38)
      double scr;
      if (DD > 0) {
        double e1i[DD > 0 ? DD : 1], e2i[DD > 0 ? DD : 1];
#pragma unroll
        for (int t = 0; t < DD; ++t) { e1i[t] = __ldg(a.E1 + (size_t)i * DD + t); e2i[t] = __ldg(a.E2 + (size_t)i * DD + t); }
        if constexpr (KIND == 0) {
          const double l1 = point_dist<DD>(e1i, e1j, 0), l2 = point_dist<DD>(e2i, e2j, 0);
          scr = euclid_score(l1, l2, a.p0, a.p1, a.p2);
        } else if constexpr (KIND == 2) {
          scr = (i < j) ? clp_invariant(e1i, e1j, e2i, e2j, DD, a.prm) : clp_invariant(e1j, e1i, e2j, e2i, DD, a.prm);
        } else {
          const double l1 = point_dist<3>(e1i, e1j, 0), l2 = point_dist<3>(e2i, e2j, 0);
          const double dot1 = __dadd_rn(__dadd_rn(__dmul_rn(e1i[3], e1j[3]), __dmul_rn(e1i[4], e1j[4])), __dmul_rn(e1i[5], e1j[5]));
          const double dot2 = __dadd_rn(__dadd_rn(__dmul_rn(e2i[3], e2j[3]), __dmul_rn(e2i[4], e2j[4])), __dmul_rn(e2i[5], e2j[5]));
          scr = pointnormal_score(l1, l2, dot1, dot2, a.p0, a.p1, a.p2, a.p3);
        }
      } else if constexpr (KIND == 2) {
        const int lo = (i < j) ? i : j, hi = (i < j) ? j : i;
        scr = clp_invariant(a.E1 + (size_t)lo * dd, a.E1 + (size_t)hi * dd, a.E2 + (size_t)lo * dd, a.E2 + (size_t)hi * dd,
                            dd, a.prm);
      } else {
        const double l1 = point_dist<0>(a.E1 + (size_t)i * dd, a.E1 + (size_t)j * dd, dd);
        const double l2 = point_dist<0>(a.E2 + (size_t)i * dd, a.E2 + (size_t)j * dd, dd);
        scr = euclid_score(l1, l2, a.p0, a.p1, a.p2);
      }
      if (keep_score(scr, a.affinityeps)) out[q][e] = encode<T>(scr, true);
    }
  }
  if (!MIRROR) {
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q) {
      const int li = lr0 + q;
      if (li < a.rows_pad && c0 < a.ld) Quad<T>::store(Mbase + (size_t)li * a.ld + c0, out[q]);
    }
    return;
  }
  // MIRROR: row0 == 0 and rows == m.  Row-wise stores of the part right of the diagonal (and the diagonal itself) ...
  const int r0 = lr0;
#pragma unroll
  for (int q = 0; q < kRowsPerWarp; ++q) {
    const int i = r0 + q;
    if (i >= a.rows_pad || c0 >= a.ld) continue;
    if (c0 > i) Quad<T>::store(Mbase + (size_t)i * a.ld + c0, out[q]);
    else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (c0 + e >= i) Mbase[(size_t)i * a.ld + c0 + e] = out[q][e];
    }
  }
  // ... and the mirror image: column j of this thread's 4 rows is 4 consecutive elements of row j
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int j = c0 + e;
    if (j >= a.rows_pad) continue;
    T col[4] = {out[0][e], out[1][e], out[2][e], out[3][e]};
    if (r0 + 3 < j && r0 + 3 < a.ld) Quad<T>::store(Mbase + (size_t)j * a.ld + r0, col);
    else {
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q)
        if (r0 + q < j && r0 + q < a.ld) Mbase[(size_t)j * a.ld + r0 + q] = col[q];
    }
  }
}

// ---- batches scored with a caller's invariant (clp_batch_solve_custom, clp_batch_max_clique_custom) ---------------------
struct BatchProblem {       // device array, one per problem; offsets into the concatenated input / output arrays
  long long d1_off, d2_off; // in doubles
  long long a_off;          // in int32 (column-major m x 2), -1: all-to-all hypothesis (utils.h:61-71)
  long long u_off;          // in doubles: u0 in, final iterate out
  int n1, n2, m, pad_;
};

// One round of such a batch: problems [first, first + count), problem first + k in scratch slot k.  batch_gather_kernel
// (clp_batch.cuh) lays out each slot's endpoints and associations as gather_endpoints_kernel does for a handle, then
// batch_score_custom_kernel scores them into the slot's fp32 matrix (rows_pad x ld, ld = round_up(m, 128), rows_pad =
// round_up(m, 4): the layout of batch_score_pairs), which the nvcc-built solve or clique kernel reads next.
struct BatchScoreArgs {
  const BatchProblem* prob;
  const long long* units;   // [nprob + 1] running count of the problems' work units (batch_tile_units)
  int first, count;
  const double* D1; const double* D2; const int* A;  // the batch's concatenated inputs
  unsigned char* scratch; size_t stride;             // slot k at scratch + k * stride
  size_t e1, e2, a, mat;    // byte offsets of the endpoint, association and matrix regions in a slot
  int d;
  double affinityeps;
  const double* prm;        // the caller's parameters (device memory)
  int* error;               // set to 2 by the gather for an association index out of range
};

// work units of an m-association problem: the 32 x 128 tiles of score_tile that touch the upper triangle, row tile by
// row tile (row tile by holds column tiles by / 4 .. ld / 128 - 1)
__host__ __device__ inline long long batch_tile_units(int m) {
  const int nct = (m + 127) / 128, nrt = (m + kRowTile - 1) / kRowTile;
  long long u = 0;
  for (int by = 0; by < nrt; ++by) u += nct - by * kRowTile / 128;
  return u;
}

// One CTA per work unit of the round, over the whole grid.  A unit is the tile (bx, by) of problem p that
// score_tile_kernel<float, 2, D, true> runs for it on an fp32 handle, and its body is that kernel's for KIND 2 and
// MIRROR: the same loads, calls with i < j, storage rule and stores, row-wise right of the diagonal and mirrored below
// it.  So problem p's matrix holds the handle's bits.
template <int D>
__global__ void __launch_bounds__(kThreads) batch_score_custom_kernel(BatchScoreArgs b) {
  const long long u = b.units[b.first] + blockIdx.x;
  int p = b.first, hi = b.first + b.count - 1;  // the problem whose units hold u (every problem has at least one)
  while (p < hi) {
    const int mid = (p + hi + 1) >> 1;
    if (b.units[mid] <= u) p = mid; else hi = mid - 1;
  }
  const int m = b.prob[p].m, nct = (m + 127) / 128;
  const int ld = nct * 128, rows_pad = (m + 3) / 4 * 4;
  long long t = u - b.units[p];
  int by = 0;
  while (t >= nct - by * kRowTile / 128) { t -= nct - by * kRowTile / 128; ++by; }
  const int bx = by * kRowTile / 128 + (int)t;
  unsigned char* sc = b.scratch + (size_t)(p - b.first) * b.stride;
  const double* E1 = reinterpret_cast<const double*>(sc + b.e1);
  const double* E2 = reinterpret_cast<const double*>(sc + b.e2);
  const int* A0 = reinterpret_cast<const int*>(sc + b.a);
  const int* A1 = A0 + m;
  float* Mbase = reinterpret_cast<float*>(sc + b.mat);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c0 = bx * 128 + lane * 4;
  const int r0 = by * kRowTile + warp * kRowsPerWarp;
  const int dd = (D > 0) ? D : b.d;

  float out[kRowsPerWarp][4];
#pragma unroll
  for (int q = 0; q < kRowsPerWarp; ++q)
#pragma unroll
    for (int e = 0; e < 4; ++e) out[q][e] = encode<float>(0.0, false);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int j = c0 + e;
    if (j >= m || j <= r0) continue;  // column not right of any of this thread's rows
    const int aj0 = __ldg(A0 + j), aj1 = __ldg(A1 + j);
    double e1j[D > 0 ? D : 1], e2j[D > 0 ? D : 1];
    if (D > 0) {
#pragma unroll
      for (int q = 0; q < D; ++q) { e1j[q] = __ldg(E1 + (size_t)j * D + q); e2j[q] = __ldg(E2 + (size_t)j * D + q); }
    }
#pragma unroll
    for (int q = 0; q < kRowsPerWarp; ++q) {
      const int i = r0 + q;
      if (i >= m || i >= j) continue;  // the lower triangle is written as the mirror of (j, i)
      const int ai0 = __ldg(A0 + i), ai1 = __ldg(A1 + i);
      if (ai0 == aj0 || ai1 == aj1) continue;  // distinctness (ref clipper.cpp:35-38)
      double scr;
      if (D > 0) {
        double e1i[D > 0 ? D : 1], e2i[D > 0 ? D : 1];
#pragma unroll
        for (int s = 0; s < D; ++s) { e1i[s] = __ldg(E1 + (size_t)i * D + s); e2i[s] = __ldg(E2 + (size_t)i * D + s); }
        scr = clp_invariant(e1i, e1j, e2i, e2j, D, b.prm);
      } else {
        scr = clp_invariant(E1 + (size_t)i * dd, E1 + (size_t)j * dd, E2 + (size_t)i * dd, E2 + (size_t)j * dd, dd, b.prm);
      }
      if (keep_score(scr, b.affinityeps)) out[q][e] = encode<float>(scr, true);
    }
  }
  // row-wise stores of the part right of the diagonal (and the diagonal itself) ...
#pragma unroll
  for (int q = 0; q < kRowsPerWarp; ++q) {
    const int i = r0 + q;
    if (i >= rows_pad || c0 >= ld) continue;
    if (c0 > i) Quad<float>::store(Mbase + (size_t)i * ld + c0, out[q]);
    else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (c0 + e >= i) Mbase[(size_t)i * ld + c0 + e] = out[q][e];
    }
  }
  // ... and the mirror image: column j of this thread's 4 rows is 4 consecutive elements of row j
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int j = c0 + e;
    if (j >= rows_pad) continue;
    float col[4] = {out[0][e], out[1][e], out[2][e], out[3][e]};
    if (r0 + 3 < j && r0 + 3 < ld) Quad<float>::store(Mbase + (size_t)j * ld + r0, col);
    else {
#pragma unroll
      for (int q = 0; q < kRowsPerWarp; ++q)
        if (r0 + q < j && r0 + q < ld) Mbase[(size_t)j * ld + r0 + q] = col[q];
    }
  }
}

}  // namespace clp
