// clp_transform.cuh -- the rigid transform that aligns selected associations (clp_estimate_transform*, DESIGN §3
// "Rigid transform").  Every call gathers the k used pairs of each problem into one packed fp64 list on the device,
// then tf_estimate_kernel<D> runs one CTA of kTfThreads per problem: the means, H, the d x d solve in one thread and the
// residual sum.  The CTA shape and every summation order are fixed, so a problem's result is the same bits whatever
// batch it sits in and whichever entry gathered it.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace clp {

constexpr int kTfThreads = 256;
constexpr int kTfWarps = kTfThreads / 32;
constexpr int kTfMaxSweeps = 32;   // one-sided Jacobi sweeps of the d x d solve (3 x 3 converges in about 6)
constexpr double kTfOrthoTol = 1e-15;  // columns count as orthogonal when |g_i . g_j| <= this * |g_i| |g_j|
constexpr double kTfGapTol = 1e-12;    // CLP_TF_DEGENERATE when gap <= this * sv[0]
// status codes, as CLP_TF_* in include/clipper_b200.h
constexpr int kTfOk = 0, kTfEmpty = 1, kTfDegenerate = 2, kTfNonfinite = 3;

// Problem p: its k pairs at pairs[off ..]: coordinate c of a_i at off + c k + i, of b_i at off + (d + c) k + i.  The
// device gather also reads its rows from rows[rows_off ..] (rows_off < 0: rows 0 .. k-1) and the sizes of its inputs.
struct TfProb {
  long long off, k, rows_off;
  long long n1, n2, m;  // m == 0: the all-to-all hypothesis, row r is (r / n2, r mod n2)
};

// what the estimate writes per problem and the host reads back; T column-major (d+1) x (d+1)
struct TfOut {
  double T[16];
  double rmse, sv[3], gap;
  int status, pad;
};

// ---- gather of the caller's strided tensors (clp_*estimate_transform_dev) -----------------------------------------
// The lowest problem with an association index out of range is kept in *bad as (kBatchBadIndex << 32 | ~p), the key
// batch_stage_points_kernel uses; nothing is written for a bad pair.
struct TfGatherArgs {
  const TfProb* prob; int nprob, d;
  const double* D1; long long s1[3];  // coordinate c of point j of problem p: D1[p s1[0] + c s1[1] + j s1[2]]
  const double* D2; long long s2[3];
  const int* A; long long sa[3];      // A(r, c): A[p sa[0] + r sa[1] + c sa[2]]; NULL: all-to-all everywhere
  const int* rows;
  double* pairs;
  unsigned long long* bad;
};

__global__ void __launch_bounds__(kTfThreads) tf_gather_kernel(TfGatherArgs g) {
  const long long t0 = (long long)blockIdx.x * kTfThreads + threadIdx.x, step = (long long)gridDim.x * kTfThreads;
  const int d = g.d;
  for (int p = blockIdx.y; p < g.nprob; p += gridDim.y) {
    const TfProb P = g.prob[p];
    int bad = 0;
    for (long long i = t0; i < P.k; i += step) {
      const long long r = P.rows_off >= 0 ? (long long)g.rows[P.rows_off + i] : i;
      long long i1, i2;
      if (!g.A || P.m == 0) {
        i1 = r / P.n2; i2 = r - i1 * P.n2;
      } else {
        const int* a = g.A + p * g.sa[0] + r * g.sa[1];
        i1 = a[0]; i2 = a[g.sa[2]];
        if (i1 < 0 || i1 >= P.n1 || i2 < 0 || i2 >= P.n2) { bad = 1; continue; }
      }
      for (int c = 0; c < d; ++c) {
        g.pairs[P.off + c * P.k + i] = g.D1[p * g.s1[0] + c * g.s1[1] + i1 * g.s1[2]];
        g.pairs[P.off + (d + c) * P.k + i] = g.D2[p * g.s2[0] + c * g.s2[1] + i2 * g.s2[2]];
      }
    }
    if (__syncthreads_or(bad) && threadIdx.x == 0)
      atomicMax(g.bad, (3ULL << 32) | (0xffffffffu - (unsigned int)p));  // 3: kBatchBadIndex (clp_batch.cuh)
  }
}

// ---- the estimate ----------------------------------------------------------------------------------------------------
// Sums of NV values over the CTA: each thread's strided partials, a butterfly over the warp (every lane ends with the
// same bits: IEEE addition commutes), then warps 0 .. kTfWarps-1 in order.  Every thread returns the totals.
template <int NV>
__device__ __forceinline__ void tf_block_sum(double (&v)[NV], double* red) {
#pragma unroll
  for (int j = 0; j < NV; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_xor_sync(0xffffffffu, v[j], o);
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < NV; ++j) red[w * NV + j] = v[j];
  __syncthreads();
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    double s = red[j];
    for (int q = 1; q < kTfWarps; ++q) s += red[q * NV + j];
    v[j] = s;
  }
  __syncthreads();
}

// Compensated sums (pass 1, the means): s + c carries the exact sum of what was added to within about one rounding
// of the result, whatever the order, so the means of a batch of 10^5 points do not depend on how they were split.
__device__ __forceinline__ void tf_two_sum(double& s, double& c, double y) {
  const double t = s + y, bp = t - s;
  c += (s - (t - bp)) + (y - bp);
  s = t;
}

template <int NV>
__device__ __forceinline__ void tf_block_sum2(double (&s)[NV], double (&c)[NV], double* red) {
#pragma unroll
  for (int j = 0; j < NV; ++j)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double so = __shfl_xor_sync(0xffffffffu, s[j], o), co = __shfl_xor_sync(0xffffffffu, c[j], o);
      // the same bits on both lanes: the lower lane's pair is always the first operand
      const bool lo = (threadIdx.x & o) == 0;
      double a = lo ? s[j] : so, ca = lo ? c[j] : co;
      tf_two_sum(a, ca, lo ? so : s[j]);
      s[j] = a; c[j] = ca + (lo ? co : c[j]);
    }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int j = 0; j < NV; ++j) { red[w * 2 * NV + j] = s[j]; red[w * 2 * NV + NV + j] = c[j]; }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < NV; ++j) {
    double a = red[j], ca = red[NV + j];
    for (int q = 1; q < kTfWarps; ++q) { tf_two_sum(a, ca, red[q * 2 * NV + j]); ca += red[q * 2 * NV + NV + j]; }
    s[j] = a + ca;
  }
  __syncthreads();
}

// a unit vector orthogonal to the unit vector u (3-D): the axis where u is smallest, minus its projection on u
__device__ __forceinline__ void tf_perp3(const double* u, double* w) {
  const int k = fabs(u[1]) < fabs(u[0]) ? (fabs(u[2]) < fabs(u[1]) ? 2 : 1) : (fabs(u[2]) < fabs(u[0]) ? 2 : 0);
  const double uk = k == 0 ? u[0] : k == 1 ? u[1] : u[2];
  double n2 = 0.0;
#pragma unroll
  for (int r = 0; r < 3; ++r) { w[r] = (r == k ? 1.0 : 0.0) - uk * u[r]; n2 += w[r] * w[r]; }
  const double s = 1.0 / sqrt(n2);
#pragma unroll
  for (int r = 0; r < 3; ++r) w[r] *= s;
}

// The d x d solve, one thread.  H is scaled by a power of two (exact) and orthogonalised by one-sided Jacobi: G = H V
// with orthogonal columns, V a product of plane rotations (at most kTfMaxSweeps sweeps).  The singular values are the
// column norms, sorted descending (ties keep column order).  With u0, u1 the unit columns of the two largest (u1 taken orthogonal to u0,
// or completed when it vanishes) and v0, v1 the matching columns of V, the proper rotation that maximises tr(R' H) is
//   d = 3: R = u0 v0' + u1 v1' + (u0 x u1)(v0 x v1')'       d = 2: R = u0 v0' + u0p v0p'  (xp: x turned by +90 degrees)
// which is U diag(1, .., 1, det U det V) V' (Umeyama) written without the smallest singular vectors.  H = 0 gives R = I.
template <int D>
__device__ int tf_solve(const double (&H)[D][D], double (&R)[D][D], double* sv, double* gap) {
  double mx = 0.0;
#pragma unroll
  for (int r = 0; r < D; ++r)
#pragma unroll
    for (int c = 0; c < D; ++c) mx = fmax(mx, fabs(H[r][c]));
#pragma unroll
  for (int r = 0; r < D; ++r)
#pragma unroll
    for (int c = 0; c < D; ++c) R[r][c] = r == c ? 1.0 : 0.0;
  sv[0] = sv[1] = sv[2] = 0.0;
  *gap = 0.0;
  if (mx == 0.0) return kTfDegenerate;
  int e = 0;
  frexp(mx, &e);
  double G[D][D], V[D][D];
#pragma unroll
  for (int r = 0; r < D; ++r)
#pragma unroll
    for (int c = 0; c < D; ++c) { G[r][c] = ldexp(H[r][c], -e); V[r][c] = r == c ? 1.0 : 0.0; }
  const double detH = D == 2 ? G[0][0] * G[1][1] - G[0][1] * G[1][0]
                             : G[0][0] * (G[1][1] * G[2][2] - G[1][2] * G[2][1]) -
                               G[0][1] * (G[1][0] * G[2][2] - G[1][2] * G[2][0]) +
                               G[0][2] * (G[1][0] * G[2][1] - G[1][1] * G[2][0]);
  for (int sweep = 0; sweep < kTfMaxSweeps; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int i = 0; i < D - 1; ++i)
#pragma unroll
      for (int j = i + 1; j < D; ++j) {
        double al = 0.0, be = 0.0, ga = 0.0;
#pragma unroll
        for (int r = 0; r < D; ++r) { al += G[r][i] * G[r][i]; be += G[r][j] * G[r][j]; ga += G[r][i] * G[r][j]; }
        if (!(fabs(ga) > kTfOrthoTol * sqrt(al) * sqrt(be))) continue;
        rotated = true;
        const double ze = (be - al) / (2.0 * ga);
        const double t = copysign(1.0, ze) / (fabs(ze) + hypot(1.0, ze));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
        for (int r = 0; r < D; ++r) {
          const double gi = G[r][i], gj = G[r][j];
          G[r][i] = c * gi - s * gj; G[r][j] = s * gi + c * gj;
          const double vi = V[r][i], vj = V[r][j];
          V[r][i] = c * vi - s * vj; V[r][j] = s * vi + c * vj;
        }
      }
    if (!rotated) break;
  }
  // rank of each column: the number of columns before it in descending order of norm (ties: the lower index first)
  double sg[D];
#pragma unroll
  for (int c = 0; c < D; ++c) {
    double n2 = 0.0;
#pragma unroll
    for (int r = 0; r < D; ++r) n2 += G[r][c] * G[r][c];
    sg[c] = sqrt(n2);
  }
  double u0[3] = {0.0, 0.0, 0.0}, v0[3] = {0.0, 0.0, 0.0}, u1[3] = {0.0, 0.0, 0.0}, v1[3] = {0.0, 0.0, 0.0}, s0 = 0.0;
#pragma unroll
  for (int c = 0; c < D; ++c) {
    int rank = 0;
#pragma unroll
    for (int q = 0; q < D; ++q) rank += (sg[q] > sg[c] || (sg[q] == sg[c] && q < c)) ? 1 : 0;
#pragma unroll
    for (int q = 0; q < D; ++q)
      if (rank == q) sv[q] = ldexp(sg[c], e);
    if (rank == 0) {
      s0 = sg[c];
#pragma unroll
      for (int r = 0; r < D; ++r) { u0[r] = G[r][c]; v0[r] = V[r][c]; }
    }
    if (rank == 1)
#pragma unroll
      for (int r = 0; r < D; ++r) { u1[r] = G[r][c]; v1[r] = V[r][c]; }
  }
  *gap = sv[D - 2] + (detH < 0.0 ? -sv[D - 1] : sv[D - 1]);
  if (sv[0] == 0.0) return kTfDegenerate;
#pragma unroll
  for (int r = 0; r < D; ++r) u0[r] /= s0;
  if (D == 2) {
    const double u0p[2] = {-u0[1], u0[0]}, v0p[2] = {-v0[1], v0[0]};
#pragma unroll
    for (int r = 0; r < D; ++r)
#pragma unroll
      for (int c = 0; c < D; ++c) R[r][c] = u0[r] * v0[c] + u0p[r] * v0p[c];
  } else {
    double pr = 0.0, n2 = 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) pr += u0[r] * u1[r];
#pragma unroll
    for (int r = 0; r < 3; ++r) { u1[r] -= pr * u0[r]; n2 += u1[r] * u1[r]; }
    if (n2 > 1e-300) {  // the scaled H has entries in [0.5, 1): below this u1 carries no direction worth keeping
      const double s = 1.0 / sqrt(n2);
#pragma unroll
      for (int r = 0; r < 3; ++r) u1[r] *= s;
    } else {
      tf_perp3(u0, u1);
    }
    const double u2[3] = {u0[1] * u1[2] - u0[2] * u1[1], u0[2] * u1[0] - u0[0] * u1[2], u0[0] * u1[1] - u0[1] * u1[0]};
    const double v2[3] = {v0[1] * v1[2] - v0[2] * v1[1], v0[2] * v1[0] - v0[0] * v1[2], v0[0] * v1[1] - v0[1] * v1[0]};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) R[r][c] = u0[r] * v0[c] + u1[r] * v1[c] + u2[r] * v2[c];
  }
  return *gap > kTfGapTol * sv[0] ? kTfOk : kTfDegenerate;
}

struct TfEstimateArgs {
  const TfProb* prob; int nprob;
  const double* pairs;
  TfOut* out;
  double* T_dev; long long ts[3];  // nullable: entry (r, c) of problem p's T also at T_dev[p ts[0] + r ts[1] + c ts[2]]
  const unsigned long long* bad;   // a gather found a bad index: nothing is written
};

template <int D>
__global__ void __launch_bounds__(kTfThreads) tf_estimate_kernel(TfEstimateArgs g) {
  constexpr int E = D + 1;
  __shared__ double red[kTfWarps * (D * D > 4 * D ? D * D : 4 * D)];
  __shared__ double sh[D * D + D];  // R | t from the solving thread
  if (*g.bad) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (int p = blockIdx.x; p < g.nprob; p += gridDim.x) {
    const TfProb P = g.prob[p];
    const long long k = P.k;
    const double* a = g.pairs + P.off;
    const double* b = a + (long long)D * k;
    // pass 1: the means, and whether every used coordinate is finite.  The sums are of x - x0, x0 the first pair's
    // coordinate: far from the origin (an offset of 10^3 on a unit spread) the terms stay at the spread's scale (the
    // subtraction is exact when x and x0 are within a factor 2), and the sums are compensated.
    double s[2 * D], sc[2 * D], x0[2 * D];
    int bad = 0;
#pragma unroll
    for (int c = 0; c < 2 * D; ++c) { s[c] = 0.0; sc[c] = 0.0; x0[c] = k > 0 ? a[c * k] : 0.0; }
    for (long long i = threadIdx.x; i < k; i += kTfThreads)
#pragma unroll
      for (int c = 0; c < 2 * D; ++c) {
        const double x = a[c * k + i];
        tf_two_sum(s[c], sc[c], x - x0[c]);
        bad |= !isfinite(x);
      }
    bad = __syncthreads_or(bad);
    tf_block_sum2<2 * D>(s, sc, red);
    double mu[2 * D];
#pragma unroll
    for (int c = 0; c < 2 * D; ++c) mu[c] = x0[c] + s[c] / (double)k;
    // pass 2: H = sum (b_i - mu_b)(a_i - mu_a)'
    double h[D * D];
#pragma unroll
    for (int c = 0; c < D * D; ++c) h[c] = 0.0;
    if (k > 0 && !bad)
      for (long long i = threadIdx.x; i < k; i += kTfThreads) {
        double x[D], y[D];
#pragma unroll
        for (int c = 0; c < D; ++c) { x[c] = a[c * k + i] - mu[c]; y[c] = b[c * k + i] - mu[D + c]; }
#pragma unroll
        for (int r = 0; r < D; ++r)
#pragma unroll
          for (int c = 0; c < D; ++c) h[r * D + c] += y[r] * x[c];
      }
    tf_block_sum<D * D>(h, red);
    // the solve, one thread; every status but NONFINITE leaves a proper rotation in R
    int status = kTfEmpty;
    double R[D][D], sv[3] = {0.0, 0.0, 0.0}, gap = 0.0;
    if (threadIdx.x == 0) {
      if (k > 0 && !bad) {
        double H[D][D];
        bool fin = true;
#pragma unroll
        for (int r = 0; r < D; ++r)
#pragma unroll
          for (int c = 0; c < D; ++c) { H[r][c] = h[r * D + c]; fin = fin && isfinite(H[r][c]); }
        if (fin) status = tf_solve<D>(H, R, sv, &gap);
        else status = kTfNonfinite;  // finite coordinates whose sums overflow
      } else if (k > 0) {
        status = kTfNonfinite;
      }
      if (status == kTfEmpty) {
#pragma unroll
        for (int r = 0; r < D; ++r)
#pragma unroll
          for (int c = 0; c < D; ++c) R[r][c] = r == c ? 1.0 : 0.0;
      }
      if (status == kTfNonfinite) {
#pragma unroll
        for (int r = 0; r < D; ++r)
#pragma unroll
          for (int c = 0; c < D; ++c) R[r][c] = nan;
        sv[0] = sv[1] = sv[2] = gap = nan;
      }
#pragma unroll
      for (int r = 0; r < D; ++r) {
        double t = mu[D + r];
#pragma unroll
        for (int c = 0; c < D; ++c) { sh[r * D + c] = R[r][c]; t -= R[r][c] * mu[c]; }
        sh[D * D + r] = status == kTfEmpty ? 0.0 : t;
      }
    }
    __syncthreads();
    double Rs[D * D];
#pragma unroll
    for (int c = 0; c < D * D; ++c) Rs[c] = sh[c];
    // pass 3: the residuals, as R (a_i - mu_a) - (b_i - mu_b)
    double q[1] = {0.0};
    if (k > 0 && !bad)
      for (long long i = threadIdx.x; i < k; i += kTfThreads) {
        double x[D];
#pragma unroll
        for (int c = 0; c < D; ++c) x[c] = a[c * k + i] - mu[c];
#pragma unroll
        for (int r = 0; r < D; ++r) {
          double z = -(b[r * k + i] - mu[D + r]);
#pragma unroll
          for (int c = 0; c < D; ++c) z += Rs[r * D + c] * x[c];
          q[0] += z * z;
        }
      }
    tf_block_sum<1>(q, red);
    if (threadIdx.x == 0) {
      TfOut& o = g.out[p];
#pragma unroll
      for (int c = 0; c < 16; ++c) o.T[c] = 0.0;
#pragma unroll
      for (int r = 0; r < D; ++r) {
#pragma unroll
        for (int c = 0; c < D; ++c) o.T[c * E + r] = sh[r * D + c];
        o.T[D * E + r] = sh[D * D + r];
      }
      o.T[D * E + D] = 1.0;
      o.rmse = status == kTfEmpty ? 0.0 : status == kTfNonfinite ? nan : sqrt(q[0] / (double)k);
      o.sv[0] = sv[0]; o.sv[1] = sv[1]; o.sv[2] = sv[2]; o.gap = gap;
      o.status = status; o.pad = 0;
      if (g.T_dev)
        for (int r = 0; r < E; ++r)
          for (int c = 0; c < E; ++c) g.T_dev[p * g.ts[0] + r * g.ts[1] + c * g.ts[2]] = o.T[c * E + r];
    }
    __syncthreads();  // sh is rewritten by the next problem's solve
  }
}

}  // namespace clp
