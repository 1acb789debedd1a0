// clp_sdp.cuh -- the semidefinite relaxation of solveAsMSRCSDR / sdp::solve (ref clipper.cpp:101-113, sdp.cpp:88-296)
// on the device: clp_sdp_solve (one problem, the handle's matrix) and clp_batch_sdp_matrices (many, given as CSC).
//
//     maximise <M, X>  subject to  X PSD, tr X = 1,  X_ij = 0 where C_ij = 0,  X_ij >= 0 where C_ij != 0
//
// Two-block ADMM on X in the spectraplex {X PSD, tr X = 1} and Z in P = {Z symmetric, 0 off the pattern of C, >= 0 on
// it} (the pattern includes the diagonal).  State Z = I/m, U = 0, rho = 1, V = I; iteration k:
//   1. W = (Z - U) + M / rho
//   2. (lambda, V) = eig(W): B = V' W V from the previous V, then cyclic Jacobi sweeps on B, every rotation applied to V
//   3. p = projection of lambda onto the unit simplex
//   4. X = V diag(p) V' over the columns with p > 0 (formed entry by entry inside step 5, never stored)
//   5. Z+ = max(X + U, 0) on the pattern, 0 off it; U = (U + X) - Z+
//   6. r_p = max|X - Z+|, r_d = rho max|Z+ - Z|; Z = Z+
//   7. stop (converged) when r_p <= ea + er max(|X|max, |Z|max), r_d <= ea + er |rho U|max and, evaluated only then,
//      |value - bound| <= ea + er max(|value|, |bound|): value = <M, X>, bound = lambda_max(M - Y~), Y = rho U,
//      Y~ = min(Y, 0) on the pattern and Y off it (the Lagrange dual of the splitting: an upper bound for any U)
//   8. every 10th iteration: r_p > 10 r_d -> rho *= 2, U /= 2; r_d > 10 r_p -> rho /= 2, U *= 2 (rho U is unchanged)
//   9. stop (timed out) once the time limit has passed
// tests/sdr_oracle.py states the same steps in numpy with eigh in place of Jacobi.
//
// One CTA of kSdpThreads owns one problem (m <= kSdpMaxM); a persistent grid draws problems from a counter.  B lives in
// shared memory (n x (n + 1) doubles, n = m rounded up to 4: 132 KB at m = 128); M, Z, U, V, the product buffer T and
// the pattern live in the CTA's scratch slot.  Jacobi: parallel cyclic order (round-robin tournament of m rounded up to
// even players, m - 1 or m rounds of disjoint pairs per sweep), rotation of Golub & Van Loan's sym.schur2; rows of B,
// barrier, columns of B and V, and the rotated pair set to exactly 0.  Sweeps stop when the off-diagonal mass is below
// 2^-52 of |B|_F (Jacobi converges quadratically: at most one sweep past the point where it matters), at most
// kSdpMaxSweeps per eigendecomposition.  Every reduction has a fixed order: a repeated call is bit-identical.
#pragma once

namespace clp {

constexpr int kSdpMaxM = 128;
constexpr int kSdpThreads = 256;
constexpr int kSdpMaxSweeps = 40;

struct SdpOut {  // per problem
  double value, bound, res_pri, res_dual, rho;
  long long n_sweeps;
  unsigned long long ns_proj;  // steps 2-3 and the selection of the columns of step 4
  int iters, converged, timed_out, pad_;
};

// The problem table is clp_batch_matrix.cuh's BatchMatProblem: m, the CSC offsets (batches) and u_off, which places the
// problem's p and evec1 (m doubles each) in p_out and e_out.  X (m x m) goes to x_out + x_off[p].
struct SdpArgs {
  const BatchMatProblem* prob;
  const long long* x_off;
  int nprob;
  const void* store; long long ld;  // the handle's dense store (element type of the kernel); null: CSC inputs below
  const long long* colptr; const int* rowidx; const double* val;
  double* x_out; double* p_out; double* e_out;
  SdpOut* out;
  int* next;
  int* flags;
  unsigned char* scratch; size_t scratch_stride;
  int max_m;
  int max_iters;
  double eps_abs, eps_rel;
  unsigned long long limit_ns;  // 0: no time limit; else measured from the start of the launch
};

__host__ __device__ inline int sdp_n(int m) { return (m + 3) & ~3; }
// per-CTA scratch: M | Z | U | V | T (n x n doubles each, V and T column-major) | pattern (n x n bytes) | fp32 store
// of a CSC problem (m rows of 128)
__host__ __device__ inline size_t sdp_slot_bytes(int max_m) {
  const size_t n = (size_t)sdp_n(max_m);
  return 5 * n * n * 8 + ((n * n + 15) & ~(size_t)15) + (size_t)max_m * 128 * 4;
}
// shared memory: B | lam | p | sorted | cos | sin | reduction table
__host__ __device__ inline size_t sdp_smem_bytes(int max_m) {
  const size_t n = (size_t)sdp_n(max_m);
  return (n * (n + 1) + 3 * n + n + kSdpThreads / 32) * 8 + (n / 2) * 2 * 4 + n * 4;
}

__device__ __forceinline__ double sdp_block_sum(double v, double* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
#pragma unroll
  for (int w = 0; w < kSdpThreads / 32; ++w) r += red[w];
  __syncthreads();
  return r;
}
__device__ __forceinline__ double sdp_block_max(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double r = 0.0;
#pragma unroll
  for (int w = 0; w < kSdpThreads / 32; ++w) r = fmax(r, red[w]);
  __syncthreads();
  return r;
}

struct SdpShared {
  double* B; double* lam; double* pr; double* srt; double* cs; double* sn; double* red;
  int* pp; int* qq; int* act;
};

// Jacobi sweeps on B (m x m of stride ldb); every rotation is also applied to the columns of Vc (column-major, n x n)
// when Vc is given.  Returns the number of sweeps; leaves the eigenvalues on the diagonal of B.
__device__ int sdp_jacobi(const SdpShared& s, int m, int n, int ldb, double* Vc) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int mp = m + (m & 1), half = mp / 2, N = mp - 1;
  double* B = s.B;
  int sweeps = 0;
  for (; sweeps < kSdpMaxSweeps; ++sweeps) {
    double off = 0.0, fro = 0.0;
    for (int e = tid; e < m * m; e += kSdpThreads) {
      const int i = e / m, j = e - i * m;
      const double b = B[i * ldb + j];
      fro += b * b;
      if (i != j) off += b * b;
    }
    off = sdp_block_sum(off, s.red);
    fro = sdp_block_sum(fro, s.red);
    if (off <= 0x1p-104 * fro) break;
    for (int r = 0; r < N; ++r) {
      if (tid < half) {  // tournament pairing of round r: (mp - 1, r), ((r + t) mod N, (r - t) mod N)
        int a = tid == 0 ? mp - 1 : (r + tid) % N, b = tid == 0 ? r : (r - tid + N) % N;
        if (a > b) { const int x = a; a = b; b = x; }
        double c = 1.0, sv = 0.0;
        if (b < m) {
          const double apq = B[a * ldb + b];
          if (apq != 0.0) {
            const double tau = (B[b * ldb + b] - B[a * ldb + a]) / (2.0 * apq);
            const double t = (tau >= 0.0 ? 1.0 : -1.0) / (fabs(tau) + sqrt(1.0 + tau * tau));
            c = 1.0 / sqrt(1.0 + t * t);
            sv = t * c;
          }
        }
        s.pp[tid] = a; s.qq[tid] = b; s.cs[tid] = c; s.sn[tid] = sv;
      }
      __syncthreads();
      for (int k = warp; k < half; k += kSdpThreads / 32) {  // rows p, q of B <- J' B
        const double sv = s.sn[k];
        if (sv == 0.0) continue;
        const double c = s.cs[k];
        double* rp = B + s.pp[k] * ldb;
        double* rq = B + s.qq[k] * ldb;
        for (int j = lane; j < m; j += 32) {
          const double bp = rp[j], bq = rq[j];
          rp[j] = c * bp - sv * bq;
          rq[j] = sv * bp + c * bq;
        }
      }
      __syncthreads();
      for (int k = warp; k < half; k += kSdpThreads / 32) {  // columns p, q of B and V <- . J
        const double sv = s.sn[k];
        if (sv == 0.0) continue;
        const double c = s.cs[k];
        const int p = s.pp[k], q = s.qq[k];
        for (int i = lane; i < m; i += 32) {
          const double bp = B[i * ldb + p], bq = B[i * ldb + q];
          B[i * ldb + p] = c * bp - sv * bq;
          B[i * ldb + q] = sv * bp + c * bq;
        }
        if (Vc) {
          double* vp = Vc + (size_t)p * n;
          double* vq = Vc + (size_t)q * n;
          for (int i = lane; i < m; i += 32) {
            const double ap = vp[i], aq = vq[i];
            vp[i] = c * ap - sv * aq;
            vq[i] = sv * ap + c * aq;
          }
        }
        __syncwarp();
        if (lane == 0) { B[p * ldb + q] = 0.0; B[q * ldb + p] = 0.0; }
      }
      __syncthreads();
    }
  }
  return sweeps;
}

// bound = lambda_max(M - Y~), Y = rho U: Y~ = min(Y, 0) on the pattern, Y off it.  Cold Jacobi without vectors.
__device__ double sdp_bound(const SdpShared& s, int m, int n, int ldb, const double* Mg, const double* U,
                            const unsigned char* pat, double rho, long long* sweeps) {
  for (int e = threadIdx.x; e < m * m; e += kSdpThreads) {
    const int i = e / m, j = e - i * m;
    const double y = rho * U[i * n + j];
    s.B[i * ldb + j] = Mg[i * n + j] - (pat[i * n + j] ? fmin(y, 0.0) : y);
  }
  __syncthreads();
  *sweeps += sdp_jacobi(s, m, n, ldb, nullptr);
  double mx = -INFINITY;
  for (int i = 0; i < m; ++i) mx = fmax(mx, s.B[i * ldb + i]);
  __syncthreads();
  return mx;
}

// x_ij of X = V diag(p) V' over the active columns (ascending), symmetric to the bit
__device__ __forceinline__ double sdp_x(const SdpShared& s, int nact, const double* Vc, int n, int i, int j) {
  double x = 0.0;
  for (int a = 0; a < nact; ++a) {
    const int k = s.act[a];
    x += s.pr[k] * (Vc[(size_t)k * n + i] * Vc[(size_t)k * n + j]);
  }
  return x;
}

template <typename T>
__device__ void sdp_load(const T* st, long long ld, int m, int n, double* Mg, unsigned char* pat) {
  for (int e = threadIdx.x; e < n * n; e += kSdpThreads) {
    const int i = e / n, j = e - i * n;
    double a = 0.0; bool c = false;
    if (i < m && j < m) {
      if (i == j) { a = 1.0; c = true; }
      else decode(st[(size_t)i * ld + j], a, c);
    }
    Mg[e] = a; pat[e] = c ? 1 : 0;
  }
}

template <typename T>
__global__ void __launch_bounds__(kSdpThreads, 1) sdp_solve_kernel(SdpArgs a) {
  extern __shared__ __align__(16) unsigned char clp_sdp_smem[];
  __shared__ int s_p, s_nact, s_stop, s_gap;
  __shared__ unsigned long long s_t0;
  const int tid = threadIdx.x;
  const int nmax = sdp_n(a.max_m);
  SdpShared s;
  s.B = reinterpret_cast<double*>(clp_sdp_smem);
  s.lam = s.B + nmax * (nmax + 1);
  s.pr = s.lam + nmax; s.srt = s.pr + nmax; s.cs = s.srt + nmax; s.sn = s.cs + nmax / 2;
  s.red = s.sn + nmax / 2;
  s.pp = reinterpret_cast<int*>(s.red + kSdpThreads / 32); s.qq = s.pp + nmax / 2; s.act = s.qq + nmax / 2;
  unsigned char* slot = a.scratch + (size_t)blockIdx.x * a.scratch_stride;
  const size_t nn = (size_t)nmax * nmax;
  double* Mg = reinterpret_cast<double*>(slot);
  double* Z = Mg + nn; double* U = Z + nn; double* Vc = U + nn; double* Tc = Vc + nn;
  unsigned char* pat = reinterpret_cast<unsigned char*>(Tc + nn);
  float* st = reinterpret_cast<float*>(pat + ((nn + 15) & ~(size_t)15));
  if (tid == 0) s_t0 = global_ns();

  for (;;) {
    __syncthreads();
    if (tid == 0) s_p = atomicAdd(a.next, 1);
    __syncthreads();
    const int p = s_p;
    if (p >= a.nprob) break;
    const BatchMatProblem P = a.prob[p];
    const int m = P.m, n = sdp_n(m), ldb = n + 1;

    // ---- the matrices: the handle's store, or a CSC problem scattered into an fp32 store exactly as
    //      clp_set_sparse_upper builds the handle's (neutral fill, M entries, then C bits)
    if (a.store) {
      sdp_load<T>(reinterpret_cast<const T*>(a.store), a.ld, m, n, Mg, pat);
    } else {
      for (int e = tid; e < m * 128; e += kSdpThreads) st[e] = -0.0f;
      __syncthreads();
      for (int pass = 0; pass < 2; ++pass) {
        const long long* cp = a.colptr + (pass ? P.cpC_off : P.cpM_off);
        const long long e0 = pass ? P.eC_off : P.eM_off;
        for (int j = tid >> 5; j < m; j += kSdpThreads / 32)
          for (long long q = cp[j] + (tid & 31); q < cp[j + 1]; q += 32) {
            if (pass == 0) scatter_csc_M_entry<float>(a.rowidx[e0 + q], j, a.val + e0 + q, st, 128, 0, m, a.flags);
            else scatter_csc_C_entry<float>(a.rowidx[e0 + q], j, a.val + e0 + q, st, 128, 0, m, a.flags);
          }
        __syncthreads();
      }
      sdp_load<float>(st, 128, m, n, Mg, pat);
    }
    for (int e = tid; e < n * n; e += kSdpThreads) {
      const int i = e / n, j = e - i * n;
      Z[e] = (i == j && i < m) ? 1.0 / m : 0.0;
      U[e] = 0.0;
      Vc[e] = i == j ? 1.0 : 0.0;
    }
    __syncthreads();

    double rho = 1.0, value = 0.0, bound = 0.0, r_p = 0.0, r_d = 0.0;
    bool have_bound = false;
    int converged = 0, timed_out = 0, k = 0, nact = 0;
    long long sweeps = 0;
    unsigned long long ns_proj = 0;
    while (k < a.max_iters) {
      ++k;
      // ---- 1. W into B
      for (int e = tid; e < n * n; e += kSdpThreads) {
        const int i = e / n, j = e - i * n;
        s.B[i * ldb + j] = (Z[e] - U[e]) + Mg[e] / rho;
      }
      __syncthreads();
      const unsigned long long t_eig = global_ns();
      // ---- 2. B = V' W V (T = W V, then B = V' T; 4 x 4 register tiles, k ascending), then Jacobi
      const int nt = n / 4;
      for (int t = tid; t < nt * nt; t += kSdpThreads) {
        const int i0 = (t / nt) * 4, j0 = (t % nt) * 4;
        double acc[4][4] = {};
        for (int l = 0; l < n; ++l) {
          double w[4], v[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) { w[r] = s.B[(i0 + r) * ldb + l]; v[r] = Vc[(size_t)(j0 + r) * n + l]; }
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = fma(w[r], v[c], acc[r][c]);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) Tc[(size_t)(j0 + c) * n + i0 + r] = acc[r][c];
      }
      __syncthreads();
      for (int t = tid; t < nt * nt; t += kSdpThreads) {
        const int i0 = (t / nt) * 4, j0 = (t % nt) * 4;
        double acc[4][4] = {};
        for (int l = 0; l < n; ++l) {
          double vi[4], tj[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) { vi[r] = Vc[(size_t)(i0 + r) * n + l]; tj[r] = Tc[(size_t)(j0 + r) * n + l]; }
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = fma(vi[r], tj[c], acc[r][c]);
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) s.B[(i0 + r) * ldb + j0 + c] = acc[r][c];
      }
      __syncthreads();
      sweeps += sdp_jacobi(s, m, n, ldb, Vc);
      // ---- 3. p = projection of the eigenvalues onto the simplex (sorted by rank, prefix sums in order)
      for (int i = tid; i < m; i += kSdpThreads) s.lam[i] = s.B[i * ldb + i];
      __syncthreads();
      for (int i = tid; i < m; i += kSdpThreads) {
        const double li = s.lam[i];
        int rank = 0;
        for (int j = 0; j < m; ++j) rank += (s.lam[j] > li || (s.lam[j] == li && j < i)) ? 1 : 0;
        s.srt[rank] = li;
      }
      __syncthreads();
      if (tid == 0) {
        double cs = 0.0, tau = 0.0;
        for (int j = 0; j < m; ++j) {
          cs += s.srt[j];
          const double t = (cs - 1.0) / (j + 1);
          if (s.srt[j] - t > 0) tau = t;
        }
        int na = 0;
        for (int i = 0; i < m; ++i) {
          const double pi = fmax(s.lam[i] - tau, 0.0);
          s.pr[i] = pi;
          if (pi > 0.0) s.act[na++] = i;
        }
        s_nact = na;
      }
      __syncthreads();
      nact = s_nact;
      ns_proj += global_ns() - t_eig;
      // ---- 4-6. X entry by entry, Z+, U, residuals, <M, X>
      double rp = 0.0, rd = 0.0, xm = 0.0, zm = 0.0, um = 0.0, val = 0.0;
      for (int e = tid; e < m * m; e += kSdpThreads) {
        const int i = e / m, j = e - i * m, f = i * n + j;
        const double x = sdp_x(s, nact, Vc, n, i, j);
        const double z0 = Z[f], u = U[f];
        const double zn = pat[f] ? fmax(x + u, 0.0) : 0.0;
        const double un = (u + x) - zn;
        rp = fmax(rp, fabs(x - zn)); rd = fmax(rd, fabs(zn - z0));
        xm = fmax(xm, fabs(x)); zm = fmax(zm, fabs(zn)); um = fmax(um, fabs(un));
        val += Mg[f] * x;
        Z[f] = zn; U[f] = un;
      }
      r_p = sdp_block_max(rp, s.red);
      r_d = rho * sdp_block_max(rd, s.red);
      xm = sdp_block_max(xm, s.red); zm = sdp_block_max(zm, s.red); um = sdp_block_max(um, s.red);
      value = sdp_block_sum(val, s.red);
      // ---- 7. stopping tests; the bound only when both residual tests pass
      have_bound = false;
      if (r_p <= a.eps_abs + a.eps_rel * fmax(xm, zm) && r_d <= a.eps_abs + a.eps_rel * rho * um) {
        bound = sdp_bound(s, m, n, ldb, Mg, U, pat, rho, &sweeps);
        have_bound = true;
        if (fabs(value - bound) <= a.eps_abs + a.eps_rel * fmax(fabs(value), fabs(bound))) { converged = 1; break; }
      }
      // ---- 8. rebalance rho (rho U, and with it the bound, is unchanged)
      if (k % 10 == 0) {
        double f = 1.0;
        if (r_p > 10.0 * r_d) { rho *= 2.0; f = 0.5; }
        else if (r_d > 10.0 * r_p) { rho *= 0.5; f = 2.0; }
        if (f != 1.0)
          for (int e = tid; e < n * n; e += kSdpThreads) U[e] *= f;
      }
      // ---- 9. time limit, decided once for the CTA
      if (a.limit_ns) {
        if (tid == 0) s_stop = global_ns() - s_t0 >= a.limit_ns;
        __syncthreads();
        if (s_stop) { timed_out = 1; break; }
      }
      __syncthreads();
    }
    __syncthreads();
    if (!have_bound) bound = sdp_bound(s, m, n, ldb, Mg, U, pat, rho, &sweeps);

    // ---- outputs of the last iterate: X, p by index, evec1 = column of the largest p, largest |entry| positive
    double* X = a.x_out + a.x_off[p];
    for (int e = tid; e < m * m; e += kSdpThreads) {
      const int i = e / m, j = e - i * m;
      X[(size_t)j * m + i] = sdp_x(s, nact, Vc, n, i, j);
    }
    if (tid == 0) {
      int top = 0;
      for (int i = 1; i < m; ++i) if (s.pr[i] > s.pr[top]) top = i;
      int big = 0;
      const double* v = Vc + (size_t)top * n;
      for (int i = 1; i < m; ++i) if (fabs(v[i]) > fabs(v[big])) big = i;
      s_gap = (v[big] < 0.0) ? 1 : 0;
      s_nact = top;
    }
    __syncthreads();
    {
      const double* v = Vc + (size_t)s_nact * n;
      const double sg = s_gap ? -1.0 : 1.0;
      for (int i = tid; i < m; i += kSdpThreads) {
        a.p_out[P.u_off + i] = s.pr[i];
        a.e_out[P.u_off + i] = sg * v[i];
      }
    }
    if (tid == 0) {
      SdpOut o;
      o.value = value; o.bound = bound; o.res_pri = r_p; o.res_dual = r_d; o.rho = rho;
      o.n_sweeps = sweeps; o.ns_proj = ns_proj;
      o.iters = k; o.converged = converged; o.timed_out = timed_out; o.pad_ = 0;
      a.out[p] = o;
    }
  }
}

}  // namespace clp
