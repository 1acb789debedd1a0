// clp_knn.cuh -- putative associations by exact k-nearest-neighbour matching on the device (the generator of the
// reference's benchmark, benchmarks/bm_utils.cpp:147-232 distance_based_correspondences): clp_correspondences(_dev).
//
// D1 (d x n1) and D2 (d x n2) are fp64, column-major.  For query i of D1 and candidate j of D2
//     sd(i, j) = sum_k (D1[k,i] - D2[k,j])^2,  k = 0 .. d-1 in order, subtract, multiply and add each rounded on its own
// (__dsub_rn / __dmul_rn / __dadd_rn: never an FMA), so a numpy restatement gives the same bits.  The neighbours of i
// are the kk = min(knn, n2) candidates of least (sd, j) in lexicographic order; a NaN sd is never one.  The pairs with
// sd <= r2 (r2 = radius * radius in fp64) are kept: as the list is sorted they are a prefix of it.
//
//   1. knn_partial_kernel<D, K>: one thread per query, kKnnThreads queries per CTA, blockIdx.y a slice of the candidates
//      (slices when n1 alone does not fill the device).  Tiles of D2 are staged in shared memory; each thread keeps its
//      running top-K (K = kk rounded up to a power of two) in registers, sorted by (sd, j), and writes its first kk.
//      D = 1, 2, 3 hold the query in registers; D = 0 (any other d) holds it in shared memory.
//   2. knn_merge_kernel<K>: per query, the slices' lists merged into one (the order is total: the result does not
//      depend on the slicing) and the count of kept pairs.
//   3. knn_scan_blocks_kernel + knn_scan_top_kernel: exclusive scan of the counts, the total is m.
//   4. knn_write_kernel: row off[i] + r = (i, j_r), column-major with leading dimension m (rows by i, then rank).
//   1-to-1 (bm_utils.cpp:214-229): per c1 the least sd of its kept pairs (atomicMin on the bits: non-negative doubles
//   order as their bits), then the least c0 among the pairs with that sd (the reference keeps the first pushed, which
//   is the smallest c0); one row per c1 that has a pair, in c1 order, by the same scan.
// Every step is deterministic: a repeated call is bit-identical.
#pragma once

namespace clp {

constexpr int kKnnMaxK = 32;          // CLP_KNN_MAX_K
constexpr int kKnnMaxD = 64;          // CLP_KNN_MAX_D
constexpr int kKnnThreads = 128;      // queries per CTA
constexpr int kKnnTileReg = 128;      // candidates per staged tile when the query is in registers (d <= 3)
constexpr int kKnnTileGen = 32;       // ... when it is in shared memory
constexpr int kKnnNone = 0x7fffffff;  // empty list slot (its sd is +inf)
constexpr int kKnnScanItems = 1024;   // counts per CTA of knn_scan_blocks_kernel (256 threads x 4)

struct KnnArgs {
  const double* D1; const double* D2;
  int d;
  long long n1, n2;
  int kk;                  // min(knn, n2): list entries written per query and slice
  int nsplit;              // candidate slices: slice s is [s * chunk, min(n2, (s + 1) * chunk))
  long long chunk;
  double* part_sd; int* part_j;  // [nsplit][kk][n1]
};

// shared memory of knn_partial_kernel<D, K>
inline size_t knn_partial_smem(int D, int d) {
  return D > 0 ? (size_t)kKnnTileReg * D * sizeof(double) : (size_t)(kKnnTileGen + kKnnThreads) * d * sizeof(double);
}

__device__ __forceinline__ bool knn_less(double a, int ja, double b, int jb) { return a < b || (a == b && ja < jb); }

// (s, j) into the sorted list if it beats the last entry; the compare-exchange pass is unrolled so the list stays in
// registers.  Returns whether it went in.
template <int K>
__device__ __forceinline__ bool knn_insert(double (&sd)[K], int (&jj)[K], double s, int j) {
  if (!knn_less(s, j, sd[K - 1], jj[K - 1])) return false;
  sd[K - 1] = s; jj[K - 1] = j;
#pragma unroll
  for (int t = K - 1; t > 0; --t) {
    if (knn_less(sd[t], jj[t], sd[t - 1], jj[t - 1])) {
      const double ts = sd[t]; sd[t] = sd[t - 1]; sd[t - 1] = ts;
      const int tj = jj[t]; jj[t] = jj[t - 1]; jj[t - 1] = tj;
    }
  }
  return true;
}

template <int K>
__device__ __forceinline__ void knn_clear(double (&sd)[K], int (&jj)[K]) {
#pragma unroll
  for (int t = 0; t < K; ++t) { sd[t] = __longlong_as_double(0x7ff0000000000000LL); jj[t] = kKnnNone; }
}

template <int D, int K>
__global__ void __launch_bounds__(kKnnThreads) knn_partial_kernel(KnnArgs a) {
  extern __shared__ double knn_smem[];
  constexpr int T = D > 0 ? kKnnTileReg : kKnnTileGen;
  const int d = D > 0 ? D : a.d;
  double* tile = knn_smem;                   // T candidates x d, as they lie in D2
  double* qs = knn_smem + (size_t)T * d;     // D = 0: the queries, coordinate-major (d x kKnnThreads)
  const long long i = (long long)blockIdx.x * kKnnThreads + threadIdx.x;
  const bool live = i < a.n1;
  double q[D > 0 ? D : 1];
  if constexpr (D > 0) {
#pragma unroll
    for (int k = 0; k < D; ++k) q[k] = live ? a.D1[i * D + k] : 0.0;
  } else {
    for (int k = 0; k < d; ++k) qs[k * kKnnThreads + threadIdx.x] = live ? a.D1[i * d + k] : 0.0;
  }
  double sd[K]; int jj[K];
  knn_clear<K>(sd, jj);
  const long long lo = (long long)blockIdx.y * a.chunk;
  const long long hi = lo + a.chunk < a.n2 ? lo + a.chunk : a.n2;
  for (long long c0 = lo; c0 < hi; c0 += T) {
    const int cnt = (int)(hi - c0 < T ? hi - c0 : T);
    __syncthreads();  // the previous tile is consumed
    const double* src = a.D2 + c0 * d;
    for (int e = threadIdx.x; e < cnt * d; e += kKnnThreads) tile[e] = src[e];
    __syncthreads();
    if (!live) continue;
    for (int c = 0; c < cnt; ++c) {
      const double* y = tile + c * d;
      double s;
      if constexpr (D > 0) {
        double t = __dsub_rn(q[0], y[0]);
        s = __dmul_rn(t, t);
#pragma unroll
        for (int k = 1; k < D; ++k) { t = __dsub_rn(q[k], y[k]); s = __dadd_rn(s, __dmul_rn(t, t)); }
      } else {
        double t = __dsub_rn(qs[threadIdx.x], y[0]);
        s = __dmul_rn(t, t);
        for (int k = 1; k < d; ++k) {
          t = __dsub_rn(qs[k * kKnnThreads + threadIdx.x], y[k]);
          s = __dadd_rn(s, __dmul_rn(t, t));
        }
      }
      knn_insert<K>(sd, jj, s, (int)(c0 + c));
    }
  }
  if (!live) return;
#pragma unroll
  for (int t = 0; t < K; ++t)
    if (t < a.kk) {
      const size_t o = ((size_t)blockIdx.y * a.kk + t) * a.n1 + i;
      a.part_sd[o] = sd[t]; a.part_j[o] = jj[t];
    }
}

// One thread per query: the slices' sorted lists merged into (out_sd, out_j) [kk][n1] (nsplit = 1: the list is the
// partial one, which is only counted), and cnt[i] = the kept pairs (sd <= r2; a prefix of the list).
template <int K>
__global__ void __launch_bounds__(256) knn_merge_kernel(KnnArgs a, double r2, double* out_sd, int* out_j, int* cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n1) return;
  if (a.nsplit == 1) {
    int c = 0;
    for (int t = 0; t < a.kk; ++t) {
      const size_t o = (size_t)t * a.n1 + i;
      if (a.part_j[o] == kKnnNone || !(a.part_sd[o] <= r2)) break;
      ++c;
    }
    cnt[i] = c;
    return;
  }
  double sd[K]; int jj[K];
  knn_clear<K>(sd, jj);
  for (int s = 0; s < a.nsplit; ++s)
    for (int t = 0; t < a.kk; ++t) {
      const size_t o = ((size_t)s * a.kk + t) * a.n1 + i;
      if (!knn_insert<K>(sd, jj, a.part_sd[o], a.part_j[o])) break;  // the rest of this sorted list is worse
    }
  int c = 0;
#pragma unroll
  for (int t = 0; t < K; ++t)
    if (t < a.kk) {
      out_sd[(size_t)t * a.n1 + i] = sd[t]; out_j[(size_t)t * a.n1 + i] = jj[t];
      c += (jj[t] != kKnnNone && sd[t] <= r2) ? 1 : 0;
    }
  cnt[i] = c;
}

// exclusive scan of kKnnScanItems counts per CTA into off; the CTA's total into bsum[blockIdx.x]
__global__ void __launch_bounds__(256) knn_scan_blocks_kernel(const int* cnt, long long n, long long* off, long long* bsum) {
  __shared__ long long ws[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long base = (long long)blockIdx.x * kKnnScanItems + threadIdx.x * 4;
  long long v[4], s = 0;
#pragma unroll
  for (int r = 0; r < 4; ++r) { v[r] = base + r < n ? cnt[base + r] : 0; s += v[r]; }
  long long x = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  if (lane == 31) ws[warp] = x;
  __syncthreads();
  long long run = x - s;
  for (int w = 0; w < warp; ++w) run += ws[w];
#pragma unroll
  for (int r = 0; r < 4; ++r) { if (base + r < n) off[base + r] = run; run += v[r]; }
  if (threadIdx.x == 255) bsum[blockIdx.x] = run;
}

// one CTA: exclusive scan of the nb block totals in place, the sum of all into *total
__global__ void __launch_bounds__(1024) knn_scan_top_kernel(long long* bsum, long long nb, long long* total) {
  __shared__ long long ws[32];
  __shared__ long long carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (long long b0 = 0; b0 < nb; b0 += 1024) {
    const long long b = b0 + threadIdx.x;
    const long long v = b < nb ? bsum[b] : 0;
    long long x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) ws[warp] = x;
    __syncthreads();
    if (warp == 0) {
      long long w = ws[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      ws[lane] = w;
    }
    __syncthreads();
    const long long excl = carry + (warp ? ws[warp - 1] : 0) + x - v;
    if (b < nb) bsum[b] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

// rows of the kNN pairs: row off[i] + bsum[i / kKnnScanItems] + r = (i, lj[r][i]), A column-major with ld = *total
__global__ void __launch_bounds__(256) knn_write_kernel(const int* cnt, const long long* off, const long long* bsum,
                                                        const int* lj, long long n1, const long long* total, int* A) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1) return;
  const long long m = *total;
  const long long row = off[i] + bsum[i / kKnnScanItems];
  const int c = cnt[i];
  for (int r = 0; r < c; ++r) { A[row + r] = (int)i; A[m + row + r] = lj[(size_t)r * n1 + i]; }
}

// 1-to-1, first pass: the least sd (as bits) of the kept pairs of every c1
__global__ void __launch_bounds__(256) knn_best_sd_kernel(const int* cnt, const double* lsd, const int* lj, long long n1,
                                                          unsigned long long* best) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1) return;
  for (int r = 0; r < cnt[i]; ++r)
    atomicMin(&best[lj[(size_t)r * n1 + i]], (unsigned long long)__double_as_longlong(lsd[(size_t)r * n1 + i]));
}

// second pass: the least c0 among the kept pairs of c1 whose sd equals that least one
__global__ void __launch_bounds__(256) knn_best_c0_kernel(const int* cnt, const double* lsd, const int* lj, long long n1,
                                                          const unsigned long long* best, unsigned int* c0best) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n1) return;
  for (int r = 0; r < cnt[i]; ++r) {
    const int j = lj[(size_t)r * n1 + i];
    if ((unsigned long long)__double_as_longlong(lsd[(size_t)r * n1 + i]) == best[j]) atomicMin(&c0best[j], (unsigned int)i);
  }
}

// one row for every c1 that has a kept pair
__global__ void __launch_bounds__(256) knn_flag_kernel(const unsigned int* c0best, long long n2, int* cnt2) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n2) cnt2[j] = c0best[j] != 0xffffffffu ? 1 : 0;
}

__global__ void __launch_bounds__(256) knn_write_1to1_kernel(const unsigned int* c0best, const long long* off,
                                                             const long long* bsum, long long n2, const long long* total,
                                                             int* A) {
  const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n2 || c0best[j] == 0xffffffffu) return;
  const long long m = *total;
  const long long row = off[j] + bsum[j / kKnnScanItems];
  A[row] = (int)c0best[j]; A[m + row] = (int)j;
}

}  // namespace clp
