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

// The running top-K (sd, jj) of query i of D1 over the candidates [lo, hi) of D2 (indices relative to D2), tiles of D2
// staged in shared memory.  Every thread of the CTA calls it with the same lo, hi and d (the barriers are the CTA's);
// live: i is a query (a thread past the last one stages tiles and keeps an empty list).
template <int D, int K>
__device__ __forceinline__ void knn_scan_candidates(const double* D1, const double* D2, int d_rt, long long i, bool live,
                                                    long long lo, long long hi, double (&sd)[K], int (&jj)[K]) {
  extern __shared__ double knn_smem[];
  constexpr int T = D > 0 ? kKnnTileReg : kKnnTileGen;
  const int d = D > 0 ? D : d_rt;
  double* tile = knn_smem;                   // T candidates x d, as they lie in D2
  double* qs = knn_smem + (size_t)T * d;     // D = 0: the queries, coordinate-major (d x kKnnThreads)
  double q[D > 0 ? D : 1];
  if constexpr (D > 0) {
#pragma unroll
    for (int k = 0; k < D; ++k) q[k] = live ? D1[i * D + k] : 0.0;
  } else {
    for (int k = 0; k < d; ++k) qs[k * kKnnThreads + threadIdx.x] = live ? D1[i * d + k] : 0.0;
  }
  knn_clear<K>(sd, jj);
  for (long long c0 = lo; c0 < hi; c0 += T) {
    const int cnt = (int)(hi - c0 < T ? hi - c0 : T);
    __syncthreads();  // the previous tile is consumed
    const double* src = D2 + c0 * d;
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
}

template <int D, int K>
__global__ void __launch_bounds__(kKnnThreads) knn_partial_kernel(KnnArgs a) {
  const long long i = (long long)blockIdx.x * kKnnThreads + threadIdx.x;
  const bool live = i < a.n1;
  const long long lo = (long long)blockIdx.y * a.chunk;
  const long long hi = lo + a.chunk < a.n2 ? lo + a.chunk : a.n2;
  double sd[K]; int jj[K];
  knn_scan_candidates<D, K>(a.D1, a.D2, a.d, i, live, lo, hi, sd, jj);
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

// ---- batches of cloud pairs (clp_batch_correspondences(_dev)) -------------------------------------------------------
// Problem p is the single call on (D1_p, D2_p), bit for bit.  The clouds are concatenated: query i of p is q_off + i of
// one query index space, candidate j of p is c_off + j of one candidate index space (the staged clouds at d * q_off
// and d * c_off).  The steps are those of the single call, each one launch for the whole batch:
//   1. knn_batch_partial_kernel<D, K>: the query CTAs of all problems one after the other along x (problem p owns
//      CTAs [cta0, cta0 + ceil(n1 / kKnnThreads))), a candidate slice along y; slice s of p is [s * chunk, (s + 1) *
//      chunk) of its own candidates, chunk = round_up(ceil(n2 / nsplit), tile).  K covers the largest kk of the batch;
//      each problem writes its own kk entries per query and slice.
//   2. knn_batch_merge_kernel<K>: the slices' lists of every query merged, cnt[q_off + i] = its kept pairs.
//   3. one exclusive scan of cnt over the whole query space (knn_scan_blocks_kernel + knn_scan_top_kernel).
//   4. knn_batch_rows_kernel: m[p] = scan(end of p) - scan(start of p) and rbase[p] = scan(start of p).
//   5. knn_batch_write_kernel: row off[q] - rbase[p] of problem p.
//   1-to-1: the atomicMin passes on the concatenated candidate space (64-bit offsets), the flags, the scan, the counts
//   and the rows the same way, by c1.
// A problem's result depends on nothing but its own clouds: the order of the lists is total, so neither the slicing
// nor the batch around a problem changes it.
struct KnnProb {
  BatchProblem bp;          // d1_off = d q_off, d2_off = d c_off, n1, n2 (0 for a problem with no rows), a_off = -1:
                            // the entry batch_stage_points_kernel reads
  long long q_off, c_off;   // first query / candidate in the concatenated index spaces
  long long cta0;           // first query CTA
  long long l_off, m_off;   // partial lists [nsplit][kk][n1] at l_off, merged lists [kk][n1] at m_off
  long long chunk;          // candidates per slice
  int kk, pad_;
};

struct KnnBatchArgs {
  const KnnProb* prob; int nprob;
  int d, nsplit;
  const double* D1; const double* D2;   // staged clouds
  double* part_sd; int* part_j;         // partial lists
  double* lsd; int* lj;                 // merged lists (the partial ones when nsplit = 1)
  double r2;
  int* cnt; long long* off; long long* bsum; long long* total; long long nscan;  // the scan and its length
  long long* mcount; long long* rbase;  // per problem: m and the scan at its first query (candidate for 1-to-1)
  unsigned long long* best; unsigned int* c0best;  // 1-to-1, per concatenated candidate
  int* A; long long as[3];              // entry (r, c) of problem p at A[p as[0] + r as[1] + c as[2]]
  int packed;                           // 1: at A[2 rbase[p] + r + c m[p]] instead (the host call's staging)
};

// the problem whose range [start, next start) holds x, for starts cta0 (F = 0), q_off (F = 1) or c_off (F = 2): the
// last one whose start is <= x (problems with empty ranges share their start with the next one)
template <int F>
__device__ __forceinline__ int knn_problem(const KnnProb* t, int nprob, long long x) {
  int lo = 0, hi = nprob - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    const long long s = F == 0 ? t[mid].cta0 : F == 1 ? t[mid].q_off : t[mid].c_off;
    if (s <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

template <int D, int K>
__global__ void __launch_bounds__(kKnnThreads, 4) knn_batch_partial_kernel(KnnBatchArgs a) {
  const KnnProb* P = a.prob + knn_problem<0>(a.prob, a.nprob, blockIdx.x);
  const long long n1 = P->bp.n1, n2 = P->bp.n2;
  const long long i = ((long long)blockIdx.x - P->cta0) * kKnnThreads + threadIdx.x;
  const bool live = i < n1;
  const long long lo = (long long)blockIdx.y * P->chunk;
  const long long hi = lo + P->chunk < n2 ? lo + P->chunk : n2;
  double sd[K]; int jj[K];
  knn_scan_candidates<D, K>(a.D1 + P->q_off * (D > 0 ? D : a.d), a.D2 + P->c_off * (D > 0 ? D : a.d), a.d, i, live, lo,
                            hi, sd, jj);
  if (!live) return;
  const long long l_off = P->l_off;  // read after the scan: fewer registers live across it
  const int kk = P->kk;
#pragma unroll
  for (int t = 0; t < K; ++t)
    if (t < kk) {
      const size_t o = l_off + ((size_t)blockIdx.y * kk + t) * n1 + i;
      a.part_sd[o] = sd[t]; a.part_j[o] = jj[t];
    }
}

// the query of this thread in the grid of knn_batch_partial_kernel (x only): its problem (returned; -1 past the
// problem's last query), the problem's entry and the local index
__device__ __forceinline__ int knn_batch_query(const KnnBatchArgs& a, KnnProb& P, long long& i) {
  const int p = knn_problem<0>(a.prob, a.nprob, blockIdx.x);
  P = a.prob[p];
  i = ((long long)blockIdx.x - P.cta0) * kKnnThreads + threadIdx.x;
  return i < P.bp.n1 ? p : -1;
}

template <int K>
__global__ void __launch_bounds__(kKnnThreads) knn_batch_merge_kernel(KnnBatchArgs a) {
  KnnProb P; long long i;
  if (knn_batch_query(a, P, i) < 0) return;
  const long long n1 = P.bp.n1;
  const int kk = P.kk;
  if (a.nsplit == 1) {
    int c = 0;
    for (int t = 0; t < kk; ++t) {
      const size_t o = P.m_off + (size_t)t * n1 + i;
      if (a.lj[o] == kKnnNone || !(a.lsd[o] <= a.r2)) break;
      ++c;
    }
    a.cnt[P.q_off + i] = c;
    return;
  }
  double sd[K]; int jj[K];
  knn_clear<K>(sd, jj);
  for (int s = 0; s < a.nsplit; ++s)
    for (int t = 0; t < kk; ++t) {
      const size_t o = P.l_off + ((size_t)s * kk + t) * n1 + i;
      if (!knn_insert<K>(sd, jj, a.part_sd[o], a.part_j[o])) break;  // the rest of this sorted list is worse
    }
  int c = 0;
#pragma unroll
  for (int t = 0; t < K; ++t)
    if (t < kk) {
      const size_t o = P.m_off + (size_t)t * n1 + i;
      a.lsd[o] = sd[t]; a.lj[o] = jj[t];
      c += (jj[t] != kKnnNone && sd[t] <= a.r2) ? 1 : 0;
    }
  a.cnt[P.q_off + i] = c;
}

// the exclusive scan at x of the scanned space (its total at the end)
__device__ __forceinline__ long long knn_scan_at(const KnnBatchArgs& a, long long x) {
  return x < a.nscan ? a.off[x] + a.bsum[x / kKnnScanItems] : *a.total;
}

// one thread per problem: m[p] and the scan at its first query (by_c1 = 0) or candidate (by_c1 = 1)
__global__ void __launch_bounds__(256) knn_batch_rows_kernel(KnnBatchArgs a, int by_c1) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= a.nprob) return;
  const KnnProb& P = a.prob[p];
  const long long x0 = by_c1 ? P.c_off : P.q_off, x1 = x0 + (by_c1 ? P.bp.n2 : P.bp.n1);
  const long long r0 = knn_scan_at(a, x0);
  a.rbase[p] = r0;
  a.mcount[p] = knn_scan_at(a, x1) - r0;
}

// the address of entry (r, c) of problem p
__device__ __forceinline__ long long knn_batch_at(const KnnBatchArgs& a, int p, long long r, int c) {
  return a.packed ? 2 * a.rbase[p] + r + c * a.mcount[p] : p * a.as[0] + r * a.as[1] + c * a.as[2];
}

__global__ void __launch_bounds__(kKnnThreads) knn_batch_write_kernel(KnnBatchArgs a) {
  KnnProb P; long long i;
  const int p = knn_batch_query(a, P, i);
  if (p < 0) return;
  const long long q = P.q_off + i;
  const long long row = knn_scan_at(a, q) - a.rbase[p];
  const int c = a.cnt[q];
  for (int r = 0; r < c; ++r) {
    a.A[knn_batch_at(a, p, row + r, 0)] = (int)i;
    a.A[knn_batch_at(a, p, row + r, 1)] = a.lj[P.m_off + (size_t)r * P.bp.n1 + i];
  }
}

// 1-to-1, first pass: the least sd (as bits) of the kept pairs of every c1 of the concatenated candidate space
__global__ void __launch_bounds__(kKnnThreads) knn_batch_best_sd_kernel(KnnBatchArgs a) {
  KnnProb P; long long i;
  if (knn_batch_query(a, P, i) < 0) return;
  const int c = a.cnt[P.q_off + i];
  for (int r = 0; r < c; ++r) {
    const size_t o = P.m_off + (size_t)r * P.bp.n1 + i;
    atomicMin(&a.best[P.c_off + a.lj[o]], (unsigned long long)__double_as_longlong(a.lsd[o]));
  }
}

// second pass: the least c0 among the kept pairs of c1 whose sd equals that least one
__global__ void __launch_bounds__(kKnnThreads) knn_batch_best_c0_kernel(KnnBatchArgs a) {
  KnnProb P; long long i;
  if (knn_batch_query(a, P, i) < 0) return;
  const int c = a.cnt[P.q_off + i];
  for (int r = 0; r < c; ++r) {
    const size_t o = P.m_off + (size_t)r * P.bp.n1 + i;
    const long long g = P.c_off + a.lj[o];
    if ((unsigned long long)__double_as_longlong(a.lsd[o]) == a.best[g]) atomicMin(&a.c0best[g], (unsigned int)i);
  }
}

// one row for every c1 that has a kept pair: the flags over the concatenated candidates (knn_flag_kernel), the scan,
// knn_batch_rows_kernel(by_c1 = 1), then the rows
__global__ void __launch_bounds__(256) knn_batch_write_1to1_kernel(KnnBatchArgs a) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.nscan || a.c0best[g] == 0xffffffffu) return;
  const int p = knn_problem<2>(a.prob, a.nprob, g);
  const long long row = knn_scan_at(a, g) - a.rbase[p];
  a.A[knn_batch_at(a, p, row, 0)] = (int)a.c0best[g];
  a.A[knn_batch_at(a, p, row, 1)] = (int)(g - a.prob[p].c_off);
}

}  // namespace clp
