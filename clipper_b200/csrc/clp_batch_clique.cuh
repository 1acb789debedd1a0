// clp_batch_clique.cuh -- maximum clique of many small graphs in a constant number of launches (clp_batch_max_clique_*).
//
// Every problem gets what clp_max_clique returns for it on an fp32 handle (clp_clique.cuh), with the host round trips
// of that path replaced by block-level steps:
//   phase A  mc_batch_prepare_kernel  one CTA per problem (problems drawn from a counter): the graph (scored with the
//            batch's arithmetic, batch_score_pairs, or scattered from the given pairs) as a bitset adjacency in the
//            problem's HBM region -> level-synchronous k-core peel with __syncthreads in place of the grid barrier ->
//            degeneracy order -> greedy heuristic with the CTA's warps as workers (mc_heu_seed, incumbent in shared
//            memory) and the replay of its winner -> later-neighbour counts, search roots and task prefix (block scan)
//   phase B  mc_batch_search_kernel   one launch over the tasks of all problems: warps draw from one counter in an
//            order that interleaves the problems (the k-th task of every problem before the (k+1)-th of any), each task
//            run by mc_search_task against its problem's incumbent; per problem: branches, completed tasks, flags
//   phase C  mc_batch_replay_kernel   one warp per problem whose search beat its heuristic replays the winning task
// Task numbering, roots, split and incumbent key are those of the single-problem path, so a proven answer is the same
// clique.
#pragma once

namespace clp {

// mc_batch_prepare_kernel<KIND, DD>: 0 Euclidean, 1 PointNormal, 2 graph given as pairs, 3 fp32 matrix already stored
// (clp_batch_max_clique_custom: the round's batch_score_custom_kernel left problem p's matrix in slot p, and `scratch`
// points at the matrix region of slot 0)
constexpr int kMcbKindGraph = 2;
constexpr int kMcbKindStored = 3;

struct McBatchProblem {   // device array, one per problem
  BatchProblem sp;        // scored problems: offsets of the inputs (sp.m is the problem's m)
  long long adj_off;      // words into the adjacency arena (m * W)
  long long v_off;        // ints into the vertex arena: core[m] | rnd[m] | roots[m] | nodes[m + 1]
  long long t_off;        // into the task-prefix arena (m + 1)
  long long e_off, ne;    // graph problems: (row, column) pairs into the edge array
};

struct McBatchOut {       // phase A results of one problem (zeroed by the host)
  unsigned long long n_edges;
  long long ntasks;
  int max_core, lb, nroots, K;
  unsigned long long ns[3];  // in-kernel time of the adjacency (scoring included), the peel, the rest
};

// per-CTA HBM scratch of a scored problem: the inputs gathered per association and the fp32 score matrix
struct McbLayout { size_t E1, E2, F1, F2, A, M, total; };
__host__ __device__ inline McbLayout mcb_layout(int max_m, int dd) {
  McbLayout L;
  const size_t mm = (size_t)max_m, ld = (mm + 127) / 128 * 128, rows_pad = (mm + 3) / 4 * 4;
  size_t o = 0;
  L.E1 = o; o = batch_align(o + mm * dd * 8);
  L.E2 = o; o = batch_align(o + mm * dd * 8);
  L.F1 = o; o = batch_align(o + mm * 16);
  L.F2 = o; o = batch_align(o + mm * 16);
  L.A = o; o = batch_align(o + 2 * mm * 4);
  L.M = o; o = batch_align(o + rows_pad * ld * 4);
  L.total = o;
  return L;
}

// dynamic shared memory: the scoring tables, then (overlaid) the clique tables
struct McbSmem { unsigned cnt, queue, tile, redf, deg, order, core, rnd, P, alive, rem, wpre, total; };
__host__ __device__ inline McbSmem mcb_smem_plan(int max_m) {
  McbSmem b;
  const unsigned mm = (unsigned)max_m, rows_pad = (mm + 3) / 4 * 4, W = (mm + 31) / 32;
  unsigned o = 0;
  b.cnt = o; o += rows_pad * 4; o = (o + 15u) & ~15u;
  b.queue = o; o += kBatchWarps * 128 * 2;
  b.tile = o; o += kBatchWarps * 128 * 4;
  b.redf = o; o += 64;
  const unsigned score = o;
  o = 0;
  b.deg = o; o += mm * 4;    // current degree during the peel, later-neighbour count after it
  b.order = o; o += mm * 4;  // degeneracy order
  b.core = o; o += mm * 4;
  b.rnd = o; o += mm * 4;
  o = (o + 15u) & ~15u;
  b.P = o; o += kBatchWarps * W * 4;
  b.alive = o; o += W * 4;
  b.rem = o; o += W * 4;
  b.wpre = o; o += (W + 1) * 4;
  b.total = (o > score ? o : score) + 16;
  return b;
}

struct McBatchArgs {
  const McBatchProblem* prob;
  int nprob;
  int run_heu;                     // HEU or EXACT
  int build_tasks;                 // EXACT with a positive time limit: roots and task prefix
  int* next;                       // problem counter
  unsigned* adj; int* vint; long long* tpre;
  McBatchOut* out;
  const int* edges;                // graph problems
  const double* D1; const double* D2; const int* A;  // scored problems
  double p0, p1, p2, p3, affinityeps;
  int* error;
  unsigned char* scratch; size_t scratch_stride;
  int max_m;
};

template <int KIND, int DD>
__global__ void __launch_bounds__(kBatchThreads) mc_batch_prepare_kernel(McBatchArgs ba) {
  extern __shared__ __align__(128) unsigned char mcb_smem[];
  __shared__ int s_p, s_K;
  __shared__ unsigned s_cnt[3];
  __shared__ unsigned s_scan[kBatchWarps + 1];
  __shared__ float s_R;
  __shared__ unsigned long long s_best, s_edges;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const McbSmem sp = mcb_smem_plan(ba.max_m);
  int* deg = reinterpret_cast<int*>(mcb_smem + sp.deg);
  int* order = reinterpret_cast<int*>(mcb_smem + sp.order);
  int* core = reinterpret_cast<int*>(mcb_smem + sp.core);
  int* rnd = reinterpret_cast<int*>(mcb_smem + sp.rnd);
  unsigned* alive = reinterpret_cast<unsigned*>(mcb_smem + sp.alive);
  unsigned* rem = reinterpret_cast<unsigned*>(mcb_smem + sp.rem);
  unsigned* wpre = reinterpret_cast<unsigned*>(mcb_smem + sp.wpre);

  for (;;) {
    __syncthreads();
    if (tid == 0) s_p = atomicAdd(ba.next, 1);
    __syncthreads();
    const int p = s_p;
    if (p >= ba.nprob) break;
    const McBatchProblem Q = ba.prob[p];
    const int m = Q.sp.m, W = (m + 31) / 32;
    unsigned* adj = ba.adj + Q.adj_off;
    int* g_core = ba.vint + Q.v_off;
    int* g_rnd = g_core + m;
    int* g_roots = g_rnd + m;
    int* g_nodes = g_roots + m;
    long long* g_tpre = ba.tpre + Q.t_off;
    const unsigned long long t0 = global_ns();

    // ---- adjacency and degrees
    if (tid == 0) s_edges = 0ull;
    if constexpr (KIND == kMcbKindGraph) {
      const int* e = ba.edges + 2 * Q.e_off;  // the region is zeroed by the host
      for (long long q = tid; q < Q.ne; q += kBatchThreads) {
        const int r = e[2 * q], c = e[2 * q + 1];
        atomicOr(&adj[(size_t)r * W + (c >> 5)], 1u << (c & 31));
        atomicOr(&adj[(size_t)c * W + (r >> 5)], 1u << (r & 31));
      }
      __syncthreads();
      for (int i = warp; i < m; i += kBatchWarps) {
        int c = 0;
        for (int w = lane; w < W; w += 32) c += __popc(__ldcg(&adj[(size_t)i * W + w]));
        c = mc_warp_sum(c);
        if (lane == 0) deg[i] = c;
      }
    } else {
      const float* M;
      if constexpr (KIND == kMcbKindStored) {  // scored by the round's batch_score_custom_kernel into slot p
        M = reinterpret_cast<const float*>(ba.scratch + (size_t)p * ba.scratch_stride);
      } else {
        const McbLayout L = mcb_layout(ba.max_m, DD);
        unsigned char* sc = ba.scratch + (size_t)blockIdx.x * ba.scratch_stride;
        float* Ms = reinterpret_cast<float*>(sc + L.M);
        batch_score_pairs<KIND, DD>(Q.sp, ba.D1 + Q.sp.d1_off, ba.D2 + Q.sp.d2_off, ba.A, ba.p0, ba.p1, ba.p2, ba.p3,
                                    ba.affinityeps, ba.error, reinterpret_cast<double*>(sc + L.E1),
                                    reinterpret_cast<double*>(sc + L.E2), reinterpret_cast<float4*>(sc + L.F1),
                                    reinterpret_cast<float4*>(sc + L.F2), reinterpret_cast<int*>(sc + L.A), Ms,
                                    reinterpret_cast<unsigned*>(mcb_smem + sp.cnt),
                                    reinterpret_cast<unsigned short*>(mcb_smem + sp.queue),
                                    reinterpret_cast<float*>(mcb_smem + sp.tile), reinterpret_cast<float*>(mcb_smem + sp.redf), s_R);
        M = Ms;
      }
      const int ld = (m + 127) / 128 * 128;
      for (int i = warp; i < m; i += kBatchWarps) {  // mc_adjacency_kernel's rule: the sign bits of row i, no diagonal
        const float* row = M + (size_t)i * ld;
        int c = 0;
        for (int w = 0; w < W; ++w) {
          const int j = w * 32 + lane;
          const bool e = (j < m && j != i) ? mc_edge<float>(row[j]) : false;
          const unsigned bits = __ballot_sync(0xffffffffu, e);
          if (lane == 0) adj[(size_t)i * W + w] = bits;
          c += __popc(bits);
        }
        if (lane == 0) deg[i] = c;
      }
    }
    __syncthreads();
    {
      unsigned long long d = 0;
      for (int i = tid; i < m; i += kBatchThreads) d += (unsigned long long)deg[i];
      for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
      if (lane == 0 && d) atomicAdd(&s_edges, d);
    }
    const unsigned long long t1 = global_ns();

    // ---- k-core peel (mc_peel_kernel's rules): iteration `it` removes every alive vertex of degree <= k; an empty
    //      iteration raises k.  The vertices removed in one iteration enter the degeneracy order by ascending index.
    for (int w = tid; w < W; w += kBatchThreads) {
      const int left = m - w * 32;
      alive[w] = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
      rem[w] = 0u;
    }
    if (tid < 3) s_cnt[tid] = 0u;
    __syncthreads();
    int k = 0, removed = 0, kmax = 0;
    for (int it = 0; removed < m && it <= 2 * m + 1; ++it) {
      unsigned* c = &s_cnt[it % 3];
      if (tid == 0) s_cnt[(it + 1) % 3] = 0u;  // last read two barriers ago
      for (int v = tid; v < m; v += kBatchThreads) {
        const unsigned bit = 1u << (v & 31);
        if ((alive[v >> 5] & bit) && deg[v] <= k) {
          core[v] = k; rnd[v] = it;
          atomicAdd(c, 1u);
          atomicAnd(&alive[v >> 5], ~bit);
          atomicOr(&rem[v >> 5], bit);
        }
      }
      __syncthreads();
      const int n = (int)*(volatile unsigned*)c;
      if (n == 0) { ++k; continue; }
      kmax = k;
      if (warp == 0) {  // exclusive prefix of the removed counts over the words
        unsigned run = 0;
        for (int w0 = 0; w0 < W; w0 += 32) {
          const int w = w0 + lane;
          const unsigned x = w < W ? (unsigned)__popc(rem[w]) : 0u;
          unsigned inc = x;
          for (int o = 1; o < 32; o <<= 1) { const unsigned y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
          if (w < W) wpre[w] = run + inc - x;
          run += __shfl_sync(0xffffffffu, inc, 31);
        }
      }
      __syncthreads();
      for (int v = tid; v < m; v += kBatchThreads) {
        const unsigned r = rem[v >> 5], bit = 1u << (v & 31);
        if (r & bit) order[removed + (int)(wpre[v >> 5] + __popc(r & (bit - 1u)))] = v;
      }
      __syncthreads();
      const int* frontier = order + removed;
      const long long work = (long long)n * W;
      for (long long q = tid; q < work; q += kBatchThreads) {
        const int f = (int)(q / W), w = (int)(q % W);
        unsigned bits = adj[(size_t)frontier[f] * W + w] & alive[w];
        while (bits) {
          const int b = __ffs(bits) - 1;
          bits &= bits - 1u;
          atomicSub(&deg[w * 32 + b], 1);
        }
      }
      for (int w = tid; w < W; w += kBatchThreads) rem[w] = 0u;
      removed += n;
      __syncthreads();
    }
    for (int v = tid; v < m; v += kBatchThreads) { g_core[v] = core[v]; g_rnd[v] = rnd[v]; }
    const unsigned long long t2 = global_ns();

    // ---- greedy heuristic over the seeds in reverse degeneracy order, then the replay of its winner
    int lb = 0;
    if (ba.run_heu) {
      if (tid == 0) s_best = 0ull;
      __syncthreads();
      unsigned* P = reinterpret_cast<unsigned*>(mcb_smem + sp.P) + (size_t)warp * W;
      for (int s = warp; s < m; s += kBatchWarps) mc_heu_seed<true>(adj, m, W, core, order[m - 1 - s], &s_best, false, nullptr, P);
      __syncthreads();
      const unsigned long long best = s_best;
      lb = (int)(best >> 32);
      if (warp == 0) mc_heu_seed<true>(adj, m, W, core, (int)(0xffffffffu - (unsigned)(best & 0xffffffffull)), &s_best, true, g_nodes, P);
    }

    // ---- search roots (core + 1 > lb, later + 1 > lb, reverse degeneracy order) and the task prefix
    int nroots = 0;
    long long ntasks = 0;
    if (ba.build_tasks && lb < kmax + 1) {
      for (int r = warp; r < m; r += kBatchWarps) {  // mc_later_count_kernel; deg[] is free after the peel
        const int rr = rnd[r];
        int cnt = 0;
        for (int w = lane; w < W; w += 32) {
          unsigned bits = adj[(size_t)r * W + w];
          while (bits) {
            const int u = w * 32 + __ffs(bits) - 1;
            bits &= bits - 1u;
            const int ru = rnd[u];
            cnt += (ru > rr || (ru == rr && u > r)) ? 1 : 0;
          }
        }
        cnt = mc_warp_sum(cnt);
        if (lane == 0) deg[r] = cnt;
      }
      if (tid == 0) s_K = 1;
      __syncthreads();
      const int per = (m + kBatchThreads - 1) / kBatchThreads, s0 = tid * per;
      unsigned nr = 0, nt = 0;
      int kmine = 1;
      for (int q = 0; q < per; ++q) {
        const int s = s0 + q;
        if (s >= m) break;
        const int v = order[m - 1 - s], later = deg[v];
        if (core[v] + 1 <= lb || later + 1 <= lb) continue;
        ++nr; nt += later > kMcSplit ? (unsigned)later : 1u;
        kmine = max(kmine, later);
      }
      atomicMax(&s_K, kmine);
      unsigned rpos = batch_block_exscan(nr, s_scan);
      nroots = (int)s_scan[kBatchWarps];
      unsigned tpos = batch_block_exscan(nt, s_scan);
      ntasks = (long long)s_scan[kBatchWarps];
      for (int q = 0; q < per; ++q) {
        const int s = s0 + q;
        if (s >= m) break;
        const int v = order[m - 1 - s], later = deg[v];
        if (core[v] + 1 <= lb || later + 1 <= lb) continue;
        g_roots[rpos] = v; g_tpre[rpos] = (long long)tpos;
        ++rpos; tpos += later > kMcSplit ? (unsigned)later : 1u;
      }
      if (tid == 0) g_tpre[nroots] = ntasks;
    }
    __syncthreads();
    if (tid == 0) {
      McBatchOut o;
      o.n_edges = s_edges / 2; o.ntasks = ntasks; o.max_core = kmax; o.lb = lb; o.nroots = nroots; o.K = nroots ? s_K : 0;
      const unsigned long long t3 = global_ns();
      o.ns[0] = t1 - t0; o.ns[1] = t2 - t1; o.ns[2] = t3 - t2;
      ba.out[p] = o;
    }
  }
}

// ---- phase B ------------------------------------------------------------------------------------------------------
// Draw d is task k of problem q: the draws are grouped in rounds (round k holds task k of every problem with more than
// k tasks, in a fixed problem order); rounds of equal width form a segment, found by binary search.
struct McBatchSearchArgs {
  const McBatchProblem* prob;
  const McBatchOut* out;
  const unsigned* adj; const int* vint; const long long* tpre;
  const int* porder;          // problems by task count, descending
  const long long* seg_start; // [nseg + 1] first draw of each segment
  const long long* seg_k0;    // [nseg] first round of each segment
  const int* seg_width;       // [nseg] problems per round
  int nseg;
  long long total;
  int K, KW;
  unsigned arena_cap;
  unsigned char* scratch; size_t stride;
  unsigned long long* best;      // [nprob] incumbent keys
  unsigned long long* branches;  // [nprob]
  unsigned long long* done;      // [nprob] completed tasks
  int* flags;                    // [nprob][2]: a task stopped at the deadline, a colour-class arena overflowed
  unsigned long long* next;
  const unsigned long long* deadline;
};

__device__ __forceinline__ McSearchArgs mcb_task_args(const McBatchSearchArgs& b, int q) {
  const McBatchProblem& P = b.prob[q];
  McSearchArgs a;
  a.m = P.sp.m; a.W = (a.m + 31) / 32;
  a.adj = b.adj + P.adj_off;
  const int* v = b.vint + P.v_off;
  a.rnd = v + a.m; a.roots = v + 2 * a.m; a.nodes_out = const_cast<int*>(v) + 3 * a.m;
  a.tprefix = b.tpre + P.t_off;
  a.nroots = b.out[q].nroots; a.ntasks = b.out[q].ntasks;
  a.K = b.K; a.KW = b.KW; a.arena_cap = b.arena_cap; a.scratch = b.scratch; a.stride = b.stride;
  a.best = b.best + q; a.next_task = nullptr; a.n_branches = nullptr; a.flags = b.flags + 2 * q; a.deadline = b.deadline;
  a.replay_task = -1; a.replay_size = 0;
  return a;
}

__global__ void __launch_bounds__(kMcSearchWarps * 32) mc_batch_search_kernel(McBatchSearchArgs b) {
  extern __shared__ unsigned mc_smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  unsigned* U = mc_smem + (size_t)wib * 2 * b.KW;
  unsigned* Q = U + b.KW;
  unsigned char* base = b.scratch + (size_t)((long long)blockIdx.x * kMcSearchWarps + wib) * b.stride;
  for (;;) {  // at most `total` draws in total
    unsigned long long d = 0;
    int stop = 0;
    if (lane == 0) { d = atomicAdd(b.next, 1ull); stop = global_ns() > *b.deadline; }
    d = __shfl_sync(0xffffffffu, d, 0);
    stop = __shfl_sync(0xffffffffu, stop, 0);
    if ((long long)d >= b.total || stop) break;
    int lo = 0, hi = b.nseg - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (b.seg_start[mid] <= (long long)d) lo = mid; else hi = mid - 1;
    }
    const long long off = (long long)d - b.seg_start[lo];
    const int wdt = b.seg_width[lo];
    const int q = b.porder[off % wdt];
    const long long t = b.seg_k0[lo] + off / wdt;
    const McSearchArgs a = mcb_task_args(b, q);
    unsigned long long nb = 0;
    const bool ok = mc_search_task(a, t, U, Q, base, &nb);
    if (lane == 0) {
      if (nb) atomicAdd(&b.branches[q], nb);
      if (ok) atomicAdd(&b.done[q], 1ull);
    }
    if (!ok) break;
  }
}

// ---- phase C: one warp per problem whose search found a clique larger than its heuristic's -------------------------
__global__ void __launch_bounds__(kMcSearchWarps * 32) mc_batch_replay_kernel(McBatchSearchArgs b, int nprob) {
  extern __shared__ unsigned mc_smem[];
  const int wib = threadIdx.x >> 5;
  unsigned* U = mc_smem + (size_t)wib * 2 * b.KW;
  unsigned* Q = U + b.KW;
  const long long worker = (long long)blockIdx.x * kMcSearchWarps + wib;
  const long long nworkers = (long long)gridDim.x * kMcSearchWarps;
  unsigned char* base = b.scratch + (size_t)worker * b.stride;
  for (long long q = worker; q < nprob; q += nworkers) {
    const unsigned long long best = b.best[q];
    const int s = (int)(best >> 32);
    if (b.out[q].ntasks == 0 || s <= b.out[q].lb) continue;
    McSearchArgs a = mcb_task_args(b, (int)q);
    a.replay_task = (long long)(0xffffffffu - (unsigned)(best & 0xffffffffull));
    a.replay_size = s;
    unsigned long long nb = 0;
    mc_search_task(a, a.replay_task, U, Q, base, &nb);
  }
}

}  // namespace clp
