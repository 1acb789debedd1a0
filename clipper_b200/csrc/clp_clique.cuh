// clp_clique.cuh -- maximum clique of the constraint graph C (solveAsMaximumClique, reference clipper.cpp:82-97 and
// maxclique.cpp:89-140).  The graph is the sign-bit pattern of the dense store without the diagonal: {i,j} is an edge
// iff the stored element s_ij has its sign bit clear (DESIGN §2), whatever M's value.
//
//   mc_adjacency_kernel  bitset adjacency (ceil(m/32) words per row, diagonal cleared) + degrees, one CTA per row
//   mc_peel_kernel       k-core peeling, level by level, in ONE cooperative launch (device-wide barriers of
//                        clp_kernels.cuh): core numbers and the removal iteration of every vertex (degeneracy order)
//   mc_heu_kernel        greedy clique from every seed (one warp per seed, P as a bitset in shared memory), the winner
//                        kept as one 64-bit atomicMax over (size, -seed); replayed by one warp for the nodes
//   mc_search_kernel     exact branch-and-bound (bitset greedy-colouring bound, BBMC / MCQ): one warp per task, tasks
//                        drawn from an atomic counter, incumbent in global memory; replayed by one warp for the nodes
// No CTA ever waits for another one outside the cooperative peel, and every loop is bounded.
#pragma once

namespace clp {

constexpr int kMcThreads = 256;     // adjacency / heuristic CTAs
constexpr int kMcPeelThreads = 512;
constexpr int kMcSearchWarps = 4;   // independent workers per CTA of the search kernel
constexpr int kMcMaxCore = 8191;    // EXACT: largest max core whose per-worker scratch the search sizes (16-bit packing)
constexpr int kMcSplit = 96;        // roots with more candidates than this are split at depth 1

template <typename T> __device__ __forceinline__ bool mc_edge(T s);
template <> __device__ __forceinline__ bool mc_edge<float>(float s) { return (__float_as_uint(s) >> 31) == 0u; }
template <> __device__ __forceinline__ bool mc_edge<double>(double s) { return ((unsigned long long)__double_as_longlong(s) >> 63) == 0ull; }

// (size, -id) packed so that a larger key is a larger clique, ties to the smaller id
__host__ __device__ __forceinline__ unsigned long long mc_key(unsigned size, unsigned id) {
  return ((unsigned long long)size << 32) | (unsigned long long)(0xffffffffu - id);
}

__device__ __forceinline__ int mc_warp_sum(int x) {
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
__device__ __forceinline__ unsigned long long mc_warp_max(unsigned long long x) {
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, o);
    x = y > x ? y : x;
  }
  return x;
}

// ---- bitset adjacency ------------------------------------------------------------------------------------------------
// Row i of the (unsharded) store is read once, coalesced; each warp turns 32 consecutive elements into one word.
template <typename T>
__global__ void __launch_bounds__(kMcThreads) mc_adjacency_kernel(const T* __restrict__ S, long long ld, int m, int W,
                                                                  unsigned* __restrict__ adj, int* __restrict__ deg) {
  __shared__ int s_cnt;
  const int i = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const T* row = S + (size_t)i * (size_t)ld;
  unsigned* arow = adj + (size_t)i * W;
  int cnt = 0;
  for (int w = warp; w < W; w += kMcThreads / 32) {
    const int j = w * 32 + lane;
    const bool e = (j < m && j != i) ? mc_edge<T>(row[j]) : false;
    const unsigned bits = __ballot_sync(0xffffffffu, e);
    if (lane == 0) { arow[w] = bits; cnt += __popc(bits); }
  }
  if (lane == 0) atomicAdd(&s_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0) deg[i] = s_cnt;
}

// ---- k-core peeling ----------------------------------------------------------------------------------------------------
struct McPeelArgs {
  const unsigned* adj;
  int m, W;
  int* deg;           // current degree (in: full degree)
  unsigned* alive;    // [W] bitset of vertices still in the graph
  int* core;          // [m] out
  int* rnd;           // [m] out: iteration in which the vertex left (degeneracy order = (rnd, index) ascending)
  int* frontier;      // [m] vertices leaving in the current iteration
  unsigned* ctr;      // [3] rotating frontier counters (zeroed by the host)
  int* out;           // [2] max core, iterations
  TreeBar bar;
};

// Iteration `it` removes every vertex whose current degree is <= k (core number k), then subtracts the removed rows
// (ANDed with the alive mask) from the neighbours' degrees; an iteration that removes nothing raises k.  Every
// iteration removes a vertex or raises k (k < m), so there are at most 2m + 1 of them.
__global__ void __launch_bounds__(kMcPeelThreads) mc_peel_kernel(McPeelArgs a) {
  __shared__ int s_flag;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nthr = gridDim.x * blockDim.x;
  for (int w = tid; w < a.W; w += nthr) {
    const int left = a.m - w * 32;
    a.alive[w] = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
  }
  unsigned long long round = 1;
  grid_barrier(a.bar, round++, &s_flag);
  int k = 0, removed = 0, kmax = 0, it = 0;
  for (; removed < a.m && it <= 2 * a.m + 1; ++it) {
    unsigned* c = a.ctr + (it % 3);
    if (tid == 0) a.ctr[(it + 1) % 3] = 0u;  // last read two barriers ago
    for (int v = tid; v < a.m; v += nthr) {
      const unsigned bit = 1u << (v & 31);
      if ((__ldcg(&a.alive[v >> 5]) & bit) && __ldcg(&a.deg[v]) <= k) {
        a.core[v] = k; a.rnd[v] = it;
        a.frontier[atomicAdd(c, 1u)] = v;
        atomicAnd(&a.alive[v >> 5], ~bit);
      }
    }
    grid_barrier(a.bar, round++, &s_flag);
    if (*(volatile int*)&a.bar.sb->error) break;
    const int n = (int)__ldcg(c);
    if (n == 0) { ++k; continue; }
    kmax = k;
    removed += n;
    const long long work = (long long)n * a.W;
    for (long long q = tid; q < work; q += nthr) {
      const int f = (int)(q / a.W), w = (int)(q % a.W);
      const int v = __ldcg(&a.frontier[f]);
      unsigned bits = a.adj[(size_t)v * a.W + w] & __ldcg(&a.alive[w]);
      while (bits) {
        const int b = __ffs(bits) - 1;
        bits &= bits - 1u;
        atomicSub(&a.deg[w * 32 + b], 1);
      }
    }
    grid_barrier(a.bar, round++, &s_flag);
    if (*(volatile int*)&a.bar.sb->error) break;
  }
  if (tid == 0) { a.out[0] = kmax; a.out[1] = it; }
}

// ---- greedy heuristic ----------------------------------------------------------------------------------------------
// Seed v: K = {v}, P = N(v); while P is not empty take the u in P of highest core number (ties: lowest index),
// K += u, P &= N(u).  The largest K wins, ties to the smaller seed.  A seed is skipped when core(v) + 1 < best size and
// abandoned when |K| + |P| cannot beat the incumbent key: neither can change the winner, whatever the schedule.
// replay_seed >= 0: one warp re-runs that seed and writes its nodes in the order they were taken.
// One seed of the heuristic, run by one warp; P is the warp's W-word bitset.  best is the incumbent key: global memory
// (read through L2) for mc_heu_kernel, shared memory (SHARED_BEST) for the batched path.
template <bool SHARED_BEST>
__device__ __forceinline__ unsigned long long mc_load_best(const unsigned long long* best) {
  return SHARED_BEST ? *(const volatile unsigned long long*)best : __ldcg(best);
}
template <bool SHARED_BEST>
__device__ __forceinline__ void mc_heu_seed(const unsigned* __restrict__ adj, int m, int W, const int* __restrict__ core,
                                            int v, unsigned long long* best, bool replay, int* nodes_out, unsigned* P) {
  const int lane = threadIdx.x & 31;
  if (!replay && core[v] + 1 < (int)(mc_load_best<SHARED_BEST>(best) >> 32)) return;
  int psize = 0;
  for (int w = lane; w < W; w += 32) { const unsigned x = adj[(size_t)v * W + w]; P[w] = x; psize += __popc(x); }
  psize = mc_warp_sum(psize);
  int ksz = 1;
  if (replay && lane == 0) nodes_out[0] = v;
  bool abandoned = false;
  while (psize > 0) {  // |P| shrinks by at least one per step
    if (!replay && mc_key((unsigned)(ksz + psize), (unsigned)v) <= mc_load_best<SHARED_BEST>(best)) { abandoned = true; break; }
    unsigned long long bk = 0ull;
    for (int w = lane; w < W; w += 32) {
      unsigned bits = P[w];
      while (bits) {
        const int u = w * 32 + __ffs(bits) - 1;
        bits &= bits - 1u;
        const unsigned long long c = mc_key((unsigned)core[u], (unsigned)u);
        bk = c > bk ? c : bk;
      }
    }
    bk = mc_warp_max(bk);
    const int u = (int)(0xffffffffu - (unsigned)(bk & 0xffffffffull));
    if (replay && lane == 0) nodes_out[ksz] = u;
    ++ksz;
    psize = 0;
    for (int w = lane; w < W; w += 32) { const unsigned x = P[w] & adj[(size_t)u * W + w]; P[w] = x; psize += __popc(x); }
    psize = mc_warp_sum(psize);
  }
  if (!replay && !abandoned && lane == 0) atomicMax(best, mc_key((unsigned)ksz, (unsigned)v));
  if (replay && lane == 0) nodes_out[m] = ksz;  // size after the m node slots
}

__global__ void __launch_bounds__(kMcThreads) mc_heu_kernel(const unsigned* __restrict__ adj, int m, int W,
                                                            const int* __restrict__ core, const int* __restrict__ seeds,
                                                            unsigned long long* best, int replay_seed, int* nodes_out) {
  extern __shared__ unsigned mc_smem[];
  const int wib = threadIdx.x >> 5;
  unsigned* P = mc_smem + (size_t)wib * W;  // word w is only ever touched by lane w % 32
  const bool replay = replay_seed >= 0;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const int n = replay ? 1 : m;
  for (int s = blockIdx.x * (blockDim.x >> 5) + wib; s < n; s += nwarps)
    mc_heu_seed<false>(adj, m, W, core, replay ? replay_seed : seeds[s], best, replay, nodes_out, P);
}

// number of later neighbours (in degeneracy order) of every vertex: the candidate count of a search root
__global__ void __launch_bounds__(kMcThreads) mc_later_count_kernel(const unsigned* __restrict__ adj, int m, int W,
                                                                    const int* __restrict__ rnd, int* __restrict__ later) {
  const int lane = threadIdx.x & 31;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  for (int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < m; r += nwarps) {
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
    if (lane == 0) later[r] = cnt;
  }
}

// ---- exact branch-and-bound --------------------------------------------------------------------------------------------
// Task t is a root r (vertices in reverse degeneracy order with core(r) + 1 > lb) whose candidates are its later
// neighbours in degeneracy order (at most core(r) of them), or -- for a root with more than kMcSplit candidates -- the
// pair (r, j): r plus its j-th candidate x, with the candidates after x adjacent to x.  The local adjacency of the
// candidates is gathered into the worker's scratch; the search colours greedily (bitsets) and branches on the vertices
// of highest colour first.  The incumbent is the key (size, -t): a branch is cut when its bound cannot beat it, so the
// winning task (largest clique, ties to the smallest task) does not depend on the schedule once the search completes.
struct McSearchArgs {
  const unsigned* adj;
  int m, W;
  const int* rnd;               // removal iteration: u is later than r iff (rnd[u], u) > (rnd[r], r)
  const int* roots;             // [nroots] in task order
  const long long* tprefix;     // [nroots + 1] first task of each root
  int nroots;
  long long ntasks;
  int K, KW;                    // capacity of a local candidate set and words per local row
  unsigned arena_cap;           // entries of the colour-class arena per worker
  unsigned char* scratch;       // per worker: members[K] | adjL[K*KW] | P[(K+1)*KW] | level[(K+1)*3] | chosen[K+1] | arena
  size_t stride;
  unsigned long long* best;     // incumbent key
  unsigned long long* next_task;
  unsigned long long* n_branches;
  int* flags;                   // [0] deadline passed, [1] a colour-class arena overflowed (result not proven)
  const unsigned long long* deadline;  // absolute %globaltimer ns
  long long replay_task;        // >= 0: one warp re-runs this task against the fixed bound `replay_size` - 1
  int replay_size;
  int* nodes_out;               // replay: nodes (global indices) then the size at nodes_out[m]
};

__host__ __device__ inline size_t mc_scratch_bytes(int K, int KW, unsigned arena_cap) {
  const size_t words = (size_t)K + (size_t)K * KW + (size_t)(K + 1) * KW + (size_t)(K + 1) * 4 + arena_cap;
  return (words * 4 + 255) / 256 * 256;
}

// greedy sequential colouring of P (BBMC): class after class, repeatedly take the lowest vertex left that has no
// neighbour in the class.  Only vertices whose colour reaches cmin are listed (the others cannot lead to a better
// clique and stay in P); entries are (colour << 16 | vertex), ascending colour.  Returns the count, or -1 on overflow.
__device__ int mc_colour(const unsigned* P, const unsigned* adjL, int KW, int KWn, unsigned* U, unsigned* Q,
                         unsigned* out, long long cap, int cmin) {
  const int lane = threadIdx.x & 31;
  bool any = false;
  for (int w = lane; w < KWn; w += 32) { U[w] = P[w]; any |= P[w] != 0u; }
  int cnt = 0;
  int col = 0;
  while (__any_sync(0xffffffffu, any)) {  // every class takes at least one vertex out of U
    ++col;
    for (int w = lane; w < KWn; w += 32) Q[w] = U[w];
    int cw = 0;
    for (;;) {  // every step takes one vertex out of Q
      int v = -1;
      for (int c = cw & ~31; c < KWn; c += 32) {
        const unsigned x = (c + lane < KWn) ? Q[c + lane] : 0u;
        const unsigned bal = __ballot_sync(0xffffffffu, x != 0u);
        if (bal) {
          const int wl = __ffs(bal) - 1;
          const unsigned xw = __shfl_sync(0xffffffffu, x, wl);
          v = (c + wl) * 32 + __ffs(xw) - 1;
          cw = c + wl;
          break;
        }
      }
      if (v < 0) break;
      const int vw = v >> 5;
      const unsigned vb = 1u << (v & 31);
      for (int w = lane; w < KWn; w += 32) {
        unsigned nb = adjL[(size_t)v * KW + w];
        if (w == vw) { nb |= vb; U[w] &= ~vb; }
        Q[w] &= ~nb;
      }
      if (col >= cmin) {
        if (cnt >= cap) return -1;
        if (lane == 0) out[cnt] = ((unsigned)col << 16) | (unsigned)v;
        ++cnt;
      }
    }
    any = false;
    for (int w = lane; w < KWn; w += 32) any |= U[w] != 0u;
  }
  __syncwarp();
  return cnt;
}

// smallest colour that can still beat `best` for a clique of dsz vertices plus the coloured ones (task t)
__device__ __forceinline__ int mc_cmin(unsigned long long best, int dsz, long long t) {
  const int bs = (int)(best >> 32);
  const unsigned mine = 0xffffffffu - (unsigned)t, theirs = (unsigned)(best & 0xffffffffull);
  const int c = bs - dsz + (mine > theirs ? 0 : 1);
  return c < 1 ? 1 : c;
}

__device__ __forceinline__ unsigned long long mc_read_best(const McSearchArgs& a, bool replay) {
  return replay ? mc_key((unsigned)(a.replay_size - 1), 0u) : __ldcg(a.best);
}

// returns false when the deadline passed
__device__ bool mc_search_task(const McSearchArgs& a, long long t, unsigned* U, unsigned* Q, unsigned char* base_ptr,
                               unsigned long long* branches) {
  const int lane = threadIdx.x & 31;
  const bool replay = a.replay_task >= 0;
  int* members = reinterpret_cast<int*>(base_ptr);
  unsigned* adjL = reinterpret_cast<unsigned*>(members + a.K);
  unsigned* Pst = adjL + (size_t)a.K * a.KW;
  int* lvl = reinterpret_cast<int*>(Pst + (size_t)(a.K + 1) * a.KW);  // (arena offset, count, cursor) per level
  int* Kst = lvl + (size_t)(a.K + 1) * 3;                               // candidate chosen at each level
  unsigned* arena = reinterpret_cast<unsigned*>(Kst + (a.K + 1));

  // decode the task: root index by binary search over the prefix
  int lo = 0, hi = a.nroots - 1;
  while (lo < hi) {  // largest i with tprefix[i] <= t
    const int mid = (lo + hi + 1) >> 1;
    if (a.tprefix[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const int r = a.roots[lo];
  const bool split = a.tprefix[lo + 1] - a.tprefix[lo] > 1;
  const int j = split ? (int)(t - a.tprefix[lo]) : -1;

  // candidates of the root: later neighbours, ascending index
  const int rr = a.rnd[r];
  int n = 0;
  for (int c = 0; c < a.W; c += 32) {
    const int w = c + lane;
    unsigned bits = w < a.W ? a.adj[(size_t)r * a.W + w] : 0u, keep = 0u;
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1u;
      const int u = w * 32 + b, ru = a.rnd[u];
      if (ru > rr || (ru == rr && u > r)) keep |= 1u << b;
    }
    int pre = __popc(keep);
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += y; }
    const int tot = __shfl_sync(0xffffffffu, pre, 31);
    if (n + tot > a.K) { if (lane == 0) atomicExch(&a.flags[1], 1); return true; }  // cannot happen: n <= core(r)
    int pos = n + pre - __popc(keep);
    while (keep) { const int b = __ffs(keep) - 1; keep &= keep - 1u; members[pos++] = w * 32 + b; }
    n += tot;
  }
  __syncwarp();
  int base = 1;
  int x = -1;
  if (split) {
    if (j >= n) return true;
    if (mc_key((unsigned)(2 + n - j - 1), (unsigned)t) <= mc_read_best(a, replay)) return true;
    x = members[j];
    int cnt = 0;
    for (int c = j + 1; c < n; c += 32) {
      const int i = c + lane;
      const int u = i < n ? members[i] : 0;
      const bool e = i < n && ((a.adj[(size_t)x * a.W + (u >> 5)] >> (u & 31)) & 1u);
      const unsigned bal = __ballot_sync(0xffffffffu, e);
      __syncwarp();
      if (e) members[cnt + __popc(bal & ((1u << lane) - 1u))] = u;
      cnt += __popc(bal);
      __syncwarp();
    }
    n = cnt;
    base = 2;
  }
  if (mc_key((unsigned)(base + n), (unsigned)t) <= mc_read_best(a, replay)) return true;
  const int KWn = (n + 31) >> 5;

  // local adjacency: row a is the candidates adjacent to candidate a
  for (int ia = 0; ia < n; ++ia) {
    const int ga = members[ia];
    for (int c = 0; c < KWn; ++c) {
      const int b = c * 32 + lane;
      bool e = false;
      if (b < n && b != ia) { const int gb = members[b]; e = (a.adj[(size_t)ga * a.W + (gb >> 5)] >> (gb & 31)) & 1u; }
      const unsigned bal = __ballot_sync(0xffffffffu, e);
      if (lane == 0) adjL[(size_t)ia * a.KW + c] = bal;
    }
  }
  for (int w = lane; w < KWn; w += 32) {
    const int left = n - w * 32;
    Pst[w] = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
  }
  __syncwarp();

  if (n == 0) {
    const unsigned long long k = mc_key((unsigned)base, (unsigned)t);
    if (k > mc_read_best(a, replay)) {
      if (!replay) { if (lane == 0) atomicMax(a.best, k); }
      else if (lane == 0) { a.nodes_out[0] = r; if (base == 2) a.nodes_out[1] = x; a.nodes_out[a.m] = base; }
    }
    return true;
  }

  // level 0
  {
    const int c0 = mc_colour(Pst, adjL, a.KW, KWn, U, Q, arena, a.arena_cap, mc_cmin(mc_read_best(a, replay), base, t));
    if (c0 < 0) { if (lane == 0) atomicExch(&a.flags[1], 1); return true; }
    if (lane == 0) { lvl[0] = 0; lvl[1] = c0; lvl[2] = c0 - 1; }
    __syncwarp();
  }
  int d = 0;
  unsigned long long steps = 0, nb = 0;
  while (d >= 0) {  // the search tree is finite: every level has a strictly smaller candidate set
    if (!replay && (++steps & 63ull) == 0ull) {
      int stop = 0;
      if (lane == 0) stop = (__ldcg(&a.flags[0]) != 0) || (global_ns() > *a.deadline);
      stop = __shfl_sync(0xffffffffu, stop, 0);
      if (stop) { if (lane == 0) atomicExch(&a.flags[0], 1); *branches += nb; return false; }
    }
    int* L = lvl + (size_t)d * 3;
    const int off = L[0], cur = L[2];
    if (cur < 0) { --d; continue; }
    const unsigned e = arena[off + cur];
    const int col = (int)(e >> 16), v = (int)(e & 0xffffu);
    const unsigned long long best = mc_read_best(a, replay);
    if (mc_key((unsigned)(base + d + col), (unsigned)t) <= best) { --d; continue; }  // the rest have colours <= col
    __syncwarp();
    ++nb;
    if (lane == 0) { L[2] = cur - 1; Kst[d] = v; }
    const unsigned* Pd = Pst + (size_t)d * a.KW;
    unsigned* Pn = Pst + (size_t)(d + 1) * a.KW;
    int cnt = 0;
    for (int w = lane; w < KWn; w += 32) {
      const unsigned p = Pd[w];
      const unsigned nw = p & adjL[(size_t)v * a.KW + w];
      Pn[w] = nw;
      cnt += __popc(nw);
      if (w == (v >> 5)) Pst[(size_t)d * a.KW + w] = p & ~(1u << (v & 31));
    }
    cnt = mc_warp_sum(cnt);
    __syncwarp();
    if (cnt == 0) {
      const unsigned long long k = mc_key((unsigned)(base + d + 1), (unsigned)t);
      if (k > best) {
        if (!replay) { if (lane == 0) atomicMax(a.best, k); }
        else {
          if (lane == 0) {
            a.nodes_out[0] = r;
            if (base == 2) a.nodes_out[1] = x;
            for (int q = 0; q <= d; ++q) a.nodes_out[base + q] = members[Kst[q]];
            a.nodes_out[a.m] = base + d + 1;
          }
          *branches += nb;
          return true;
        }
      }
      continue;
    }
    if (mc_key((unsigned)(base + d + 1 + cnt), (unsigned)t) <= best) continue;
    if (d + 1 >= a.K) { if (lane == 0) atomicExch(&a.flags[1], 1); continue; }  // cannot happen: depth < n
    const int noff = off + L[1];
    const int c = mc_colour(Pn, adjL, a.KW, KWn, U, Q, arena + noff, (long long)a.arena_cap - noff,
                            mc_cmin(mc_read_best(a, replay), base + d + 1, t));
    if (c < 0) { if (lane == 0) atomicExch(&a.flags[1], 1); continue; }
    if (c == 0) continue;
    if (lane == 0) { int* N = L + 3; N[0] = noff; N[1] = c; N[2] = c - 1; }
    __syncwarp();
    ++d;
  }
  *branches += nb;
  return true;
}

__global__ void __launch_bounds__(kMcSearchWarps * 32) mc_search_kernel(McSearchArgs a) {
  extern __shared__ unsigned mc_smem[];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  unsigned* U = mc_smem + (size_t)wib * 2 * a.KW;
  unsigned* Q = U + a.KW;
  const long long worker = (long long)blockIdx.x * kMcSearchWarps + wib;
  unsigned char* base = a.scratch + (size_t)worker * a.stride;
  unsigned long long branches = 0;
  if (a.replay_task >= 0) {
    if (worker == 0) mc_search_task(a, a.replay_task, U, Q, base, &branches);
    return;
  }
  for (;;) {  // at most ntasks draws in total
    unsigned long long t = 0;
    if (lane == 0) t = atomicAdd(a.next_task, 1ull);
    t = __shfl_sync(0xffffffffu, t, 0);
    if ((long long)t >= a.ntasks) break;
    if (!mc_search_task(a, (long long)t, U, Q, base, &branches)) break;
  }
  if (lane == 0) atomicAdd(a.n_branches, branches);
}

__global__ void mc_deadline_kernel(unsigned long long* deadline, unsigned long long limit_ns) {
  const unsigned long long now = global_ns();
  *deadline = (limit_ns > ~0ull - now) ? ~0ull : now + limit_ns;
}

}  // namespace clp
