// clp_batch.cuh -- many small problems in ONE launch (SURVEY.md section 8f rank 4).
//
// The reference's own operating point is m <= 2048 associations per registration (benchmarks/main.cpp:206-208, README.md:85)
// and its benchmark solves such problems one after the other (main.cpp:254-270).  One problem of that size cannot fill
// an H100: as a stand-alone launch it pays a device-wide synchronisation per objective evaluation and leaves most of
// the 132 SMs idle.  Here ONE CTA owns one problem from the raw inputs to the final iterate:
//     gather the association endpoints -> score all pairs (fp32 screening, exact fp64 for the survivors: the arithmetic
//     of score_tile_kernel) into a per-CTA fp32 scratch matrix -> build the full-row sliced-ELL copy (counting sort of
//     the rows by length, item lengths, scan, item-wise fill: the steps of clp_sparse.cuh as device functions) ->
//     run findDenseClique with the resident-vector solver body (clp_resident.cuh, SOLO: every "device-wide" exchange is
//     a __syncthreads-level block reduction)
// and the CTAs of a persistent grid draw problems from a counter: hundreds of problems per launch, no host in
// between, no device-wide barrier anywhere.  Each problem's result is bit-identical to what the single-problem path
// (sweep mode 6) computes for it with one CTA.
#pragma once

namespace clp {

constexpr int kBatchThreads = 256;
constexpr int kBatchWarps = kBatchThreads / 32;
constexpr int kBatchMaxM = 4096;      // largest problem a batch may hold (shared-memory tables of the in-CTA build)
constexpr int kBatchU = 2, kBatchD = 3;

struct BatchProblem {       // device array, one per problem; offsets into the concatenated input / output arrays
  long long d1_off, d2_off; // in doubles
  long long a_off;          // in int32 (column-major m x 2), -1: all-to-all hypothesis (utils.h:61-71)
  long long u_off;          // in doubles: u0 in, final iterate out
  int n1, n2, m, pad_;
};

// per-CTA scratch in HBM, sized for the largest problem of the batch
struct BatchLayout {
  size_t E1, E2, F1, F2, A, M, rowid, itemptr, ctafirst, val, idx, vecs, cand, pieces, total;
  int ld_max, rows_pad_max;
};
__host__ __device__ inline size_t batch_align(size_t x) { return (x + 255) & ~(size_t)255; }
__host__ __device__ inline BatchLayout batch_layout(int max_m, int dd) {
  BatchLayout L;
  const size_t mm = (size_t)max_m;
  L.ld_max = (int)((mm + 127) / 128 * 128);
  L.rows_pad_max = (int)((mm + 3) / 4 * 4);
  const size_t ni = (size_t)L.rows_pad_max / 4;
  size_t o = 0;
  L.E1 = o; o = batch_align(o + mm * dd * 8);
  L.E2 = o; o = batch_align(o + mm * dd * 8);
  L.F1 = o; o = batch_align(o + mm * 16);
  L.F2 = o; o = batch_align(o + mm * 16);
  L.A = o; o = batch_align(o + 2 * mm * 4);
  L.M = o; o = batch_align(o + (size_t)L.rows_pad_max * L.ld_max * 4);
  L.rowid = o; o = batch_align(o + (size_t)L.rows_pad_max * 4);
  L.itemptr = o; o = batch_align(o + (ni + 1) * 4);
  L.ctafirst = o; o = batch_align(o + 16);
  const size_t cap = (size_t)L.rows_pad_max * ((mm + 3) / 4 * 4) + 64;  // entries: every row padded to whole chunks
  L.val = o; o = batch_align(o + cap * 4);
  L.idx = o; o = batch_align(o + cap * 2);
  const size_t mpad = (mm + 127) / 128 * 128;
  L.vecs = o; o = batch_align(o + (size_t)R_SLOTS * mpad * 8);
  L.cand = o; o = batch_align(o + 4 * mpad * 8);
  L.pieces = o; o = batch_align(o + (ni + kBatchWarps + 8) * kPieceVals * 8);
  L.total = o;
  return L;
}

// dynamic shared memory of a batch CTA: the solver's plan (clp_resident.cuh) and the build tables overlay each other
struct BatchSmem { unsigned int cnt, queue, tile, hist, scan, ring, total; };
__host__ __device__ inline BatchSmem batch_smem_plan(int max_m) {
  BatchSmem b;
  const unsigned int rows_pad = (unsigned int)((max_m + 3) / 4 * 4);
  const unsigned int nb = (unsigned int)(((max_m + 127) / 128 * 128) / 4 + 2);
  unsigned int o = 0;
  b.cnt = o; o += rows_pad * 4; o = (o + 15u) & ~15u;            // kept entries per row
  b.queue = o; o += kBatchWarps * 128 * 2;                         // scoring: survivor queue per warp
  b.tile = o; o += kBatchWarps * 128 * 4;                          // scoring: 128 columns of the row per warp
  b.hist = o; o += (nb + 1) * 4; o = (o + 15u) & ~15u;            // counting sort of the rows by length
  b.scan = o; o += 64;                                             // block scan scratch
  b.ring = o; o += kFillWarps * 4 * kRing * (4 + 2);               // item-wise fill rings
  const unsigned int solve = res_smem_plan(max_m, kBatchWarps).total;
  b.total = (o > solve ? o : solve) + 128;
  return b;
}

struct BatchArgs {
  const BatchProblem* prob;
  int nprob;
  const double* D1; const double* D2; const int* A; const double* u0;
  double* u_out;
  SolverOut* out;          // [nprob]
  unsigned int* nnz_out;   // [nprob] kept entries (i != j, both triangles) -- diagnostics
  int* next;               // problem counter
  unsigned long long* prof;  // nullable: [nprob][4] ns spent in gather+score, build, solve, whole problem -- diagnostics
  unsigned char* scratch; size_t scratch_stride;
  int max_m, kind, dd;     // kind 0: EuclideanDistance (dd = 2, 3), 1: PointNormalDistance (dd = 6)
  SolverParams prm;
  double p0, p1, p2, p3, affinityeps;
  SyncBlock* sb;
  long long spin_limit;
};

// block-wide exclusive scan of x over the threads (256), result for this thread; total in *total_out (shared)
__device__ __forceinline__ unsigned int batch_block_exscan(unsigned int x, unsigned int* sc /*[kBatchWarps + 1]*/) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned int inc = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
  __syncthreads();
  if (lane == 31) sc[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int run = 0;
    for (int q = 0; q < kBatchWarps; ++q) { const unsigned int t = sc[q]; sc[q] = run; run += t; }
    sc[kBatchWarps] = run;
  }
  __syncthreads();
  return sc[w] + (inc - x);
}

template <int KIND, int DD>
__global__ void __launch_bounds__(kBatchThreads, 3) batch_solve_kernel(BatchArgs ba) {
  extern __shared__ __align__(128) unsigned char clp_batch_smem[];
  unsigned char* smem = clp_batch_smem;
  __shared__ ResArgs sa;
  __shared__ int s_p;
  __shared__ float s_R;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const BatchLayout L = batch_layout(ba.max_m, DD);
  unsigned char* sc = ba.scratch + (size_t)blockIdx.x * ba.scratch_stride;
  double* E1 = reinterpret_cast<double*>(sc + L.E1);
  double* E2 = reinterpret_cast<double*>(sc + L.E2);
  float4* F1 = reinterpret_cast<float4*>(sc + L.F1);
  float4* F2 = reinterpret_cast<float4*>(sc + L.F2);
  int* Ag = reinterpret_cast<int*>(sc + L.A);
  float* M = reinterpret_cast<float*>(sc + L.M);
  unsigned int* rowid = reinterpret_cast<unsigned int*>(sc + L.rowid);
  unsigned int* itemptr = reinterpret_cast<unsigned int*>(sc + L.itemptr);
  unsigned int* ctafirst = reinterpret_cast<unsigned int*>(sc + L.ctafirst);
  float* val = reinterpret_cast<float*>(sc + L.val);
  unsigned short* idx = reinterpret_cast<unsigned short*>(sc + L.idx);

  for (;;) {
    __syncthreads();
    if (tid == 0) s_p = atomicAdd(ba.next, 1);
    __syncthreads();
    const int p = s_p;
    if (p >= ba.nprob) break;
    const BatchProblem P = ba.prob[p];
    const unsigned long long t_begin = global_ns();
    const int m = P.m;
    const int ld = (m + 127) / 128 * 128;
    const int rows_pad = (m + 3) / 4 * 4;
    const int NI = rows_pad / 4;
    const double* D1 = ba.D1 + P.d1_off;
    const double* D2 = ba.D2 + P.d2_off;

    // ---- 1. endpoints of every association (gather_endpoints_kernel), fp32 positions, R = max |coordinate|
    float big = 0.f;
    int bad = 0;
    for (int i = tid; i < m; i += kBatchThreads) {
      int a0, a1;
      if (P.a_off >= 0) { a0 = ba.A[P.a_off + i]; a1 = ba.A[P.a_off + m + i]; }
      else { a0 = i / P.n2; a1 = i % P.n2; }
      Ag[i] = a0; Ag[m + i] = a1;
      if (a0 < 0 || a0 >= P.n1 || a1 < 0 || a1 >= P.n2) { bad = 1; a0 = 0; a1 = 0; }
      float f1[3] = {0.f, 0.f, 0.f}, f2[3] = {0.f, 0.f, 0.f};
#pragma unroll
      for (int q = 0; q < DD; ++q) {
        const double x1 = D1[(size_t)a0 * DD + q], x2 = D2[(size_t)a1 * DD + q];
        E1[(size_t)i * DD + q] = x1; E2[(size_t)i * DD + q] = x2;
        if (q < 3) {
          f1[q] = (float)x1; f2[q] = (float)x2;
          const float m1 = fabsf(f1[q]), m2 = fabsf(f2[q]);
          big = fmaxf(big, (m1 == m1) ? m1 : __int_as_float(0x7f800000));
          big = fmaxf(big, (m2 == m2) ? m2 : __int_as_float(0x7f800000));
        }
      }
      F1[i] = make_float4(f1[0], f1[1], f1[2], 0.f);
      F2[i] = make_float4(f2[0], f2[1], f2[2], 0.f);
    }
    if (bad) atomicExch(&ba.sb->error, 2);
    {
      float* redf = reinterpret_cast<float*>(smem + batch_smem_plan(ba.max_m).scan);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) big = fmaxf(big, __shfl_xor_sync(0xffffffffu, big, o));
      if (lane == 0) redf[warp] = big;
      __syncthreads();
      if (tid == 0) { float t = 0.f; for (int w = 0; w < kBatchWarps; ++w) t = fmaxf(t, redf[w]); s_R = t; }
      __syncthreads();
    }

    // ---- 2. scoring: warp per row, 128 columns per step; screening + survivor queue as in score_tile_kernel.
    //      A row's warp evaluates its diagonal block of 128 columns and the blocks to the right of it; an entry kept in
    //      a block right of the diagonal block is also stored transposed (the pair functions are symmetric bit for bit:
    //      squared differences and commutative products), so every pair outside the diagonal blocks is evaluated once
    //      (ref clipper.cpp:31-56 fills the upper triangle and mirrors it).
    const BatchSmem bs = batch_smem_plan(ba.max_m);
    unsigned int* cnt = reinterpret_cast<unsigned int*>(smem + bs.cnt);                          // [rows_pad]
    unsigned short* queue = reinterpret_cast<unsigned short*>(smem + bs.queue) + warp * 128;
    float* tile = reinterpret_cast<float*>(smem + bs.tile) + warp * 128;
    for (int i = tid; i < rows_pad; i += kBatchThreads) cnt[i] = 0u;
    {
      const float4 neutral4 = make_float4(-0.0f, -0.0f, -0.0f, -0.0f);
      for (int i = 128 + warp; i < m; i += kBatchWarps) {  // the blocks left of the diagonal block: transposed stores only
        const int jd = i & ~127;
        for (int j = lane * 4; j < jd; j += 128) *reinterpret_cast<float4*>(M + (size_t)i * ld + j) = neutral4;
      }
    }
    __syncthreads();
    {
      const float R = s_R;
      const double eps = ba.p1;  // epsilon (Euclidean) / epsp (PointNormal): the position-consistency bound
      const float thr = __double2float_ru((eps + 1024.0 * 5.9604644775390625e-08 * (double)R) * (1.0 + 9.5367431640625e-07));
      for (int i = warp; i < rows_pad; i += kBatchWarps) {
        unsigned int kept = 0;
        if (i < m) {
          const int ai0 = Ag[i], ai1 = Ag[m + i];
          const float4 f1i = F1[i], f2i = F2[i];
          const int jdiag = i & ~127;
          for (int j0 = jdiag; j0 < ld; j0 += 128) {
            unsigned int qn = 0;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int j = j0 + lane * 4 + e;
              tile[lane * 4 + e] = -0.0f;
              bool cand = false;
              if (j < m && j != i) {
                const int aj0 = Ag[j], aj1 = Ag[m + j];
                const float4 f1j = F1[j], f2j = F2[j];
                const float x1 = f1i.x - f1j.x, y1 = f1i.y - f1j.y, z1 = f1i.z - f1j.z;
                const float x2 = f2i.x - f2j.x, y2 = f2i.y - f2j.y, z2 = f2i.z - f2j.z;
                const float l1 = sqrt_approx(fmaf(z1, z1, fmaf(y1, y1, x1 * x1)));
                const float l2 = sqrt_approx(fmaf(z2, z2, fmaf(y2, y2, x2 * x2)));
                cand = ai0 != aj0 && ai1 != aj1 && !(fabsf(l1 - l2) >= thr);  // distinctness: ref clipper.cpp:35-38
              }
              const unsigned int vote = __ballot_sync(0xffffffffu, cand);
              if (cand) queue[qn + __popc(vote & ((1u << lane) - 1u))] = (unsigned short)((e << 5) | lane);
              qn += __popc(vote);
            }
            __syncwarp();
            for (unsigned int k = lane; k < qn; k += 32) {
              const unsigned int code = queue[k];
              const int e = code >> 5, l = code & 31;
              const int j = j0 + l * 4 + e;
              double e1i[DD], e2i[DD], e1j[DD], e2j[DD];
#pragma unroll
              for (int t = 0; t < DD; ++t) {
                e1i[t] = E1[(size_t)i * DD + t]; e2i[t] = E2[(size_t)i * DD + t];
                e1j[t] = E1[(size_t)j * DD + t]; e2j[t] = E2[(size_t)j * DD + t];
              }
              double scr;
              if (KIND == 0) {
                const double l1 = point_dist<DD>(e1i, e1j, 0), l2 = point_dist<DD>(e2i, e2j, 0);
                scr = euclid_score(l1, l2, ba.p0, ba.p1, ba.p2);
              } else {
                const double l1 = point_dist<3>(e1i, e1j, 0), l2 = point_dist<3>(e2i, e2j, 0);
                const double dot1 = __dadd_rn(__dadd_rn(__dmul_rn(e1i[3 % DD], e1j[3 % DD]), __dmul_rn(e1i[4 % DD], e1j[4 % DD])), __dmul_rn(e1i[5 % DD], e1j[5 % DD]));
                const double dot2 = __dadd_rn(__dadd_rn(__dmul_rn(e2i[3 % DD], e2j[3 % DD]), __dmul_rn(e2i[4 % DD], e2j[4 % DD])), __dmul_rn(e2i[5 % DD], e2j[5 % DD]));
                scr = pointnormal_score(l1, l2, dot1, dot2, ba.p0, ba.p1, ba.p2, ba.p3);
              }
              if (scr > ba.affinityeps) {  // ref clipper.cpp:53-55
                const float enc = encode<float>(scr, true);
                tile[l * 4 + e] = enc;
                if (j0 != jdiag) { M[(size_t)j * ld + i] = enc; atomicAdd(&cnt[j], 1u); }
              }
            }
            __syncwarp();
            const float4 o4 = *reinterpret_cast<const float4*>(tile + lane * 4);
            *reinterpret_cast<float4*>(M + (size_t)i * ld + j0 + lane * 4) = o4;
            kept += (is_neutral<float>(o4.x) ? 0u : 1u) + (is_neutral<float>(o4.y) ? 0u : 1u) +
                    (is_neutral<float>(o4.z) ? 0u : 1u) + (is_neutral<float>(o4.w) ? 0u : 1u);
            __syncwarp();
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
        }
        if (lane == 0 && kept) atomicAdd(&cnt[i], kept);
      }
    }
    __syncthreads();

    const unsigned long long t_scored = global_ns();
    // ---- 3. full-row sliced-ELL copy: sort rows by length (longest first), items of four, scan, fill
    const int nb = ld / 4 + 2;
    unsigned int* hist = reinterpret_cast<unsigned int*>(smem + bs.hist);                         // [nb + 1]
    unsigned int* scs = reinterpret_cast<unsigned int*>(smem + bs.scan);
    {
      unsigned int mine = 0;
      for (int i = tid; i <= nb; i += kBatchThreads) hist[i] = 0u;
      __syncthreads();
      for (int r = tid; r < rows_pad; r += kBatchThreads) { mine += cnt[r]; atomicAdd(&hist[min((cnt[r] + 3u) >> 2, (unsigned int)(nb - 1))], 1u); }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
      if (lane == 0 && mine) atomicAdd(&ba.nnz_out[p], mine);
      __syncthreads();
      // start of every length class, longest first: exclusive scan of the histogram read backwards
      const int per = (nb + kBatchThreads - 1) / kBatchThreads;
      const int r0 = tid * per;
      unsigned int local = 0;
      for (int q = 0; q < per; ++q) { const int r = r0 + q; if (r < nb) local += hist[nb - 1 - r]; }
      unsigned int run = batch_block_exscan(local, scs);
      for (int q = 0; q < per; ++q) {
        const int r = r0 + q;
        if (r < nb) { const unsigned int hc = hist[nb - 1 - r]; hist[nb - 1 - r] = run; run += hc; }
      }
      __syncthreads();
      // stable placement, as in sell_sort_kernel: tiles of 256 rows in row order, the warps take turns
      for (int base = 0; base < rows_pad; base += kBatchThreads) {
        const int r = base + tid;
        const bool have = r < rows_pad;
        const unsigned int cls = have ? min((cnt[r] + 3u) >> 2, (unsigned int)(nb - 1)) : 0xffffffffu;
        const unsigned int peers = __match_any_sync(0xffffffffu, cls);
        const int leader = __ffs(peers) - 1;
        const unsigned int before = __popc(peers & ((1u << lane) - 1u));
        unsigned int start = 0u;
        for (int w = 0; w < kBatchWarps; ++w) {
          if (warp == w && have && lane == leader) { start = hist[cls]; hist[cls] = start + __popc(peers); }
          __syncthreads();
        }
        start = __shfl_sync(0xffffffffu, start, leader);
        if (have) rowid[start + before] = (unsigned int)r;
      }
      __syncthreads();
      // item lengths (4 x the longest = first member), exclusive scan into itemptr[0..NI]
      const int peri = (NI + 1 + kBatchThreads - 1) / kBatchThreads;
      const int i0 = tid * peri;
      unsigned int loc = 0;
      for (int q = 0; q < peri; ++q) { const int it = i0 + q; if (it < NI) loc += 4u * ((cnt[rowid[4 * it]] + 3u) >> 2); }
      unsigned int runi = batch_block_exscan(loc, scs);
      for (int q = 0; q < peri; ++q) {
        const int it = i0 + q;
        if (it <= NI) { itemptr[it] = runi; if (it < NI) runi += 4u * ((cnt[rowid[4 * it]] + 3u) >> 2); }
      }
      if (tid == 0) { ctafirst[0] = 0u; ctafirst[1] = (unsigned int)NI; }
      __syncthreads();
    }
    {
      // item-wise fill by the first kFillWarps warps
      unsigned char* ringbase = smem + bs.ring;
      float (*ringv)[4][kRing] = reinterpret_cast<float (*)[4][kRing]>(ringbase);
      unsigned short (*ringo)[4][kRing] = reinterpret_cast<unsigned short (*)[4][kRing]>(ringbase + (size_t)kFillWarps * 4 * kRing * 4);
      if (warp < kFillWarps) {
        for (int it = warp; it < NI; it += kFillWarps) {
          unsigned int r[4];
#pragma unroll
          for (int s_ = 0; s_ < 4; ++s_) r[s_] = rowid[4 * it + s_];
          sell_fill_item_warp<float>(M, ld, m, 0, m, itemptr[it], itemptr[it + 1], r, val, idx, 0, (unsigned int)m,
                                     ringv[warp], ringo[warp]);
        }
      }
    }
    __threadfence_block();
    __syncthreads();

    // ---- 4. the solver (clp_resident.cuh, SOLO): arguments in shared memory
    if (tid == 0) {
      ResArgs a;
      a.sp.val = val; a.sp.off16 = idx; a.sp.itemptr = itemptr; a.sp.rowid = rowid; a.sp.rows_pad = rows_pad; a.sp.plain = 1;
      a.sp.cta_first = ctafirst;
      a.m = m; a.row0 = 0; a.rows = m; a.rows_pad = rows_pad; a.NI = NI; a.G = 1;
      a.prm = ba.prm;
      a.u0 = ba.u0 + P.u_off;
      a.vecs = reinterpret_cast<double*>(sc + L.vecs);
      a.cand = reinterpret_cast<double*>(sc + L.cand);
      a.ll = nullptr;
      a.mpad = (long long)ld;
      a.pieces = reinterpret_cast<double*>(sc + L.pieces);
      a.sb = ba.sb;
      a.u_final = ba.u_out + P.u_off;
      a.out = ba.out + p;
      a.rank = 0; a.world = 1;
      for (int r = 0; r < kMaxPeers; ++r) { a.peer_ll[r] = nullptr; a.peer_comm[r] = nullptr; }
      a.comm = nullptr; a.seq0 = 0; a.spin_limit = ba.spin_limit; a.pieces_cap = 0u; a.state_cap = 0u; a.redll = nullptr; a.prof_cta = nullptr; a.prof_laps = 0;
      sa = a;
    }
    __syncthreads();
    const unsigned long long t_built = global_ns();
    res_solve_body<float, kBatchThreads, kBatchU, kBatchD, false, true, /*coherent loads*/ true>(sa, smem);
    if (ba.prof && tid == 0) {
      const unsigned long long t_end = global_ns();
      ba.prof[(size_t)p * 4 + 0] = t_scored - t_begin; ba.prof[(size_t)p * 4 + 1] = t_built - t_scored;
      ba.prof[(size_t)p * 4 + 2] = t_end - t_built; ba.prof[(size_t)p * 4 + 3] = t_end - t_begin;
    }
  }
}

}  // namespace clp
