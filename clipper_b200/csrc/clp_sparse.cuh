// clp_sparse.cuh -- compact copy of the affinity matrix and its sweep (SURVEY section 8f rank 3).
//
// The consistency graph is sparse (14.9 % at BASELINE.json's config 2), so after the dense build the
// non-neutral entries (everything except the -0.0 "inconsistent" code) of every local row are compacted into
//      val[]  : the stored element itself (fp32 / fp64; sign bit = constraint bit, as in the dense store)
//      off16[]: 8 * (column - first column of its segment) -- the byte offset of v[column] inside the
//               shared-memory copy of the segment (segments are <= 4096 columns wide)
// = 6 bytes per kept entry (fp32 storage) instead of 4 bytes per matrix element.
//
// Layout (a sliced-ELL variant: SELL-4 with the sort window = one whole column segment):
//  * the columns are cut into the NSEG segments of the Plan; a "slice" is one row x one segment, stored in
//    CHUNKS of 4 entries (16-byte value load + 8-byte offset load); the last chunk is padded with neutral
//    entries that point at a zero slot behind the staged segment;
//  * inside a segment the rows are SORTED by slice length (descending) and taken four at a time: an ITEM.
//    The four slices of an item are padded to the longest of them (neighbours in sorted order: < 1 % padding)
//    and interleaved chunk by chunk: chunk k of member s sits at chunk position 4 k + s of the item.
//    An item is therefore ONE contiguous run of HBM that a warp streams with perfectly coalesced loads
//    (lane l reads chunks l, l+32, ... -> always member l & 3), each lane keeps just two accumulators, and
//    the row sums need a 3-step butterfly over the 8 lanes of a member instead of the 18 shuffles of the
//    row-major variant; the registers saved buy a deeper unroll (more bytes in flight per warp).
//  * items of segment 0, then segment 1, ...: one stream, itemptr[seg][i] = first chunk of item i
//    (cumulative over everything before it), rowid[seg][4 i + s] = local row of member s.
// Row densities differ a lot (config 2: 93 +- 24 chunks per slice), which is why the rows are sorted and why
// the sweep is split by bytes, not by row count (sparse_partition_kernel).
// The sum of a row does not depend on which item it landed in nor on the (atomic, unordered) tie-breaking of
// the sort: its chunks k go to accumulator lane k mod 8 in increasing k, then the fixed butterfly.
// "plain" matrices (every kept entry has M > 0 and C = 1 -- always true after scorePairwiseConsistency) take
// a shorter path: Chat v is then just the sum of the gathered v.
// Algorithmic bytes per objective evaluation: 6 * stored entries + 20 * NSEG * rows / 4.
// Whole-row layout of a plain fp32 matrix (the resident solver's): PACKED 4-byte entries instead (column delta + exponent
// code + mantissa, no off16; see pack_word below), which needs one filler per empty 16-column window of a row: the
// counting pass records the occupied windows and the exponent range, the sort and the item lengths count the fillers
// when the matrix qualifies (PackCount, decided on the device; the host reads the decision back with the totals).
#pragma once

namespace clp {

constexpr unsigned int kZeroSlot = kSegMax * 8;  // byte offset of the zero element behind the staged segment
constexpr int kSellUnroll = 3;                   // chunks per lane and round; two rounds are in flight
constexpr unsigned int kItemCost = 128;          // fixed cost of an item (pointer fetch, pipeline restart, reduction, store) in chunks;
                                                 // too small a charge leaves the CTAs holding many short items running long;
                                                 // irrelevant for the whole-row layout

struct SparseView {
  const void* val;               // T [4 * chunks]
  const unsigned short* off16;   // [4 * chunks]
  const unsigned int* itemptr;   // [NSEG][NI + 1], NI = rows_pad / 4
  const unsigned int* rowid;     // [NSEG][rows_pad]
  int rows_pad;
  int plain;                     // every kept entry has M > 0 and C = 1
  const unsigned int* cta_first; // [G + 1] first item of every CTA (balanced by bytes), see sparse_partition_kernel
  int packed;                    // whole-row layout with 4-byte entries (val holds the words, no off16; see pack_word)
  unsigned int ebias;            // packed: (fp32 exponent of code 0) << 23
};

// ---- packed whole-row entries (resident layout, fp32, plain matrices) -------------------------------------------
// One 32-bit word per entry:  [31:27] column delta - 1 (31: same column) | [26:23] exponent code | [22:0] mantissa.
// The column of entry k of a row slice is the column of entry k - 1 plus its delta (entry 0 counts from column -1);
// exponent code c in 1..15 stands for the fp32 exponent c + bias, code 0 (mantissa 0) is a FILLER: it contributes
// nothing.  Every aligned 16-column window of a row that holds no kept entry gets one filler at its first column, so two
// consecutive stored columns are never more than 31 apart.  Item padding is "same column, code 0".  Applies when every
// kept entry is positive (plain) and every kept exponent lies in the 15 binades below the largest (no subnormal).
constexpr unsigned int kPackPad = 0xF8000000u;
constexpr int kWinCols = 16;
// ehi: largest kept exponent, elo: 255 - smallest (0, 0: no kept entry); returns false when the values do not fit
__host__ __device__ inline bool pack_window(unsigned int ehi, unsigned int elo, unsigned int* bias) {
  const unsigned int b = ehi > 15u ? ehi - 15u : 0u;
  if (bias) *bias = b;
  return (ehi | elo) == 0u || 255u - elo >= b + 1u;
}
__device__ __forceinline__ unsigned int pack_word(unsigned int delta, float x, unsigned int bias) {  // x > 0 or filler +0
  const unsigned int bits = __float_as_uint(x);
  const unsigned int ec = bits ? ((bits >> 23) - bias) << 23 : 0u;
  return ((delta - 1u) << 27) | ec | (bits & 0x7fffffu);
}
// the counts of a packed build: kept entries + empty windows of the row when the device-side gate holds
struct PackCount {
  const unsigned int* win;  // [rows_pad][wwords] occupied-window bitmap, null: never packed
  int wwords, nwin, rows;   // nwin = windows that start below m
  const SyncBlock* sb;      // counts[1] (non-plain entries) and expo of the matrix
  __device__ __forceinline__ bool on() const {
    return win && sb->counts[1] == 0ull && pack_window(sb->expo[0], sb->expo[1], nullptr);
  }
  __device__ __forceinline__ unsigned int fillers(int r) const {
    if (r >= rows) return 0u;
    unsigned int occ = 0u;
    for (int k = 0; k < wwords; ++k) occ += __popc(win[(size_t)r * wwords + k]);
    return (unsigned int)nwin - occ;
  }
};

template <typename T> __device__ __forceinline__ void load4(const T* p, T (&x)[4]);
template <> __device__ __forceinline__ void load4<float>(const float* p, float (&x)[4]) {
  const float4 v = *reinterpret_cast<const float4*>(p); x[0] = v.x; x[1] = v.y; x[2] = v.z; x[3] = v.w;
}
template <> __device__ __forceinline__ void load4<double>(const double* p, double (&x)[4]) {
  const double2 a = reinterpret_cast<const double2*>(p)[0], b = reinterpret_cast<const double2*>(p)[1];
  x[0] = a.x; x[1] = a.y; x[2] = b.x; x[3] = b.y;
}

template <typename T> __device__ __forceinline__ bool is_plain(T s) { return s > T(0); }

// pass 1: one warp per (padded) local row counts the kept entries per column segment:
//   cnt4[seg * (rows_pad + 1) + row] = kept entries of slice (row, seg)   (the scoring kernel can produce the
//   same array on the fly: ScoreArgs::cnt)
//   totals[0] += kept entries, totals[1] += kept entries that are not "plain"
//   win (nullable, whole-row layout of fp32 storage): occupied 16-column windows and kept exponent range, see PackCount
template <typename T>
__global__ void sparse_count_kernel(const T* M, long long ld, int m, int rows, int rows_pad, int W, int nseg,
                                    unsigned int* cnt4, unsigned long long* totals, unsigned int* win, int wwords,
                                    unsigned int* expo) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows_pad) return;
  unsigned int real = 0, odd = 0, ehi = 0, elo = 0;
  for (int s = 0; s < nseg; ++s) {
    unsigned int c = 0, o = 0;
    if (warp < rows) {
      const int c0 = s * W, c1 = min(m, c0 + W);
      for (int j0 = c0; j0 < c1; j0 += 128) {  // warp-uniform trip count (the window ballot below)
        const int j = j0 + lane * 4;
        T x[4];
        if (j < c1) load4<T>(M + (size_t)warp * ld + j, x);  // j + 3 < ld: ld is a multiple of 128
        unsigned int any = 0;
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (j + e < c1 && !is_neutral<T>(x[e])) {
            ++c; o += is_plain<T>(x[e]) ? 0u : 1u; any = 1;
            if constexpr (sizeof(T) == 4) {
              const unsigned int xe = (__float_as_uint(x[e]) >> 23) & 0xffu;
              ehi = max(ehi, xe); elo = max(elo, 255u - xe);
            }
          }
        if (win) {
          const unsigned int v = __ballot_sync(0xffffffffu, any);
          unsigned int wm = 0u;
#pragma unroll
          for (int w = 0; w < 8; ++w) wm |= ((v >> (4 * w)) & 0xfu) ? (1u << w) : 0u;
          if (lane == 0 && wm) atomicOr(win + (size_t)warp * wwords + j0 / 512, wm << ((j0 / kWinCols) & 31));
        }
      }
    }
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) { c += __shfl_xor_sync(0xffffffffu, c, k); o += __shfl_xor_sync(0xffffffffu, o, k); }
    if (lane == 0) cnt4[(size_t)s * (rows_pad + 1) + warp] = c;
    real += c; odd += o;
  }
  if (lane == 0) {
    if (real) atomicAdd(&totals[0], (unsigned long long)real);
    if (odd) atomicAdd(&totals[1], (unsigned long long)odd);
  }
  if (win) {
    ehi = __reduce_max_sync(0xffffffffu, ehi); elo = __reduce_max_sync(0xffffffffu, elo);
    if (lane == 0 && (ehi | elo)) { atomicMax(expo, ehi); atomicMax(expo + 1, elo); }
  }
}

// pass 2: one block (1024 threads) per column segment sorts the rows by slice length, longest first (counting sort
// over the nb = W/4 + 2 possible lengths in chunks; ties in row order: a stable sort, so the layout is reproducible).
//   rowid[seg][pos] = row at sorted position pos
// Dynamic shared memory: (nb + 1) counters.
// Packed builds (pc.on()) sort by kept entries + fillers: the stored length.
__global__ void sell_sort_kernel(const unsigned int* cnt4, int rows_pad, int nb, unsigned int* rowid,
                                 unsigned long long* total_entries /* nullable: += kept entries */, PackCount pc) {
  extern __shared__ unsigned int hist[];
  __shared__ unsigned int wsum[32];
  const unsigned int* c = cnt4 + (size_t)blockIdx.x * (rows_pad + 1);
  const bool pk = pc.on();
  auto len = [&](int r) { return c[r] + (pk ? pc.fillers(r) : 0u); };
  for (int i = threadIdx.x; i <= nb; i += blockDim.x) hist[i] = 0u;
  __syncthreads();
  unsigned long long mine = 0;
  for (int r = threadIdx.x; r < rows_pad; r += blockDim.x) { mine += c[r]; atomicAdd(&hist[min((len(r) + 3u) >> 2, (unsigned int)(nb - 1))], 1u); }
  if (total_entries) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(total_entries, mine);
  }
  __syncthreads();
  {  // start of every length class, longest class first: exclusive scan of the histogram read backwards
    const int per = (nb + (int)blockDim.x - 1) / (int)blockDim.x;
    const int r0 = (int)threadIdx.x * per;          // reversed positions [r0, r0 + per): bin = nb - 1 - r
    unsigned int local = 0;
    for (int q = 0; q < per; ++q) { const int r = r0 + q; if (r < nb) local += hist[nb - 1 - r]; }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    unsigned int inc = local;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    if (w == 0) {
      unsigned int v = wsum[lane], t = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
      wsum[lane] = t - v;
    }
    __syncthreads();
    unsigned int run = wsum[w] + (inc - local);
    for (int q = 0; q < per; ++q) {
      const int r = r0 + q;
      if (r < nb) { const unsigned int hcount = hist[nb - 1 - r]; hist[nb - 1 - r] = run; run += hcount; }
    }
  }
  __syncthreads();
  // STABLE placement (ties in row order): the layout -- hence the grouping of every fp64 sum downstream -- must not
  // depend on the arrival order of atomics, or two runs on the same input differ in the last bit.  Rows are taken in
  // tiles of blockDim.x in row order; inside a tile the warps take turns (one __syncthreads per turn); inside a warp
  // __match_any_sync ranks the lanes of equal length class.
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  for (int base = 0; base < rows_pad; base += blockDim.x) {
    const int r = base + threadIdx.x;
    const bool have = r < rows_pad;
    const unsigned int cls = have ? min((len(r) + 3u) >> 2, (unsigned int)(nb - 1)) : 0xffffffffu;
    const unsigned int peers = __match_any_sync(0xffffffffu, cls);
    const int leader = __ffs(peers) - 1;
    const unsigned int before = __popc(peers & ((1u << lane) - 1u));
    unsigned int start = 0u;
    for (int w = 0; w < nwarp; ++w) {   // the warps of the tile take turns (passing a ticket through shared memory
      if (warp == w && have && lane == leader) { start = hist[cls]; hist[cls] = start + __popc(peers); }  // with
      __syncthreads();                  // spinning warps was several times slower)
    }
    start = __shfl_sync(0xffffffffu, start, leader);
    if (have) rowid[(size_t)blockIdx.x * rows_pad + start + before] = (unsigned int)r;
  }
}

// pass 3: chunks of every item = 4 x its longest member (the first one in sorted order); scanned in place by
// the two scan kernels below into itemptr[seg][0..NI]
__global__ void sell_itemlen_kernel(const unsigned int* cnt4, const unsigned int* rowid, int rows_pad, int nseg,
                                    unsigned int* itemptr, PackCount pc) {
  const int NI = rows_pad >> 2;
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)nseg * (NI + 1)) return;
  const int seg = (int)(t / (NI + 1)), i = (int)(t - (long long)seg * (NI + 1));
  unsigned int len = 0u;
  if (i < NI) {
    const unsigned int r = rowid[(size_t)seg * rows_pad + 4 * i];
    len = 4u * ((cnt4[(size_t)seg * (rows_pad + 1) + r] + (pc.on() ? pc.fillers((int)r) : 0u) + 3u) >> 2);
  }
  itemptr[t] = len;
}

// pass 3a: one block per column segment: exclusive scan (in place) of that segment's item lengths, walking the
// array in coalesced tiles of 1024; the segment total goes to segtot[seg]
__global__ void sparse_scan_seg_kernel(unsigned int* cnt4, int n, unsigned long long* segtot) {
  __shared__ unsigned int wsum[32];
  __shared__ unsigned int carry_s;
  unsigned int* a = cnt4 + (size_t)blockIdx.x * n;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  unsigned long long carry = 0;
  for (int base = 0; base < n; base += 1024) {
    const int i = base + t;
    const unsigned int x = (i < n) ? a[i] : 0u;
    unsigned int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) wsum[w] = inc;
    __syncthreads();
    if (w == 0) {
      unsigned int v = wsum[lane], s = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, s, o); if (lane >= o) s += y; }
      wsum[lane] = s - v;                 // exclusive prefix of the warp sums
      if (lane == 31) carry_s = s;        // tile total
    }
    __syncthreads();
    if (i < n) a[i] = (unsigned int)(carry + wsum[w] + (inc - x));
    carry += carry_s;
    __syncthreads();
  }
  if (t == 0) segtot[blockIdx.x] = carry;
}

// pass 3b: add the start of each segment (prefix of the segment totals); block 0 also publishes the grand total
__global__ void sparse_scan_fix_kernel(unsigned int* cnt4, int n, int nseg, const unsigned long long* segtot,
                                       unsigned long long* total4) {
  unsigned long long base = 0;
  for (int s = 0; s < (int)blockIdx.x; ++s) base += segtot[s];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned long long tot = 0;
    for (int s = 0; s < nseg; ++s) tot += segtot[s];
    *total4 = tot;
  }
  if (base == 0) return;
  unsigned int* a = cnt4 + (size_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) a[i] += (unsigned int)base;
}

// pass 4: one warp per item reads its four member rows together and compacts them through four shared-memory
// rings; chunk k of all four members is then 64 contiguous bytes of val (32 of off16), so a flush of 8 chunks per
// member is one fully coalesced 512-byte store.
constexpr int kFillWarps = 4;
constexpr int kRing = 256;  // entries per member ring: < 36 left after a flush + <= 128 new ones per step
// one warp: the item whose chunks are [b, e) of the stream and whose members are rows r[0..3]; columns [c0, c1)
// PACK (fp32, whole rows): one filler (+0.0) at the first column of every empty 16-column window of a real row, and
// the chunks are written as packed words (pack_word; the column delta reads the previous entry from the ring)
template <typename T, bool PACK = false>
__device__ __forceinline__ void sell_fill_item_warp(const T* M, long long ld, int rows, int c0, int c1, unsigned int b, unsigned int e,
                                                    const unsigned int (&r)[4], T* val, unsigned short* off16, int off_shift,
                                                    unsigned int pad_off, T (*rv)[kRing], unsigned short (*ro)[kRing],
                                                    unsigned int bias = 0u) {
  const int lane = threadIdx.x & 31;
  const unsigned int L = (e - b) >> 2;  // chunks per member
  if (L == 0u) return;
  unsigned int n[4] = {0u, 0u, 0u, 0u}, f[4] = {0u, 0u, 0u, 0u};
  const int g = lane >> 2, ms = lane & 3;  // flush role: chunk f + g of member ms
  // writes chunk k of member ms (entries beyond the member's n are neutral padding)
  auto put_chunk = [&](unsigned int k, unsigned int nm) {
    if constexpr (PACK) {
      unsigned int wd[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const unsigned int w = 4u * k + q;
        wd[q] = kPackPad;
        if (w < nm) {
          const int prev = w ? (int)ro[ms][(w - 1u) & (kRing - 1)] : -1;  // < 165 entries back: still in the ring
          wd[q] = pack_word((unsigned int)((int)ro[ms][w & (kRing - 1)] - prev), rv[ms][w & (kRing - 1)], bias);
        }
      }
      *reinterpret_cast<uint4*>(reinterpret_cast<unsigned int*>(val) + 4ull * (b + 4ull * k + ms)) = make_uint4(wd[0], wd[1], wd[2], wd[3]);
    } else {
      T x[4]; unsigned short o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const unsigned int w = 4u * k + q;
        const bool have = w < nm;
        x[q] = have ? rv[ms][w & (kRing - 1)] : encode<T>(0.0, false);
        o[q] = have ? ro[ms][w & (kRing - 1)] : (unsigned short)pad_off;
      }
      const unsigned long long at = 4ull * (b + 4ull * k + ms);
      Quad<T>::store(val + at, x);
      *reinterpret_cast<uint2*>(off16 + at) = make_uint2((unsigned int)o[0] | ((unsigned int)o[1] << 16), (unsigned int)o[2] | ((unsigned int)o[3] << 16));
    }
  };
  for (int j0 = c0; j0 < c1; j0 += 128) {
    const int j = j0 + lane * 4;
    // the four members' 128 columns: all loads first, then ONE warp scan for the four kept-entry counts (packed
    // as four 8-bit fields: a member keeps at most 128 entries per step)
    T x[4][4];
    unsigned int keep[4], packed = 0u;
#pragma unroll
    for (int s_ = 0; s_ < 4; ++s_) {
      if (r[s_] < (unsigned int)rows) load4<T>(M + (size_t)r[s_] * ld + j, x[s_]);  // j + 3 < ld: ld is a multiple of 128
      else { x[s_][0] = x[s_][1] = x[s_][2] = x[s_][3] = encode<T>(0.0, false); }
    }
#pragma unroll
    for (int s_ = 0; s_ < 4; ++s_) {
      keep[s_] = 0u;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (j + q >= c1) x[s_][q] = encode<T>(0.0, false);
        keep[s_] |= (!is_neutral<T>(x[s_][q]) ? 1u : 0u) << q;
      }
      if (PACK && r[s_] < (unsigned int)rows) {  // warp-uniform
        const unsigned int v = __ballot_sync(0xffffffffu, keep[s_] != 0u);
        if ((lane & 3) == 0 && ((v >> lane) & 0xfu) == 0u && j < c1) { keep[s_] |= 1u; x[s_][0] = T(0); }
      }
      packed |= (unsigned int)__popc(keep[s_]) << (8 * s_);
    }
    unsigned int pre = packed;  // inclusive scan over lanes, four fields at once (no carry: every field stays <= 128)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int y = __shfl_up_sync(0xffffffffu, pre, o);
      if (lane >= o) pre += y;
    }
    const unsigned int total = __shfl_sync(0xffffffffu, pre, 31);
    const unsigned int excl = pre - packed;
#pragma unroll
    for (int s_ = 0; s_ < 4; ++s_) {
      unsigned int w = n[s_] + ((excl >> (8 * s_)) & 0xffu);
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (keep[s_] & (1u << q)) { rv[s_][w & (kRing - 1)] = x[s_][q]; ro[s_][w & (kRing - 1)] = (unsigned short)((j + q - c0) << off_shift); ++w; }
      n[s_] += (total >> (8 * s_)) & 0xffu;
    }
    __syncwarp();
    // flush 8 complete chunks of every member that has them (members of an item have almost the same length:
    // usually all four flush together and the store is one contiguous 512-byte run)
    for (;;) {
      const unsigned int nm = ms == 0 ? n[0] : ms == 1 ? n[1] : ms == 2 ? n[2] : n[3];
      const unsigned int fm = ms == 0 ? f[0] : ms == 1 ? f[1] : ms == 2 ? f[2] : f[3];
      const bool can = (nm >> 2) >= fm + 8u;
      const unsigned int vote = __ballot_sync(0xffffffffu, can);
      if (vote == 0u) break;
      if (can) put_chunk(fm + g, nm);
#pragma unroll
      for (int s_ = 0; s_ < 4; ++s_) if (vote & (1u << s_)) f[s_] += 8u;  // lanes 0..3 are (g = 0, member s_)
    }
    __syncwarp();
  }
  // the rest of every member: remaining chunks, the partial one, then padding up to the item's length
  {
    const unsigned int nm = ms == 0 ? n[0] : ms == 1 ? n[1] : ms == 2 ? n[2] : n[3];
    const unsigned int fm = ms == 0 ? f[0] : ms == 1 ? f[1] : ms == 2 ? f[2] : f[3];
    for (unsigned int k = fm + g; k < L; k += 8u) put_chunk(k, nm);
  }
  __syncwarp();
}

template <typename T, bool PACK = false>
__global__ void __launch_bounds__(kFillWarps * 32)
sparse_fill_items_kernel(const T* M, long long ld, int m, int rows, int rows_pad, int W, int nseg,
                         const unsigned int* itemptr, const unsigned int* rowid, T* val, unsigned short* off16,
                         int off_shift /* 3: byte offset of v[col] in the staged segment; 0: column index */,
                         unsigned int pad_off /* offset stored in padding entries: a slot that holds 0.0 */,
                         unsigned int bias = 0u /* PACK: exponent bias of the codes */) {
  __shared__ __align__(16) T ringv[kFillWarps][4][kRing];
  __shared__ __align__(8) unsigned short ringo[kFillWarps][4][kRing];
  const int wic = threadIdx.x >> 5;
  const int NI = rows_pad >> 2;
  const long long gw = (long long)blockIdx.x * kFillWarps + wic;
  if (gw >= (long long)nseg * NI) return;
  const int seg = (int)(gw / NI), it = (int)(gw - (long long)seg * NI);
  const unsigned int b = itemptr[(size_t)seg * (NI + 1) + it], e = itemptr[(size_t)seg * (NI + 1) + it + 1];
  unsigned int r[4];
#pragma unroll
  for (int s_ = 0; s_ < 4; ++s_) r[s_] = rowid[(size_t)seg * rows_pad + 4 * it + s_];
  const int c0 = seg * W, c1 = min(m, c0 + W);
  sell_fill_item_warp<T, PACK>(M, ld, rows, c0, c1, b, e, r, val, off16, off_shift, pad_off, ringv[wic], ringo[wic], bias);
}

// 4 entries of one row slice
template <typename T> struct Entry4;
template <> struct Entry4<float> {
  float4 x; uint2 k;
  __device__ __forceinline__ void load(const float* val, const unsigned short* off, unsigned long long at) {
    x = ldg_stream(reinterpret_cast<const float4*>(val + at));
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(k.x), "=r"(k.y) : "l"(off + at));
  }
  __device__ __forceinline__ void load_cg(const float* val, const unsigned short* off, unsigned long long at) {  // L2-coherent
    asm volatile("ld.global.cg.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(x.x), "=f"(x.y), "=f"(x.z), "=f"(x.w) : "l"(val + at));
    asm volatile("ld.global.cg.v2.u32 {%0,%1}, [%2];" : "=r"(k.x), "=r"(k.y) : "l"(off + at));
  }
  __device__ __forceinline__ float get(int e) const { return e == 0 ? x.x : e == 1 ? x.y : e == 2 ? x.z : x.w; }
  __device__ __forceinline__ void neutral() { x = make_float4(-0.f, -0.f, -0.f, -0.f); k = make_uint2(kZeroSlot | (kZeroSlot << 16), kZeroSlot | (kZeroSlot << 16)); }
  __device__ __forceinline__ void neutral_at(unsigned int kk) { x = make_float4(-0.f, -0.f, -0.f, -0.f); k = make_uint2(kk, kk); }
};
template <> struct Entry4<double> {
  double2 a, b; uint2 k;
  __device__ __forceinline__ void load(const double* val, const unsigned short* off, unsigned long long at) {
    a = ldg_stream(reinterpret_cast<const double2*>(val + at));
    b = ldg_stream(reinterpret_cast<const double2*>(val + at) + 1);
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(k.x), "=r"(k.y) : "l"(off + at));
  }
  __device__ __forceinline__ void load_cg(const double* val, const unsigned short* off, unsigned long long at) {
    asm volatile("ld.global.cg.v2.f64 {%0,%1}, [%2];" : "=d"(a.x), "=d"(a.y) : "l"(val + at));
    asm volatile("ld.global.cg.v2.f64 {%0,%1}, [%2];" : "=d"(b.x), "=d"(b.y) : "l"(val + at + 2));
    asm volatile("ld.global.cg.v2.u32 {%0,%1}, [%2];" : "=r"(k.x), "=r"(k.y) : "l"(off + at));
  }
  __device__ __forceinline__ double get(int e) const { return e == 0 ? a.x : e == 1 ? a.y : e == 2 ? b.x : b.y; }
  __device__ __forceinline__ void neutral() { a = make_double2(-0.0, -0.0); b = a; k = make_uint2(kZeroSlot | (kZeroSlot << 16), kZeroSlot | (kZeroSlot << 16)); }
  __device__ __forceinline__ void neutral_at(unsigned int kk) { a = make_double2(-0.0, -0.0); b = a; k = make_uint2(kk, kk); }
};
__device__ __forceinline__ unsigned int off_of(const uint2& k, int e) {
  return e == 0 ? (k.x & 0xffffu) : e == 1 ? (k.x >> 16) : e == 2 ? (k.y & 0xffffu) : (k.y >> 16);
}
__device__ __forceinline__ double vs_at(const double* vs, unsigned int byte_off) {
  return *reinterpret_cast<const double*>(reinterpret_cast<const char*>(vs) + byte_off);
}

// A ROUND is kSellUnroll * 32 consecutive chunks of an item: lane l takes chunks l, l + 32, ... of the round
// (always member l & 3 of the item because items start at a multiple of 4).
// vs holds the segment of v in natural order, vs[kSegMax] == 0.
template <typename T>
__device__ __forceinline__ void sell_load_round(const SparseView& sp, Entry4<T> (&E)[kSellUnroll], unsigned int j, unsigned int e) {
  const T* val = reinterpret_cast<const T*>(sp.val);
#pragma unroll
  for (int u = 0; u < kSellUnroll; ++u) {
    if (j + 32u * u < e) E[u].load(val, sp.off16, 4ull * (j + 32u * u));
    else E[u].neutral();
  }
}
// aM/aC: this lane's share of its member's |M| v and C v (two interleaved accumulators each)
template <typename T, bool PLAIN>
__device__ __forceinline__ void sell_apply_round(const Entry4<T> (&E)[kSellUnroll], const double* vs, double (&aM)[2], double (&aC)[2]) {
#pragma unroll
  for (int u = 0; u < kSellUnroll; ++u)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const double v = vs_at(vs, off_of(E[u].k, q));
      if (PLAIN) {
        aM[u & 1] = fma((double)E[u].get(q), v, aM[u & 1]);  // padding: -0.0 * 0.0
        aC[u & 1] += v;
      } else {
        double dummyM = 0.0, dummyC = 0.0;
        apply_elem<false>(E[u].get(q), v, 0.0, aM[u & 1], aC[u & 1], dummyM, dummyC);
      }
    }
}

// Work split of one sweep: every CTA gets a CONTIGUOUS range of the item stream holding 1/G of the cost
// (chunks + kItemCost per item), found by bisection on itemptr; inside a CTA the warps draw items from a
// shared-memory counter.  (Dealing 32-row tiles round-robin, as the dense sweep does, left the slowest CTA
// with 1.23x the mean bytes at config 2.)
__device__ __forceinline__ unsigned long long sparse_item_cost(const unsigned int* itemptr, int NI, int nseg, unsigned int g) {
  const unsigned int seg = g / (unsigned int)NI, it = g - seg * (unsigned int)NI;
  const unsigned int at = (seg >= (unsigned int)nseg) ? itemptr[(size_t)(nseg - 1) * (NI + 1) + NI]
                                                      : itemptr[(size_t)seg * (NI + 1) + it];
  return (unsigned long long)at + (unsigned long long)kItemCost * g;
}

__global__ void sparse_partition_kernel(const unsigned int* itemptr, int rows_pad, int nseg, int G, unsigned int* cta_first) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > G) return;
  const int NI = rows_pad >> 2;
  const unsigned int N = (unsigned int)nseg * (unsigned int)NI;
  const unsigned long long total = sparse_item_cost(itemptr, NI, nseg, N);
  const unsigned long long target = total * (unsigned long long)b / (unsigned long long)G;  // total < 2^34, b <= G <= 3 CTAs x SMs
  unsigned int lo = 0, hi = N;  // smallest g with cost(g) >= target
  while (lo < hi) {
    const unsigned int mid = lo + ((hi - lo) >> 1);
    if (sparse_item_cost(itemptr, NI, nseg, mid) >= target) hi = mid; else lo = mid + 1;
  }
  if (b == G) lo = N;
  cta_first[b] = lo;
}

// whole sparse pass of one CTA: same partial layout as matvec_phase (partM/partC [NSEG][rows_pad]).
// vs must hold kSegMax + 1 doubles.
// (Tried and dropped: a plain-only instance capped at 64 registers for 4 CTAs/SM -- what the sweep gained, the
// two synchronisation steps of the evaluation lost again with the larger grid; a bulk L2 prefetch of the next
// item (cp.async.bulk.prefetch.L2) -- slower.)
template <typename T>
__device__ void sparse_phase(const MatView& mv, const Plan& p, const StageArgs& st, const SparseView& sp,
                             double* partM, double* partC, double* vs, double* red_smem) {
  __shared__ int next_item;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NI = sp.rows_pad >> 2;
  unsigned int g = sp.cta_first[blockIdx.x];
  const unsigned int gend = sp.cta_first[blockIdx.x + 1];
  if (threadIdx.x == 0) vs[kSegMax] = 0.0;
  for (int seg = (int)(g / (unsigned int)NI); g < gend; ++seg) {
    const int it0 = (int)(g - (unsigned int)seg * NI);
    const int it1 = (int)min(gend - (unsigned int)seg * NI, (unsigned int)NI);
    if (threadIdx.x == 0) next_item = it0 + kWarps;
    // the CTA that holds the first item of a segment publishes the staged vector and its sum
    stage_segment<double>(st, p, mv.m, seg, it0 == 0, vs, red_smem);  // <double>: natural (unpermuted) order
    const unsigned int* ipseg = sp.itemptr + (size_t)seg * (NI + 1);
    const unsigned int* rowseg = sp.rowid + (size_t)seg * sp.rows_pad;
    // lanes 0,1: chunk range of the item; lanes 2..5: its member rows
    auto fetch = [&](int it) -> unsigned int {
      if (it >= it1) return 0u;
      if (lane < 2) return ipseg[it + lane];
      if (lane < 6) return rowseg[4 * it + lane - 2];
      return 0u;
    };
    // The warp walks its items as one stream of rounds, software-pipelined: the loads of the NEXT round -- the
    // first round of the next item when the current one ends -- are issued before the current round is applied,
    // so a warp always has a round in flight (a sweep that loads, waits, then computes leaves HBM idle while
    // the 24 warps of an SM work through their 7-way bank-conflicted gathers).
    int it = it0 + warp;
    if (it < it1) {
      unsigned int q0 = fetch(it);
      int itn = 0;
      if (lane == 0) itn = atomicAdd(&next_item, 1);
      itn = __shfl_sync(0xffffffffu, itn, 0);
      unsigned int q1 = fetch(itn);
      unsigned int e = __shfl_sync(0xffffffffu, q0, 1), row = __shfl_sync(0xffffffffu, q0, 2 + (lane & 3));
      unsigned int j = __shfl_sync(0xffffffffu, q0, 0) + lane;  // this lane's first chunk of the current round
      double aM[2] = {0.0, 0.0}, aC[2] = {0.0, 0.0};
      Entry4<T> A[kSellUnroll], B[kSellUnroll];
      sell_load_round<T>(sp, A, j, e);
      // applies round X of the current item after issuing the loads of the following round into Y;
      // returns true when the warp has run out of items
      auto step = [&](Entry4<T> (&X)[kSellUnroll], Entry4<T> (&Y)[kSellUnroll]) -> bool {
        const bool last = (j - lane) + 32u * kSellUnroll >= e;  // warp-uniform
        unsigned int jn = j + 32u * kSellUnroll, en = e, rown = row;
        if (last) {
          jn = __shfl_sync(0xffffffffu, q1, 0) + lane; en = __shfl_sync(0xffffffffu, q1, 1);
          rown = __shfl_sync(0xffffffffu, q1, 2 + (lane & 3));
          if (itn >= it1) en = jn - lane;  // no next item: nothing to load
        }
        sell_load_round<T>(sp, Y, jn, en);
        if (sp.plain) sell_apply_round<T, true>(X, vs, aM, aC);
        else sell_apply_round<T, false>(X, vs, aM, aC);
        if (last) {
          double accM = aM[0] + aM[1], accC = aC[0] + aC[1];
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            accM += __shfl_xor_sync(0xffffffffu, accM, o);
            accC += __shfl_xor_sync(0xffffffffu, accC, o);
          }
          if (lane < 4) {
            partM[(size_t)seg * mv.rows_pad + row] = accM;
            partC[(size_t)seg * mv.rows_pad + row] = accC;
          }
          if (itn >= it1) return true;
          aM[0] = aM[1] = aC[0] = aC[1] = 0.0;
          it = itn;
          if (lane == 0) itn = atomicAdd(&next_item, 1);
          itn = __shfl_sync(0xffffffffu, itn, 0);
          q1 = fetch(itn);
        }
        j = jn; e = en; row = rown;
        return false;
      };
      for (;;) {
        if (step(A, B)) break;
        if (step(B, A)) break;
      }
    }
    __syncthreads();  // vs and next_item are re-used by the next segment pass
    g = (unsigned int)(seg + 1) * NI;
  }
}


}  // namespace clp
