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

// pass 2: a device-wide stable counting sort of the rows of every segment by slice length, longest first (the
// nb = W/4 + 2 possible lengths in chunks are the classes; ties in row order, so the layout -- hence the grouping of
// every fp64 sum downstream -- is reproducible), in tiles of kSortTile rows, segment-major:
//   sell_hist_kernel   class histogram of every (segment, tile) into hist[seg][nb - 1 - class][tile]
//   sparse_scan_*      exclusive scan of hist in that order: the sorted position of the tile's first row of the class,
//                      counted from the start of rowid (every segment holds rows_pad rows)
//   sell_place_kernel  stable placement inside the tile: rowid[seg][pos] = row at sorted position pos; the first row of
//                      every item also writes the item's length (4 x its chunks), scanned by sparse_scan_* into itemptr
// Packed builds (pc.on()) sort by kept entries + fillers: the stored length.  The class of a row is its stored length
// in chunks, at most ceil(W / 4) <= nb - 2 (a packed row holds at most one entry or filler per column).
constexpr int kSortTile = 256;

// class of row base + threadIdx.x (0xffffffff past rows_pad); occ: kSortTile shared words
__device__ __forceinline__ unsigned int sell_tile_class(const unsigned int* c, int base, int rows_pad, int nb, const PackCount& pc,
                                                        bool pk, unsigned int* occ) {
  const int r = base + (int)threadIdx.x;
  if (pk) {  // occupied windows of the tile's rows: the bitmap words are contiguous, read them coalesced
    occ[threadIdx.x] = 0u;
    __syncthreads();
    const int nr = min(kSortTile, max(0, pc.rows - base));
    const unsigned int* w = pc.win + (size_t)base * pc.wwords;
    for (int k = threadIdx.x; k < nr * pc.wwords; k += blockDim.x) {
      const unsigned int x = __popc(w[k]);
      if (x) atomicAdd(&occ[k / pc.wwords], x);
    }
    __syncthreads();
  }
  if (r >= rows_pad) return 0xffffffffu;
  const unsigned int len = c[r] + ((pk && r < pc.rows) ? (unsigned int)pc.nwin - occ[threadIdx.x] : 0u);
  return min((len + 3u) >> 2, (unsigned int)(nb - 1));
}

// grid (tiles, nseg), kSortTile threads; dynamic shared memory: nb counters
__global__ void __launch_bounds__(kSortTile) sell_hist_kernel(const unsigned int* cnt4, int rows_pad, int nb, int ntile, unsigned int* hist,
                                                              unsigned long long* total_entries /* nullable: += kept entries */, PackCount pc) {
  extern __shared__ unsigned int h[];
  __shared__ unsigned int occ[kSortTile];
  const int seg = blockIdx.y, base = blockIdx.x * kSortTile;
  const unsigned int* c = cnt4 + (size_t)seg * (rows_pad + 1);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) h[i] = 0u;
  const unsigned int cls = sell_tile_class(c, base, rows_pad, nb, pc, pc.on(), occ);  // synchronises when packed
  __syncthreads();
  if (cls != 0xffffffffu) atomicAdd(&h[cls], 1u);
  if (total_entries) {
    unsigned long long mine = cls != 0xffffffffu ? c[base + threadIdx.x] : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(total_entries, mine);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nb; i += blockDim.x) hist[((size_t)seg * nb + (nb - 1 - i)) * ntile + blockIdx.x] = h[i];
}

// grid (tiles, nseg), kSortTile threads; dynamic shared memory: nb counters.  hist: scanned by sparse_scan_*.
// items: [nseg][NI + 1] item lengths in chunks (entry NI = 0), scanned by sparse_scan_* into itemptr
__global__ void __launch_bounds__(kSortTile) sell_place_kernel(const unsigned int* cnt4, int rows_pad, int nb, int ntile, const unsigned int* hist,
                                                               unsigned int* rowid, unsigned int* items, PackCount pc) {
  extern __shared__ unsigned int taken[];
  __shared__ unsigned int occ[kSortTile];
  const int seg = blockIdx.y, base = blockIdx.x * kSortTile;
  const unsigned int* c = cnt4 + (size_t)seg * (rows_pad + 1);
  const int NI = rows_pad >> 2;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) taken[i] = 0u;
  if (blockIdx.x == 0 && threadIdx.x == 0) items[(size_t)seg * (NI + 1) + NI] = 0u;
  const unsigned int cls = sell_tile_class(c, base, rows_pad, nb, pc, pc.on(), occ);
  __syncthreads();
  // inside the tile the warps take turns in row order; __match_any_sync ranks the lanes of equal class
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned int peers = __match_any_sync(0xffffffffu, cls);
  const int leader = __ffs(peers) - 1;
  const unsigned int before = __popc(peers & ((1u << lane) - 1u));
  unsigned int start = 0u;
  for (int w = 0; w < kSortTile / 32; ++w) {
    if (warp == w && cls != 0xffffffffu && lane == leader) { start = taken[cls]; taken[cls] = start + __popc(peers); }
    __syncthreads();
  }
  start = __shfl_sync(0xffffffffu, start, leader);
  if (cls == 0xffffffffu) return;
  const unsigned int pos = hist[((size_t)seg * nb + (nb - 1 - cls)) * ntile + blockIdx.x] + start + before - (unsigned int)seg * rows_pad;
  rowid[(size_t)seg * rows_pad + pos] = (unsigned int)(base + threadIdx.x);
  if ((pos & 3u) == 0u) items[(size_t)seg * (NI + 1) + (pos >> 2)] = 4u * cls;  // the longest member: chunks of the item
}

// pass 3: exclusive scan in place of a flat array of n words (sorted positions, then item pointers), in blocks of
// kScanBlock words: sparse_scan_reduce_kernel sums every block, sparse_scan_down_kernel adds the sums of the blocks
// before its own to the scan of its block; block 0 publishes the grand total.  Block sums and the total are 64-bit,
// so a total past 2^32 (the scanned words wrap) is seen by the host, which then keeps the dense sweep
constexpr int kScanThreads = 1024, kScanPer = 4, kScanBlock = kScanThreads * kScanPer;

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long x, unsigned long long* wsum) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  __syncthreads();
  if (lane == 0) wsum[w] = x;
  __syncthreads();
  unsigned long long t = lane < (int)(blockDim.x >> 5) ? wsum[lane] : 0ull;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

__global__ void __launch_bounds__(kScanThreads) sparse_scan_reduce_kernel(const unsigned int* a, long long n, unsigned long long* bsum) {
  __shared__ unsigned long long wsum[32];
  const long long i0 = (long long)blockIdx.x * kScanBlock + (long long)threadIdx.x * kScanPer;
  unsigned long long x = 0;
#pragma unroll
  for (int q = 0; q < kScanPer; ++q) if (i0 + q < n) x += a[i0 + q];
  x = block_sum_u64(x, wsum);
  if (threadIdx.x == 0) bsum[blockIdx.x] = x;
}

__global__ void __launch_bounds__(kScanThreads) sparse_scan_down_kernel(unsigned int* a, long long n, const unsigned long long* bsum, int nblk,
                                                                        unsigned long long* total /* nullable */) {
  __shared__ unsigned long long wsum[32];
  __shared__ unsigned int wex[32];
  unsigned long long off = 0;  // sums of the blocks before this one (block 0: of all blocks, for the total)
  const int upto = blockIdx.x == 0 ? nblk : (int)blockIdx.x;
  for (int k = threadIdx.x; k < upto; k += blockDim.x) off += bsum[k];
  off = block_sum_u64(off, wsum);
  if (blockIdx.x == 0) { if (total && threadIdx.x == 0) *total = off; off = 0; }
  const long long i0 = (long long)blockIdx.x * kScanBlock + (long long)threadIdx.x * kScanPer;
  unsigned int x[kScanPer], mine = 0u;
#pragma unroll
  for (int q = 0; q < kScanPer; ++q) { x[q] = (i0 + q < n) ? a[i0 + q] : 0u; mine += x[q]; }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned int inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
  if (lane == 31) wex[w] = inc;
  __syncthreads();
  if (w == 0) {
    const unsigned int v = wex[lane];
    unsigned int t = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, t, o); if (lane >= o) t += y; }
    wex[lane] = t - v;
  }
  __syncthreads();
  unsigned int run = (unsigned int)off + wex[w] + (inc - mine);
#pragma unroll
  for (int q = 0; q < kScanPer; ++q) if (i0 + q < n) { a[i0 + q] = run; run += x[q]; }
}

// pass 4: one warp per item reads its four member rows together and compacts them through four shared-memory
// rings; chunk k of all four members is then 64 contiguous bytes of val (32 of off16), so a flush of 8 chunks per
// member is one fully coalesced 512-byte store.
constexpr int kFillWarps = 4;  // warps of the batched solver's fill (clp_batch.cuh)
constexpr int kRing = 256;  // entries per member ring: < 36 left after a flush + <= 128 new ones per step
// one warp: the item whose chunks are [b, e) of the stream and whose members are rows r[0..3]; columns [c0, c1)
// PACK (fp32, whole rows): one filler (+0.0) at the first column of every empty 16-column window of a real row, and
// the chunks are written as packed words (pack_word; the column delta reads the previous entry from the ring)
// PIPE: the loads of the next 128-column step are issued (streaming, no L1 allocation) before the current step is
// scanned and flushed, so a warp always has one step of its rows in flight
template <typename T, bool PACK = false, bool PIPE = false>
__device__ __forceinline__ void sell_fill_item_warp(const T* M, long long ld, int rows, int c0, int c1, unsigned int b, unsigned int e,
                                                    const unsigned int (&r)[4], T* val, unsigned short* off16, int off_shift,
                                                    unsigned int pad_off, T (*rv)[kRing], unsigned short (*ro)[kRing],
                                                    unsigned int bias = 0u) {
  const int lane = threadIdx.x & 31;
  const unsigned int L = (e - b) >> 2;  // chunks per member
  if (L == 0u) return;
  T xn[4][4];  // PIPE: the step after the current one
  auto load_step = [&](int jj, T (&y)[4][4]) {
#pragma unroll
    for (int s_ = 0; s_ < 4; ++s_) {
      if (r[s_] < (unsigned int)rows) {  // jj + 3 < ld: ld is a multiple of 128
        if constexpr (sizeof(T) == 4) {
          const float4 v = ldg_stream(reinterpret_cast<const float4*>(M + (size_t)r[s_] * ld + jj));
          y[s_][0] = v.x; y[s_][1] = v.y; y[s_][2] = v.z; y[s_][3] = v.w;
        } else {
          load4<T>(M + (size_t)r[s_] * ld + jj, y[s_]);
        }
      } else { y[s_][0] = y[s_][1] = y[s_][2] = y[s_][3] = encode<T>(0.0, false); }
    }
  };
  if constexpr (PIPE) load_step(c0 + lane * 4, xn);
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
    if constexpr (PIPE) {
#pragma unroll
      for (int s_ = 0; s_ < 4; ++s_)
#pragma unroll
        for (int q = 0; q < 4; ++q) x[s_][q] = xn[s_][q];
      if (j0 + 128 < c1) load_step(j + 128, xn);
    } else {
#pragma unroll
      for (int s_ = 0; s_ < 4; ++s_) {
        if (r[s_] < (unsigned int)rows) load4<T>(M + (size_t)r[s_] * ld + j, x[s_]);  // j + 3 < ld: ld is a multiple of 128
        else { x[s_][0] = x[s_][1] = x[s_][2] = x[s_][3] = encode<T>(0.0, false); }
      }
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

// One warp per item.  The packed whole-row build (PACK, config 2's) is PERSISTENT: the grid holds at most one wave of
// CTAs, and every warp draws items in stream order from the zeroed counter next_item until none is left, loading the
// next 128-column step while it scans and flushes the current one (sell_fill_item_warp<..., PIPE>).  Every item reads
// whole rows of the dense store, so all cost about the same.  fill_grid (clp_capi.cu) keeps the number of rounds a
// full wave would need but spreads the items over as few warps as that takes, so every round is about equally full:
// at config 2 (5 000 items, 4 752 warps in a wave) about 2 500 warps take two items each, where one warp per item left
// 248 items to a second wave on an idle GPU.  The 6-byte builds (column segments: config 4's 400 000 short items)
// keep one CTA slot per item: there the persistent, pipelined variant measured 8 % slower (12.31 against 11.38 ms).
// The ring size is shared with the batched solver's fill and already the smallest power of two above what a step
// needs; the warps per CTA are this kernel's own (kDevFillWarps; 2 and 4 measured the same at config 2).
constexpr int kDevFillWarps = 4;
template <typename T, bool PACK = false>
__global__ void __launch_bounds__(kDevFillWarps * 32)
sparse_fill_items_kernel(const T* M, long long ld, int m, int rows, int rows_pad, int W, int nseg,
                         const unsigned int* itemptr, const unsigned int* rowid, T* val, unsigned short* off16,
                         int off_shift /* 3: byte offset of v[col] in the staged segment; 0: column index */,
                         unsigned int pad_off /* offset stored in padding entries: a slot that holds 0.0 */,
                         unsigned int* next_item /* PACK */, unsigned int bias = 0u /* PACK: exponent bias of the codes */) {
  __shared__ __align__(16) T ringv[kDevFillWarps][4][kRing];
  __shared__ __align__(8) unsigned short ringo[kDevFillWarps][4][kRing];
  const int wic = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NI = rows_pad >> 2;
  const unsigned int N = (unsigned int)nseg * (unsigned int)NI;
  unsigned int g = (unsigned int)blockIdx.x * kDevFillWarps + wic;
  for (;;) {
    if constexpr (PACK) {
      g = 0u;
      if (lane == 0) g = atomicAdd(next_item, 1u);
      g = __shfl_sync(0xffffffffu, g, 0);
    }
    if (g >= N) return;
    const int seg = (int)(g / (unsigned int)NI), it = (int)(g - (unsigned int)seg * NI);
    const unsigned int b = itemptr[(size_t)seg * (NI + 1) + it], e = itemptr[(size_t)seg * (NI + 1) + it + 1];
    unsigned int r[4];
#pragma unroll
    for (int s_ = 0; s_ < 4; ++s_) r[s_] = rowid[(size_t)seg * rows_pad + 4 * it + s_];
    const int c0 = seg * W, c1 = min(m, c0 + W);
    sell_fill_item_warp<T, PACK, PACK>(M, ld, rows, c0, c1, b, e, r, val, off16, off_shift, pad_off, ringv[wic], ringo[wic], bias);
    if constexpr (!PACK) return;
  }
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
