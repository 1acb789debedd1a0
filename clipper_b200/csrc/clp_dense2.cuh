// clp_dense2.cuh -- second-generation dense pass over M ("stripe" decomposition).
//
// Included by clp_kernels.cuh (needs MatView, StageArgs, staged_value, ldg_stream, decode).
//
// The matrix is cut into column stripes of 2048 columns (8 warps x 256 columns).  A CTA walks a
// contiguous run of 32-row tiles inside a stripe; warp w owns columns [256w, 256w+256) of the stripe
// for ALL rows of the run, lane l owns 2 x 4 consecutive columns (two 128-column steps).
//   * the lane's 8 entries of v stay in REGISTERS for the whole run (no shared-memory staging of v);
//   * row sums: per 4-row chunk each warp reduces its 8 partial sums with a halving butterfly
//     (18 SHFL), the 8 warps of the CTA are added through 4 KB of shared memory once per 32-row tile;
//   * only tiles of the UPPER triangle are read (single GPU: the store holds the whole symmetric matrix).
//     Every element s = M_ij (i<j) is applied twice in-tile:  y_i += |s| v_j  (row sum) and
//     y_j += |s| v_i  (column sum, 16 register accumulators per lane that live across the whole run).
//     HBM traffic per objective evaluation drops from 4 m^2 to ~2 m^2 bytes (fp32 storage).
//     Inside the diagonal 2048 x 2048 block the strict-upper mask c > r is applied per element and
//     chunks that lie entirely below the diagonal are skipped.
// Work is split by enumerating all (stripe, row-tile) items stripe-major and giving every CTA an
// equal contiguous share (perfect balance up to one tile).  All partial results are written to
// fixed slots and added in a fixed order by the combine step -> bit-reproducible.
#pragma once

namespace clp {

constexpr int kStripe = 2048;    // columns per stripe
constexpr int kWarpCols = 256;   // columns per warp inside a stripe (2 steps of 128)
constexpr int kMaxStripes = 128; // m <= 262144

struct Plan2 {
  int G;        // CTAs
  int NST;      // stripes
  int KMAX;     // max number of stripes one CTA's run touches (column-partial slots per CTA)
  int NRT;      // local 32-row tiles
  long long T;  // total items
  const long long* tile_prefix;  // [NST+1] first item index of each stripe
  const int* cta_first_stripe;   // [G] stripe that contains the first item of CTA b
  const int* stripe_cta_lo;      // [NST] first / last CTA whose run intersects stripe J
  const int* stripe_cta_hi;
  const int* cta_has_items;      // [G] 0 for CTAs without items (problems with fewer items than CTAs)
  const int* slot_begin;         // [NST+1] range in slot_list of the column-partial slots of stripe J
  const int* slot_list;          // slot = cta * KMAX + (J - first stripe of cta), in CTA order
};

struct Dense2Buffers {
  double* rowM;   // [NST][rows_pad]  row-type partial products  (M and C)
  double* rowC;
  double* colM;   // [G*KMAX][kStripe] column-type partial products
  double* colC;
  double* sumpart;  // [G] per-CTA partial sums of the staged vector
};

// sum 8 values over the 32 lanes with a halving butterfly; the total of value q ends up in the four
// lanes whose bits (4,3,2) spell q.  18 shuffles instead of 80.
__device__ __forceinline__ double warp_reduce8(const double (&v)[8]) {
  const unsigned lane = threadIdx.x & 31u;
  double w[4], x[2], y;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const double send = (lane & 16u) ? v[i] : v[i + 4];
    const double keep = (lane & 16u) ? v[i + 4] : v[i];
    w[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const double send = (lane & 8u) ? w[i] : w[i + 2];
    const double keep = (lane & 8u) ? w[i + 2] : w[i];
    x[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  {
    const double send = (lane & 4u) ? x[0] : x[1];
    const double keep = (lane & 4u) ? x[1] : x[0];
    y = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  y += __shfl_xor_sync(0xffffffffu, y, 2);
  y += __shfl_xor_sync(0xffffffffu, y, 1);
  return y;
}

template <typename T> struct Elem4;  // 4 consecutive stored elements
template <> struct Elem4<float> {
  float4 v;
  __device__ __forceinline__ void load(const float* p) { v = ldg_stream(reinterpret_cast<const float4*>(p)); }
  __device__ __forceinline__ void neutral() { v = make_float4(-0.f, -0.f, -0.f, -0.f); }
  __device__ __forceinline__ float get(int e) const { return e == 0 ? v.x : e == 1 ? v.y : e == 2 ? v.z : v.w; }
};
template <> struct Elem4<double> {
  double2 a, b;
  __device__ __forceinline__ void load(const double* p) {
    a = ldg_stream(reinterpret_cast<const double2*>(p));
    b = ldg_stream(reinterpret_cast<const double2*>(p) + 1);
  }
  __device__ __forceinline__ void neutral() { a = make_double2(-0.0, -0.0); b = a; }
  __device__ __forceinline__ double get(int e) const { return e == 0 ? a.x : e == 1 ? a.y : e == 2 ? b.x : b.y; }
};

// one stored element applied to the row sums (and, SYM, to the column sums).  The C bit is
// turned into the double 1.0 / 0.0 with two integer instructions ({~(bits>>31) & 0x3ff00000, 0}) and the
// constraint sums are plain FMAs -- ptxas turns predicated fp64 adds into DADD + 2 FSEL, which costs more.
__device__ __forceinline__ double cbit_as_double(int hibits) {
  return __hiloint2double(~(hibits >> 31) & 0x3ff00000, 0);
}
template <bool SYM>
__device__ __forceinline__ void apply_elem(float x, double vcol, double vrow, double& rM, double& rC, double& cM, double& cC) {
  const double t = (double)fabsf(x);
  const double cf = cbit_as_double(__float_as_int(x));
  rM = fma(t, vcol, rM);
  rC = fma(cf, vcol, rC);
  if (SYM) {
    cM = fma(t, vrow, cM);
    cC = fma(cf, vrow, cC);
  }
}
template <bool SYM>
__device__ __forceinline__ void apply_elem(double x, double vcol, double vrow, double& rM, double& rC, double& cM, double& cC) {
  const double t = fabs(x);
  const double cf = cbit_as_double(__double2hiint(x));
  rM = fma(t, vcol, rM);
  rC = fma(cf, vcol, rC);
  if (SYM) {
    cM = fma(t, vrow, cM);
    cC = fma(cf, vrow, cC);
  }
}
__device__ __forceinline__ float neutral_if(bool kill, float x) { return kill ? -0.0f : x; }
__device__ __forceinline__ double neutral_if(bool kill, double x) { return kill ? -0.0 : x; }

// 4 rows x 4 columns of one lane (one 128-column step): apply to the row and column accumulators
template <typename T, bool DIAG>
__device__ __forceinline__ void dense2_apply(const Elem4<T> (&a)[4], const double (&vc)[4], const double (&vr)[4],
                                             int gi, int cfirst, double (&acc)[8], double (&colM)[4], double (&colC)[4]) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      auto x = a[r].get(e);
      if (DIAG) x = neutral_if((cfirst + e) <= (gi + r), x);  // keep the strict upper part only
      apply_elem<true>(x, vc[e], vr[r], acc[r], acc[4 + r], colM[e], colC[e]);
    }
}

// One 32-row tile for one warp: 8 chunks of 4 rows x 256 columns, software-pipelined at the granularity of
// one 128-column step (the loads of the next step are in flight while the current one is consumed).
template <typename T, bool DIAG>
__device__ __forceinline__ void dense2_tile(const T* prow, long long ld, bool ok1, int qend, const double (&vc)[2][4],
                                            const double* vr_tile, int gi0, int c0, double (&colM)[2][4],
                                            double (&colC)[2][4], double* rowpart_warp) {
  const int lane = threadIdx.x & 31;
  Elem4<T> A[4], B[4];
  if (qend > 0) {
#pragma unroll
    for (int r = 0; r < 4; ++r) A[r].load(prow + (size_t)r * ld);
  }
#pragma unroll 1
  for (int q = 0; q < qend; ++q) {
    const T* p = prow + (size_t)(4 * q) * ld;
    const int gi = gi0 + 4 * q;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (ok1) B[r].load(p + (size_t)r * ld + 128);
      else B[r].neutral();
    }
    double vr[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) vr[r] = vr_tile[4 * q + r];
    double acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.0;
    dense2_apply<T, DIAG>(A, vc[0], vr, gi, c0, acc, colM[0], colC[0]);
    if (q + 1 < qend) {
#pragma unroll
      for (int r = 0; r < 4; ++r) A[r].load(p + (size_t)(4 + r) * ld);
    }
    dense2_apply<T, DIAG>(B, vc[1], vr, gi, c0 + 128, acc, colM[1], colC[1]);
    const double tot = warp_reduce8(acc);
    if ((lane & 3) == 0) {
      const int qv = lane >> 2;  // 0..3: M of row qv, 4..7: C of row qv-4
      rowpart_warp[(4 * q + (qv & 3)) * 2 + (qv >> 2)] = tot;
    }
  }
  // chunks this warp skips (no columns, or entirely below the diagonal) contribute zeros
  for (int q = qend; q < kRowTile / 4; ++q)
    if (lane < 8) rowpart_warp[(4 * q + (lane & 3)) * 2 + (lane >> 2)] = 0.0;
}

// One run of row tiles [rt_a, rt_b) inside stripe J.
// smem: rowpart[2][8 warps][32 rows][2] + vr[2][32] doubles (double-buffered: one CTA sync per tile).
template <typename T>
__device__ void dense2_run(const MatView& mv, const StageArgs& st, double nrm, int J, int rt_a, int rt_b,
                           const Dense2Buffers& buf, size_t col_slot, double* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double* rowpart = smem;                // [2][8][32][2]
  double* vr_s = smem + 2 * 8 * 32 * 2;  // [2][32]
  const int cw = J * kStripe + warp * kWarpCols;  // first column of this warp
  const int c0 = cw + lane * 4;
  const bool has_cols = cw < mv.ld;
  const bool ok1 = cw + 128 < mv.ld;
  const long long ld = mv.ld;
  const T* Mbase = reinterpret_cast<const T*>(mv.M);

  // the lane's 8 entries of the staged vector, kept in registers for the whole run
  double vc[2][4];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = c0 + s * 128 + e;
      vc[s][e] = (c < mv.m) ? staged_value(st, c, nrm) : 0.0;
    }
  double colM[2][4], colC[2][4];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int e = 0; e < 4; ++e) { colM[s][e] = 0.0; colC[s][e] = 0.0; }

  // entries of the staged vector for the 32 rows of a tile (the column sums need v_row)
  auto stage_rows = [&](int rt, int bufi) {
    if (threadIdx.x < kRowTile) {
      const int g = mv.row0 + rt * kRowTile + threadIdx.x;
      vr_s[bufi * kRowTile + threadIdx.x] = (g < mv.m) ? staged_value(st, g, nrm) : 0.0;
    }
  };
  stage_rows(rt_a, 0);
  __syncthreads();

  int pb = 0;
  for (int rt = rt_a; rt < rt_b; ++rt, pb ^= 1) {
    if (rt + 1 < rt_b) stage_rows(rt + 1, pb ^ 1);  // for the next tile; published by this tile's sync
    const int lr0 = rt * kRowTile;          // local row of the tile
    const int gi0 = mv.row0 + lr0;          // global row
    const bool diag = gi0 >= J * kStripe;   // tile lies inside the diagonal block of the stripe
    // number of 4-row chunks that can hold a strict-upper element (c > r) for this warp's columns
    int qend = has_cols ? kRowTile / 4 : 0;
    if (diag && has_cols) {
      const int span = cw + kWarpCols - 1 - gi0;  // rows gi with gi < cw+255 take part
      qend = span <= 0 ? 0 : min(kRowTile / 4, (span + 3) / 4);
    }
    const T* prow = Mbase + (size_t)lr0 * ld + c0;
    double* rp = rowpart + (size_t)(pb * kWarps + warp) * kRowTile * 2;
    if (diag) dense2_tile<T, true>(prow, ld, ok1, qend, vc, vr_s + pb * kRowTile, gi0, c0, colM, colC, rp);
    else dense2_tile<T, false>(prow, ld, ok1, qend, vc, vr_s + pb * kRowTile, gi0, c0, colM, colC, rp);
    __syncthreads();
    if (threadIdx.x < 2 * kRowTile) {  // add the 8 warps in order, publish the row-type partials of this tile
      const int row = threadIdx.x >> 1, which = threadIdx.x & 1;
      double t = 0.0;
#pragma unroll
      for (int w = 0; w < kWarps; ++w) t += rowpart[((size_t)(pb * kWarps + w) * kRowTile + row) * 2 + which];
      double* dst = which ? buf.rowC : buf.rowM;
      dst[(size_t)J * mv.rows_pad + lr0 + row] = t;
    }
  }
  __syncthreads();  // the next run (or phase) reuses the buffers
  // column-type partials of the whole run
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    const size_t off = col_slot * kStripe + warp * kWarpCols + s * 128 + lane * 4;
    *reinterpret_cast<double4*>(buf.colM + off) = make_double4(colM[s][0], colM[s][1], colM[s][2], colM[s][3]);
    *reinterpret_cast<double4*>(buf.colC + off) = make_double4(colC[s][0], colC[s][1], colC[s][2], colC[s][3]);
  }
}

// whole dense pass of one CTA: (1) its slice of the staged vector -> st.dst and the partial sum,
// (2) its contiguous share of the (stripe, row tile) items
template <typename T>
__device__ __forceinline__ void dense2_phase(const MatView& mv, const Plan2& p, const StageArgs& st, const Dense2Buffers& buf,
                             double* smem) {
  const double nrm = sqrt(st.z);
  // (1) publish the staged vector and its sum (every CTA a contiguous slice, fixed order inside)
  {
    const int per = (mv.m + p.G - 1) / p.G;
    const int j0 = blockIdx.x * per, j1 = min(mv.m, j0 + per);
    double part = 0.0;
    for (int j = j0 + threadIdx.x; j < j1; j += kThreads) {
      const double v = staged_value(st, j, nrm);
      if (st.dst) st.dst[j] = v;
      part += v;
    }
    part = warp_sum(part);
    if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += smem[w];
      buf.sumpart[blockIdx.x] = t;
    }
    __syncthreads();
  }
  // (2) items [t0, t1)
  const long long t0 = p.T * blockIdx.x / p.G, t1 = p.T * (blockIdx.x + 1) / p.G;
  if (t0 >= t1) return;
  int J = p.cta_first_stripe[blockIdx.x];
  long long t = t0;
  int k = 0;
  while (t < t1) {
    const long long sbeg = p.tile_prefix[J], send = p.tile_prefix[J + 1];
    const long long tend = t1 < send ? t1 : send;
    dense2_run<T>(mv, st, nrm, J, (int)(t - sbeg), (int)(tend - sbeg), buf,
                       (size_t)blockIdx.x * p.KMAX + k, smem);
    t = tend; ++J; ++k;
  }
}

// Mhat v, Chat v of local row lr: row-type partials of every stripe that holds the row, then the column-type
// partials of every CTA run that crossed the row's own stripe -- always in the same order
__device__ __forceinline__ void dense2_gather(const MatView& mv, const Plan2& p, const Dense2Buffers& buf, int lr,
                                              double& Mv, double& Cv) {
  const int i = mv.row0 + lr;
  const int Ji = i / kStripe;
  double a = 0.0, c = 0.0;
  for (int J = Ji; J < p.NST; ++J) {
    a += buf.rowM[(size_t)J * mv.rows_pad + lr];
    c += buf.rowC[(size_t)J * mv.rows_pad + lr];
  }
  const int s0 = p.slot_begin[Ji], s1 = p.slot_begin[Ji + 1];
  const size_t col = (size_t)(i - Ji * kStripe);
  int t = s0;
  for (; t + 4 <= s1; t += 4) {  // independent loads in batches of 4, added in list order
    const size_t o0 = (size_t)p.slot_list[t] * kStripe + col, o1 = (size_t)p.slot_list[t + 1] * kStripe + col;
    const size_t o2 = (size_t)p.slot_list[t + 2] * kStripe + col, o3 = (size_t)p.slot_list[t + 3] * kStripe + col;
    const double m0 = buf.colM[o0], m1 = buf.colM[o1], m2 = buf.colM[o2], m3 = buf.colM[o3];
    const double c0 = buf.colC[o0], c1 = buf.colC[o1], c2 = buf.colC[o2], c3 = buf.colC[o3];
    a += m0; a += m1; a += m2; a += m3;
    c += c0; c += c1; c += c2; c += c3;
  }
  for (; t < s1; ++t) {
    const size_t o = (size_t)p.slot_list[t] * kStripe + col;
    a += buf.colM[o];
    c += buf.colC[o];
  }
  Mv = a; Cv = c;
}

// sum of n doubles in a fixed order, identical on every CTA (all threads call; smem >= kWarps doubles)
__device__ __forceinline__ double block_sum_ordered(const double* src, int n, double* smem) {
  double t = 0.0;
  for (int b = threadIdx.x; b < n; b += kThreads) t += __ldcg(src + b);
  t = warp_sum(t);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) smem[threadIdx.x >> 5] = t;
  __syncthreads();
  double r = 0.0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) r += smem[w];
  __syncthreads();
  return r;
}

}  // namespace clp
