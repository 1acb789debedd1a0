// clp_capi.cu -- host side of the C-ABI declared in include/clipper_b200.h.
//
// One handle = one CUDA device + one stream + the dense M store + the solver workspace.
// There is NO CPU implementation of the hot path in this library: every scoring / mat-vec /
// solve call launches the sm_90a kernels of clp_kernels.cuh or fails with an error code.
#include "clp_kernels.cuh"
#include "clp_clique.cuh"
#include "clp_batch_clique.cuh"
#include "clp_batch_matrix.cuh"
#include "clp_sdp.cuh"
#include "clp_knn.cuh"
#include "clp_transform.cuh"
#include "clp_host_utils.h"
#include "clp_jit.h"
#include "../../include/clipper_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>
#include <unistd.h>

#ifndef CLP_VERSION
#define CLP_VERSION "0.1.0"
#endif

using namespace clp;

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) { cudaFree(p); p = nullptr; cap = 0; }
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <typename U> U* as() const { return reinterpret_cast<U*>(p); }
};

struct PinnedBuf {  // page-locked host staging: the asynchronous copies from and to it do not wait for the host
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) { cudaFreeHost(p); p = nullptr; cap = 0; }
    cudaError_t e = cudaMallocHost(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
  template <typename U> U* as() const { return reinterpret_cast<U*>(p); }
};

// layout of the compact copy (compact_shape): whole rows for the resident sweep (one segment W = ld wide, column
// indices; padding entries point at column m of the staged vector), else the plan's column segments (byte offsets)
struct CompactShape {
  bool resident = false;
  int nseg = 0, W = 0;
};

}  // namespace

static int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return (v && *v) ? std::atoi(v) : dflt;
}

// Rounding::DSD_HEU keeps the round(F) largest entries of u (ref clipper.cpp:302-308).  The reference converts with
// (int)std::round(F), which is undefined for NaN (u0 = 0) and for F >= 2^31 (weights near 1e10); here round(F) is
// clamped to [0, m] first and NaN keeps no node.
static int32_t heu_omega(double F, int64_t m) {
  const double r = std::round(F);
  if (!(r >= 1.0)) return 0;
  return r >= (double)m ? (int32_t)m : (int32_t)r;
}

struct clp_handle_s {
  int device = 0;
  int storage = CLP_STORE_F32;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  clp_params prm;
  std::string err;
  int sm_count = 0;
  int ctas_per_sm = 2;       // dense sweeps (and the user cap set by clp_set_ctas_per_sm)
  int ctas_sparse = 3;       // compact-row sweep: latency-bound, few registers -> 3 CTAs per SM
  int ctas_cap = 3;          // user cap (clp_set_ctas_per_sm)
  int ctas_for(int mode) const { return std::min(ctas_cap, mode == 3 ? ctas_sparse : ctas_per_sm); }
  int grid_cap = 0;          // > 0: at most this many CTAs in the persistent kernels (clp_set_grid_cap)
  int spin_seconds = env_int("CLP_SPIN_SECONDS", 4);  // bound of every in-kernel wait of the resident solver
  int grid_for(int ctas) const { const int g = sm_count * ctas; return grid_cap > 0 ? std::min(g, grid_cap) : g; }

  // sharding (row block [row0,row0+rows) of the m x m matrix lives here)
  int rank = 0, world = 1;
  DevBuf comm;                          // CommBlock, mapped into every peer
  uint4* peer_ll[kMaxPeers] = {};       // every rank's LL block
  CommBlock* peer_comm[kMaxPeers] = {};
  bool peer_opened[kMaxPeers] = {};     // pointers obtained with cudaIpcOpenMemHandle
  void* peer_open_ptr[kMaxPeers][2] = {};
  bool shard_ready = false;
  unsigned long long seq = 0;           // exchange sequence number (monotonic across solves)
  void* exported_ll = nullptr;          // llbuf.p at export time (peers hold this mapping)

  // problem
  long long m = 0;
  int row0 = 0, rows = 0, rows_pad = 0;
  long long ld = 0;
  bool has_matrix = false;
  DevBuf Mbuf;
  bool has_A = false;
  bool A_host_valid = false;
  std::vector<int32_t> A_host;  // column-major m x 2
  DevBuf A_dev;                 // int32 [2m]
  DevBuf E1, E2, D1dev, D2dev, F12;  // F12: fp32 positions of both endpoints (screening pass of the scoring kernel)
  DevBuf inv_prm;                    // parameters of a CUDA-source invariant (CLP_INV_MAX_PARAMS doubles)
  int prof_ctas = env_int("CLP_PROF_CTAS", 0);      // print the per-CTA phase times of every resident solve (stderr)
  int prof_host = env_int("CLP_PROF_HOST", 0);      // print wall-clock marks of the scoring / solve calls (stderr)
  int prof_laps = env_int("CLP_PROF_LAPS", 1);      // in-kernel phase timers (the split reported in clp_solution.prof_*)
  DevBuf prof_buf;
  // resident-vector solver (clp_resident.cuh): the default whenever the whole trial vector fits shared memory
  int res_G = 0;                                    // CTAs of the resident kernels for the current matrix
  int res_NI = 0;
  int smem_optin = 0;                               // cudaDevAttrMaxSharedMemoryPerBlockOptin
  int l2_bytes = 0;                                 // cudaDevAttrL2CacheSize
  int pack = env_int("CLP_PACK", 1);              // resident layout of plain fp32 matrices with 4-byte entries (0: always 6 bytes)

  // solver workspace
  DevBuf vecs;    // V_SLOTS x mpad doubles: U0 U1 MV0 MV1 CV0 CV1 (local only)
  DevBuf llbuf;   // L_SLOTS x mpad LL cells (16 B): X G0 G1 -- replicated across shards via peer stores
  DevBuf parts;   // partM | partC : 2 x NSEG x rows_pad
  DevBuf small;   // segsum[kMaxSeg] | red[2][G][kRedVals]
  DevBuf result;  // SolverOut (256 B) | u_final[mpad]
  DevBuf u0dev;   // [mpad]
  DevBuf ybuf;    // matvec scratch: v | y | Mv | Cv  (4 x mpad)
  DevBuf sync;    // counter (u64) | error (int) | flags (int) | counts (2 x u64)
  DevBuf res_vecs, res_cand, res_pieces, res_redll;  // resident solver: plain vectors | candidate points | piece table | LL sums
  DevBuf panel;   // staging panels for get/set dense
  DevBuf cscbuf;
  PinnedBuf pinned;
  Plan plan{};
  long long mpad = 0;
  // stripe decomposition (clp_dense2.cuh)
  int dense_mode = 4;     // requested: 0 segments, 2 stripes/upper-triangle two-sided (one GPU),
                          //            3 compact rows (segmented), 6 compact rows + resident vector,
                          //            4 auto (6 if the vector fits shared memory, else 3, when the graph is sparse enough; else 2 / 0)
  int dense_mode_eff = 2; // effective, decided when the matrix is finalised
  // compact-row copy (clp_sparse.cuh)
  DevBuf sp_val, sp_col, sp_ptr4, sp_part, sp_item, sp_rowid;  // sp_ptr4: kept entries per (segment, row)
  DevBuf sp_hist, sp_bsum;  // compact build: class histograms of the row tiles | block sums of the scans
  DevBuf sp_win, res_wcol;  // packed layout: occupied 16-column windows per row | members' columns where every warp starts
  // packed layout on one GPU: the resident solver's restricted copy (values | columns | slot offsets | row lengths | S' of
  // every CTA | row products), sized once per build for the largest S' that can be taken
  DevBuf res_rval, res_rcol, res_roff, res_rlen, res_rbits, res_rprod;
  bool res_restrict = false;
  ResSweeps last_sweeps{};  // sweep counters of the last solve
  unsigned long long sp_nnz = 0, sp_nnz_real = 0;
  CompactShape sp_shape{};  // layout of the last compact copy built
  SparseView sp{};
  Plan2 plan2{};
  Dense2Buffers d2{};
  DevBuf d2buf, plan2buf;
  // maximum clique (clp_clique.cuh): the bitset adjacency is built on the first call and dropped with the matrix
  DevBuf mc_adj, mc_work, mc_scratch;
  bool mc_adj_valid = false;
  // semidefinite relaxation (clp_sdp.cuh): problem table | X offset | counter | SdpOut | p | evec1 | X | scratch slot
  DevBuf sdp_buf;
  // putative associations (clp_knn.cuh): staged clouds | partial lists | merged lists | counts and scans | staged A
  DevBuf knn_buf;
  // rigid transform (clp_transform.cuh): bad key | problem table | rows | packed pairs | results; its pinned staging
  DevBuf tf_buf;
  PinnedBuf tf_pinned;

  size_t esize() const { return storage == CLP_STORE_F64 ? 8 : 4; }
  int entry_bytes() const { return sp.packed ? 4 : (int)esize() + 2; }  // compact copy: bytes per stored entry
  int wwords() const { return (int)((ld + 511) / 512); }  // 32-bit words of a row's window bitmap
  // the packed layout may be built: whole rows, fp32, one GPU, not switched off
  bool pack_candidate() const { return pack && storage == CLP_STORE_F32 && world == 1; }
};

namespace {

// the message of the last failed create on this thread, one per handle type (clp_handle_s, clp_batch_s): what
// clp_last_error(nullptr) and clp_batch_last_error(nullptr) return
template <typename H>
std::string& create_error() {
  thread_local std::string msg;
  return msg;
}

// records msg on the handle (or, without one, as the failed create's message) and returns code
template <typename H>
int fail(H* h, int code, const std::string& msg) {
  (h ? h->err : create_error<H>()) = msg;
  return code;
}

#define CLP_CUDA(h, call)                                                                  \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess)                                                                \
      return fail(h, e__ == cudaErrorMemoryAllocation ? CLP_ERR_ALLOC : CLP_ERR_CUDA,      \
                  std::string(#call) + ": " + cudaGetErrorString(e__));                    \
  } while (0)

inline long long round_up(long long x, long long q) { return (x + q - 1) / q * q; }
// element strides of a dense device matrix (clp_set_dense_dev, clp_batch_solve_dense_dev): one is 1, the other >= 1
inline bool dense_strides_ok(long long rs, long long cs) { return (rs == 1 && cs >= 1) || (cs == 1 && rs >= 1); }
int reset_sync(clp_handle h);

// f(T{}) with T the handle's storage type (float or double)
template <typename F>
decltype(auto) with_storage(clp_handle h, F&& f) {
  return h->storage == CLP_STORE_F64 ? f(double{}) : f(float{});
}

// nothing may propagate out of an extern "C" entry point (the library is loaded into Python and into C callers)
template <typename H, typename F>
int guarded(H* h, F&& f) {
  try { return f(); }
  catch (const std::bad_alloc&) { return fail(h, CLP_ERR_ALLOC, "host allocation failed"); }
  catch (const std::exception& e) { return fail(h, CLP_ERR_INVALID, std::string("internal error: ") + e.what()); }
  catch (...) { return fail(h, CLP_ERR_INVALID, "internal error"); }
}

// the checks clp_create and clp_batch_create share: the ordinal names a device, and that device is an sm_90
template <typename H>
int probe_device(int device, cudaDeviceProp* prop) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail<H>(nullptr, CLP_ERR_CUDA, std::string("no usable CUDA device: ") + cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail<H>(nullptr, CLP_ERR_INVALID, "device ordinal out of range");
  if ((e = cudaGetDeviceProperties(prop, device)) != cudaSuccess) return fail<H>(nullptr, CLP_ERR_CUDA, cudaGetErrorString(e));
  if (prop->major != 9 || prop->minor != 0)
    return fail<H>(nullptr, CLP_ERR_CUDA, "clipper_b200 is built for sm_90a only; device is sm_" + std::to_string(prop->major) +
                                              std::to_string(prop->minor));
  return CLP_OK;
}

SolverParams solver_params(const clp_params& P) {
  SolverParams prm;
  prm.tol_u = P.tol_u; prm.tol_F = P.tol_F; prm.beta = P.beta; prm.eps = P.eps;
  prm.maxiniters = P.maxiniters; prm.maxoliters = P.maxoliters; prm.maxlsiters = P.maxlsiters;
  prm.rescale_u0 = P.rescale_u0 ? 1 : 0;
  return prm;
}

void shard_rows(long long m, int rank, int world, int* row0, int* rows) {
  // row tiles of 32 are never split between shards
  const long long tiles = (m + kRowTile - 1) / kRowTile;
  const long long t0 = tiles * rank / world, t1 = tiles * (rank + 1) / world;
  long long r0 = t0 * kRowTile, r1 = std::min<long long>(t1 * kRowTile, m);
  if (r0 > m) r0 = m;
  *row0 = (int)r0; *rows = (int)std::max<long long>(0, r1 - r0);
}

// choose the CTA / segment decomposition of the mat-vec for this problem size.  The column segmentation
// (NSEG, W) depends on m only -- the compact-row copy is cut along it -- while SG / RG follow the grid size.
Plan make_plan(long long m, int rows_pad, int G) {
  Plan p;
  p.G = G;
  const long long cols128 = (m + 127) / 128;
  int sgmax = 1;
  for (int cand : {8, 4, 2, 1}) if (cand <= std::max<long long>(1, cols128)) { sgmax = cand; break; }
  const long long nseg_min = (m + kSegMax - 1) / kSegMax;
  long long NSEG = sgmax * std::max<long long>(1, (nseg_min + sgmax - 1) / sgmax);
  long long W = round_up((m + NSEG - 1) / NSEG, 128);
  if (W < 128) W = 128;
  NSEG = std::max<long long>(sgmax, round_up((m + W - 1) / W, sgmax));
  int SG = 1;
  for (int cand : {8, 4, 2, 1}) if (cand <= sgmax && G % cand == 0) { SG = cand; break; }
  p.SG = SG; p.RG = G / SG; p.NSEG = (int)NSEG; p.W = (int)W; p.NRT = rows_pad / kRowTile;
  return p;
}

// stripe decomposition of the upper triangle: item enumeration, per-CTA runs, buffers (clp_dense2.cuh)
int build_plan2(clp_handle h) {
  const int G = h->plan.G;
  Plan2& p = h->plan2;
  p.G = G;
  p.NST = (int)((h->m + kStripe - 1) / kStripe);
  p.NRT = h->rows_pad / kRowTile;
  std::vector<long long> prefix((size_t)p.NST + 1, 0);
  for (int J = 0; J < p.NST; ++J) {  // stripe J holds the row tiles up to its diagonal block
    const long long nt = std::min<long long>(p.NRT, (long long)(J + 1) * (kStripe / kRowTile));
    prefix[(size_t)J + 1] = prefix[(size_t)J] + nt;
  }
  p.T = prefix[(size_t)p.NST];
  std::vector<int> first((size_t)G, 0), lo((size_t)p.NST, G), hi((size_t)p.NST, -1), has((size_t)G, 0);
  int kmax = 1;
  for (int b = 0; b < G; ++b) {
    const long long t0 = p.T * b / G, t1 = p.T * (b + 1) / G;
    if (t0 >= t1) continue;
    has[(size_t)b] = 1;
    int J = 0;
    while (prefix[(size_t)J + 1] <= t0) ++J;
    first[(size_t)b] = J;
    int k = 0;
    long long t = t0;
    while (t < t1) {
      lo[(size_t)J] = std::min(lo[(size_t)J], b); hi[(size_t)J] = std::max(hi[(size_t)J], b);
      t = std::min(t1, prefix[(size_t)J + 1]); ++J; ++k;
    }
    kmax = std::max(kmax, k);
  }
  p.KMAX = kmax;
  // per stripe, the ordered list of column-partial slots (one per CTA run crossing the stripe)
  std::vector<int> slot_begin((size_t)p.NST + 1, 0), slot_list;
  for (int J = 0; J < p.NST; ++J) {
    slot_begin[(size_t)J] = (int)slot_list.size();
    for (int b = lo[(size_t)J]; b <= hi[(size_t)J]; ++b)
      if (has[(size_t)b]) slot_list.push_back(b * kmax + (J - first[(size_t)b]));
  }
  slot_begin[(size_t)p.NST] = (int)slot_list.size();
  // device copies of the small integer tables
  const size_t b_prefix = ((size_t)p.NST + 1) * sizeof(long long);
  const size_t b_int = (2 * (size_t)G + 2 * (size_t)p.NST + slot_begin.size() + slot_list.size()) * sizeof(int);
  CLP_CUDA(h, h->plan2buf.ensure(b_prefix + b_int + 64));
  char* base = h->plan2buf.as<char>();
  std::vector<int> ints;
  ints.insert(ints.end(), first.begin(), first.end());
  ints.insert(ints.end(), lo.begin(), lo.end());
  ints.insert(ints.end(), hi.begin(), hi.end());
  ints.insert(ints.end(), has.begin(), has.end());
  ints.insert(ints.end(), slot_begin.begin(), slot_begin.end());
  ints.insert(ints.end(), slot_list.begin(), slot_list.end());
  CLP_CUDA(h, cudaMemcpyAsync(base, prefix.data(), b_prefix, cudaMemcpyHostToDevice, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(base + b_prefix, ints.data(), b_int, cudaMemcpyHostToDevice, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));  // the host vectors go out of scope
  p.tile_prefix = reinterpret_cast<const long long*>(base);
  p.cta_first_stripe = reinterpret_cast<const int*>(base + b_prefix);
  p.stripe_cta_lo = p.cta_first_stripe + G;
  p.stripe_cta_hi = p.stripe_cta_lo + p.NST;
  p.cta_has_items = p.stripe_cta_hi + p.NST;
  p.slot_begin = p.cta_has_items + G;
  p.slot_list = p.slot_begin + p.NST + 1;
  // partial-product buffers
  const size_t n_row = (size_t)p.NST * h->rows_pad;
  const size_t n_col = (size_t)G * p.KMAX * kStripe;
  CLP_CUDA(h, h->d2buf.ensure((2 * n_row + 2 * n_col + (size_t)G) * sizeof(double) + 64));
  double* d = h->d2buf.as<double>();
  h->d2.rowM = d; h->d2.rowC = d + n_row;
  h->d2.colM = d + 2 * n_row; h->d2.colC = h->d2.colM + n_col;
  h->d2.sumpart = h->d2.colC + n_col;
  return CLP_OK;
}


// ------------------------------------------------------------------------------------------
// resident-vector solver (clp_resident.cuh): one load pipeline per handle type (ResShape)
// ------------------------------------------------------------------------------------------
struct ResKernels { const void* solver; const void* matvec; int NT; };
template <typename T>
ResKernels res_kernels(clp_handle h) {
  if (h->world > 1)
    return {(const void*)solver_resident_kernel<T, true>, (const void*)matvec_resident_kernel<T, ResShape<T, true>>, ResShape<T, true>::NT};
  using S = ResShape<T, false>;
  if constexpr (sizeof(T) == 4)
    if (h->sp.packed)
      return {h->res_restrict ? (const void*)solver_resident_kernel<T, false, true, true> : (const void*)solver_resident_kernel<T, false, true>,
              (const void*)matvec_resident_kernel<T, S, true>, S::NT};
  return {(const void*)solver_resident_kernel<T, false>, (const void*)matvec_resident_kernel<T, S>, S::NT};
}
int res_warps(clp_handle h) {
  return with_storage(h, [&](auto t) { return res_kernels<decltype(t)>(h); }).NT / 32;
}

// On-chip tables behind the plan's minimum: the CTA's piece table and per-row solver state, sized for 1.5x the mean
// CTA (a CTA that exceeds them falls back to the HBM copies on its own).  Kept to a few KB on purpose: launching with
// all 227 KB leaves no L1 for the streaming sweep.
void res_pick_caps(clp_handle h, unsigned int* pieces_cap, unsigned int* state_cap) {
  *pieces_cap = 0; *state_cap = 0;
  if (h->res_G < 1) return;
  const int NW = res_warps(h);
  const unsigned int items = (unsigned int)((h->res_NI + h->res_G - 1) / h->res_G);
  // the partition is balanced by bytes, so CTAs holding short rows hold more items than the mean: 2x the mean + slack
  unsigned int pc = 2 * items + 8 + (unsigned int)NW, sc = 4 * (2 * items + 8);
  const unsigned int base = res_smem_plan((int)h->m, NW).total;
  const unsigned int budget = std::min<unsigned int>(32u << 10, (unsigned int)std::max(0, h->smem_optin - (int)base - 256));
  if (pc * 64u + sc * 72u > budget) {  // keep the piece table first, then as much row state as fits -- or none
    if (pc * 64u > budget) return;
    sc = 0;
  }
  *pieces_cap = pc; *state_cap = sc;
}
unsigned int res_launch_smem(clp_handle h) {
  unsigned int pc, sc;
  res_pick_caps(h, &pc, &sc);
  return res_smem_plan((int)h->m, res_warps(h), pc, sc).total_ext;
}

// The one decision of the compact layout for the current m, requested mode and plan: whole rows when the resident
// solver can take the problem (mode 4 or 6, the vector fits shared memory), else the plan's column segments.  The
// scoring kernel counts for this layout and the build cuts along it; the plan's NSEG and W depend on m only.
CompactShape compact_shape(clp_handle h) {
  const bool resident = h->m <= kResMaxM && h->m <= 65535 && (h->dense_mode == 4 || h->dense_mode == 6) &&
                        (long long)res_smem_plan((int)h->m, kResThreads / 32).total <= (long long)h->smem_optin;
  if (resident) return {true, 1, (int)h->ld};
  return {false, h->plan.NSEG, h->plan.W};
}

template <typename T>
cudaError_t res_set_attrs(clp_handle h) {
  // [storage][sharded][packed][restricted][device]: set once per process (handles may live on different host threads)
  static std::atomic<bool> done[2][2][2][2][8];
  std::atomic<bool>& flag = done[sizeof(T) == 8 ? 1 : 0][h->world > 1 ? 1 : 0][h->sp.packed ? 1 : 0][h->res_restrict ? 1 : 0][h->device & 7];
  if (flag.load(std::memory_order_acquire)) return cudaSuccess;
  // the attribute is a per-function PERMISSION shared by every handle of the process (two shards in one process ask
  // for different sizes): always the device maximum; the carve-out follows what each launch actually requests
  const ResKernels k = res_kernels<T>(h);
  cudaError_t rc = cudaFuncSetAttribute(k.matvec, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin);
  if (rc == cudaSuccess) rc = cudaFuncSetAttribute(k.solver, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin);
  if (rc == cudaSuccess) flag.store(true, std::memory_order_release);
  return rc;
}

// the result buffer's 256-byte header: SolverOut, then the resident solver's sweep counters
constexpr size_t kSweepsAt = 128;
static_assert(sizeof(SolverOut) <= kSweepsAt && kSweepsAt + sizeof(ResSweeps) <= 256, "result header layout");

ResArgs res_args(clp_handle h) {
  ResArgs a;
  std::memset(&a, 0, sizeof(a));
  a.sp = h->sp;
  a.m = (int)h->m; a.row0 = h->row0; a.rows = h->rows; a.rows_pad = h->rows_pad; a.NI = h->res_NI; a.G = h->res_G;
  a.prm = solver_params(h->prm);
  a.u0 = h->u0dev.as<double>();
  a.vecs = h->res_vecs.as<double>();
  a.cand = h->res_cand.as<double>();
  a.ll = h->llbuf.as<uint4>();
  a.mpad = h->mpad;
  a.pieces = h->res_pieces.as<double>();
  a.sb = h->sync.as<SyncBlock>();
  a.u_final = reinterpret_cast<double*>(reinterpret_cast<char*>(h->result.p) + 256);
  a.out = reinterpret_cast<SolverOut*>(h->result.p);
  a.rank = h->rank; a.world = h->world; a.seq0 = h->seq;
  a.comm = h->comm.as<CommBlock>();
  for (int r = 0; r < kMaxPeers; ++r) { a.peer_ll[r] = h->peer_ll[r]; a.peer_comm[r] = h->peer_comm[r]; }
  a.spin_limit = (long long)h->spin_seconds * 1900000000LL;
  res_pick_caps(h, &a.pieces_cap, &a.state_cap);
  a.redll = h->res_redll.as<uint4>();
  a.prof_cta = h->prof_ctas ? h->prof_buf.as<double>() : nullptr;
  a.prof_laps = (h->prof_ctas || h->prof_laps) ? 1 : 0;
  a.wcol = h->res_wcol.as<int>();
  if (h->res_restrict) {
    a.rval = h->res_rval.as<float>(); a.rcol = h->res_rcol.as<unsigned short>(); a.roff = h->res_roff.as<unsigned int>();
    a.rlen = h->res_rlen.as<unsigned int>(); a.rbits = h->res_rbits.as<unsigned int>(); a.rprod = h->res_rprod.as<uint4>();
  }
  a.sweeps = reinterpret_cast<ResSweeps*>(reinterpret_cast<char*>(h->result.p) + kSweepsAt);
  return a;
}

template <typename T>
cudaError_t launch_resident_solver(clp_handle h, ResArgs& a) {
  const ResKernels k = res_kernels<T>(h);
  void* args[] = {&a};
  return cudaLaunchCooperativeKernel(k.solver, dim3(a.G), dim3(k.NT), args, res_launch_smem(h), h->stream);
}

template <typename T>
cudaError_t launch_resident_matvec(clp_handle h, const double* v, double d, double* y, double* Mv, double* Cv) {
  const ResKernels k = res_kernels<T>(h);
  ResArgs a = res_args(h);
  void* args[] = {&a, &v, &d, &y, &Mv, &Cv};
  return cudaLaunchKernel(k.matvec, dim3(a.G), dim3(k.NT), args, res_launch_smem(h), h->stream);
}

constexpr int kKeepDense = -1;  // build_sparse: the compact copy would not pay off (NOT an error code)

// CTAs of the persistent packed fill (sparse_fill_items_kernel<float, true>): at most one wave, and only as many warps
// as the items need in the rounds a full wave would take, so that every round is about equally full.  The occupancy is
// asked once per device.
unsigned packed_fill_grid(clp_handle h, long long items) {
  static std::atomic<int> occ_of[8];  // 0: not asked yet
  std::atomic<int>& slot = occ_of[h->device & 7];
  int occ = slot.load(std::memory_order_relaxed);
  if (occ == 0) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, sparse_fill_items_kernel<float, true>, kDevFillWarps * 32, 0) != cudaSuccess ||
        occ < 1)
      occ = 1;
    slot.store(occ, std::memory_order_relaxed);
  }
  const long long cap = (long long)occ * h->sm_count * kDevFillWarps;  // warps of one wave
  const long long rounds = std::max<long long>(1, (items + cap - 1) / cap);
  const long long warps = (items + rounds - 1) / rounds;
  return (unsigned)std::max<long long>(1, (warps + kDevFillWarps - 1) / kDevFillWarps);
}

// What a scoring launch hands to the compact build of the same call; every other build passes {}.
struct ScoreHandoff {
  // the sync block still carries the scoring launch's error flag (read back with the build's totals: one host
  // synchronisation per scoring call) and zeroed counters
  bool after_score = false;
  // the scoring kernel counted the kept entries for compact_shape(h) into sp_ptr4, and for the packed layout also
  // the occupied windows (sp_win) and the exponent range: the build skips its counting pass
  bool counted = false;
};

// Called once the dense store holds the new matrix: build the compact copy of layout s.
template <typename T>
int build_sparse(clp_handle h, bool force, const CompactShape& s, ScoreHandoff ho) {
  const int nseg = s.nseg;
  const long long nptr = (long long)nseg * (h->rows_pad + 1);
  h->res_restrict = false;  // decided below with the layout; a build that keeps the dense sweep leaves it off
  if (!ho.after_score) { if (int rc = reset_sync(h)) return rc; }
  SyncBlock* sb = h->sync.as<SyncBlock>();
  const T* M = h->Mbuf.as<T>();
  const unsigned blocks = (unsigned)(((size_t)h->rows_pad * 32 + 255) / 256);
  // packed layout (whole rows, fp32): the counts also describe the occupied 16-column windows and the exponent range;
  // the sort and the item lengths then decide on the device whether the fillers count (PackCount::on), the host reads
  // the same decision back with the totals
  const bool want_pack = s.resident && h->pack_candidate();
  const int wwords = h->wwords();
  if (!ho.counted) {
    CLP_CUDA(h, h->sp_ptr4.ensure((size_t)nptr * sizeof(unsigned int)));
    CLP_CUDA(h, cudaMemsetAsync(h->sp_ptr4.p, 0, (size_t)nptr * sizeof(unsigned int), h->stream));
    if (want_pack) {
      CLP_CUDA(h, h->sp_win.ensure((size_t)h->rows_pad * wwords * sizeof(unsigned int)));
      CLP_CUDA(h, cudaMemsetAsync(h->sp_win.p, 0, (size_t)h->rows_pad * wwords * sizeof(unsigned int), h->stream));
    }
    sparse_count_kernel<T><<<blocks, 256, 0, h->stream>>>(M, h->ld, (int)h->m, h->rows, h->rows_pad, s.W, nseg,
                                                          h->sp_ptr4.as<unsigned int>(), &sb->counts[0],
                                                          want_pack ? h->sp_win.as<unsigned int>() : nullptr, wwords, &sb->expo[0]);
    CLP_CUDA(h, cudaGetLastError());
  }
  const PackCount pc{want_pack ? h->sp_win.as<unsigned int>() : nullptr, wwords, (int)((h->m + kWinCols - 1) / kWinCols), h->rows, sb};
  // sort the rows of every segment by slice length, group them four at a time, scan the item lengths
  const int NI = h->rows_pad / 4;
  const long long nitem = (long long)nseg * (NI + 1);
  CLP_CUDA(h, h->sp_rowid.ensure((size_t)nseg * h->rows_pad * sizeof(unsigned int)));
  CLP_CUDA(h, h->sp_item.ensure((size_t)nitem * sizeof(unsigned int)));
  const int nb = s.W / 4 + 2;  // possible slice lengths in chunks
  const int ntile = (h->rows_pad + kSortTile - 1) / kSortTile;
  const long long nhist = (long long)nseg * nb * ntile;
  const long long nblk = (std::max(nhist, nitem) + kScanBlock - 1) / kScanBlock;
  CLP_CUDA(h, h->sp_hist.ensure((size_t)nhist * sizeof(unsigned int)));
  CLP_CUDA(h, h->sp_bsum.ensure((size_t)nblk * sizeof(unsigned long long)));
  unsigned long long* total4_d = reinterpret_cast<unsigned long long*>(&sb->leaf[0][0]);  // scratch words of the sync block
  // exclusive scan in place of n words; total: nullable
  auto scan = [&](unsigned int* a, long long n, unsigned long long* total) -> int {
    const unsigned g = (unsigned)((n + kScanBlock - 1) / kScanBlock);
    sparse_scan_reduce_kernel<<<g, kScanThreads, 0, h->stream>>>(a, n, h->sp_bsum.as<unsigned long long>());
    CLP_CUDA(h, cudaGetLastError());
    sparse_scan_down_kernel<<<g, kScanThreads, 0, h->stream>>>(a, n, h->sp_bsum.as<unsigned long long>(), (int)g, total);
    CLP_CUDA(h, cudaGetLastError());
    return CLP_OK;
  };
  const dim3 tiles((unsigned)ntile, (unsigned)nseg);
  sell_hist_kernel<<<tiles, kSortTile, (size_t)nb * sizeof(unsigned int), h->stream>>>(
      h->sp_ptr4.as<unsigned int>(), h->rows_pad, nb, ntile, h->sp_hist.as<unsigned int>(), ho.counted ? &sb->counts[0] : nullptr, pc);
  CLP_CUDA(h, cudaGetLastError());
  if (int rc = scan(h->sp_hist.as<unsigned int>(), nhist, nullptr)) return rc;
  sell_place_kernel<<<tiles, kSortTile, (size_t)nb * sizeof(unsigned int), h->stream>>>(
      h->sp_ptr4.as<unsigned int>(), h->rows_pad, nb, ntile, h->sp_hist.as<unsigned int>(), h->sp_rowid.as<unsigned int>(),
      h->sp_item.as<unsigned int>(), pc);
  CLP_CUDA(h, cudaGetLastError());
  if (int rc = scan(h->sp_item.as<unsigned int>(), nitem, total4_d)) return rc;
  unsigned long long host[3] = {0, 0, 0};
  unsigned int hexpo[2] = {0u, 0u};
  int host_err = 0;
  CLP_CUDA(h, cudaMemcpyAsync(&host[0], total4_d, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(&host[1], &sb->counts[0], 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  if (want_pack) CLP_CUDA(h, cudaMemcpyAsync(hexpo, &sb->expo[0], sizeof(hexpo), cudaMemcpyDeviceToHost, h->stream));
  if (ho.after_score) CLP_CUDA(h, cudaMemcpyAsync(&host_err, &sb->error, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  if (host_err == 2) return fail(h, CLP_ERR_INVALID, "association index out of range of D1/D2");
  const unsigned long long n4 = host[0];
  if (n4 >= 0xffffffffull) { if (force) return fail(h, CLP_ERR_UNSUPPORTED, "compact rows: too many entries"); return kKeepDense; }
  h->sp_nnz = 4 * n4;        // stored entries (incl. the padding of slices and items): what one pass reads
  h->sp_nnz_real = host[1];  // non-neutral entries of the local rows
  h->sp.plain = host[2] == 0 ? 1 : 0;
  unsigned int bias = 0u;
  h->sp.packed = (want_pack && h->sp.plain && pack_window(hexpo[0], hexpo[1], &bias)) ? 1 : 0;  // = pc.on() on the device
  h->sp.ebias = bias << 23;
  // worth it?  compare with the bytes of the best dense sweep (upper triangle two-sided on one GPU, full rows when sharded)
  const double sparse_bytes = (double)h->sp_nnz * h->entry_bytes();
  const double dense_bytes = (h->world > 1) ? (double)sizeof(T) * h->rows * (double)h->m : 0.5 * sizeof(T) * (double)h->m * (double)h->m;
  if (!force && !(sparse_bytes < 0.8 * dense_bytes)) return kKeepDense;  // keep a dense sweep
  CLP_CUDA(h, h->sp_val.ensure((size_t)std::max<unsigned long long>(h->sp_nnz, 4) * sizeof(T)));
  if (!h->sp.packed) CLP_CUDA(h, h->sp_col.ensure((size_t)std::max<unsigned long long>(h->sp_nnz, 4) * sizeof(unsigned short)));
  unsigned int* next_item = reinterpret_cast<unsigned int*>(&sb->leaf[5][0]);  // zeroed with the sync block
  if (h->sp.packed) {  // whole rows (nseg = 1), fp32 only
    if constexpr (sizeof(T) == 4)
      sparse_fill_items_kernel<T, true><<<packed_fill_grid(h, NI), kDevFillWarps * 32, 0, h->stream>>>(
          M, h->ld, (int)h->m, h->rows, h->rows_pad, s.W, nseg, h->sp_item.as<unsigned int>(), h->sp_rowid.as<unsigned int>(),
          h->sp_val.as<T>(), nullptr, 0, 0u, next_item, bias);
  } else {
    const long long nwarp = (long long)nseg * NI;  // one warp per item
    sparse_fill_items_kernel<T><<<(unsigned)((nwarp + kDevFillWarps - 1) / kDevFillWarps), kDevFillWarps * 32, 0, h->stream>>>(
        M, h->ld, (int)h->m, h->rows, h->rows_pad, s.W, nseg, h->sp_item.as<unsigned int>(), h->sp_rowid.as<unsigned int>(),
        h->sp_val.as<T>(), h->sp_col.as<unsigned short>(), s.resident ? 0 : 3, s.resident ? (unsigned int)h->m : kZeroSlot, nullptr);
  }
  CLP_CUDA(h, cudaGetLastError());
  h->sp.val = h->sp_val.p; h->sp.off16 = h->sp.packed ? nullptr : h->sp_col.as<unsigned short>();
  h->sp.itemptr = h->sp_item.as<unsigned int>(); h->sp.rowid = h->sp_rowid.as<unsigned int>(); h->sp.rows_pad = h->rows_pad;
  // byte-balanced contiguous item range of every CTA (depends on the grid size: rebuilt with the plan)
  int G = h->plan.G;
  if (s.resident) {
    // one fat CTA per SM; small problems use fewer CTAs -- every CTA should stream at least ~32 KB per sweep, since
    // with more CTAs the per-evaluation exchange costs more than the sweep saves; shards sharing a GPU honour the cap
    h->res_NI = NI;
    const long long by_bytes = (long long)((double)h->sp_nnz * h->entry_bytes() / (32.0 * 1024.0));
    G = (int)std::max<long long>(1, std::min<long long>(std::min<long long>(h->grid_cap > 0 ? std::min(h->grid_cap, h->sm_count) : h->sm_count, NI / 2),
                                                        std::max<long long>(1, by_bytes)));
    h->res_G = G;
    // sweeps over the support of the trial vector (the restricted copy, allocated below): packed copy on one GPU,
    // only when it does not fit L2 -- a copy that does is served from L2 after the first pass anyway, and there the
    // streamed full sweep beat the per-row restricted one (config 1: 3.3 against 4.0 ms per solve, DESIGN.md section 6)
    h->res_restrict = h->sp.packed && h->world == 1 && (double)h->sp_nnz * sizeof(T) > (double)h->l2_bytes;
    CLP_CUDA(h, res_set_attrs<T>(h));
    const int NW = res_warps(h);
    CLP_CUDA(h, h->res_vecs.ensure((size_t)R_SLOTS * h->mpad * sizeof(double)));
    CLP_CUDA(h, h->res_cand.ensure((size_t)4 * h->mpad * sizeof(double)));
    CLP_CUDA(h, h->res_pieces.ensure(((size_t)NI + (size_t)G * NW + 8) * kPieceVals * sizeof(double)));
    CLP_CUDA(h, h->res_redll.ensure((size_t)2 * G * kRedVals * sizeof(uint4)));
  }
  CLP_CUDA(h, h->sp_part.ensure(((size_t)G + 1) * sizeof(unsigned int)));
  sparse_partition_kernel<<<(G + 1 + 255) / 256, 256, 0, h->stream>>>(h->sp.itemptr, h->rows_pad, nseg, G, h->sp_part.as<unsigned int>());
  CLP_CUDA(h, cudaGetLastError());
  h->sp.cta_first = h->sp_part.as<unsigned int>();
  if (h->sp.packed) {  // where every warp of the resident kernels starts: once per build, not per sweep
    const int NW = res_warps(h);
    CLP_CUDA(h, h->res_wcol.ensure((size_t)G * NW * 4 * sizeof(int)));
    res_warp_cols_kernel<<<(unsigned)((G * NW * 32 + 255) / 256), 256, 0, h->stream>>>(h->sp, G, NW, h->res_wcol.as<int>());
    CLP_CUDA(h, cudaGetLastError());
  }
  // the restricted copy: every row slot sized for the largest S' a rebuild takes
  if (h->res_restrict) {
    const unsigned long long ent = std::max<unsigned long long>(
        4, std::min<unsigned long long>(h->sp_nnz, (unsigned long long)h->rows_pad * res_restrict_cap(~0u, (int)h->m)));
    CLP_CUDA(h, h->res_rval.ensure((size_t)ent * sizeof(float)));
    CLP_CUDA(h, h->res_rcol.ensure((size_t)ent * sizeof(unsigned short)));
    CLP_CUDA(h, h->res_roff.ensure(((size_t)NI + 1) * sizeof(unsigned int)));
    CLP_CUDA(h, h->res_rlen.ensure((size_t)h->rows_pad * sizeof(unsigned int)));
    CLP_CUDA(h, h->res_rbits.ensure((size_t)G * ((h->m + 31) / 32) * sizeof(unsigned int)));
    CLP_CUDA(h, h->res_rprod.ensure((size_t)h->rows_pad * 2 * sizeof(uint4)));
    res_restrict_caps_kernel<<<(unsigned)((NI + 1 + 255) / 256), 256, 0, h->stream>>>(h->sp.itemptr, NI, (int)h->m, h->res_roff.as<unsigned int>());
    CLP_CUDA(h, cudaGetLastError());
    if (int rc = scan(h->res_roff.as<unsigned int>(), (long long)NI + 1, nullptr)) return rc;
  }
  h->sp_shape = s;
  return CLP_OK;
}

int set_plan_for(clp_handle h, int mode) {
  int ctas = h->ctas_for(mode);
  if (mode == 3) {
    // more than 2 CTAs/SM only pay off when every CTA still gets several 32-row tiles
    while (ctas > 2) {
      const Plan pc = make_plan(h->m, h->rows_pad, h->grid_for(ctas));
      if (pc.NRT >= 4 * pc.RG) break;
      --ctas;
    }
  }
  h->plan = make_plan(h->m, h->rows_pad, h->grid_for(ctas));
  CLP_CUDA(h, h->parts.ensure((size_t)2 * h->plan.NSEG * h->rows_pad * sizeof(double)));
  CLP_CUDA(h, h->small.ensure(((size_t)kMaxSeg + (size_t)2 * h->plan.G * kRedVals) * sizeof(double)));
  return CLP_OK;
}

// the plan of the requested mode, before a matrix decides the effective one: auto (4) plans for the compact sweep
int plan_requested(clp_handle h) { return set_plan_for(h, h->dense_mode == 3 || h->dense_mode == 4 ? 3 : h->dense_mode); }

// modes 3, 4 and 6 try the compact copy first
bool compact_requested(clp_handle h) { return h->dense_mode == 3 || h->dense_mode == 4 || h->dense_mode == 6; }

int finalize_matrix_impl(clp_handle h, ScoreHandoff ho) {
  int eff = h->dense_mode;
  if (compact_requested(h)) {
    h->sp.plain = 0; h->sp.packed = 0;
    if (int rc = set_plan_for(h, 3)) return rc;
    const CompactShape s = compact_shape(h);
    const bool force = (eff == 3) || (eff == 6);
    const int rc = with_storage(h, [&](auto t) { return build_sparse<decltype(t)>(h, force, s, ho); });
    if (rc == CLP_OK) eff = s.resident ? 6 : 3;
    else if (rc == kKeepDense) eff = (h->world > 1) ? 0 : 2;
    else return rc;
  }
  if (eff == 2 && h->world > 1) eff = 0;  // a shard holds row blocks, not the whole upper triangle
  if (eff != 3 && eff != 6) { if (int rc = set_plan_for(h, eff)) return rc; }
  h->dense_mode_eff = eff;
  if (eff == 2) { if (int rc = build_plan2(h)) return rc; }
  return CLP_OK;
}

int finalize_matrix(clp_handle h, ScoreHandoff ho = {}) { return guarded(h, [&] { return finalize_matrix_impl(h, ho); }); }

// (re)allocate the matrix store for problem size m under the current shard config
int ensure_matrix(clp_handle h, long long m) {
  if (m <= 0) return fail(h, CLP_ERR_INVALID, "number of associations must be positive");
  if (m > (long long)kMaxSeg * kSegMax) return fail(h, CLP_ERR_INVALID, "m exceeds the supported maximum (262144)");
  CLP_CUDA(h, cudaSetDevice(h->device));
  h->mc_adj_valid = false;  // the max-clique adjacency describes the previous matrix
  h->mc_adj.release();
  h->mc_scratch.release();
  h->m = m;
  shard_rows(m, h->rank, h->world, &h->row0, &h->rows);
  h->rows_pad = (int)round_up(std::max(h->rows, 1), kRowTile);
  h->ld = round_up(m, 128);
  h->mpad = round_up(m, 128);
  CLP_CUDA(h, h->Mbuf.ensure((size_t)h->rows_pad * (size_t)h->ld * h->esize()));
  // workspace
  CLP_CUDA(h, h->vecs.ensure((size_t)V_SLOTS * h->mpad * sizeof(double)));
  {
    void* before = h->llbuf.p;
    CLP_CUDA(h, h->llbuf.ensure((size_t)5 * h->mpad * sizeof(uint4)));  // 3 vectors (segmented solver) / 5 (resident solver)
    if (h->llbuf.p != before) {  // fresh cells carry tag 0 == "never written"
      CLP_CUDA(h, cudaMemset(h->llbuf.p, 0, h->llbuf.cap));
      h->shard_ready = false;
    }
  }
  if (int rc = plan_requested(h)) return rc;
  CLP_CUDA(h, h->result.ensure(256 + (size_t)h->mpad * sizeof(double)));
  CLP_CUDA(h, h->u0dev.ensure((size_t)h->mpad * sizeof(double)));
  CLP_CUDA(h, h->ybuf.ensure((size_t)4 * h->mpad * sizeof(double)));
  CLP_CUDA(h, h->pinned.ensure(256 + (size_t)h->mpad * sizeof(double)));
  h->has_matrix = false;
  return CLP_OK;
}

MatView mat_view(clp_handle h) {
  MatView mv;
  mv.M = h->Mbuf.p; mv.ld = h->ld; mv.m = (int)h->m; mv.row0 = h->row0; mv.rows = h->rows; mv.rows_pad = h->rows_pad;
  return mv;
}

int reset_sync(clp_handle h) {
  CLP_CUDA(h, cudaMemsetAsync(h->sync.p, 0, sizeof(SyncBlock), h->stream));
  return CLP_OK;
}

int read_sync(clp_handle h, SyncBlock* sb) {
  CLP_CUDA(h, cudaMemcpyAsync(sb, h->sync.p, sizeof(SyncBlock), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  return CLP_OK;
}

// fp32 storage and (PointNormal, or Euclidean with d = 2 or 3): the scoring kernel screens every pair in fp32 first
// and also counts the kept entries (first pass of the compact build); every other case runs the plain kernel.  The
// screened kernel's shared-memory block is sized for fp32 storage.
bool screened_scoring(clp_handle h, int kind, int d) {
  return h->storage == CLP_STORE_F32 && kind != 2 && (kind == 1 || d == 2 || d == 3);
}

// The persistent screened kernel runs one wave: as many CTAs as fit on the device at once.  The shared-memory opt-in
// (more than 48 KB) is a property of the current device's context and is set on every launch; the occupancy is asked
// once per device ordinal (ordinals past the table are asked every time).
template <int KIND, int D, bool MIRROR>
int launch_score_runs(clp_handle h, const ScoreArgs& a) {
  const auto kernel = score_tile_kernel_runs<KIND, D, MIRROR>;
  constexpr int smem = (int)sizeof(ScoreRunSmem<KIND == 1 ? 6 : D>);
  CLP_CUDA(h, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  constexpr int kCachedDevices = 64;
  static std::atomic<int> occ_of[kCachedDevices];  // 0: not asked yet
  const bool cached = h->device >= 0 && h->device < kCachedDevices;
  int occ = cached ? occ_of[h->device].load(std::memory_order_relaxed) : 0;
  if (occ == 0) {
    CLP_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, kThreads, smem));
    if (occ < 1) return fail(h, CLP_ERR_CUDA, "the screened scoring kernel does not fit on an SM");
    if (cached) occ_of[h->device].store(occ, std::memory_order_relaxed);
  }
  const int nruns = (int)((h->ld / 128 + kRunTiles - 1) / kRunTiles), nrb = h->rows_pad / kRowTile;
  const long long units = score_units_before<MIRROR>(nrb, nruns);
  const unsigned grid = (unsigned)std::min<long long>(units, (long long)occ * h->sm_count);
  kernel<<<grid, kThreads, smem, h->stream>>>(a);
  CLP_CUDA(h, cudaGetLastError());
  return CLP_OK;
}

template <typename T, bool MIRROR>
int launch_score_m(clp_handle h, int kind, int d, const ScoreArgs& a, const void* custom) {
  dim3 grid((unsigned)(h->ld / 128), (unsigned)(h->rows_pad / kRowTile));
  if (kind == 2) {  // score_tile_kernel<T, 2, D, MIRROR> compiled for the caller's invariant (clp_jit.cpp)
    void* args[] = {const_cast<ScoreArgs*>(&a)};
    CLP_CUDA(h, cudaLaunchKernel(custom, grid, dim3(kThreads), args, 0, h->stream));
  } else if constexpr (sizeof(T) == 4) {
    if (!screened_scoring(h, kind, d)) score_tile_kernel<T, 0, 0, MIRROR><<<grid, kThreads, 0, h->stream>>>(a);
    else if (kind == 1) return launch_score_runs<1, 6, MIRROR>(h, a);
    else if (d == 3) return launch_score_runs<0, 3, MIRROR>(h, a);
    else return launch_score_runs<0, 2, MIRROR>(h, a);
  } else {
    if (kind == 1) score_tile_kernel<T, 1, 6, MIRROR><<<grid, kThreads, 0, h->stream>>>(a);
    else if (d == 3) score_tile_kernel<T, 0, 3, MIRROR><<<grid, kThreads, 0, h->stream>>>(a);
    else if (d == 2) score_tile_kernel<T, 0, 2, MIRROR><<<grid, kThreads, 0, h->stream>>>(a);
    else score_tile_kernel<T, 0, 0, MIRROR><<<grid, kThreads, 0, h->stream>>>(a);
  }
  CLP_CUDA(h, cudaGetLastError());
  return CLP_OK;
}
template <typename T>
int launch_score(clp_handle h, int kind, int d, const ScoreArgs& a, const void* custom) {
  // an unsharded handle holds the whole symmetric matrix: compute the upper triangle, mirror the rest
  return (h->world == 1) ? launch_score_m<T, true>(h, kind, d, a, custom) : launch_score_m<T, false>(h, kind, d, a, custom);
}

// common tail of the scoring entry points: D1/D2/A already on the device.  kind 0 Euclidean, 1 PointNormal, 2 a
// CUDA-source invariant: `custom` is its compiled kernel, its parameters are in h->inv_prm.
int score_on_device(clp_handle h, int kind, const double* D1d, int d, long long n1, const double* D2d,
                    long long n2, const int32_t* Ad, long long m, double p0, double p1, double p2, double p3,
                    const void* custom) {
  const auto tp0 = std::chrono::steady_clock::now();
  if (int rc = ensure_matrix(h, m)) return rc;
  CLP_CUDA(h, h->E1.ensure((size_t)m * d * sizeof(double)));
  CLP_CUDA(h, h->E2.ensure((size_t)m * d * sizeof(double)));
  CLP_CUDA(h, h->F12.ensure((size_t)2 * m * sizeof(float4)));
  if (int rc = reset_sync(h)) return rc;
  SyncBlock* sb = h->sync.as<SyncBlock>();
  const int tb = 256;
  gather_endpoints_kernel<<<(unsigned)((m + tb - 1) / tb), tb, 0, h->stream>>>(
      D1d, D2d, Ad, Ad + m, (int)m, d, n1, n2, h->E1.as<double>(), h->E2.as<double>(), h->F12.as<float4>(),
      h->F12.as<float4>() + m, &sb->scale_bits, &sb->error);
  CLP_CUDA(h, cudaGetLastError());
  ScoreArgs a;
  a.E1 = h->E1.as<double>(); a.E2 = h->E2.as<double>();
  a.A0 = Ad; a.A1 = Ad + m;
  a.M = h->Mbuf.p; a.ld = h->ld; a.m = (int)m; a.row0 = h->row0; a.rows = h->rows; a.rows_pad = h->rows_pad;
  a.F1 = h->F12.as<float4>(); a.F2 = a.F1 + m; a.scale_bits = &sb->scale_bits;
  const CompactShape s = compact_shape(h);  // the layout the build of this call cuts (finalize_matrix_impl)
  const bool compact = compact_requested(h);
  a.cnt = nullptr; a.W = s.W; a.win = nullptr; a.wwords = 0; a.expo = nullptr; a.next_unit = &sb->score_next;
  if (compact && screened_scoring(h, kind, d)) {
    // the screened scoring kernel also counts the kept entries per (segment, row): first pass of the compact build
    const size_t nptr = (size_t)s.nseg * (h->rows_pad + 1);
    CLP_CUDA(h, h->sp_ptr4.ensure(nptr * sizeof(unsigned int)));
    CLP_CUDA(h, cudaMemsetAsync(h->sp_ptr4.p, 0, nptr * sizeof(unsigned int), h->stream));
    a.cnt = h->sp_ptr4.as<unsigned int>();
    // and what the packed layout needs (occupied windows, exponent range), under the build's own condition (want_pack)
    if (s.resident && h->pack_candidate()) {
      const size_t nw = (size_t)h->rows_pad * h->wwords();
      CLP_CUDA(h, h->sp_win.ensure(nw * sizeof(unsigned int)));
      CLP_CUDA(h, cudaMemsetAsync(h->sp_win.p, 0, nw * sizeof(unsigned int), h->stream));
      a.win = h->sp_win.as<unsigned int>(); a.wwords = h->wwords(); a.expo = &sb->expo[0];
    }
  }
  a.d = d; a.p0 = p0; a.p1 = p1; a.p2 = p2; a.p3 = p3; a.affinityeps = h->prm.affinityeps;
  a.prm = (kind == 2) ? h->inv_prm.as<double>() : nullptr;
  int rc = with_storage(h, [&](auto t) { return launch_score<decltype(t)>(h, kind, d, a, custom); });
  if (rc) return rc;
  if (!compact) {  // dense sweeps: nothing else synchronises with the scoring launch
    SyncBlock host;
    if ((rc = read_sync(h, &host))) return rc;
    if (host.error == 2) return fail(h, CLP_ERR_INVALID, "association index out of range of D1/D2");
  }
  const auto tp1 = std::chrono::steady_clock::now();
  if ((rc = finalize_matrix(h, ScoreHandoff{compact, a.cnt != nullptr}))) return rc;
  h->has_matrix = true;
  h->has_A = true;
  if (h->prof_host) {
    const auto tp2 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[clp host] score call: scoring kernel done after %.3f ms, build enqueued after %.3f ms (total)\n",
                 1e3 * std::chrono::duration<double>(tp1 - tp0).count(), 1e3 * std::chrono::duration<double>(tp2 - tp0).count());
  }
  return CLP_OK;
}

// a CUDA-source invariant (kind 2): its source and parameters
struct CustomInvariant {
  const char* source;
  const double* prm;  // host, nprm doubles
  int nprm;
};

// the scoring entry points: D1, D2 and A on the host (clp_score_*) or on the device (clp_score_*_dev)
int score(clp_handle h, bool on_device, int kind, const double* D1, int d, long long n1, const double* D2,
          long long n2, const int32_t* A, long long m, double p0, double p1, double p2, double p3,
          const CustomInvariant* inv = nullptr) {
  if (!h) return CLP_ERR_INVALID;
  if (!D1 || !D2 || d <= 0 || n1 <= 0 || n2 <= 0 || (on_device && (m < 0 || (A && m == 0))))
    return fail(h, CLP_ERR_INVALID, on_device ? "bad device arguments" : "bad data set arguments");
  CLP_CUDA(h, cudaSetDevice(h->device));
  const bool all_to_all = (A == nullptr || m == 0);  // all-to-all hypothesis (ref clipper.cpp:24, utils.h:61-71)
  if (all_to_all) {
    m = n1 * n2;
    if (m > (long long)kMaxSeg * kSegMax) return fail(h, CLP_ERR_INVALID, "all-to-all hypothesis too large");
  } else if (m < 0) return fail(h, CLP_ERR_INVALID, "negative m");
  const void* custom = nullptr;
  if (kind == 2) {  // compiled and loaded before anything of the handle changes: a failure leaves its matrix as it was
    std::string err;
    if (int rc = jit_score_kernel(JitKernel::kScoreTile, inv->source, d, h->storage == CLP_STORE_F64, h->world == 1, h->device, &custom, &err))
      return fail(h, rc, err);
    CLP_CUDA(h, h->inv_prm.ensure(CLP_INV_MAX_PARAMS * sizeof(double)));
    if (inv->nprm > 0)
      CLP_CUDA(h, cudaMemcpyAsync(h->inv_prm.p, inv->prm, (size_t)inv->nprm * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  }
  CLP_CUDA(h, h->A_dev.ensure((size_t)2 * m * sizeof(int32_t)));
  if (!on_device) {
    CLP_CUDA(h, h->D1dev.ensure((size_t)d * n1 * sizeof(double)));
    CLP_CUDA(h, h->D2dev.ensure((size_t)d * n2 * sizeof(double)));
  }
  if (all_to_all) {  // generated on the device: A never crosses PCIe; the host copy is fetched only if asked for
    all_to_all_kernel<<<(unsigned)std::min<long long>((m + 255) / 256, 4096), 256, 0, h->stream>>>(n1, n2, h->A_dev.as<int32_t>());
    CLP_CUDA(h, cudaGetLastError());
  } else if (on_device) {
    CLP_CUDA(h, cudaMemcpyAsync(h->A_dev.p, A, (size_t)2 * m * sizeof(int32_t), cudaMemcpyDeviceToDevice, h->stream));
  } else {
    h->A_host.assign(A, A + (size_t)2 * m);
    CLP_CUDA(h, cudaMemcpyAsync(h->A_dev.p, h->A_host.data(), (size_t)2 * m * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  }
  h->A_host_valid = !all_to_all && !on_device;
  if (!on_device) {
    CLP_CUDA(h, cudaMemcpyAsync(h->D1dev.p, D1, (size_t)d * n1 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CLP_CUDA(h, cudaMemcpyAsync(h->D2dev.p, D2, (size_t)d * n2 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    D1 = h->D1dev.as<double>(); D2 = h->D2dev.as<double>();
  }
  return score_on_device(h, kind, D1, d, n1, D2, n2, h->A_dev.as<int32_t>(), m, p0, p1, p2, p3, custom);
}

// clp_score_custom(_dev): the built-ins' argument checks, plus the source and the parameter count
int score_custom(clp_handle h, bool on_device, const char* source, const double* prm, int32_t nprm, const double* D1,
                 int32_t d, int64_t n1, const double* D2, int64_t n2, const int32_t* A, int64_t m) {
  if (!h) return CLP_ERR_INVALID;
  if (!source || !*source) return fail(h, CLP_ERR_INVALID, "empty invariant source");
  if (nprm < 0 || nprm > CLP_INV_MAX_PARAMS || (nprm > 0 && !prm))
    return fail(h, CLP_ERR_INVALID, "invariant parameters: 0 to " + std::to_string(CLP_INV_MAX_PARAMS) + " doubles");
  const CustomInvariant inv{source, prm, nprm};
  return score(h, on_device, 2, D1, d, n1, D2, n2, A, m, 0.0, 0.0, 0.0, 0.0, &inv);
}

// opens a load of a caller-given matrix (clp_set_dense, clp_set_sparse_upper): the store for m, no associations, a
// clean sync block for the flags the load raises, every entry neutral
int begin_load(clp_handle h, long long m) {
  if (int rc = ensure_matrix(h, m)) return rc;
  h->has_A = false; h->A_host_valid = false;
  if (int rc = reset_sync(h)) return rc;
  const size_t total = (size_t)h->rows_pad * (size_t)h->ld;
  with_storage(h, [&](auto t) {
    using T = decltype(t);
    fill_neutral_kernel<T><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<T>(), total);
  });
  CLP_CUDA(h, cudaGetLastError());
  return CLP_OK;
}

struct LoadCheck { int flag, code; const char* msg; };  // a flag the load may raise, and the error it makes

// closes it: the first raised flag in the order of checks fails the call, else the matrix is built for its sweep
int end_load(clp_handle h, std::initializer_list<LoadCheck> checks) {
  SyncBlock host;
  if (int rc = read_sync(h, &host)) return rc;
  for (const LoadCheck& c : checks)
    if (host.flags & c.flag) return fail(h, c.code, c.msg);
  if (int rc = finalize_matrix(h)) return rc;
  h->has_matrix = true;
  return CLP_OK;
}

// after a change of the grid knobs: rebuild the loaded matrix for the new grid, or only re-plan
int apply_grid_knobs(clp_handle h) {
  if (h->m == 0) return CLP_OK;
  CLP_CUDA(h, cudaSetDevice(h->device));
  return h->has_matrix ? finalize_matrix(h) : plan_requested(h);
}

template <typename T>
int launch_matvec(clp_handle h, const StageArgs& st, const double* v, double d, double* y, double* Mv, double* Cv) {
  if (h->dense_mode_eff == 6) {  // resident layout: stage, sweep and per-row epilogue in one launch
    CLP_CUDA(h, launch_resident_matvec<T>(h, v, d, y, Mv, Cv));
    return CLP_OK;
  }
  const unsigned cb = (unsigned)((h->rows + 255) / 256);
  if (h->dense_mode_eff == 0 || h->dense_mode_eff == 3) {
    const Plan& p = h->plan;
    double* partM = h->parts.as<double>();
    double* partC = partM + (size_t)p.NSEG * h->rows_pad;
    if (h->dense_mode_eff == 3) matvec_sparse_partials_kernel<T><<<p.G, kThreads, 0, h->stream>>>(mat_view(h), p, st, h->sp, partM, partC);
    else matvec_partials_kernel<T><<<p.G, kThreads, 0, h->stream>>>(mat_view(h), p, st, partM, partC);
    CLP_CUDA(h, cudaGetLastError());
    matvec_combine_kernel<<<cb, 256, 0, h->stream>>>(mat_view(h), p, partM, partC, h->small.as<double>(), v, d, y, Mv, Cv);
  } else {
    matvec2_partials_kernel<T><<<h->plan2.G, kThreads, 0, h->stream>>>(mat_view(h), h->plan2, st, h->d2);
    CLP_CUDA(h, cudaGetLastError());
    matvec2_combine_kernel<<<cb, 256, 0, h->stream>>>(mat_view(h), h->plan2, h->d2, v, d, y, Mv, Cv);
  }
  CLP_CUDA(h, cudaGetLastError());
  return CLP_OK;
}

int matvec_enqueue(clp_handle h, const double* v_dev, double d, double* y_dev, double* Mv_dev, double* Cv_dev) {
  StageArgs st;
  st.mode = STAGE_RAW; st.srcA = v_dev; st.llA = nullptr; st.llB = nullptr; st.tag = 0;
  st.error = &h->sync.as<SyncBlock>()->error; st.alpha = 0.0; st.z = 1.0; st.dst = nullptr;
  st.segsum = h->small.as<double>();
  return with_storage(h, [&](auto t) { return launch_matvec<decltype(t)>(h, st, v_dev, d, y_dev, Mv_dev, Cv_dev); });
}

template <typename T>
cudaError_t launch_solver(clp_handle h, SolverArgs& a) {
  void* args[] = {&a};
  const void* fn = h->dense_mode_eff == 3 ? (const void*)solver_kernel<T, 3>
                 : h->dense_mode_eff == 2 ? (const void*)solver_kernel<T, 2> : (const void*)solver_kernel<T, 0>;
  return cudaLaunchCooperativeKernel(fn, dim3(h->plan.G), dim3(kThreads), args, 0, h->stream);
}

struct ResultHeader {  // first 256 bytes of the result buffer
  SolverOut out;
};

// u0 already in h->u0dev; runs the persistent kernel, brings back scalars + u, rounds on the host
int solve_core(clp_handle h, clp_solution* out, double* u_out_host, double* u_out_dev, int32_t* nodes_out,
               std::chrono::steady_clock::time_point t_begin) {
  const clp_params& P = h->prm;
  if (P.maxlsiters < 1) return fail(h, CLP_ERR_INVALID, "maxlsiters must be >= 1");
  SolverArgs a;
  a.mv = mat_view(h);
  a.plan = h->plan;
  a.prm = solver_params(P);
  SyncBlock* sb = h->sync.as<SyncBlock>();
  a.bar.sb = sb; a.bar.nleaf = std::min(32, h->plan.G); a.bar.G = h->plan.G;
  a.u0 = h->u0dev.as<double>();
  a.vecs = h->vecs.as<double>();
  a.ll = h->llbuf.as<uint4>();
  a.mpad = h->mpad;
  a.partM = h->parts.as<double>();
  a.partC = a.partM + (size_t)h->plan.NSEG * h->rows_pad;
  a.segsum = h->small.as<double>();
  a.red = h->small.as<double>() + kMaxSeg;
  a.plan2 = h->plan2; a.d2 = h->d2; a.sp = h->sp;
  a.out = reinterpret_cast<SolverOut*>(h->result.p);
  a.u_final = reinterpret_cast<double*>(reinterpret_cast<char*>(h->result.p) + 256);
  a.rank = h->rank; a.world = h->world; a.seq0 = h->seq;
  a.comm = h->comm.as<CommBlock>();
  for (int r = 0; r < kMaxPeers; ++r) { a.peer_ll[r] = h->peer_ll[r]; a.peer_comm[r] = h->peer_comm[r]; }
  if (h->world > 1) {
    if (!h->shard_ready || h->exported_ll != h->llbuf.p)
      return fail(h, CLP_ERR_COMM, "sharded solve: peer buffers not connected (clp_shard_export/import after scoring)");
  }

  if (int rc = reset_sync(h)) return rc;
  CLP_CUDA(h, cudaEventRecord(h->ev0, h->stream));
  cudaError_t le;
  if (h->dense_mode_eff == 6) {
    if (h->prof_ctas) CLP_CUDA(h, h->prof_buf.ensure((size_t)h->res_G * 8 * sizeof(double)));
    // the per-CTA partial sums travel as LL cells tagged with the launch-local round number: start from tag 0
    CLP_CUDA(h, cudaMemsetAsync(h->res_redll.p, 0, (size_t)2 * h->res_G * kRedVals * sizeof(uint4), h->stream));
    // so are the row products of the restricted sweeps
    if (h->res_restrict) CLP_CUDA(h, cudaMemsetAsync(h->res_rprod.p, 0, (size_t)h->rows_pad * 2 * sizeof(uint4), h->stream));
    ResArgs ra = res_args(h);
    le = with_storage(h, [&](auto t) { return launch_resident_solver<decltype(t)>(h, ra); });
  } else {
    le = with_storage(h, [&](auto t) { return launch_solver<decltype(t)>(h, a); });
  }
  CLP_CUDA(h, le);
  CLP_CUDA(h, cudaEventRecord(h->ev1, h->stream));
  const size_t rbytes = 256 + (size_t)h->m * sizeof(double);
  CLP_CUDA(h, cudaMemcpyAsync(h->pinned.p, h->result.p, rbytes, cudaMemcpyDeviceToHost, h->stream));
  if (u_out_dev)
    CLP_CUDA(h, cudaMemcpyAsync(u_out_dev, a.u_final, (size_t)h->m * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  const auto tp_sync = std::chrono::steady_clock::now();
  float ms = 0.f;
  CLP_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));

  const SolverOut so = *h->pinned.as<const SolverOut>();
  h->seq = so.seq_end;
  h->last_sweeps = ResSweeps{so.n_evals, 0, 0, 0ull, 0ull, 0};
  if (h->dense_mode_eff == 6 && h->res_restrict)
    h->last_sweeps = *reinterpret_cast<const ResSweeps*>(h->pinned.as<const char>() + kSweepsAt);
  if (h->prof_ctas && h->dense_mode_eff == 6) {  // diagnostics: spread of the per-CTA phase times
    std::vector<double> pc((size_t)h->res_G * 8);
    CLP_CUDA(h, cudaMemcpy(pc.data(), h->prof_buf.p, pc.size() * sizeof(double), cudaMemcpyDeviceToHost));
    if (h->prof_ctas >= 2) {  // one line per CTA: index, ms in sweeps / epilogues / exchanges / staging, items, chunks
                              // (+ restricted entries swept and how far the costliest warp range of the restricted split lies above
                              // its share, in costliest slots: below 1)
      for (int b = 0; b < h->res_G; ++b) {
        std::fprintf(stderr, "[clp cta] %d %.4f %.4f %.4f %.4f %.0f %.0f", b, 1e-6 * pc[(size_t)b * 8], 1e-6 * pc[(size_t)b * 8 + 1],
                     1e-6 * pc[(size_t)b * 8 + 2], 1e-6 * pc[(size_t)b * 8 + 3], pc[(size_t)b * 8 + 4], pc[(size_t)b * 8 + 5]);
        if (h->res_restrict) std::fprintf(stderr, " %.0f %.4f", pc[(size_t)b * 8 + 6], pc[(size_t)b * 8 + 7]);
        std::fprintf(stderr, "\n");
      }
    }
    if (h->res_restrict) {  // the restricted entries each CTA swept (the split of res_restrict_split balances them)
      double lo = 1e300, hi = 0, sum = 0, over = -1;
      for (int b = 0; b < h->res_G; ++b) {
        const double x = pc[(size_t)b * 8 + 6];
        lo = std::min(lo, x); hi = std::max(hi, x); sum += x; over = std::max(over, pc[(size_t)b * 8 + 7]);
      }
      std::fprintf(stderr, "[clp prof] restricted entries per solve: min %.0f  mean %.1f  max %.0f over %d CTAs (split: costliest warp range "
                   "above its share by %.3f costliest slots)\n", lo, sum / h->res_G, hi, h->res_G, over);
    }
    const char* nm[4] = {"sweeps", "epilogues", "exchanges", "staging"};
    for (int q = 0; q < 4; ++q) {
      double lo = 1e300, hi = 0, sum = 0;
      for (int b = 0; b < h->res_G; ++b) { const double x = pc[(size_t)b * 8 + q]; lo = std::min(lo, x); hi = std::max(hi, x); sum += x; }
      std::fprintf(stderr, "[clp prof] %-9s per solve: min %.3f  mean %.3f  max %.3f ms over %d CTAs (%lld evaluations)\n", nm[q],
                   1e-6 * lo, 1e-6 * sum / h->res_G, 1e-6 * hi, h->res_G, (long long)so.n_evals);
    }
  }
  if (so.status != 0) {
    h->shard_ready = false;  // sequence numbers may have diverged between ranks
    return fail(h, CLP_ERR_TIMEOUT, "solver kernel: device-wide barrier / peer exchange timed out");
  }
  const double* u = reinterpret_cast<const double*>(h->pinned.as<const char>() + 256);

  // rounding (ref clipper.cpp:287-310) on the device-produced u
  std::vector<int32_t> nodes;
  if (P.rounding == CLP_ROUND_NONZERO) {
    nodes.resize((size_t)h->m);
    nodes.resize((size_t)clp_find_above(u, h->m, 0.0, nodes.data()));
  } else if (P.rounding == CLP_ROUND_DSD_HEU) {
    const int32_t omega = heu_omega(so.F, h->m);
    if (omega >= 1) {
      nodes.resize((size_t)omega);
      nodes.resize((size_t)clp_find_k_largest(u, h->m, omega, nodes.data()));
    }
  } else if (P.rounding == CLP_ROUND_DSD) {
    std::vector<int32_t> S((size_t)h->m);
    S.resize((size_t)clp_find_above(u, h->m, 0.0, S.data()));
    const int k = (int)S.size();
    if (k > 0 && h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "Rounding::DSD on a sharded handle");
    if (k > 8192) return fail(h, CLP_ERR_UNSUPPORTED, "Rounding::DSD: support(u) larger than 8192 nodes");
    if (k > 0) {
      // ship only the k x k sub-block of M induced by support(u) (SURVEY 8f rank 1)
      CLP_CUDA(h, h->cscbuf.ensure((size_t)k * sizeof(int32_t) + (size_t)k * k * sizeof(double) + 16));
      double* sub_d = h->cscbuf.as<double>();
      int32_t* S_d = reinterpret_cast<int32_t*>(sub_d + (size_t)k * k);
      CLP_CUDA(h, cudaMemcpyAsync(S_d, S.data(), (size_t)k * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
      dim3 g((unsigned)((k + 127) / 128), (unsigned)k);
      with_storage(h, [&](auto t) {
        using T = decltype(t);
        gather_subblock_kernel<T><<<g, 128, 0, h->stream>>>(h->Mbuf.as<T>(), h->ld, S_d, k, sub_d);
      });
      CLP_CUDA(h, cudaGetLastError());
      std::vector<double> sub((size_t)k * k);
      CLP_CUDA(h, cudaMemcpyAsync(sub.data(), sub_d, sub.size() * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
      CLP_CUDA(h, cudaStreamSynchronize(h->stream));
      // n_total = m: the reference runs dsd::solve on the full M_ restricted to S (clipper.cpp:299)
      const std::vector<int32_t> sel = clp::densest_subgraph_dense(sub.data(), k, h->m);
      nodes.resize(sel.size());
      for (size_t i = 0; i < sel.size(); ++i) nodes[i] = S[(size_t)sel[i]];
    }
  } else {
    return fail(h, CLP_ERR_INVALID, "unknown rounding mode");
  }

  if (u_out_host) std::memcpy(u_out_host, u, (size_t)h->m * sizeof(double));
  if (nodes_out && !nodes.empty()) std::memcpy(nodes_out, nodes.data(), nodes.size() * sizeof(int32_t));
  if (out) {
    out->ifinal = so.ifinal; out->n_nodes = (int32_t)nodes.size(); out->score = so.F; out->d_final = so.d;
    out->n_evals = so.n_evals; out->n_matvec = so.n_matvec; out->n_inner = so.n_inner; out->kernel_ms = ms;
    out->prof_matvec_ms = 1e-6 * (double)so.ns_matvec; out->prof_combine_ms = 1e-6 * (double)so.ns_combine;
    out->prof_exchange_ms = 1e-6 * (double)so.ns_exchange;

    out->t = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  }
  if (h->prof_host)
    std::fprintf(stderr, "[clp host] solve call: results on the host after %.3f ms (solver kernel %.3f ms), rounding done after %.3f ms\n",
                 1e3 * std::chrono::duration<double>(tp_sync - t_begin).count(), ms,
                 1e3 * std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count());
  return CLP_OK;
}

// ------------------------------------------------------------------------------------------
// maximum clique (clp_clique.cuh)
// ------------------------------------------------------------------------------------------
struct McLayout {  // int32 regions of mc_work, then 8-byte ones
  int *deg0, *deg, *core, *rnd, *frontier, *later, *seeds, *roots, *nodes;
  unsigned *alive, *ctr;
  int *out, *flags;
  long long* tprefix;
  unsigned long long *best, *next, *branches, *deadline;
};

size_t mc_layout(long long m, int W, char* base, McLayout* L) {
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base + off; off += (bytes + 15) / 16 * 16; return p; };
  const size_t mi = (size_t)m * sizeof(int);
  L->deg0 = (int*)take(mi); L->deg = (int*)take(mi); L->core = (int*)take(mi); L->rnd = (int*)take(mi);
  L->frontier = (int*)take(mi); L->later = (int*)take(mi); L->seeds = (int*)take(mi); L->roots = (int*)take(mi);
  L->nodes = (int*)take(mi + sizeof(int));
  L->alive = (unsigned*)take((size_t)W * sizeof(unsigned)); L->ctr = (unsigned*)take(4 * sizeof(unsigned));
  L->out = (int*)take(4 * sizeof(int)); L->flags = (int*)take(4 * sizeof(int));
  L->tprefix = (long long*)take(((size_t)m + 1) * sizeof(long long));
  L->best = (unsigned long long*)take(8); L->next = (unsigned long long*)take(8);
  L->branches = (unsigned long long*)take(8); L->deadline = (unsigned long long*)take(8);
  return off;
}

struct McPeeled {
  std::vector<int32_t> core, rnd;
  int max_core = 0;
  long long n_edges = 0;
  float adj_ms = 0.f, peel_ms = 0.f;
};

struct McEvents {  // timing of one call; destroyed with the call
  cudaEvent_t e[8] = {};
  ~McEvents() { for (cudaEvent_t x : e) if (x) cudaEventDestroy(x); }
};

float mc_elapsed(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  return cudaEventElapsedTime(&ms, a, b) == cudaSuccess ? ms : 0.f;
}

// EXACT search over tasks of at most K candidates (mc_search_kernel, mc_batch_search_kernel): words of a candidate
// bitset, node arena, scratch bytes per worker, workers (two per SM warp slot, no more than half of free_b holds, whole
// CTAs; fewer than one CTA means the scratch does not fit) and the nanoseconds left of time_limit_s since t0.
struct McSearchSetup {
  int KW;
  unsigned arena_cap;
  size_t stride;
  long long nworkers;
  unsigned long long limit_ns;
};

McSearchSetup mc_search_setup(int K, size_t free_b, int sm_count, double time_limit_s, std::chrono::steady_clock::time_point t0) {
  McSearchSetup s;
  s.KW = (K + 31) / 32;
  s.arena_cap = (unsigned)std::min<long long>((long long)K * (K + 1) / 2 + 64, 1ll << 18);
  s.stride = mc_scratch_bytes(K, s.KW, s.arena_cap);
  const long long want = (long long)sm_count * 2 * kMcSearchWarps;
  s.nworkers = std::min<long long>(want, (long long)(free_b / 2 / s.stride));
  s.nworkers = s.nworkers / kMcSearchWarps * kMcSearchWarps;
  const double left = time_limit_s - std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  const double left_ns = std::max(0.0, left) * 1e9;
  s.limit_ns = left_ns >= 1.8e19 ? ~0ull : (unsigned long long)left_ns;
  return s;
}

// bitset adjacency (built once per matrix) + k-core peel; core numbers and removal iterations come back to the host
int mc_prepare(clp_handle h, McLayout* L, McPeeled* out, McEvents& ev) {
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "maximum clique before any affinity matrix was scored or set");
  if (h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "maximum clique on a sharded handle (a rank holds only its own rows)");
  CLP_CUDA(h, cudaSetDevice(h->device));
  const long long m = h->m;
  const int W = (int)((m + 31) / 32);
  McLayout probe;
  const size_t work = mc_layout(m, W, nullptr, &probe);
  CLP_CUDA(h, h->mc_work.ensure(work));
  mc_layout(m, W, h->mc_work.as<char>(), L);
  for (cudaEvent_t& x : ev.e) CLP_CUDA(h, cudaEventCreate(&x));
  CLP_CUDA(h, cudaEventRecord(ev.e[0], h->stream));
  const bool rebuild = !h->mc_adj_valid;
  if (rebuild) {
    CLP_CUDA(h, h->mc_adj.ensure((size_t)m * W * sizeof(unsigned)));
    with_storage(h, [&](auto t) {
      using T = decltype(t);
      mc_adjacency_kernel<T><<<(unsigned)m, kMcThreads, 0, h->stream>>>(h->Mbuf.as<T>(), h->ld, (int)m, W, h->mc_adj.as<unsigned>(), L->deg0);
    });
    CLP_CUDA(h, cudaGetLastError());
  }
  CLP_CUDA(h, cudaEventRecord(ev.e[1], h->stream));
  // peel: one cooperative launch, every CTA co-resident
  int occ = 0;
  CLP_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, mc_peel_kernel, kMcPeelThreads, 0));
  if (occ < 1) return fail(h, CLP_ERR_CUDA, "k-core peel kernel cannot be resident");
  const int G = h->sm_count * std::min(occ, 2);
  CLP_CUDA(h, cudaMemcpyAsync(L->deg, L->deg0, (size_t)m * sizeof(int), cudaMemcpyDeviceToDevice, h->stream));
  CLP_CUDA(h, cudaMemsetAsync(L->ctr, 0, 4 * sizeof(unsigned), h->stream));
  if (int rc = reset_sync(h)) return rc;
  McPeelArgs pa;
  pa.adj = h->mc_adj.as<unsigned>(); pa.m = (int)m; pa.W = W;
  pa.deg = L->deg; pa.alive = L->alive; pa.core = L->core; pa.rnd = L->rnd; pa.frontier = L->frontier;
  pa.ctr = L->ctr; pa.out = L->out;
  pa.bar.sb = h->sync.as<SyncBlock>(); pa.bar.nleaf = std::min(32, G); pa.bar.G = G;
  void* args[] = {&pa};
  CLP_CUDA(h, cudaLaunchCooperativeKernel((const void*)mc_peel_kernel, dim3(G), dim3(kMcPeelThreads), args, 0, h->stream));
  CLP_CUDA(h, cudaEventRecord(ev.e[2], h->stream));
  out->core.resize((size_t)m); out->rnd.resize((size_t)m);
  std::vector<int32_t> deg0((size_t)m);
  int hout[4] = {0, 0, 0, 0};
  CLP_CUDA(h, cudaMemcpyAsync(out->core.data(), L->core, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(out->rnd.data(), L->rnd, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(deg0.data(), L->deg0, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(hout, L->out, sizeof(hout), cudaMemcpyDeviceToHost, h->stream));
  SyncBlock sb;
  if (int rc = read_sync(h, &sb)) return rc;  // synchronises the stream
  if (sb.error) return fail(h, CLP_ERR_TIMEOUT, "k-core peel: device-wide barrier timed out");
  h->mc_adj_valid = true;
  out->max_core = hout[0];
  long long deg_sum = 0;
  for (int32_t x : deg0) deg_sum += x;
  out->n_edges = deg_sum / 2;
  out->adj_ms = rebuild ? mc_elapsed(ev.e[0], ev.e[1]) : 0.f;
  out->peel_ms = mc_elapsed(ev.e[1], ev.e[2]);
  return CLP_OK;
}

int mc_solve(clp_handle h, int method, double time_limit_s, int32_t* nodes_out, clp_mc_info* info) {
  const auto t0 = std::chrono::steady_clock::now();
  if (method < CLP_MC_EXACT || method > CLP_MC_KCORE) return fail(h, CLP_ERR_INVALID, "unknown maximum-clique method");
  McLayout L;
  McPeeled pk;
  McEvents ev;
  if (int rc = mc_prepare(h, &L, &pk, ev)) return rc;
  const long long m = h->m;
  const int W = (int)((m + 31) / 32);
  const unsigned* adj = h->mc_adj.as<unsigned>();
  std::vector<int32_t> nodes;
  int lb = 0, proven = 0, timed_out = 0;
  long long branches = 0;
  float heu_ms = 0.f, search_ms = 0.f;
  if (method == CLP_MC_KCORE) {  // maxclique.cpp:89-100
    for (long long v = 0; v < m; ++v) if (pk.core[(size_t)v] >= pk.max_core) nodes.push_back((int32_t)v);
  } else {
    // degeneracy order: (removal iteration, index) ascending; seeds and roots run in reverse (descending core)
    std::vector<int32_t> order((size_t)m);
    for (long long v = 0; v < m; ++v) order[(size_t)v] = (int32_t)v;
    std::stable_sort(order.begin(), order.end(), [&](int32_t x, int32_t y) { return pk.rnd[(size_t)x] < pk.rnd[(size_t)y]; });
    std::vector<int32_t> rev(order.rbegin(), order.rend());
    CLP_CUDA(h, cudaMemcpyAsync(L.seeds, rev.data(), (size_t)m * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CLP_CUDA(h, cudaMemsetAsync(L.best, 0, sizeof(unsigned long long), h->stream));
    const size_t row_bytes = (size_t)W * sizeof(unsigned);
    if (row_bytes > (size_t)h->smem_optin) return fail(h, CLP_ERR_UNSUPPORTED, "maximum clique: m too large for the heuristic's shared-memory bitset");
    const int wpc = (int)std::max<size_t>(1, std::min<size_t>(kMcThreads / 32, (size_t)(h->smem_optin - 1024) / row_bytes));
    const size_t smem = (size_t)wpc * row_bytes;
    CLP_CUDA(h, cudaFuncSetAttribute(mc_heu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(smem, row_bytes)));
    const unsigned grid = (unsigned)std::min<long long>((m + wpc - 1) / wpc, (long long)h->sm_count * 16);
    CLP_CUDA(h, cudaEventRecord(ev.e[3], h->stream));
    mc_heu_kernel<<<grid, wpc * 32, smem, h->stream>>>(adj, (int)m, W, L.core, L.seeds, L.best, -1, L.nodes);
    CLP_CUDA(h, cudaGetLastError());
    unsigned long long best = 0;
    CLP_CUDA(h, cudaMemcpyAsync(&best, L.best, sizeof(best), cudaMemcpyDeviceToHost, h->stream));
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));
    const int seed = (int)(0xffffffffu - (unsigned)(best & 0xffffffffull));
    mc_heu_kernel<<<1, 32, row_bytes, h->stream>>>(adj, (int)m, W, L.core, L.seeds, L.best, seed, L.nodes);
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaEventRecord(ev.e[4], h->stream));
    lb = (int)(best >> 32);
    nodes.resize((size_t)lb);
    int replay_size = 0;
    CLP_CUDA(h, cudaMemcpyAsync(nodes.data(), L.nodes, (size_t)lb * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CLP_CUDA(h, cudaMemcpyAsync(&replay_size, L.nodes + m, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));
    heu_ms = mc_elapsed(ev.e[3], ev.e[4]);
    if (replay_size != lb) return fail(h, CLP_ERR_CUDA, "maximum clique: heuristic replay disagrees with its winner");
    const int ub = pk.max_core + 1;
    proven = (lb == ub) ? 1 : 0;
    if (method == CLP_MC_EXACT && lb < ub && time_limit_s > 0) {
      if (pk.max_core > kMcMaxCore)
        return fail(h, CLP_ERR_UNSUPPORTED, "maximum clique EXACT: max core " + std::to_string(pk.max_core) +
                                                " exceeds the search's limit of " + std::to_string(kMcMaxCore) + " (use HEU or KCORE)");
      // roots: core + 1 > lb, reverse degeneracy order; a root with many candidates becomes one task per candidate
      const int nwl = kMcThreads / 32;
      mc_later_count_kernel<<<(unsigned)std::min<long long>((m + nwl - 1) / nwl, (long long)h->sm_count * 16), kMcThreads, 0, h->stream>>>(
          adj, (int)m, W, L.rnd, L.later);
      CLP_CUDA(h, cudaGetLastError());
      std::vector<int32_t> later((size_t)m);
      CLP_CUDA(h, cudaMemcpyAsync(later.data(), L.later, (size_t)m * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
      CLP_CUDA(h, cudaStreamSynchronize(h->stream));
      std::vector<int32_t> roots;
      std::vector<long long> tprefix(1, 0);
      for (int32_t v : rev) {
        if (pk.core[(size_t)v] + 1 <= lb || later[(size_t)v] + 1 <= lb) continue;
        roots.push_back(v);
        tprefix.push_back(tprefix.back() + (later[(size_t)v] > kMcSplit ? later[(size_t)v] : 1));
      }
      const long long ntasks = tprefix.back();
      unsigned long long best_s = mc_key((unsigned)lb, 0u);
      unsigned hflags[4] = {0u, 0u, 0u, 0u};
      if (ntasks > 0) {
        int K = 1;
        for (int32_t v : roots) K = std::max(K, (int)later[(size_t)v]);
        size_t free_b = 0, total_b = 0;
        CLP_CUDA(h, cudaMemGetInfo(&free_b, &total_b));
        const McSearchSetup ss = mc_search_setup(K, free_b, h->sm_count, time_limit_s, t0);
        if (ss.nworkers < kMcSearchWarps)
          return fail(h, CLP_ERR_ALLOC, "maximum clique EXACT: not enough device memory for the search scratch");
        CLP_CUDA(h, h->mc_scratch.ensure((size_t)ss.nworkers * ss.stride));
        CLP_CUDA(h, cudaMemcpyAsync(L.roots, roots.data(), roots.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
        CLP_CUDA(h, cudaMemcpyAsync(L.tprefix, tprefix.data(), tprefix.size() * sizeof(long long), cudaMemcpyHostToDevice, h->stream));
        CLP_CUDA(h, cudaMemcpyAsync(L.best, &best_s, sizeof(best_s), cudaMemcpyHostToDevice, h->stream));
        CLP_CUDA(h, cudaMemsetAsync(L.next, 0, sizeof(unsigned long long), h->stream));
        CLP_CUDA(h, cudaMemsetAsync(L.branches, 0, sizeof(unsigned long long), h->stream));
        CLP_CUDA(h, cudaMemsetAsync(L.flags, 0, 4 * sizeof(int), h->stream));
        McSearchArgs sa;
        sa.adj = adj; sa.m = (int)m; sa.W = W; sa.rnd = L.rnd; sa.roots = L.roots; sa.tprefix = L.tprefix;
        sa.nroots = (int)roots.size(); sa.ntasks = ntasks; sa.K = K; sa.KW = ss.KW; sa.arena_cap = ss.arena_cap;
        sa.scratch = h->mc_scratch.as<unsigned char>(); sa.stride = ss.stride;
        sa.best = L.best; sa.next_task = L.next; sa.n_branches = L.branches; sa.flags = L.flags; sa.deadline = L.deadline;
        sa.replay_task = -1; sa.replay_size = 0; sa.nodes_out = L.nodes;
        const size_t ssmem = (size_t)kMcSearchWarps * 2 * ss.KW * sizeof(unsigned);
        CLP_CUDA(h, cudaFuncSetAttribute(mc_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssmem));
        CLP_CUDA(h, cudaEventRecord(ev.e[5], h->stream));
        mc_deadline_kernel<<<1, 1, 0, h->stream>>>(L.deadline, ss.limit_ns);
        mc_search_kernel<<<(unsigned)(ss.nworkers / kMcSearchWarps), kMcSearchWarps * 32, ssmem, h->stream>>>(sa);
        CLP_CUDA(h, cudaGetLastError());
        unsigned long long hb[2] = {0ull, 0ull};
        CLP_CUDA(h, cudaMemcpyAsync(&hb[0], L.best, 8, cudaMemcpyDeviceToHost, h->stream));
        CLP_CUDA(h, cudaMemcpyAsync(&hb[1], L.branches, 8, cudaMemcpyDeviceToHost, h->stream));
        CLP_CUDA(h, cudaMemcpyAsync(hflags, L.flags, sizeof(hflags), cudaMemcpyDeviceToHost, h->stream));
        CLP_CUDA(h, cudaStreamSynchronize(h->stream));
        best_s = hb[0]; branches = (long long)hb[1];
        const int s = (int)(best_s >> 32);
        if (s > lb) {  // a task beat the heuristic: replay it for the nodes
          sa.replay_task = (long long)(0xffffffffu - (unsigned)(best_s & 0xffffffffull));
          sa.replay_size = s;
          mc_search_kernel<<<1, 32, 2 * ss.KW * sizeof(unsigned), h->stream>>>(sa);
          CLP_CUDA(h, cudaGetLastError());
          int got = 0;
          CLP_CUDA(h, cudaMemcpyAsync(&got, L.nodes + m, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
          CLP_CUDA(h, cudaStreamSynchronize(h->stream));
          if (got < s || got > m) return fail(h, CLP_ERR_CUDA, "maximum clique: search replay did not reproduce its clique");
          nodes.resize((size_t)got);
          CLP_CUDA(h, cudaMemcpyAsync(nodes.data(), L.nodes, (size_t)got * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
        }
        CLP_CUDA(h, cudaEventRecord(ev.e[6], h->stream));
        CLP_CUDA(h, cudaStreamSynchronize(h->stream));
        search_ms = mc_elapsed(ev.e[5], ev.e[6]);
      }
      timed_out = hflags[0] ? 1 : 0;
      proven = (hflags[0] == 0u && hflags[1] == 0u) ? 1 : 0;
    }
    std::sort(nodes.begin(), nodes.end());
  }
  if (nodes_out && !nodes.empty()) std::memcpy(nodes_out, nodes.data(), nodes.size() * sizeof(int32_t));
  if (info) {
    info->n_nodes = (int32_t)nodes.size();
    info->max_core = pk.max_core;
    info->lower_bound = lb;
    info->upper_bound = pk.max_core + 1;
    info->proven = proven;
    info->timed_out = timed_out;
    info->n_edges = pk.n_edges;
    info->n_branches = branches;
    info->adjacency_ms = pk.adj_ms; info->peel_ms = pk.peel_ms; info->heuristic_ms = heu_ms; info->search_ms = search_ms;
    info->kernel_ms = pk.adj_ms + pk.peel_ms + heu_ms + search_ms;
    info->t = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
  return CLP_OK;
}

// ---- semidefinite relaxation (clp_sdp.cuh) ------------------------------------------------------------------------
template <typename H>
int sdp_check_params(H* h, const clp_sdp_params* p, const void* info) {
  if (!p || !info) return fail(h, CLP_ERR_INVALID, "sdp: params and info are required");
  if (p->max_iters < 1) return fail(h, CLP_ERR_INVALID, "sdp: max_iters must be >= 1");
  if (!(p->eps_abs >= 0.0) || !(p->eps_rel >= 0.0) || !(p->time_limit_s >= 0.0))
    return fail(h, CLP_ERR_INVALID, "sdp: eps_abs, eps_rel and time_limit_s must be >= 0 and not NaN");
  return CLP_OK;
}

// the in-kernel time limit: what is left of the call's budget at the launch (0: none)
unsigned long long sdp_limit_ns(const clp_sdp_params& p, std::chrono::steady_clock::time_point t0) {
  if (!(p.time_limit_s > 0.0)) return 0;
  const double left = p.time_limit_s - std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return (unsigned long long)std::max(1.0, std::min(left * 1e9, 1e18));
}

// the answer read out of the last iterate (ref sdp.cpp:249-262): thr = max|evec1| / 2, nodes = {i : |evec1_i| > thr};
// lambdas = p ascending.  info->t is left to the caller.
void sdp_result(const SdpOut& o, int m, const double* pv, const double* ev, float ms, clp_sdp_info* info, int32_t* nodes_out,
                double* lambdas_out, double* evec1_out) {
  double mx = 0.0;
  for (int i = 0; i < m; ++i) mx = std::max(mx, std::fabs(ev[i]));
  const double thr = mx / 2;
  int nn = 0;
  for (int i = 0; i < m; ++i)
    if (std::fabs(ev[i]) > thr) { if (nodes_out) nodes_out[nn] = i; ++nn; }
  if (lambdas_out) { std::memcpy(lambdas_out, pv, (size_t)m * 8); std::sort(lambdas_out, lambdas_out + m); }
  if (evec1_out) std::memcpy(evec1_out, ev, (size_t)m * 8);
  std::memset(info, 0, sizeof(*info));
  info->iters = o.iters; info->converged = o.converged; info->timed_out = o.timed_out; info->n_nodes = nn;
  info->value = o.value; info->bound = o.bound; info->res_pri = o.res_pri; info->res_dual = o.res_dual; info->rho = o.rho;
  info->thr = thr; info->n_sweeps = o.n_sweeps; info->kernel_ms = ms; info->proj_ms = 1e-6 * (double)o.ns_proj;
}

int sdp_solve(clp_handle h, const clp_sdp_params* prm, clp_sdp_info* info, int32_t* nodes_out, double* X_out,
              double* lambdas_out, double* evec1_out) {
  const auto t0 = std::chrono::steady_clock::now();
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "sdp: no affinity matrix has been scored or set");
  if (int rc = sdp_check_params(h, prm, info)) return rc;
  if (h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "sdp: not available on a sharded handle");
  if (h->m > kSdpMaxM)
    return fail(h, CLP_ERR_UNSUPPORTED, "sdp: m = " + std::to_string(h->m) + " exceeds CLP_SDP_MAX_M = " + std::to_string(kSdpMaxM));
  CLP_CUDA(h, cudaSetDevice(h->device));
  const int m = (int)h->m;
  const size_t nv = (size_t)((m + 1) & ~1);
  // device layout: problem table (0) | X offset (64) | counter (128) | SdpOut (256) | p | evec1 | X | scratch slot
  const size_t o_p = 512, o_e = o_p + nv * 8, o_x = o_e + nv * 8, o_slot = (o_x + (size_t)m * m * 8 + 255) & ~(size_t)255;
  CLP_CUDA(h, h->sdp_buf.ensure(o_slot + sdp_slot_bytes(m)));
  char* d = h->sdp_buf.as<char>();
  unsigned char hdr[256] = {};
  BatchMatProblem P{};
  P.m = m;
  std::memcpy(hdr, &P, sizeof(P));
  CLP_CUDA(h, cudaMemcpyAsync(d, hdr, sizeof(hdr), cudaMemcpyHostToDevice, h->stream));
  SdpArgs a{};
  a.prob = reinterpret_cast<const BatchMatProblem*>(d); a.x_off = reinterpret_cast<const long long*>(d + 64); a.nprob = 1;
  a.store = h->Mbuf.p; a.ld = h->ld;
  a.x_out = reinterpret_cast<double*>(d + o_x); a.p_out = reinterpret_cast<double*>(d + o_p);
  a.e_out = reinterpret_cast<double*>(d + o_e); a.out = reinterpret_cast<SdpOut*>(d + 256);
  a.next = reinterpret_cast<int*>(d + 128);
  a.scratch = reinterpret_cast<unsigned char*>(d + o_slot); a.scratch_stride = sdp_slot_bytes(m); a.max_m = m;
  a.max_iters = prm->max_iters; a.eps_abs = prm->eps_abs; a.eps_rel = prm->eps_rel;
  const size_t smem = sdp_smem_bytes(m);
  int rc = with_storage(h, [&](auto t) -> int {
    using T = decltype(t);
    CLP_CUDA(h, cudaFuncSetAttribute(sdp_solve_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    a.limit_ns = sdp_limit_ns(*prm, t0);
    CLP_CUDA(h, cudaEventRecord(h->ev0, h->stream));
    sdp_solve_kernel<T><<<1, kSdpThreads, smem, h->stream>>>(a);
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaEventRecord(h->ev1, h->stream));
    return CLP_OK;
  });
  if (rc) return rc;
  SdpOut o;
  std::vector<double> pe(2 * nv);
  CLP_CUDA(h, cudaMemcpyAsync(&o, d + 256, sizeof(o), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(pe.data(), d + o_p, 2 * nv * 8, cudaMemcpyDeviceToHost, h->stream));
  if (X_out) CLP_CUDA(h, cudaMemcpyAsync(X_out, d + o_x, (size_t)m * m * 8, cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  float ms = 0.f;
  CLP_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  sdp_result(o, m, pe.data(), pe.data() + nv, ms, info, nodes_out, lambdas_out, evec1_out);
  info->t = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  return CLP_OK;
}

// ---- putative associations (clp_knn.cuh) --------------------------------------------------------------------------
static_assert(kKnnMaxK == CLP_KNN_MAX_K && kKnnMaxD == CLP_KNN_MAX_D, "clp_knn.cuh and clipper_b200.h disagree on the caps");
template <int D, int K>
cudaError_t knn_partial(dim3 grid, size_t smem, cudaStream_t s, const KnnArgs& a) {
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(knn_partial_kernel<D, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  knn_partial_kernel<D, K><<<grid, kKnnThreads, smem, s>>>(a);
  return cudaGetLastError();
}

template <int D>
cudaError_t knn_partial_k(int K, dim3 grid, size_t smem, cudaStream_t s, const KnnArgs& a) {
  switch (K) {
    case 1: return knn_partial<D, 1>(grid, smem, s, a);
    case 2: return knn_partial<D, 2>(grid, smem, s, a);
    case 4: return knn_partial<D, 4>(grid, smem, s, a);
    case 8: return knn_partial<D, 8>(grid, smem, s, a);
    case 16: return knn_partial<D, 16>(grid, smem, s, a);
    default: return knn_partial<D, 32>(grid, smem, s, a);
  }
}

cudaError_t knn_merge(int K, unsigned blocks, cudaStream_t s, const KnnArgs& a, double r2, double* lsd, int* lj, int* cnt) {
  switch (K) {
    case 1: knn_merge_kernel<1><<<blocks, 256, 0, s>>>(a, r2, lsd, lj, cnt); break;
    case 2: knn_merge_kernel<2><<<blocks, 256, 0, s>>>(a, r2, lsd, lj, cnt); break;
    case 4: knn_merge_kernel<4><<<blocks, 256, 0, s>>>(a, r2, lsd, lj, cnt); break;
    case 8: knn_merge_kernel<8><<<blocks, 256, 0, s>>>(a, r2, lsd, lj, cnt); break;
    case 16: knn_merge_kernel<16><<<blocks, 256, 0, s>>>(a, r2, lsd, lj, cnt); break;
    default: knn_merge_kernel<32><<<blocks, 256, 0, s>>>(a, r2, lsd, lj, cnt); break;
  }
  return cudaGetLastError();
}

// clp_correspondences(_dev): D1, D2 on the host (staged in knn_buf, A read back into A_out) or on the device (A written
// into A_out).  Nothing of the handle but knn_buf, its stream and its error string is touched.
int correspondences(clp_handle h, bool on_device, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2,
                    int32_t knn, double radius, int enforce_1to1, int32_t* A_out, int64_t capacity, int64_t* m_out) {
  if (!h) return CLP_ERR_INVALID;
  if (!m_out) return fail(h, CLP_ERR_INVALID, "correspondences: m_out is required");
  *m_out = 0;
  if (knn < 1) return fail(h, CLP_ERR_INVALID, "correspondences: knn must be >= 1");
  if (d < 1) return fail(h, CLP_ERR_INVALID, "correspondences: d must be >= 1");
  if (n1 < 0 || n2 < 0) return fail(h, CLP_ERR_INVALID, "correspondences: negative n1 or n2");
  if ((n1 > 0 && !D1) || (n2 > 0 && !D2)) return fail(h, CLP_ERR_INVALID, "correspondences: NULL point cloud");
  if (knn > kKnnMaxK)
    return fail(h, CLP_ERR_UNSUPPORTED, "correspondences: knn = " + std::to_string(knn) + " exceeds CLP_KNN_MAX_K = " +
                                            std::to_string(kKnnMaxK));
  if (d > kKnnMaxD)
    return fail(h, CLP_ERR_UNSUPPORTED, "correspondences: d = " + std::to_string(d) + " exceeds CLP_KNN_MAX_D = " +
                                            std::to_string(kKnnMaxD));
  if (n1 >= kKnnNone || n2 >= kKnnNone)
    return fail(h, CLP_ERR_UNSUPPORTED, "correspondences: n1 and n2 must be below 2^31 - 1 (int32 indices)");
  const int kk = (int)std::min<int64_t>(knn, n2);
  const long long rows = (long long)n1 * kk;
  if (capacity < rows || (rows > 0 && !A_out))
    return fail(h, CLP_ERR_INVALID, "correspondences: A_out holds " + std::to_string(capacity) + " rows, n1 * min(knn, n2) = " +
                                        std::to_string(rows) + " are required");
  if (rows == 0) return CLP_OK;
  CLP_CUDA(h, cudaSetDevice(h->device));
  const cudaStream_t st = h->stream;
  int K = 1;
  while (K < kk) K *= 2;
  const int D = d <= 3 ? d : 0;
  const int T = D > 0 ? kKnnTileReg : kKnnTileGen;
  // candidate slices: enough CTAs for every SM several times over, each slice at least 1024 candidates
  const long long qblocks = (n1 + kKnnThreads - 1) / kKnnThreads;
  const long long want = (4LL * h->sm_count + qblocks - 1) / qblocks;
  const long long nsplit0 = std::max<long long>(1, std::min<long long>({want, (n2 + 1023) / 1024, 1024}));
  const long long chunk = round_up((n2 + nsplit0 - 1) / nsplit0, T);
  const int nsplit = (int)((n2 + chunk - 1) / chunk);
  // scratch layout, every region 256-byte aligned
  const long long nmax = std::max<long long>(n1, n2);
  const long long nb = (nmax + kKnnScanItems - 1) / kKnnScanItems;
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at = (at + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_d1 = on_device ? 0 : take((size_t)d * n1 * 8), o_d2 = on_device ? 0 : take((size_t)d * n2 * 8);
  const size_t lsize = (size_t)nsplit * kk * n1;
  const size_t o_psd = take(lsize * 8), o_pj = take(lsize * 4);
  const size_t o_lsd = nsplit > 1 ? take((size_t)kk * n1 * 8) : o_psd, o_lj = nsplit > 1 ? take((size_t)kk * n1 * 4) : o_pj;
  const size_t o_cnt = take((size_t)nmax * 4), o_off = take((size_t)nmax * 8), o_bsum = take((size_t)nb * 8), o_tot = take(8);
  const size_t o_best = enforce_1to1 ? take((size_t)n2 * 8) : 0, o_c0 = enforce_1to1 ? take((size_t)n2 * 4) : 0;
  const size_t o_a = on_device ? 0 : take((size_t)2 * rows * 4);
  CLP_CUDA(h, h->knn_buf.ensure(at));
  char* base = h->knn_buf.as<char>();
  auto at_ = [&](size_t o) { return reinterpret_cast<void*>(base + o); };
  if (!on_device) {
    CLP_CUDA(h, cudaMemcpyAsync(at_(o_d1), D1, (size_t)d * n1 * 8, cudaMemcpyHostToDevice, st));
    CLP_CUDA(h, cudaMemcpyAsync(at_(o_d2), D2, (size_t)d * n2 * 8, cudaMemcpyHostToDevice, st));
    D1 = static_cast<const double*>(at_(o_d1)); D2 = static_cast<const double*>(at_(o_d2));
  }
  int32_t* A = on_device ? A_out : static_cast<int32_t*>(at_(o_a));
  KnnArgs a{};
  a.D1 = D1; a.D2 = D2; a.d = d; a.n1 = n1; a.n2 = n2; a.kk = kk; a.nsplit = nsplit; a.chunk = chunk;
  a.part_sd = static_cast<double*>(at_(o_psd)); a.part_j = static_cast<int*>(at_(o_pj));
  double* lsd = static_cast<double*>(at_(o_lsd));
  int* lj = static_cast<int*>(at_(o_lj));
  int* cnt = static_cast<int*>(at_(o_cnt));
  long long* off = static_cast<long long*>(at_(o_off));
  long long* bsum = static_cast<long long*>(at_(o_bsum));
  long long* total = static_cast<long long*>(at_(o_tot));
  const dim3 grid((unsigned)qblocks, (unsigned)nsplit);
  const size_t smem = knn_partial_smem(D, d);
  cudaError_t e;
  switch (D) {
    case 1: e = knn_partial_k<1>(K, grid, smem, st, a); break;
    case 2: e = knn_partial_k<2>(K, grid, smem, st, a); break;
    case 3: e = knn_partial_k<3>(K, grid, smem, st, a); break;
    default: e = knn_partial_k<0>(K, grid, smem, st, a); break;
  }
  CLP_CUDA(h, e);
  const double r2 = radius * radius;  // bm_utils.cpp:192: NaN keeps nothing, inf keeps every neighbour
  const unsigned b1 = (unsigned)((n1 + 255) / 256), b2 = (unsigned)((n2 + 255) / 256);
  CLP_CUDA(h, knn_merge(K, b1, st, a, r2, lsd, lj, cnt));
  if (!enforce_1to1) {
    knn_scan_blocks_kernel<<<(unsigned)((n1 + kKnnScanItems - 1) / kKnnScanItems), 256, 0, st>>>(cnt, n1, off, bsum);
    knn_scan_top_kernel<<<1, 1024, 0, st>>>(bsum, (n1 + kKnnScanItems - 1) / kKnnScanItems, total);
    knn_write_kernel<<<b1, 256, 0, st>>>(cnt, off, bsum, lj, n1, total, A);
  } else {
    auto* best = static_cast<unsigned long long*>(at_(o_best));
    auto* c0best = static_cast<unsigned int*>(at_(o_c0));
    CLP_CUDA(h, cudaMemsetAsync(best, 0xff, (size_t)n2 * 8, st));
    CLP_CUDA(h, cudaMemsetAsync(c0best, 0xff, (size_t)n2 * 4, st));
    knn_best_sd_kernel<<<b1, 256, 0, st>>>(cnt, lsd, lj, n1, best);
    knn_best_c0_kernel<<<b1, 256, 0, st>>>(cnt, lsd, lj, n1, best, c0best);
    knn_flag_kernel<<<b2, 256, 0, st>>>(c0best, n2, cnt);
    knn_scan_blocks_kernel<<<(unsigned)((n2 + kKnnScanItems - 1) / kKnnScanItems), 256, 0, st>>>(cnt, n2, off, bsum);
    knn_scan_top_kernel<<<1, 1024, 0, st>>>(bsum, (n2 + kKnnScanItems - 1) / kKnnScanItems, total);
    knn_write_1to1_kernel<<<b2, 256, 0, st>>>(c0best, off, bsum, n2, total, A);
  }
  CLP_CUDA(h, cudaGetLastError());
  long long m = 0;
  CLP_CUDA(h, cudaMemcpyAsync(&m, total, sizeof(m), cudaMemcpyDeviceToHost, st));
  CLP_CUDA(h, cudaStreamSynchronize(st));
  if (!on_device && m > 0) {
    CLP_CUDA(h, cudaMemcpyAsync(A_out, A, (size_t)2 * m * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CLP_CUDA(h, cudaStreamSynchronize(st));
  }
  *m_out = m;
  return CLP_OK;
}

}  // namespace

// ==========================================================================================
// C-ABI
// ==========================================================================================
extern "C" {

const char* clp_version(void) { return "clipper_b200 " CLP_VERSION " (sm_90a, dense f32/f64 store, fp64 solver)"; }

void clp_default_params(clp_params* p) {
  if (!p) return;
  p->tol_u = 1e-8; p->tol_F = 1e-9; p->tol_Fop = 1e-10;
  p->maxiniters = 200; p->maxoliters = 1000;
  p->beta = 0.25; p->maxlsiters = 99;
  p->eps = 1e-9; p->affinityeps = 1e-4;
  p->rescale_u0 = 1; p->rounding = CLP_ROUND_DSD_HEU;
}

int clp_create(int device, int storage, clp_handle* out) {
  if (!out) return CLP_ERR_INVALID;
  *out = nullptr;
  if (storage != CLP_STORE_F32 && storage != CLP_STORE_F64) return fail<clp_handle_s>(nullptr, CLP_ERR_INVALID, "unknown storage type");
  cudaDeviceProp prop;
  if (int rc = probe_device<clp_handle_s>(device, &prop)) return rc;
  if (!prop.cooperativeLaunch) return fail<clp_handle_s>(nullptr, CLP_ERR_CUDA, "device lacks cooperative launch");
  clp_handle h = new (std::nothrow) clp_handle_s();
  if (!h) return fail<clp_handle_s>(nullptr, CLP_ERR_ALLOC, "host allocation failed");
  h->device = device; h->storage = storage; h->sm_count = prop.multiProcessorCount;
  clp_default_params(&h->prm);
  auto bail = [&](const char* what, cudaError_t ce) {
    clp_destroy(h);
    return fail<clp_handle_s>(nullptr, CLP_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(ce));
  };
  cudaError_t e;
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  if ((e = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaEventCreate(&h->ev0)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaEventCreate(&h->ev1)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = h->sync.ensure(sizeof(SyncBlock))) != cudaSuccess) return bail("cudaMalloc", e);
  int occ = 0, occ3 = 0;
  {
    int o0 = 0, o2 = 0;
    if (storage == CLP_STORE_F64) {
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o0, solver_kernel<double, 0>, kThreads, 0);
      if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o2, solver_kernel<double, 2>, kThreads, 0);
      if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ3, solver_kernel<double, 3>, kThreads, 0);
    } else {
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o0, solver_kernel<float, 0>, kThreads, 0);
      if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o2, solver_kernel<float, 2>, kThreads, 0);
      if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ3, solver_kernel<float, 3>, kThreads, 0);
    }
    occ = std::min(o0, o2);
  }
  if (e != cudaSuccess || occ < 1 || occ3 < 1) return bail("occupancy query (is the sm_90a image loadable?)", e);
  h->ctas_per_sm = std::min(occ, 2);
  h->ctas_sparse = std::min(occ3, 3);
  if ((e = cudaDeviceGetAttribute(&h->l2_bytes, cudaDevAttrL2CacheSize, device)) != cudaSuccess)
    return bail("cudaDeviceGetAttribute", e);
  if ((e = cudaDeviceGetAttribute(&h->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device)) != cudaSuccess)
    return bail("cudaDeviceGetAttribute", e);

  *out = h;
  return CLP_OK;
}

int clp_destroy(clp_handle h) {
  if (!h) return CLP_OK;
  cudaSetDevice(h->device);
  for (int r = 0; r < kMaxPeers; ++r)
    if (h->peer_opened[r]) { cudaIpcCloseMemHandle(h->peer_open_ptr[r][0]); cudaIpcCloseMemHandle(h->peer_open_ptr[r][1]); }
  h->comm.release();
  for (DevBuf* b : {&h->Mbuf, &h->A_dev, &h->E1, &h->E2, &h->F12, &h->inv_prm, &h->D1dev, &h->D2dev, &h->vecs, &h->llbuf, &h->d2buf, &h->plan2buf, &h->sp_val, &h->sp_col, &h->sp_ptr4, &h->sp_part, &h->sp_item, &h->sp_rowid, &h->parts, &h->small,
                    &h->result, &h->u0dev, &h->ybuf, &h->sync, &h->panel, &h->cscbuf, &h->res_vecs, &h->res_cand, &h->res_pieces, &h->res_redll, &h->prof_buf,
                    &h->res_rval, &h->res_rcol, &h->res_roff, &h->res_rlen, &h->res_rbits, &h->res_rprod,
                    &h->mc_adj, &h->mc_work, &h->mc_scratch, &h->sdp_buf, &h->knn_buf, &h->tf_buf})
    b->release();
  h->pinned.release();
  h->tf_pinned.release();
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream && h->own_stream) cudaStreamDestroy(h->stream);
  delete h;
  return CLP_OK;
}

const char* clp_last_error(clp_handle h) { return h ? h->err.c_str() : create_error<clp_handle_s>().c_str(); }

int clp_set_params(clp_handle h, const clp_params* p) {
  if (!h || !p) return CLP_ERR_INVALID;
  if (p->rounding < 0 || p->rounding > 2) return fail(h, CLP_ERR_INVALID, "unknown rounding mode");
  h->prm = *p;
  return CLP_OK;
}
int clp_get_params(clp_handle h, clp_params* p) {
  if (!h || !p) return CLP_ERR_INVALID;
  *p = h->prm;
  return CLP_OK;
}

int clp_set_stream(clp_handle h, void* cuda_stream) {
  if (!h) return CLP_ERR_INVALID;
  CLP_CUDA(h, cudaSetDevice(h->device));
  if (h->stream && h->own_stream) { cudaStreamSynchronize(h->stream); cudaStreamDestroy(h->stream); }
  if (cuda_stream) { h->stream = reinterpret_cast<cudaStream_t>(cuda_stream); h->own_stream = false; }
  else { CLP_CUDA(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true; }
  return CLP_OK;
}

// ---- scoring ------------------------------------------------------------------------------
int clp_score_euclidean(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2,
                        const int32_t* A, int64_t m, double sigma, double epsilon, double mindist) {
  return guarded(h, [&] { return score(h, false, 0, D1, d, n1, D2, n2, A, m, sigma, epsilon, mindist, 0.0); });
}
int clp_score_pointnormal(clp_handle h, const double* D1, int64_t n1, const double* D2, int64_t n2,
                          const int32_t* A, int64_t m, double sigp, double epsp, double sign, double epsn) {
  return guarded(h, [&] { return score(h, false, 1, D1, 6, n1, D2, n2, A, m, sigp, epsp, sign, epsn); });
}
int clp_score_euclidean_dev(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2,
                            const int32_t* A, int64_t m, double sigma, double epsilon, double mindist) {
  return guarded(h, [&] { return score(h, true, 0, D1, d, n1, D2, n2, A, m, sigma, epsilon, mindist, 0.0); });
}
int clp_score_pointnormal_dev(clp_handle h, const double* D1, int64_t n1, const double* D2, int64_t n2,
                              const int32_t* A, int64_t m, double sigp, double epsp, double sign, double epsn) {
  return guarded(h, [&] { return score(h, true, 1, D1, 6, n1, D2, n2, A, m, sigp, epsp, sign, epsn); });
}


int clp_score_custom(clp_handle h, const char* source, const double* prm, int32_t nprm, const double* D1, int32_t d,
                     int64_t n1, const double* D2, int64_t n2, const int32_t* A, int64_t m) {
  return guarded(h, [&] { return score_custom(h, false, source, prm, nprm, D1, d, n1, D2, n2, A, m); });
}
int clp_score_custom_dev(clp_handle h, const char* source, const double* prm, int32_t nprm, const double* D1_dev,
                         int32_t d, int64_t n1, const double* D2_dev, int64_t n2, const int32_t* A_dev, int64_t m) {
  return guarded(h, [&] { return score_custom(h, true, source, prm, nprm, D1_dev, d, n1, D2_dev, n2, A_dev, m); });
}

int clp_invariant_check(const char* source, int32_t d, char* log, int64_t log_bytes) {
  std::string msg;
  int rc = CLP_ERR_INVALID;
  if (!source || !*source) msg = "empty invariant source";
  else if (d <= 0) msg = "dimension must be positive";
  else {
    try { rc = jit_check(source, d, &msg); }
    catch (const std::exception& e) { msg = std::string("internal error: ") + e.what(); rc = CLP_ERR_INVALID; }
  }
  if (log && log_bytes > 0) {
    const size_t n = std::min<size_t>(msg.size(), (size_t)log_bytes - 1);
    std::memcpy(log, msg.data(), n);
    log[n] = '\0';
  }
  return rc;
}

int clp_jit_stats(int64_t* compiles, double* compile_ms) {
  long long c = 0;
  jit_stats(&c, compile_ms);
  if (compiles) *compiles = c;
  return CLP_OK;
}

// ---- get / set ----------------------------------------------------------------------------
int clp_set_dense(clp_handle h, const double* M, const double* C, int64_t m) {
  if (!h || !M || !C) return CLP_ERR_INVALID;
  if (int rc = begin_load(h, m)) return rc;
  SyncBlock* sb = h->sync.as<SyncBlock>();
  // column panels of at most 32 MB per matrix
  const long long pc = std::max<long long>(1, std::min<long long>(m, (32ll << 20) / (8 * m)));
  CLP_CUDA(h, h->panel.ensure((size_t)2 * pc * m * sizeof(double)));
  double* Mp = h->panel.as<double>();
  double* Cp = Mp + (size_t)pc * m;
  for (long long j0 = 0; j0 < m; j0 += pc) {
    const long long j1 = std::min<long long>(m, j0 + pc);
    CLP_CUDA(h, cudaMemcpyAsync(Mp, M + (size_t)j0 * m, (size_t)(j1 - j0) * m * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    CLP_CUDA(h, cudaMemcpyAsync(Cp, C + (size_t)j0 * m, (size_t)(j1 - j0) * m * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    dim3 grid((unsigned)((m + 255) / 256), (unsigned)(j1 - j0));
    with_storage(h, [&](auto t) {
      using T = decltype(t);
      encode_dense_panel_kernel<T><<<grid, 256, 0, h->stream>>>(Mp, Cp, (int)m, (int)j0, (int)j1, h->Mbuf.as<T>(), h->ld, h->row0, h->rows, &sb->flags);
    });
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));  // the panel buffer is reused
  }
  return end_load(h, {{1, CLP_ERR_UNSUPPORTED, "affinity matrix has negative entries (contract: M in [0,1], ref clipper.h:166-171)"},
                      {2, CLP_ERR_UNSUPPORTED, "constraint matrix is not binary (contract: ref clipper.h:176)"}});
}

int clp_set_dense_dev(clp_handle h, const void* M, const void* C, int64_t m, int dtype, int64_t row_stride, int64_t col_stride) {
  if (!h || !M || !C) return CLP_ERR_INVALID;
  if (dtype != CLP_IN_F32 && dtype != CLP_IN_F64) return fail(h, CLP_ERR_INVALID, "unknown input dtype (CLP_IN_F32 or CLP_IN_F64)");
  if (!dense_strides_ok(row_stride, col_stride)) return fail(h, CLP_ERR_INVALID, "one of row_stride, col_stride must be 1 and the other >= 1");
  if (h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "clp_set_dense_dev on a sharded handle (a rank would need the whole matrix)");
  return guarded(h, [&] {
    if (int rc = begin_load(h, m)) return rc;
    SyncBlock* sb = h->sync.as<SyncBlock>();
    const unsigned nt = (unsigned)((m + 31) / 32);
    with_storage(h, [&](auto t) {
      using T = decltype(t);
      if (dtype == CLP_IN_F32)
        load_dense_dev_kernel<T, float><<<dim3(nt, nt), 256, 0, h->stream>>>(static_cast<const float*>(M), static_cast<const float*>(C), (int)m,
                                                                          row_stride, col_stride, h->Mbuf.as<T>(), h->ld, &sb->flags);
      else
        load_dense_dev_kernel<T, double><<<dim3(nt, nt), 256, 0, h->stream>>>(static_cast<const double*>(M), static_cast<const double*>(C), (int)m,
                                                                           row_stride, col_stride, h->Mbuf.as<T>(), h->ld, &sb->flags);
    });
    CLP_CUDA(h, cudaGetLastError());
    return end_load(h, {{1, CLP_ERR_UNSUPPORTED, "affinity matrix has negative entries (contract: M in [0,1], ref clipper.h:166-171)"},
                        {2, CLP_ERR_UNSUPPORTED, "constraint matrix is not binary (contract: ref clipper.h:176)"}});
  });
}

int clp_set_sparse_upper(clp_handle h, int64_t m, const int64_t* cpM, const int32_t* riM, const double* vM,
                         const int64_t* cpC, const int32_t* riC, const double* vC) {
  if (!h || !cpM || !cpC) return CLP_ERR_INVALID;
  if (int rc = begin_load(h, m)) return rc;
  SyncBlock* sb = h->sync.as<SyncBlock>();
  for (int which = 0; which < 2; ++which) {
    const int64_t* cp = which ? cpC : cpM; const int32_t* ri = which ? riC : riM; const double* vv = which ? vC : vM;
    const long long nnz = cp[m];
    if (nnz < 0) return fail(h, CLP_ERR_INVALID, "bad CSC column pointer");
    const size_t b_cp = (size_t)(m + 1) * sizeof(long long), b_v = (size_t)std::max<long long>(nnz, 1) * sizeof(double);
    const size_t b_ri = (size_t)std::max<long long>(nnz, 1) * sizeof(int32_t);
    CLP_CUDA(h, h->cscbuf.ensure(b_cp + b_v + b_ri + 64));
    char* base = h->cscbuf.as<char>();
    long long* cp_d = reinterpret_cast<long long*>(base);
    double* v_d = reinterpret_cast<double*>(base + b_cp);
    int32_t* ri_d = reinterpret_cast<int32_t*>(base + b_cp + b_v);
    CLP_CUDA(h, cudaMemcpyAsync(cp_d, cp, b_cp, cudaMemcpyHostToDevice, h->stream));
    if (nnz > 0) {
      CLP_CUDA(h, cudaMemcpyAsync(v_d, vv, (size_t)nnz * sizeof(double), cudaMemcpyHostToDevice, h->stream));
      CLP_CUDA(h, cudaMemcpyAsync(ri_d, ri, (size_t)nnz * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    }
    with_storage(h, [&](auto t) {
      using T = decltype(t);
      if (which == 0) scatter_csc_M_kernel<T><<<(unsigned)m, 128, 0, h->stream>>>(cp_d, ri_d, v_d, (int)m, h->Mbuf.as<T>(), h->ld, h->row0, h->rows, &sb->flags);
      else scatter_csc_C_kernel<T><<<(unsigned)m, 128, 0, h->stream>>>(cp_d, ri_d, v_d, (int)m, h->Mbuf.as<T>(), h->ld, h->row0, h->rows, &sb->flags);
    });
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return end_load(h, {{4, CLP_ERR_INVALID, "sparse input is not strictly upper triangular (ref clipper.h:137-138)"},
                      {1, CLP_ERR_UNSUPPORTED, "affinity matrix has negative entries"},
                      {2, CLP_ERR_UNSUPPORTED, "constraint matrix is not binary"}});
}

int clp_get_dense(clp_handle h, int which, double* out) {
  if (!h || !out) return CLP_ERR_INVALID;
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "no affinity matrix has been scored or set");
  if (h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "clp_get_dense on a sharded handle");
  CLP_CUDA(h, cudaSetDevice(h->device));
  const long long m = h->m;
  const long long pc = std::max<long long>(1, std::min<long long>(m, (64ll << 20) / (8 * m)));
  CLP_CUDA(h, h->panel.ensure((size_t)pc * m * sizeof(double)));
  double* P = h->panel.as<double>();
  for (long long j0 = 0; j0 < m; j0 += pc) {
    const long long j1 = std::min<long long>(m, j0 + pc);
    dim3 grid((unsigned)((m + 255) / 256), (unsigned)(j1 - j0));
    with_storage(h, [&](auto t) {
      using T = decltype(t);
      decode_dense_panel_kernel<T><<<grid, 256, 0, h->stream>>>(h->Mbuf.as<T>(), h->ld, (int)m, (int)j0, (int)j1, which, P);
    });
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaMemcpyAsync(out + (size_t)j0 * m, P, (size_t)(j1 - j0) * m * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  return CLP_OK;
}

int clp_num_associations(clp_handle h, int64_t* m) {
  if (!h || !m) return CLP_ERR_INVALID;
  *m = h->has_matrix ? h->m : 0;
  return CLP_OK;
}

int clp_get_associations(clp_handle h, int32_t* A) {
  if (!h || !A) return CLP_ERR_INVALID;
  if (!h->has_A) return fail(h, CLP_ERR_INVALID, "no associations: the matrix was not built by scorePairwiseConsistency");
  if (!h->A_host_valid) {
    try { h->A_host.resize((size_t)2 * h->m); } catch (...) { return fail(h, CLP_ERR_ALLOC, "host allocation failed"); }
    CLP_CUDA(h, cudaSetDevice(h->device));
    CLP_CUDA(h, cudaMemcpyAsync(h->A_host.data(), h->A_dev.p, (size_t)2 * h->m * sizeof(int32_t), cudaMemcpyDeviceToHost, h->stream));
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));
    h->A_host_valid = true;
  }
  std::memcpy(A, h->A_host.data(), (size_t)2 * h->m * sizeof(int32_t));
  return CLP_OK;
}

int clp_count_nonzeros(clp_handle h, int64_t* nnzM, int64_t* nnzC) {
  if (!h) return CLP_ERR_INVALID;
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "no affinity matrix");
  CLP_CUDA(h, cudaSetDevice(h->device));
  if (int rc = reset_sync(h)) return rc;
  SyncBlock* sb = h->sync.as<SyncBlock>();
  with_storage(h, [&](auto t) {
    using T = decltype(t);
    count_upper_kernel<T><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<T>(), h->ld, (int)h->m, h->row0, h->rows, sb->counts);
  });
  CLP_CUDA(h, cudaGetLastError());
  SyncBlock host;
  if (int rc = read_sync(h, &host)) return rc;
  if (nnzM) *nnzM = (int64_t)host.counts[0];
  if (nnzC) *nnzC = (int64_t)host.counts[1];
  return CLP_OK;
}

// ---- solve --------------------------------------------------------------------------------
int clp_solve(clp_handle h, const double* u0, clp_solution* out, double* u_out, int32_t* nodes_out, double* u0_out) {
  if (!h) return CLP_ERR_INVALID;
  const auto t0 = std::chrono::steady_clock::now();
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "solve() before any affinity matrix was scored or set");
  CLP_CUDA(h, cudaSetDevice(h->device));
  double* stage = reinterpret_cast<double*>(h->pinned.as<char>() + 256);
  if (u0) {
    std::memcpy(stage, u0, (size_t)h->m * sizeof(double));
  } else {  // utils::randvec (ref utils.cpp:22-29): U[0,1) seeded from std::random_device
    if (h->world > 1)
      return fail(h, CLP_ERR_INVALID, "sharded solve needs an explicit u0: every rank must start from the same vector");
    std::random_device rd;
    std::mt19937 gen(rd());
    std::uniform_real_distribution<double> dis(0, 1);
    for (long long i = 0; i < h->m; ++i) stage[i] = dis(gen);
  }
  if (u0_out) std::memcpy(u0_out, stage, (size_t)h->m * sizeof(double));
  CLP_CUDA(h, cudaMemcpyAsync(h->u0dev.p, stage, (size_t)h->m * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  return guarded(h, [&] { return solve_core(h, out, u_out, nullptr, nodes_out, t0); });
}

int clp_solve_dev(clp_handle h, const double* u0_dev, clp_solution* out, double* u_out_dev, int32_t* nodes_out) {
  if (!h || !u0_dev) return CLP_ERR_INVALID;
  const auto t0 = std::chrono::steady_clock::now();
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "solve() before any affinity matrix was scored or set");
  CLP_CUDA(h, cudaSetDevice(h->device));
  CLP_CUDA(h, cudaMemcpyAsync(h->u0dev.p, u0_dev, (size_t)h->m * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  return guarded(h, [&] { return solve_core(h, out, nullptr, u_out_dev, nodes_out, t0); });
}

// ---- maximum clique -------------------------------------------------------------------------
int clp_max_clique(clp_handle h, int method, double time_limit_s, int32_t* nodes_out, clp_mc_info* info) {
  if (!h) return CLP_ERR_INVALID;
  return guarded(h, [&] { return mc_solve(h, method, time_limit_s, nodes_out, info); });
}

void clp_sdp_default_params(clp_sdp_params* p) {
  if (!p) return;
  p->max_iters = 2000; p->eps_abs = 1e-3; p->eps_rel = 1e-3; p->time_limit_s = 0.0;
}

int clp_sdp_solve(clp_handle h, const clp_sdp_params* p, clp_sdp_info* info, int32_t* nodes_out, double* X_out,
                  double* lambdas_out, double* evec1_out) {
  if (!h) return CLP_ERR_INVALID;
  return guarded(h, [&] { return sdp_solve(h, p, info, nodes_out, X_out, lambdas_out, evec1_out); });
}

int clp_correspondences(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2, int32_t knn,
                        double radius, int enforce_1to1, int32_t* A_out, int64_t capacity, int64_t* m) {
  return guarded(h, [&] { return correspondences(h, false, D1, d, n1, D2, n2, knn, radius, enforce_1to1, A_out, capacity, m); });
}

int clp_correspondences_dev(clp_handle h, const double* D1_dev, int32_t d, int64_t n1, const double* D2_dev, int64_t n2,
                            int32_t knn, double radius, int enforce_1to1, int32_t* A_dev, int64_t capacity, int64_t* m) {
  return guarded(h, [&] {
    return correspondences(h, true, D1_dev, d, n1, D2_dev, n2, knn, radius, enforce_1to1, A_dev, capacity, m);
  });
}

int clp_core_numbers(clp_handle h, int32_t* core_out) {
  if (!h || !core_out) return CLP_ERR_INVALID;
  return guarded(h, [&] {
    McLayout L;
    McPeeled pk;
    McEvents ev;
    if (int rc = mc_prepare(h, &L, &pk, ev)) return rc;
    std::memcpy(core_out, pk.core.data(), pk.core.size() * sizeof(int32_t));
    return CLP_OK;
  });
}

// ---- mat-vec ------------------------------------------------------------------------------
int clp_matvec(clp_handle h, const double* v, double d, double* y, double* Mv, double* Cv) {
  if (!h || !v) return CLP_ERR_INVALID;
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "no affinity matrix");
  if (h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "clp_matvec on a sharded handle");
  CLP_CUDA(h, cudaSetDevice(h->device));
  double* b = h->ybuf.as<double>();
  const size_t vb = (size_t)h->m * sizeof(double);
  CLP_CUDA(h, cudaMemcpyAsync(b, v, vb, cudaMemcpyHostToDevice, h->stream));
  if (int rc = matvec_enqueue(h, b, d, b + h->mpad, b + 2 * h->mpad, b + 3 * h->mpad)) return rc;
  if (y) CLP_CUDA(h, cudaMemcpyAsync(y, b + h->mpad, vb, cudaMemcpyDeviceToHost, h->stream));
  if (Mv) CLP_CUDA(h, cudaMemcpyAsync(Mv, b + 2 * h->mpad, vb, cudaMemcpyDeviceToHost, h->stream));
  if (Cv) CLP_CUDA(h, cudaMemcpyAsync(Cv, b + 3 * h->mpad, vb, cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  return CLP_OK;
}

int clp_matvec_dev(clp_handle h, const double* v_dev, double d, double* y_dev, double* Mv_dev, double* Cv_dev,
                   int reps, double* ms_per_launch) {
  if (!h || !v_dev || reps < 1) return CLP_ERR_INVALID;
  if (!h->has_matrix) return fail(h, CLP_ERR_INVALID, "no affinity matrix");
  if (h->world > 1) return fail(h, CLP_ERR_UNSUPPORTED, "clp_matvec_dev on a sharded handle");
  CLP_CUDA(h, cudaSetDevice(h->device));
  if ((reinterpret_cast<uintptr_t>(v_dev) & 15u) != 0) {  // the kernels read v with 16-byte loads
    CLP_CUDA(h, cudaMemcpyAsync(h->ybuf.p, v_dev, (size_t)h->m * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    v_dev = h->ybuf.as<double>();
  }
  CLP_CUDA(h, cudaEventRecord(h->ev0, h->stream));
  for (int r = 0; r < reps; ++r)
    if (int rc = matvec_enqueue(h, v_dev, d, y_dev, Mv_dev, Cv_dev)) return rc;
  CLP_CUDA(h, cudaEventRecord(h->ev1, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  float ms = 0.f;
  CLP_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));
  if (ms_per_launch) *ms_per_launch = (double)ms / reps;
  return CLP_OK;
}

// ---- multi-GPU (row-block sharding) --------------------------------------------------------
namespace {
struct ShardBlob {  // opaque to the caller; 256 bytes
  cudaIpcMemHandle_t ll;     // 64 B  (LL-cell block)
  cudaIpcMemHandle_t comm;   // 64 B
  unsigned long long pid;
  void* ll_ptr;              // valid only inside the exporting process (same-process peers)
  void* comm_ptr;
  long long mpad;
  int rank, world, device, pad;
  unsigned long long seq;    // exchange sequence number of the exporting rank
};
static_assert(sizeof(ShardBlob) <= 256, "blob too large");
}  // namespace

int clp_shard_config(clp_handle h, int rank, int world) {
  if (!h || world < 1 || world > kMaxPeers || rank < 0 || rank >= world)
    return fail(h, CLP_ERR_INVALID, "bad shard configuration (1 <= world <= 8)");
  CLP_CUDA(h, cudaSetDevice(h->device));
  // h->seq is NOT reset: LL tags must never repeat on cells that may still hold values of earlier solves (after a
  // timed-out solve the ranks' sequence numbers can differ; clp_shard_import re-synchronises them to the maximum)
  h->rank = rank; h->world = world; h->has_matrix = false; h->shard_ready = false;
  CLP_CUDA(h, h->comm.ensure(sizeof(CommBlock)));
  CLP_CUDA(h, cudaMemset(h->comm.p, 0, sizeof(CommBlock)));
  if (h->llbuf.p) CLP_CUDA(h, cudaMemset(h->llbuf.p, 0, h->llbuf.cap));  // tag 0 == "never written"
  return CLP_OK;
}

void clp_shard_rows(int64_t m, int rank, int world, int64_t* row0, int64_t* rows) {
  int r0 = 0, n = 0;
  shard_rows(m, rank, world, &r0, &n);
  if (row0) *row0 = r0;
  if (rows) *rows = n;
}

int64_t clp_shard_blob_bytes(void) { return 256; }

int clp_shard_export(clp_handle h, void* blob, int64_t blob_bytes, int64_t* written) {
  if (!h || !blob || blob_bytes < 256) return CLP_ERR_INVALID;
  if (h->world < 2) return fail(h, CLP_ERR_INVALID, "clp_shard_export on an unsharded handle");
  if (!h->llbuf.p) return fail(h, CLP_ERR_INVALID, "clp_shard_export before the first scoring / set call");
  CLP_CUDA(h, cudaSetDevice(h->device));
  ShardBlob b;
  std::memset(&b, 0, sizeof(b));
  CLP_CUDA(h, cudaIpcGetMemHandle(&b.ll, h->llbuf.p));
  CLP_CUDA(h, cudaIpcGetMemHandle(&b.comm, h->comm.p));
  b.pid = (unsigned long long)getpid();
  b.ll_ptr = h->llbuf.p; b.comm_ptr = h->comm.p; b.mpad = h->mpad;
  b.rank = h->rank; b.world = h->world; b.device = h->device; b.seq = h->seq;
  std::memset(blob, 0, 256);
  std::memcpy(blob, &b, sizeof(b));
  if (written) *written = 256;
  h->exported_ll = h->llbuf.p;
  return CLP_OK;
}

int clp_shard_import(clp_handle h, const void* blobs, int64_t blob_bytes_each, int world) {
  if (!h || !blobs || blob_bytes_each < 256) return CLP_ERR_INVALID;
  if (world != h->world) return fail(h, CLP_ERR_INVALID, "clp_shard_import: world size mismatch");
  CLP_CUDA(h, cudaSetDevice(h->device));
  for (int r = 0; r < kMaxPeers; ++r)
    if (h->peer_opened[r]) {
      cudaIpcCloseMemHandle(h->peer_open_ptr[r][0]); cudaIpcCloseMemHandle(h->peer_open_ptr[r][1]);
      h->peer_opened[r] = false;
    }
  unsigned long long seq_max = h->seq;
  for (int r = 0; r < world; ++r) {
    ShardBlob b;
    std::memcpy(&b, reinterpret_cast<const char*>(blobs) + (size_t)r * blob_bytes_each, sizeof(b));
    seq_max = std::max(seq_max, b.seq);
    if (b.rank != r || b.world != world) return fail(h, CLP_ERR_COMM, "clp_shard_import: blobs are not in rank order");
    if (b.mpad != h->mpad) return fail(h, CLP_ERR_COMM, "clp_shard_import: ranks disagree on the problem size");
    if (r == h->rank) {
      h->peer_ll[r] = h->llbuf.as<uint4>(); h->peer_comm[r] = h->comm.as<CommBlock>();
      continue;
    }
    if (b.pid == (unsigned long long)getpid()) {  // peer handle lives in this process: plain P2P
      if (b.device != h->device) {
        int can = 0;
        CLP_CUDA(h, cudaDeviceCanAccessPeer(&can, h->device, b.device));
        if (!can) return fail(h, CLP_ERR_COMM, "no P2P access between the shards' devices");
        cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CLP_CUDA(h, e);
        cudaGetLastError();
      }
      h->peer_ll[r] = reinterpret_cast<uint4*>(b.ll_ptr);
      h->peer_comm[r] = reinterpret_cast<CommBlock*>(b.comm_ptr);
    } else {
      void *pv = nullptr, *pc = nullptr;
      CLP_CUDA(h, cudaIpcOpenMemHandle(&pv, b.ll, cudaIpcMemLazyEnablePeerAccess));
      CLP_CUDA(h, cudaIpcOpenMemHandle(&pc, b.comm, cudaIpcMemLazyEnablePeerAccess));
      h->peer_ll[r] = reinterpret_cast<uint4*>(pv);
      h->peer_comm[r] = reinterpret_cast<CommBlock*>(pc);
      h->peer_opened[r] = true; h->peer_open_ptr[r][0] = pv; h->peer_open_ptr[r][1] = pc;
    }
  }
  // all ranks continue from the same sequence number, beyond every tag any of them has used (a timed-out solve
  // leaves them different); skipping ahead keeps stale cells from ever validating
  h->seq = seq_max + 16;
  h->shard_ready = true;
  return CLP_OK;
}

int clp_set_grid_cap(clp_handle h, int n_ctas) {
  if (!h || n_ctas < 0) return fail(h, CLP_ERR_INVALID, "grid cap must be >= 0 (0 = whole GPU)");
  h->grid_cap = n_ctas;
  return apply_grid_knobs(h);
}

int clp_set_ctas_per_sm(clp_handle h, int n) {
  if (!h || n < 1 || n > 3) return fail(h, CLP_ERR_INVALID, "ctas_per_sm must be 1, 2 or 3");
  h->ctas_cap = n;
  return apply_grid_knobs(h);
}

int clp_sparse_info(clp_handle h, int64_t* nnz_kept, int64_t* bytes_per_pass) {
  if (!h) return CLP_ERR_INVALID;
  if (nnz_kept) *nnz_kept = (int64_t)h->sp_nnz_real;
  if (bytes_per_pass)
    *bytes_per_pass = (int64_t)(h->sp_nnz * h->entry_bytes() +
                                (unsigned long long)(h->rows_pad / 4) * (h->sp_shape.resident ? 1 : h->plan.NSEG) * 20);
  return CLP_OK;
}

int clp_last_solve_sweeps(clp_handle h, int64_t* counts) {
  if (!h || !counts) return CLP_ERR_INVALID;
  const ResSweeps& r = h->last_sweeps;
  counts[0] = r.full; counts[1] = r.rebuild; counts[2] = r.restricted;
  counts[3] = (int64_t)r.entries; counts[4] = (int64_t)r.padding; counts[5] = r.fallback;
  return CLP_OK;
}

int clp_get_dense_mode(clp_handle h, int* requested, int* effective) {
  if (!h) return CLP_ERR_INVALID;
  if (requested) *requested = h->dense_mode;
  if (effective) *effective = h->dense_mode_eff;
  return CLP_OK;
}

int clp_set_dense_mode(clp_handle h, int mode) {
  if (!h || mode < 0 || mode > 6 || mode == 1 || mode == 5) return fail(h, CLP_ERR_INVALID, "sweep mode must be 0, 2, 3, 4 or 6");
  h->dense_mode = mode;
  if (h->has_matrix) {
    CLP_CUDA(h, cudaSetDevice(h->device));
    if (int rc = finalize_matrix(h)) return rc;
  }
  return CLP_OK;
}

}  // extern "C"

// ==========================================================================================
// batches of small problems (clp_batch.cuh)
// ==========================================================================================
struct clp_batch_s {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_up = nullptr;
  clp_params prm;
  std::string err;
  int sm_count = 0, smem_optin = 0;
  DevBuf in_d1, in_d2, in_a, in_u0, out_u, probs, outs, nnz, sync, scratch, prof;
  DevBuf mat_in;  // batched matrices: column pointers | values | u0 | row indices | problem table
  DevBuf custom_in;  // batches scored with a caller's invariant: parameters | work units | problem table
  // batched maximum clique: problem table, edges, per-problem regions, per-problem search state, task rounds, scratch
  DevBuf mc_probs, mc_edges, mc_adj, mc_vint, mc_tpre, mc_out, mc_state, mc_rounds, mc_pscratch, mc_sscratch;
  DevBuf sdp_out;  // batched relaxation: X offsets | SdpOut | p | evec1 | X
  // putative associations (clp_knn.cuh): problem table | staged clouds | lists | scan | counts | 1-to-1 | staged A
  DevBuf knn_buf;
  PinnedBuf knn_pinned;     // the table and host clouds going up, the counts and host A coming back
  DevBuf tf_buf;            // rigid transform (clp_transform.cuh), as clp_handle_s::tf_buf
  PinnedBuf tf_pinned;
  int prof_on = env_int("CLP_PROF_BATCH", 0);
  PinnedBuf pinned;         // the caller's other inputs, then the results
  PinnedBuf pinned_points;  // D1 | D2 | A of scored problems (stage_points)
  int last_ctas = 0; long long last_scratch = 0, last_nnz = 0;
};

namespace {

template <int KIND, int DD>
int batch_launch(clp_batch b, BatchArgs& ba, int grid, size_t smem) {
  CLP_CUDA(b, cudaFuncSetAttribute(batch_solve_kernel<KIND, DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  batch_solve_kernel<KIND, DD><<<grid, kBatchThreads, smem, b->stream>>>(ba);
  CLP_CUDA(b, cudaGetLastError());
  return CLP_OK;
}
template <int KIND, int DD>
int batch_occupancy(clp_batch b, size_t smem, int* occ) {
  CLP_CUDA(b, cudaFuncSetAttribute(batch_solve_kernel<KIND, DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CLP_CUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, batch_solve_kernel<KIND, DD>, kBatchThreads, smem));
  return CLP_OK;
}

// per-problem results of a batched solve: rounding (NONZERO or DSD_HEU) and the outputs of clp_batch_solve_*.
// Prob: BatchProblem or BatchMatProblem (m, u_off).  sols[p].t is left to the caller.
template <typename Prob>
void batch_results(const clp_params& P, const std::vector<Prob>& probs, const double* h_u, const SolverOut* h_out, float ms,
                   clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  std::vector<int32_t> nodes;
  for (int p = 0; p < (int)probs.size(); ++p) {
    const Prob& q = probs[(size_t)p];
    const SolverOut& so = h_out[p];
    const double* u = h_u + q.u_off;
    nodes.clear();
    if (P.rounding == CLP_ROUND_NONZERO) {
      nodes.resize((size_t)q.m);
      nodes.resize((size_t)clp_find_above(u, q.m, 0.0, nodes.data()));
    } else {  // DSD_HEU, ref clipper.cpp:302-308
      const int32_t omega = heu_omega(so.F, q.m);
      if (omega >= 1) {
        nodes.resize((size_t)omega);
        nodes.resize((size_t)clp_find_k_largest(u, q.m, omega, nodes.data()));
      }
    }
    clp_solution& s = sols[p];
    std::memset(&s, 0, sizeof(s));
    s.ifinal = so.ifinal; s.n_nodes = (int32_t)nodes.size(); s.score = so.F; s.d_final = so.d;
    s.n_evals = so.n_evals; s.n_matvec = so.n_matvec; s.n_inner = so.n_inner; s.kernel_ms = ms;
    s.prof_matvec_ms = 1e-6 * (double)so.ns_matvec; s.prof_combine_ms = 1e-6 * (double)so.ns_combine;
    s.prof_exchange_ms = 1e-6 * (double)so.ns_exchange;
    if (u_out && u_out[p]) std::memcpy(u_out[p], u, (size_t)q.m * 8);
    if (nodes_out && nodes_out[p] && !nodes.empty()) std::memcpy(nodes_out[p], nodes.data(), nodes.size() * 4);
  }
}

// Inputs of the batch C-ABI calls.  Scored problems: D1, n1, D2, n2, A, m and the invariant's parameters p, or for
// clp_batch_*_custom the caller's invariant inv; graphs given as strictly-upper CSC patterns: m, colptr and rowidx.
// clp_batch_*_dev: the points and associations are in dev (n1, n2 and m are its host arrays), and the solves take u0
// from u0_dev and write u to u_out_dev (nullable).
struct BatchInput {
  const double* const* D1 = nullptr; const int64_t* n1 = nullptr;
  const double* const* D2 = nullptr; const int64_t* n2 = nullptr;
  const int32_t* const* A = nullptr; const int64_t* m = nullptr;
  const int64_t* const* colptr = nullptr; const int32_t* const* rowidx = nullptr;
  double p[4] = {0.0, 0.0, 0.0, 0.0};
  const CustomInvariant* inv = nullptr;
  const clp_points_dev* dev = nullptr;
  const double* u0_dev = nullptr; int64_t u0_stride = 0;
  double* u_out_dev = nullptr; int64_t u_out_stride = 0;
};

// problem p of a scored batch takes the all-to-all hypothesis: no associations are given for it
bool all_to_all(const BatchInput& in, int p) {
  return (in.dev ? in.dev->A == nullptr : (in.A == nullptr || in.A[p] == nullptr)) || in.m[p] == 0;
}

// the checks of problem p of a scored batch (CLP_ERR_INVALID): its data and its association count *mp (n1 n2 for the
// all-to-all hypothesis)
int point_problem_check(clp_batch b, const BatchInput& in, int p, long long* mp) {
  if ((!in.dev && (!in.D1[p] || !in.D2[p])) || in.n1[p] <= 0 || in.n2[p] <= 0)
    return fail(b, CLP_ERR_INVALID, "bad problem in the batch (null data)");
  *mp = all_to_all(in, p) ? (long long)in.n1[p] * in.n2[p] : (long long)in.m[p];
  if (*mp <= 0 || *mp > kBatchMaxM) return fail(b, CLP_ERR_INVALID, "batched problems need 1 <= m <= 4096 associations");
  return CLP_OK;
}

// the `kind` of batch_solve and batch_max_clique for problems scored with a caller's invariant (clp_batch_*_custom):
// the clique's prepare kernel reads the stored matrix (0, 1: the built-ins, kMcbKindGraph: graphs)
constexpr int kBatchKindCustom = kMcbKindStored;

// ---- batches scored with a caller's invariant ---------------------------------------------------------------------
// The scoring is compiled at run time (batch_score_custom_kernel, clp_jit.cpp); the build, the solve and the clique
// steps are the nvcc-built kernels.  The problems go in rounds over the scratch slots batch_grid sized: round r gathers
// and scores problems [rG, rG + G) into slots 0 .. G - 1 with the whole grid, then the stored-matrix kernel runs one CTA
// per problem of the round.  Every round is enqueued on the batch's stream; the results are read once at the end.

// the checks of a custom batch that come before everything else (CLP_ERR_INVALID): the source, the parameter count,
// the dimension and every problem's m (plan_points repeats the last)
int custom_check(clp_batch b, const CustomInvariant& inv, int32_t nprob, int dd, const BatchInput& in) {
  if (!inv.source || !*inv.source) return fail(b, CLP_ERR_INVALID, "empty invariant source");
  if (inv.nprm < 0 || inv.nprm > CLP_INV_MAX_PARAMS || (inv.nprm > 0 && !inv.prm))
    return fail(b, CLP_ERR_INVALID, "invariant parameters: 0 to " + std::to_string(CLP_INV_MAX_PARAMS) + " doubles");
  if (dd < 1) return fail(b, CLP_ERR_INVALID, "dimension must be positive");
  for (int p = 0; p < nprob; ++p) {
    long long mp = 0;
    if (int rc = point_problem_check(b, in, p, &mp)) return rc;
  }
  return CLP_OK;
}

// the compiled scoring of a custom batch and what its rounds read
struct CustomRounds {
  const void* fn = nullptr;      // batch_score_custom_kernel<D> for the caller's source
  BatchScoreArgs sa{};
  std::vector<long long> units;  // host copy of sa.units
  int max_m = 1;
};

// compiles (or finds in the cache) the scoring kernel for inv and dimension d: CLP_ERR_INVALID with the compiler's log
int custom_compile(clp_batch b, const CustomInvariant& inv, int d, CustomRounds* cr) {
  std::string err;
  if (int rc = jit_score_kernel(JitKernel::kBatchScore, inv.source, d, false, true, b->device, &cr->fn, &err))
    return fail(b, rc, err);
  return CLP_OK;
}

// uploads the parameters, the running count of work units and the problem table, and sets the arguments every round
// shares: slots of `stride` bytes at `scratch`, their regions at the offsets of batch_layout / mcb_layout
int custom_stage(clp_batch b, const CustomInvariant& inv, int d, const std::vector<BatchProblem>& probs, unsigned char* scratch,
                 size_t stride, size_t e1, size_t e2, size_t a, size_t mat, CustomRounds* cr) {
  const size_t nprob = probs.size();
  cr->units.assign(nprob + 1, 0);
  for (size_t p = 0; p < nprob; ++p) {
    cr->units[p + 1] = cr->units[p] + batch_tile_units(probs[p].m);
    cr->max_m = std::max(cr->max_m, probs[p].m);
  }
  const size_t units_at = CLP_INV_MAX_PARAMS * 8, table_at = batch_align(units_at + (nprob + 1) * 8);
  std::vector<unsigned char> h(table_at + nprob * sizeof(BatchProblem));
  if (inv.nprm > 0) std::memcpy(h.data(), inv.prm, (size_t)inv.nprm * 8);
  std::memcpy(h.data() + units_at, cr->units.data(), (nprob + 1) * 8);
  std::memcpy(h.data() + table_at, probs.data(), nprob * sizeof(BatchProblem));
  CLP_CUDA(b, b->custom_in.ensure(h.size()));
  CLP_CUDA(b, cudaMemcpyAsync(b->custom_in.p, h.data(), h.size(), cudaMemcpyHostToDevice, b->stream));
  BatchScoreArgs& sa = cr->sa;
  unsigned char* base = b->custom_in.as<unsigned char>();
  sa.prob = reinterpret_cast<const BatchProblem*>(base + table_at);
  sa.units = reinterpret_cast<const long long*>(base + units_at);
  sa.D1 = b->in_d1.as<double>(); sa.D2 = b->in_d2.as<double>(); sa.A = b->in_a.as<int>();
  sa.scratch = scratch; sa.stride = stride;
  sa.e1 = e1; sa.e2 = e2; sa.a = a; sa.mat = mat;
  sa.d = d; sa.affinityeps = b->prm.affinityeps;
  sa.prm = reinterpret_cast<const double*>(base);
  sa.error = &b->sync.as<SyncBlock>()->error;
  return CLP_OK;
}

// enqueues the gather and the scoring of problems [first, first + count) into slots 0 .. count - 1
int custom_score_round(clp_batch b, CustomRounds& cr, int first, int count) {
  cr.sa.first = first; cr.sa.count = count;
  batch_gather_kernel<<<dim3((unsigned)((cr.max_m + kBatchThreads - 1) / kBatchThreads), (unsigned)count), kBatchThreads, 0,
                        b->stream>>>(cr.sa);
  CLP_CUDA(b, cudaGetLastError());
  const long long units = cr.units[(size_t)(first + count)] - cr.units[(size_t)first];
  void* args[] = {&cr.sa};
  CLP_CUDA(b, cudaLaunchKernel(cr.fn, dim3((unsigned)units), dim3(kThreads), args, 0, b->stream));
  return CLP_OK;
}

// The concatenated point inputs of a scored batch (in_d1, in_d2, in_a), decided once for both fills: one BatchProblem
// per problem with the offsets of its D1, D2 and A (a_off -1 and m = n1 n2 for the all-to-all hypothesis; u_off 0),
// and the element counts of the three arrays.
struct PointsPlan {
  std::vector<BatchProblem> probs;
  long long nd1 = 0, nd2 = 0, na = 0;
};

// checks every problem, host association indices included (device ones are checked by batch_stage_points_kernel),
// fills the plan and sizes in_d1, in_d2 and in_a
int plan_points(clp_batch b, int dd, int32_t nprob, const BatchInput& in, PointsPlan* pl) {
  pl->probs.assign((size_t)nprob, BatchProblem{});
  long long nd1 = 0, nd2 = 0, na = 0;
  for (int p = 0; p < nprob; ++p) {
    BatchProblem& q = pl->probs[(size_t)p];
    long long mp = 0;
    if (int rc = point_problem_check(b, in, p, &mp)) return rc;
    const bool a2a = all_to_all(in, p);
    if (!a2a && !in.dev)
      for (long long i = 0; i < mp; ++i) {
        const int32_t a0 = in.A[p][i], a1 = in.A[p][mp + i];
        if (a0 < 0 || a0 >= in.n1[p] || a1 < 0 || a1 >= in.n2[p])
          return fail(b, CLP_ERR_INVALID, "association index out of range of D1/D2 in a batched problem");
      }
    q.d1_off = nd1; q.d2_off = nd2; q.a_off = a2a ? -1 : na;
    q.n1 = (int)in.n1[p]; q.n2 = (int)in.n2[p]; q.m = (int)mp;
    nd1 += (long long)dd * in.n1[p]; nd2 += (long long)dd * in.n2[p]; if (!a2a) na += 2 * mp;
  }
  pl->nd1 = nd1; pl->nd2 = nd2; pl->na = na;
  CLP_CUDA(b, b->in_d1.ensure((size_t)nd1 * 8 + 16));
  CLP_CUDA(b, b->in_d2.ensure((size_t)nd2 * 8 + 16));
  CLP_CUDA(b, b->in_a.ensure((size_t)na * 4 + 16));
  return CLP_OK;
}

// Fills the planned arrays, enqueued on the batch's stream: host inputs through pinned_points and three uploads;
// device inputs (in.dev) with batch_stage_points_kernel, which reads the problem table at `table` (device, one entry
// every table_stride bytes, u_off set) and also stages u0 into in_u0 when in.u0_dev is given.  *bytes: the bytes
// uploaded.
int fill_points(clp_batch b, int dd, const BatchInput& in, const PointsPlan& pl, const void* table, size_t table_stride,
                size_t* bytes) {
  const int nprob = (int)pl.probs.size();
  if (in.dev) {
    const clp_points_dev& s = *in.dev;
    BatchStageArgs g;
    std::memset(&g, 0, sizeof(g));
    g.prob = static_cast<const unsigned char*>(table); g.prob_stride = table_stride;
    g.nprob = nprob; g.dd = dd;
    g.D1 = s.D1; g.D2 = s.D2; g.A = s.A;
    for (int k = 0; k < 3; ++k) { g.s1[k] = s.d1_strides[k]; g.s2[k] = s.d2_strides[k]; g.sa[k] = s.a_strides[k]; }
    g.u0_in = in.u0_dev; g.u0_stride = in.u0_stride;
    g.d1 = b->in_d1.as<double>(); g.d2 = b->in_d2.as<double>(); g.a = b->in_a.as<int>(); g.u0 = b->in_u0.as<double>();
    g.bad = &b->sync.as<SyncBlock>()->counts[1];
    long long most = 1;
    for (const BatchProblem& q : pl.probs) most = std::max({most, (long long)dd * std::max(q.n1, q.n2), 2LL * q.m});
    const dim3 grid((unsigned)std::min<long long>(64, (most + kBatchThreads - 1) / kBatchThreads), (unsigned)std::min(nprob, 65535));
    batch_stage_points_kernel<<<grid, kBatchThreads, 0, b->stream>>>(g);
    CLP_CUDA(b, cudaGetLastError());
    *bytes = 0;
    return CLP_OK;
  }
  const long long nd1 = pl.nd1, nd2 = pl.nd2, na = pl.na;
  *bytes = (size_t)(nd1 + nd2) * 8 + (size_t)na * 4;
  CLP_CUDA(b, b->pinned_points.ensure(*bytes + 16));
  double* h_d1 = b->pinned_points.as<double>();
  double* h_d2 = h_d1 + nd1;
  int32_t* h_a = reinterpret_cast<int32_t*>(h_d2 + nd2);
  for (int p = 0; p < nprob; ++p) {
    const BatchProblem& q = pl.probs[(size_t)p];
    std::memcpy(h_d1 + q.d1_off, in.D1[p], (size_t)dd * q.n1 * 8);
    std::memcpy(h_d2 + q.d2_off, in.D2[p], (size_t)dd * q.n2 * 8);
    if (q.a_off >= 0) std::memcpy(h_a + q.a_off, in.A[p], (size_t)2 * q.m * 4);
  }
  CLP_CUDA(b, cudaMemcpyAsync(b->in_d1.p, h_d1, (size_t)nd1 * 8, cudaMemcpyHostToDevice, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(b->in_d2.p, h_d2, (size_t)nd2 * 8, cudaMemcpyHostToDevice, b->stream));
  if (na) CLP_CUDA(b, cudaMemcpyAsync(b->in_a.p, h_a, (size_t)na * 4, cudaMemcpyHostToDevice, b->stream));
  return CLP_OK;
}

// the error of a problem a device check found bad: SyncBlock::counts[1] holds (kind << 32 | ~p) of the lowest such
// problem p (0: none).  Kinds 1 and 2: a C or M value (batch_dense_solve_kernel); kBatchBadIndex: an association index
// (batch_stage_points_kernel).
int bad_problem(clp_batch b, unsigned long long key) {
  if (key == 0) return CLP_OK;
  const unsigned long long kind = key >> 32;
  const std::string p = "problem " + std::to_string(0xffffffffu - (unsigned int)(key & 0xffffffffu));
  if (kind == kBatchBadIndex) return fail(b, CLP_ERR_INVALID, p + ": association index out of range of D1/D2");
  return fail(b, CLP_ERR_UNSUPPORTED, p + (kind == 2 ? ", M: affinity matrix has negative entries" : ", C: constraint matrix is not binary"));
}

// CTAs of a persistent batch launch, each with a scratch slot of `stride` bytes in `scratch` (stride 0: none): as many
// as are co-resident at occ per SM, no more than there are problems, and no more than 80 % of the free device memory
// holds slots for (the slots `scratch` holds count as free).  Ensures the scratch.  When not one slot fits, no_room is
// the CLP_ERR_ALLOC message, or without one, one CTA is tried.
int batch_grid(clp_batch b, int occ, int32_t nprob, size_t stride, DevBuf& scratch, const char* no_room, int* grid) {
  long long g = std::min<long long>(nprob, (long long)occ * b->sm_count);
  if (stride > 0) {
    size_t free_b = 0, total_b = 0;
    CLP_CUDA(b, cudaMemGetInfo(&free_b, &total_b));
    const long long by_mem = (long long)((double)(free_b + scratch.cap) * 0.8 / (double)stride);
    if (by_mem < 1 && no_room) return fail(b, CLP_ERR_ALLOC, no_room);
    g = std::max<long long>(1, std::min(g, by_mem));
    CLP_CUDA(b, scratch.ensure((size_t)g * stride));
  }
  *grid = (int)g;
  return CLP_OK;
}

// Tail of the batched solves, from the launch on: reads u (nu doubles), the SolverOut and the kept-entry count of every
// problem and the sync block into the staging buffer with one synchronisation, prints the CLP_PROF_BATCH line, maps the
// device's error words (batch_matrix_solve_kernel sets flags, batch_solve_kernel error 2, both time out with error 1),
// and fills the results.  `label` names the call and `first` its first in-kernel phase in the profile line.
// batch_dense_solve_kernel and batch_stage_points_kernel leave their first bad problem in counts[1] (bad_problem); it is
// reported first.
template <typename Prob>
int batch_finish(clp_batch b, const char* label, const char* first, const std::vector<Prob>& probs, long long nu, int max_m,
                 int grid, size_t stride, size_t bytes_in, std::chrono::steady_clock::time_point t_begin, clp_solution* sols,
                 double* const* u_out, int32_t* const* nodes_out) {
  const int nprob = (int)probs.size();
  CLP_CUDA(b, cudaEventRecord(b->ev1, b->stream));
  double* h_u = b->pinned.as<double>();
  SolverOut* h_out = reinterpret_cast<SolverOut*>(h_u + nu);
  unsigned int* h_nnz = reinterpret_cast<unsigned int*>(h_out + nprob);
  SyncBlock h_sb;
  CLP_CUDA(b, cudaMemcpyAsync(h_u, b->out_u.p, (size_t)nu * 8, cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(h_out, b->outs.p, (size_t)nprob * sizeof(SolverOut), cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(h_nnz, b->nnz.p, (size_t)nprob * 4, cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(&h_sb, b->sync.p, sizeof(SyncBlock), cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaStreamSynchronize(b->stream));
  float ms = 0.f, up_ms = 0.f;
  CLP_CUDA(b, cudaEventElapsedTime(&ms, b->ev0, b->ev1));
  CLP_CUDA(b, cudaEventElapsedTime(&up_ms, b->ev_up, b->ev0));
  if (b->prof_on) {
    std::vector<unsigned long long> pr((size_t)nprob * 4);
    CLP_CUDA(b, cudaMemcpy(pr.data(), b->prof.p, pr.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    double acc[4] = {0, 0, 0, 0};
    for (int p = 0; p < nprob; ++p) for (int q = 0; q < 4; ++q) acc[q] += 1e-6 * (double)pr[(size_t)p * 4 + q];
    std::fprintf(stderr, "[clp %s prof] %d problems (max m %d), %d CTAs, upload %zu bytes %.3f ms, kernel %.3f ms; "
                 "mean per problem: %s %.3f  build %.3f  solve %.3f  total %.3f ms\n",
                 label, nprob, max_m, grid, bytes_in, up_ms, ms, first, acc[0] / nprob, acc[1] / nprob, acc[2] / nprob, acc[3] / nprob);
  }
  if (int rc = bad_problem(b, h_sb.counts[1])) return rc;
  if (h_sb.flags != 0) return fail(b, CLP_ERR_CUDA, "batched matrices: the device found an entry the host check passed");
  if (h_sb.error == 2) return fail(b, CLP_ERR_INVALID, "association index out of range of D1/D2 in a batched problem");
  if (h_sb.error != 0) return fail(b, CLP_ERR_TIMEOUT, "batch kernel: an in-kernel wait timed out");
  b->last_ctas = grid; b->last_scratch = (long long)grid * (long long)stride; b->last_nnz = 0;
  for (int p = 0; p < nprob; ++p) b->last_nnz += h_nnz[p] / 2;
  batch_results(b->prm, probs, h_u, h_out, ms, sols, u_out, nodes_out);
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  for (int p = 0; p < nprob; ++p) sols[p].t = wall / nprob;
  return CLP_OK;
}

int batch_solve(clp_batch b, int kind, int dd, int32_t nprob, const BatchInput& in, const double* const* u0, clp_solution* sols,
                double* const* u_out, int32_t* const* nodes_out) {
  if (!b) return CLP_ERR_INVALID;
  if (nprob <= 0 || (!in.dev && (!in.D1 || !in.D2 || !u0)) || !in.n1 || !in.n2 || !in.m || (in.dev && !in.u0_dev) || !sols)
    return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  const bool custom = kind == kBatchKindCustom;
  if (custom) {
    for (int p = 0; p < nprob && !in.dev; ++p)
      if (!u0[p]) return fail(b, CLP_ERR_INVALID, "bad problem in the batch (null u0)");
    if (int rc = custom_check(b, *in.inv, nprob, dd, in)) return rc;
  } else if (!((kind == 0 && (dd == 2 || dd == 3)) || (kind == 1 && dd == 6))) {
    return fail(b, CLP_ERR_UNSUPPORTED, "batched scoring supports EuclideanDistance with d = 2, 3 and PointNormalDistance");
  }
  const clp_params& P = b->prm;
  if (P.rounding == CLP_ROUND_DSD) return fail(b, CLP_ERR_UNSUPPORTED, "Rounding::DSD is not available in a batch");
  if (P.maxlsiters < 1) return fail(b, CLP_ERR_INVALID, "maxlsiters must be >= 1");
  const auto t_begin = std::chrono::steady_clock::now();
  CLP_CUDA(b, cudaSetDevice(b->device));
  CustomRounds cr;
  if (custom)
    if (int rc = custom_compile(b, *in.inv, dd, &cr)) return rc;
  // ---- problem table and concatenated inputs
  for (int p = 0; p < nprob && !in.dev; ++p)
    if (!u0[p]) return fail(b, CLP_ERR_INVALID, "bad problem in the batch (null u0)");
  CLP_CUDA(b, cudaEventRecord(b->ev_up, b->stream));
  PointsPlan pl;
  if (int rc = plan_points(b, dd, nprob, in, &pl)) return rc;
  std::vector<BatchProblem>& probs = pl.probs;
  long long nu = 0;
  int max_m = 1;
  for (BatchProblem& q : probs) {
    q.u_off = nu;
    nu += (q.m + 1) & ~1LL;  // every problem's u0 / u slot starts on a 16-byte boundary (the kernels use 16-byte loads)
    max_m = std::max(max_m, q.m);
  }
  // host u0 goes up with the table; device u0 is staged with the points
  const long long nu0 = in.dev ? 0 : nu;
  const size_t bytes_table = (size_t)nu0 * 8 + (size_t)nprob * sizeof(BatchProblem);
  const size_t bytes_out = (size_t)nu * 8 + (size_t)nprob * (sizeof(SolverOut) + 4);
  CLP_CUDA(b, b->pinned.ensure(std::max(bytes_table, bytes_out) + 4096));
  double* h_u0 = b->pinned.as<double>();
  BatchProblem* h_pr = reinterpret_cast<BatchProblem*>(h_u0 + nu0);
  for (int p = 0; p < nprob && !in.dev; ++p) std::memcpy(h_u0 + probs[(size_t)p].u_off, u0[p], (size_t)probs[(size_t)p].m * 8);
  std::memcpy(h_pr, probs.data(), (size_t)nprob * sizeof(BatchProblem));
  CLP_CUDA(b, b->in_u0.ensure((size_t)nu * 8 + 16));
  CLP_CUDA(b, b->out_u.ensure((size_t)nu * 8 + 16));
  CLP_CUDA(b, b->probs.ensure((size_t)nprob * sizeof(BatchProblem)));
  CLP_CUDA(b, b->outs.ensure((size_t)nprob * sizeof(SolverOut)));
  CLP_CUDA(b, b->nnz.ensure((size_t)nprob * 4 + 16));
  if (nu0) CLP_CUDA(b, cudaMemcpyAsync(b->in_u0.p, h_u0, (size_t)nu0 * 8, cudaMemcpyHostToDevice, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(b->probs.p, h_pr, (size_t)nprob * sizeof(BatchProblem), cudaMemcpyHostToDevice, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->nnz.p, 0, (size_t)nprob * 4 + 16, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->outs.p, 0, (size_t)nprob * sizeof(SolverOut), b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->sync.p, 0, sizeof(SyncBlock), b->stream));
  size_t bytes_in = 0;
  if (int rc = fill_points(b, dd, in, pl, b->probs.p, sizeof(BatchProblem), &bytes_in)) return rc;
  bytes_in += bytes_table;
  // ---- grid: as many CTAs as are co-resident (and as there are problems), each with its own scratch slot
  const BatchSmem bs = batch_smem_plan(max_m);
  if ((long long)bs.total > (long long)b->smem_optin) return fail(b, CLP_ERR_UNSUPPORTED, "batch: shared memory plan exceeds the device limit");
  int occ = 0;
  int rc = CLP_OK;
  if (custom) {
    CLP_CUDA(b, cudaFuncSetAttribute(batch_stored_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bs.total));
    CLP_CUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, batch_stored_solve_kernel, kBatchThreads, bs.total));
  } else {
    rc = (kind == 1) ? batch_occupancy<1, 6>(b, bs.total, &occ) : (dd == 3 ? batch_occupancy<0, 3>(b, bs.total, &occ) : batch_occupancy<0, 2>(b, bs.total, &occ));
    if (rc) return rc;
  }
  if (occ < 1) return fail(b, CLP_ERR_CUDA, "batch kernel does not fit an SM");
  const BatchLayout L = batch_layout(max_m, dd);
  int grid = 0;
  rc = batch_grid(b, occ, nprob, L.total, b->scratch, nullptr, &grid);
  if (rc) return rc;
  BatchArgs ba;
  std::memset(&ba, 0, sizeof(ba));
  ba.prob = b->probs.as<BatchProblem>(); ba.nprob = nprob;
  ba.D1 = b->in_d1.as<double>(); ba.D2 = b->in_d2.as<double>(); ba.A = b->in_a.as<int>(); ba.u0 = b->in_u0.as<double>();
  ba.u_out = b->out_u.as<double>(); ba.out = b->outs.as<SolverOut>(); ba.nnz_out = b->nnz.as<unsigned int>();
  ba.next = reinterpret_cast<int*>(&b->sync.as<SyncBlock>()->counts[0]);
  ba.scratch = b->scratch.as<unsigned char>(); ba.scratch_stride = L.total;
  ba.max_m = max_m; ba.kind = kind; ba.dd = dd;
  ba.prm = solver_params(P);
  ba.p0 = in.p[0]; ba.p1 = in.p[1]; ba.p2 = in.p[2]; ba.p3 = in.p[3]; ba.affinityeps = P.affinityeps;
  ba.sb = b->sync.as<SyncBlock>(); ba.spin_limit = 4LL * 1900000000LL;
  if (b->prof_on) { CLP_CUDA(b, b->prof.ensure((size_t)nprob * 4 * sizeof(unsigned long long))); ba.prof = b->prof.as<unsigned long long>(); }
  // after the launches: device u out (clp_batch_solve_*_dev), then the common tail
  auto finish = [&](const char* label, const char* first) -> int {
    if (in.u_out_dev) {
      const dim3 g((unsigned)((max_m + kBatchThreads - 1) / kBatchThreads), (unsigned)std::min(nprob, 65535));
      batch_copy_u_kernel<<<g, kBatchThreads, 0, b->stream>>>(ba.prob, nprob, ba.u_out, in.u_out_dev, in.u_out_stride);
      CLP_CUDA(b, cudaGetLastError());
    }
    return batch_finish(b, label, first, probs, nu, max_m, grid, L.total, bytes_in, t_begin, sols, u_out, nodes_out);
  };
  if (custom) {
    if ((rc = custom_stage(b, *in.inv, dd, probs, ba.scratch, L.total, L.E1, L.E2, L.A, L.M, &cr))) return rc;
    CLP_CUDA(b, cudaEventRecord(b->ev0, b->stream));
    for (int first = 0; first < nprob; first += grid) {
      const int count = std::min(grid, nprob - first);
      if ((rc = custom_score_round(b, cr, first, count))) return rc;
      batch_stored_solve_kernel<<<count, kBatchThreads, bs.total, b->stream>>>(ba, first);
      CLP_CUDA(b, cudaGetLastError());
    }
    return finish("batch custom", "count");
  }
  CLP_CUDA(b, cudaEventRecord(b->ev0, b->stream));
  rc = (kind == 1) ? batch_launch<1, 6>(b, ba, grid, bs.total) : (dd == 3 ? batch_launch<0, 3>(b, ba, grid, bs.total) : batch_launch<0, 2>(b, ba, grid, bs.total));
  if (rc) return rc;
  return finish("batch", "score");
}

// ---- batched solve of given matrices (clp_batch_matrix.cuh) -------------------------------------------------------
// Problem p: strictly-upper CSC M and C of m[p] columns, as clp_set_sparse_upper takes them.  Validated on the host with
// that call's predicates while the entries are copied into the pinned staging buffer; the error of the whole call is
// the first structural error of any problem (CLP_ERR_INVALID), else the first negative affinity, else the first
// constraint value outside {0, 1} (CLP_ERR_UNSUPPORTED): the single path's order, flag 4 before 1 before 2.
struct MatCheck { int kind = -1; std::string msg; };  // kind 0: structure, 1: M value, 2: C value

// validate one CSC matrix of problem p and copy its row indices and values to ri_dst / v_dst; sets chk on the first
// problem found (structure errors replace a value error found earlier)
void mat_check_copy(int p, const char* what, int which, long long m, const int64_t* cp, const int32_t* ri, const double* v,
                    int32_t* ri_dst, double* v_dst, MatCheck& chk) {
  const std::string tag = "problem " + std::to_string(p) + ", " + what + ": ";
  for (long long c = 0; c < m; ++c) {
    long long prev = -1;
    for (int64_t k = cp[c]; k < cp[c + 1]; ++k) {
      const int32_t r = ri[k];
      if (r < 0 || r >= c) {
        chk.kind = 0;
        chk.msg = tag + "entry (" + std::to_string(r) + ", " + std::to_string(c) + ") is not strictly upper triangular (row < column)";
        return;
      }
      if (r <= prev) {
        chk.kind = 0;
        chk.msg = tag + "rows of column " + std::to_string(c) + " are not strictly ascending (row " + std::to_string(r) + ")";
        return;
      }
      prev = r;
      const double x = v[k];
      if (chk.kind < 0 && (which == 0 ? (x < 0.0) : (x != 0.0 && x != 1.0))) {
        chk.kind = which + 1;
        chk.msg = tag + (which == 0 ? "affinity matrix has negative entries" : "constraint matrix is not binary");
      }
      ri_dst[k] = r; v_dst[k] = x;
    }
  }
}

int batch_launch_matrices(clp_batch b, BatchMatArgs& ba, int grid, size_t smem) {
  CLP_CUDA(b, cudaFuncSetAttribute(batch_matrix_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  batch_matrix_solve_kernel<<<grid, kBatchThreads, smem, b->stream>>>(ba);
  CLP_CUDA(b, cudaGetLastError());
  return CLP_OK;
}

// The host path of the batches given as CSC matrices (clp_batch_solve_matrices, clp_batch_sdp_matrices): the problem
// table, the checks in their order, the staging (column pointers | values | u0 | row indices | problem table) and one
// upload to mat_in after ev_up.  u0 == nullptr: the call takes none (no u0 region, no u0 check).  m[p] > m_limit is
// CLP_ERR_UNSUPPORTED with limit_msg, after the range check of m[p].  The pinned buffer holds at least bytes_out.
struct MatStaging {
  std::vector<BatchMatProblem> probs;
  long long nu = 0;
  int max_m = 1;
  size_t o_val = 0, o_u0 = 0, o_ri = 0, o_pr = 0, bytes_in = 0;
};

int stage_matrices(clp_batch b, int32_t nprob, const int64_t* m, const int64_t* const* cpM, const int32_t* const* riM,
                   const double* const* vM, const int64_t* const* cpC, const int32_t* const* riC, const double* const* vC,
                   const double* const* u0, int m_limit, const char* limit_msg, size_t bytes_out_per_u, size_t bytes_out_per_prob,
                   MatStaging* st) {
  // ---- problem table: sizes and column pointers (the entries are checked while they are copied)
  std::vector<BatchMatProblem>& probs = st->probs;
  probs.assign((size_t)nprob, BatchMatProblem{});
  long long ncp = 0, ne = 0, nu = 0;
  int max_m = 1;
  for (int p = 0; p < nprob; ++p) {
    BatchMatProblem& q = probs[(size_t)p];
    const std::string tag = "problem " + std::to_string(p) + ": ";
    const long long mp = (long long)m[p];
    if (mp < 1 || mp > kBatchMaxM) return fail(b, CLP_ERR_INVALID, tag + "batched problems need 1 <= m <= 4096");
    if (mp > m_limit) return fail(b, CLP_ERR_UNSUPPORTED, tag + limit_msg);
    if (u0 && !u0[p]) return fail(b, CLP_ERR_INVALID, tag + "null u0");
    long long nz[2] = {0, 0};
    for (int which = 0; which < 2; ++which) {
      const int64_t* cp = which ? cpC[p] : cpM[p];
      const char* what = which ? "C" : "M";
      if (!cp || cp[0] != 0) return fail(b, CLP_ERR_INVALID, tag + what + " column pointer must start at 0");
      for (long long c = 0; c < mp; ++c)
        if (cp[c + 1] < cp[c]) return fail(b, CLP_ERR_INVALID, tag + what + " column pointer decreases at column " + std::to_string(c));
      nz[which] = cp[mp];
      if (nz[which] > 0 && (which ? (!riC[p] || !vC[p]) : (!riM[p] || !vM[p])))
        return fail(b, CLP_ERR_INVALID, tag + what + " has entries but null row indices or values");
    }
    q.cpM_off = ncp; q.cpC_off = ncp + mp + 1; ncp += 2 * (mp + 1);
    q.eM_off = ne; q.eC_off = ne + nz[0]; ne += nz[0] + nz[1];
    q.u_off = nu; nu += (mp + 1) & ~1LL;  // 16-byte aligned u0 / u slots (the kernels use 16-byte loads)
    q.m = (int)mp; q.pad_ = 0;
    max_m = std::max(max_m, (int)mp);
  }
  // ---- staging: column pointers | values | u0 | row indices | problem table, one upload
  const long long nu0 = u0 ? nu : 0;
  const size_t o_val = (size_t)ncp * 8, o_u0 = (o_val + (size_t)ne * 8 + 15) & ~(size_t)15, o_ri = o_u0 + (size_t)nu0 * 8;
  const size_t o_pr = (o_ri + (size_t)ne * 4 + 15) & ~(size_t)15;
  const size_t bytes_in = o_pr + (size_t)nprob * sizeof(BatchMatProblem);
  const size_t bytes_out = (size_t)nu * bytes_out_per_u + (size_t)nprob * bytes_out_per_prob;
  CLP_CUDA(b, b->pinned.ensure(std::max(bytes_in, bytes_out) + 4096));
  char* hp = b->pinned.as<char>();
  int64_t* h_cp = reinterpret_cast<int64_t*>(hp);
  double* h_val = reinterpret_cast<double*>(hp + o_val);
  double* h_u0 = reinterpret_cast<double*>(hp + o_u0);
  int32_t* h_ri = reinterpret_cast<int32_t*>(hp + o_ri);
  // validate and copy, problems spread over host threads; the verdict does not depend on the split
  std::vector<MatCheck> chk((size_t)nprob);
  auto work = [&](int p0, int p1) {
    for (int p = p0; p < p1; ++p) {
      const BatchMatProblem& q = probs[(size_t)p];
      std::memcpy(h_cp + q.cpM_off, cpM[p], (size_t)(q.m + 1) * 8);
      std::memcpy(h_cp + q.cpC_off, cpC[p], (size_t)(q.m + 1) * 8);
      if (u0) std::memcpy(h_u0 + q.u_off, u0[p], (size_t)q.m * 8);
      MatCheck cm, cc;
      mat_check_copy(p, "M", 0, q.m, cpM[p], riM[p], vM[p], h_ri + q.eM_off, h_val + q.eM_off, cm);
      if (cm.kind != 0) mat_check_copy(p, "C", 1, q.m, cpC[p], riC[p], vC[p], h_ri + q.eC_off, h_val + q.eC_off, cc);
      chk[(size_t)p] = (cm.kind == 0 || cc.kind == 0) ? (cm.kind == 0 ? cm : cc) : (cm.kind >= 0 ? cm : cc);
    }
  };
  {
    const unsigned hw = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    const int nth = (int)std::min<long long>(hw, std::max<long long>(1, ne / (1 << 20)));  // ~1M entries per thread at least
    if (nth <= 1 || nprob == 1) work(0, nprob);
    else {
      std::vector<std::thread> th;
      for (int t = 0; t < nth; ++t) th.emplace_back(work, (int)((long long)nprob * t / nth), (int)((long long)nprob * (t + 1) / nth));
      for (std::thread& x : th) x.join();
    }
  }
  for (int kind = 0; kind < 3; ++kind)
    for (int p = 0; p < nprob; ++p)
      if (chk[(size_t)p].kind == kind) return fail(b, kind == 0 ? CLP_ERR_INVALID : CLP_ERR_UNSUPPORTED, chk[(size_t)p].msg);
  std::memcpy(hp + o_pr, probs.data(), (size_t)nprob * sizeof(BatchMatProblem));
  // the device copy keeps the staging offsets (u0 starts on a 16-byte boundary, the base is cudaMalloc-aligned)
  CLP_CUDA(b, b->mat_in.ensure(bytes_in + 16));
  CLP_CUDA(b, cudaEventRecord(b->ev_up, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(b->mat_in.p, hp, bytes_in, cudaMemcpyHostToDevice, b->stream));
  st->nu = nu; st->max_m = max_m;
  st->o_val = o_val; st->o_u0 = o_u0; st->o_ri = o_ri; st->o_pr = o_pr; st->bytes_in = bytes_in;
  return CLP_OK;
}

int batch_solve_matrices(clp_batch b, int32_t nprob, const int64_t* m, const int64_t* const* cpM, const int32_t* const* riM,
                         const double* const* vM, const int64_t* const* cpC, const int32_t* const* riC,
                         const double* const* vC, const double* const* u0, clp_solution* sols, double* const* u_out,
                         int32_t* const* nodes_out) {
  if (!b) return CLP_ERR_INVALID;
  if (nprob <= 0 || !m || !cpM || !riM || !vM || !cpC || !riC || !vC || !u0 || !sols) return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  const clp_params& P = b->prm;
  if (P.rounding == CLP_ROUND_DSD) return fail(b, CLP_ERR_UNSUPPORTED, "Rounding::DSD is not available in a batch");
  if (P.maxlsiters < 1) return fail(b, CLP_ERR_INVALID, "maxlsiters must be >= 1");
  const auto t_begin = std::chrono::steady_clock::now();
  CLP_CUDA(b, cudaSetDevice(b->device));
  MatStaging st;
  if (int rc = stage_matrices(b, nprob, m, cpM, riM, vM, cpC, riC, vC, u0, kBatchMaxM, "", 8, sizeof(SolverOut) + 4, &st))
    return rc;
  const std::vector<BatchMatProblem>& probs = st.probs;
  const long long nu = st.nu;
  const int max_m = st.max_m;
  const size_t o_val = st.o_val, o_u0 = st.o_u0, o_ri = st.o_ri, o_pr = st.o_pr, bytes_in = st.bytes_in;
  CLP_CUDA(b, b->out_u.ensure((size_t)nu * 8 + 16));
  CLP_CUDA(b, b->outs.ensure((size_t)nprob * sizeof(SolverOut)));
  CLP_CUDA(b, b->nnz.ensure((size_t)nprob * 4 + 16));
  CLP_CUDA(b, cudaMemsetAsync(b->nnz.p, 0, (size_t)nprob * 4 + 16, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->outs.p, 0, (size_t)nprob * sizeof(SolverOut), b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->sync.p, 0, sizeof(SyncBlock), b->stream));
  // ---- grid: as many CTAs as are co-resident (and as there are problems), each with its own scratch slot
  const BatchSmem bs = batch_smem_plan(max_m);
  if ((long long)bs.total > (long long)b->smem_optin) return fail(b, CLP_ERR_UNSUPPORTED, "batch: shared memory plan exceeds the device limit");
  int occ = 0;
  CLP_CUDA(b, cudaFuncSetAttribute(batch_matrix_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bs.total));
  CLP_CUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, batch_matrix_solve_kernel, kBatchThreads, bs.total));
  if (occ < 1) return fail(b, CLP_ERR_CUDA, "batch kernel does not fit an SM");
  const BatchLayout L = batch_layout(max_m, 0, /*points*/ false);
  int grid = 0;
  if (int rc = batch_grid(b, occ, nprob, L.total, b->scratch, nullptr, &grid)) return rc;
  const char* din = b->mat_in.as<char>();
  BatchMatArgs ba;
  std::memset(&ba, 0, sizeof(ba));
  ba.prob = reinterpret_cast<const BatchMatProblem*>(din + o_pr); ba.nprob = nprob;
  ba.colptr = reinterpret_cast<const long long*>(din); ba.val = reinterpret_cast<const double*>(din + o_val);
  ba.u0 = reinterpret_cast<const double*>(din + o_u0); ba.rowidx = reinterpret_cast<const int*>(din + o_ri);
  ba.u_out = b->out_u.as<double>(); ba.out = b->outs.as<SolverOut>(); ba.nnz_out = b->nnz.as<unsigned int>();
  ba.next = reinterpret_cast<int*>(&b->sync.as<SyncBlock>()->counts[0]);
  ba.scratch = b->scratch.as<unsigned char>(); ba.scratch_stride = L.total;
  ba.max_m = max_m;
  ba.prm = solver_params(P);
  ba.sb = b->sync.as<SyncBlock>(); ba.spin_limit = 4LL * 1900000000LL;
  if (b->prof_on) { CLP_CUDA(b, b->prof.ensure((size_t)nprob * 4 * sizeof(unsigned long long))); ba.prof = b->prof.as<unsigned long long>(); }
  CLP_CUDA(b, cudaEventRecord(b->ev0, b->stream));
  if (int rc = batch_launch_matrices(b, ba, grid, bs.total)) return rc;
  return batch_finish(b, "batch matrices", "scatter", probs, nu, max_m, grid, L.total, bytes_in, t_begin, sols, u_out, nodes_out);
}

// ---- batched semidefinite relaxations of given matrices (clp_sdp.cuh) ---------------------------------------------
// The host path of clp_batch_solve_matrices (stage_matrices), then sdp_solve_kernel<float> with the CSC inputs: each
// CTA scatters its problem into an fp32 store as clp_set_sparse_upper does, so problem p gets what an fp32 handle gets.
int batch_sdp_matrices(clp_batch b, int32_t nprob, const int64_t* m, const int64_t* const* cpM, const int32_t* const* riM,
                       const double* const* vM, const int64_t* const* cpC, const int32_t* const* riC, const double* const* vC,
                       const clp_sdp_params* prm, clp_sdp_info* infos, int32_t* const* nodes_out, double* const* X_out,
                       double* const* lambdas_out, double* const* evec1_out) {
  if (!b) return CLP_ERR_INVALID;
  if (nprob <= 0 || !m || !cpM || !riM || !vM || !cpC || !riC || !vC) return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  if (int rc = sdp_check_params(b, prm, infos)) return rc;
  const auto t_begin = std::chrono::steady_clock::now();
  CLP_CUDA(b, cudaSetDevice(b->device));
  // read back: p and evec1 (2 per u slot), X (m^2 <= 128 * slot), SdpOut
  MatStaging st;
  const std::string limit_msg = "the relaxation needs m <= CLP_SDP_MAX_M = " + std::to_string(kSdpMaxM);
  if (int rc = stage_matrices(b, nprob, m, cpM, riM, vM, cpC, riC, vC, nullptr, kSdpMaxM, limit_msg.c_str(),
                              (2 + kSdpMaxM) * 8, sizeof(SdpOut), &st))
    return rc;
  const long long nu = st.nu;
  std::vector<long long> x_off((size_t)nprob);
  long long nx = 0;
  for (int p = 0; p < nprob; ++p) { x_off[(size_t)p] = nx; nx += (long long)st.probs[(size_t)p].m * st.probs[(size_t)p].m; }
  // device outputs: X offsets | SdpOut | p | evec1 | X
  const size_t o_out = ((size_t)nprob * 8 + 255) & ~(size_t)255, o_p = o_out + (((size_t)nprob * sizeof(SdpOut) + 255) & ~(size_t)255);
  const size_t o_e = o_p + (size_t)nu * 8, o_x = o_e + (size_t)nu * 8, bytes_out = o_x + (size_t)nx * 8;
  CLP_CUDA(b, b->sdp_out.ensure(bytes_out));
  char* d = b->sdp_out.as<char>();
  CLP_CUDA(b, cudaMemcpyAsync(d, x_off.data(), (size_t)nprob * 8, cudaMemcpyHostToDevice, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->sync.p, 0, sizeof(SyncBlock), b->stream));
  const size_t smem = sdp_smem_bytes(st.max_m);
  int occ = 0;
  CLP_CUDA(b, cudaFuncSetAttribute(sdp_solve_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CLP_CUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, sdp_solve_kernel<float>, kSdpThreads, smem));
  if (occ < 1) return fail(b, CLP_ERR_CUDA, "sdp kernel does not fit an SM");
  int grid = 0;
  if (int rc = batch_grid(b, occ, nprob, sdp_slot_bytes(st.max_m), b->scratch, nullptr, &grid)) return rc;
  const char* din = b->mat_in.as<char>();
  SdpArgs a{};
  a.prob = reinterpret_cast<const BatchMatProblem*>(din + st.o_pr); a.x_off = reinterpret_cast<const long long*>(d);
  a.nprob = nprob;
  a.colptr = reinterpret_cast<const long long*>(din); a.val = reinterpret_cast<const double*>(din + st.o_val);
  a.rowidx = reinterpret_cast<const int*>(din + st.o_ri);
  a.x_out = reinterpret_cast<double*>(d + o_x); a.p_out = reinterpret_cast<double*>(d + o_p);
  a.e_out = reinterpret_cast<double*>(d + o_e); a.out = reinterpret_cast<SdpOut*>(d + o_out);
  a.next = reinterpret_cast<int*>(&b->sync.as<SyncBlock>()->counts[0]);
  a.flags = &b->sync.as<SyncBlock>()->flags;
  a.scratch = b->scratch.as<unsigned char>(); a.scratch_stride = sdp_slot_bytes(st.max_m); a.max_m = st.max_m;
  a.max_iters = prm->max_iters; a.eps_abs = prm->eps_abs; a.eps_rel = prm->eps_rel;
  a.limit_ns = sdp_limit_ns(*prm, t_begin);
  CLP_CUDA(b, cudaEventRecord(b->ev0, b->stream));
  sdp_solve_kernel<float><<<grid, kSdpThreads, smem, b->stream>>>(a);
  CLP_CUDA(b, cudaGetLastError());
  CLP_CUDA(b, cudaEventRecord(b->ev1, b->stream));
  char* hp = b->pinned.as<char>();
  SyncBlock h_sb;
  CLP_CUDA(b, cudaMemcpyAsync(hp, d + o_out, bytes_out - o_out, cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(&h_sb, b->sync.p, sizeof(SyncBlock), cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaStreamSynchronize(b->stream));
  if (h_sb.flags != 0) return fail(b, CLP_ERR_CUDA, "batched matrices: the device found an entry the host check passed");
  float ms = 0.f;
  CLP_CUDA(b, cudaEventElapsedTime(&ms, b->ev0, b->ev1));
  b->last_ctas = grid; b->last_scratch = (long long)grid * (long long)a.scratch_stride; b->last_nnz = 0;
  const SdpOut* h_out = reinterpret_cast<const SdpOut*>(hp);
  const double* h_p = reinterpret_cast<const double*>(hp + (o_p - o_out));
  const double* h_e = h_p + nu;
  const double* h_x = h_e + nu;
  for (int p = 0; p < nprob; ++p) {
    const BatchMatProblem& q = st.probs[(size_t)p];
    sdp_result(h_out[p], q.m, h_p + q.u_off, h_e + q.u_off, ms, &infos[p], nodes_out ? nodes_out[p] : nullptr,
               lambdas_out ? lambdas_out[p] : nullptr, evec1_out ? evec1_out[p] : nullptr);
    if (X_out && X_out[p]) std::memcpy(X_out[p], h_x + x_off[(size_t)p], (size_t)q.m * q.m * 8);
  }
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  for (int p = 0; p < nprob; ++p) infos[p].t = wall / nprob;
  return CLP_OK;
}

// ---- batched solve of dense device tensors (batch_dense_solve_kernel) ---------------------------------------------
// The values are checked on the device (batch_finish maps what the kernel found); only the sizes, pointers, strides and
// dtype are checked here.  Only the problem table is uploaded.
template <typename In>
int batch_launch_dense(clp_batch b, BatchDenseArgs& ba, size_t smem, int nprob, size_t stride, int* grid) {
  int occ = 0;
  CLP_CUDA(b, cudaFuncSetAttribute(batch_dense_solve_kernel<In>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CLP_CUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, batch_dense_solve_kernel<In>, kBatchThreads, smem));
  if (occ < 1) return fail(b, CLP_ERR_CUDA, "batch kernel does not fit an SM");
  if (int rc = batch_grid(b, occ, nprob, stride, b->scratch, nullptr, grid)) return rc;
  ba.scratch = b->scratch.as<unsigned char>();
  CLP_CUDA(b, cudaEventRecord(b->ev0, b->stream));
  batch_dense_solve_kernel<In><<<*grid, kBatchThreads, smem, b->stream>>>(ba);
  CLP_CUDA(b, cudaGetLastError());
  return CLP_OK;
}

int batch_solve_dense_dev(clp_batch b, int32_t nprob, const int64_t* m, int dtype, const void* M, const void* Cm, int64_t bstride,
                          int64_t rs, int64_t cs, const double* u0, int64_t u0_stride, clp_solution* sols, double* u_out_dev,
                          int64_t u_out_stride, int32_t* const* nodes_out) {
  if (!b) return CLP_ERR_INVALID;
  if (nprob <= 0 || !m || !M || !Cm || !sols) return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  if (!u0) return fail(b, CLP_ERR_INVALID, "null u0");
  int max_m = 1;
  for (int p = 0; p < nprob; ++p) {
    if (m[p] < 1 || m[p] > kBatchMaxM) return fail(b, CLP_ERR_INVALID, "problem " + std::to_string(p) + ": batched problems need 1 <= m <= 4096");
    max_m = std::max(max_m, (int)m[p]);
  }
  if (!dense_strides_ok(rs, cs) || bstride < 1 || u0_stride < 1 || (u_out_dev && u_out_stride < max_m))
    return fail(b, CLP_ERR_INVALID, "bad strides (one of row_stride, col_stride must be 1 and the other >= 1; batch_stride, "
                                    "u0_stride >= 1; u_out_stride >= the largest m)");
  if (dtype != CLP_IN_F32 && dtype != CLP_IN_F64) return fail(b, CLP_ERR_INVALID, "unknown input dtype (CLP_IN_F32 or CLP_IN_F64)");
  const clp_params& P = b->prm;
  if (P.rounding == CLP_ROUND_DSD) return fail(b, CLP_ERR_UNSUPPORTED, "Rounding::DSD is not available in a batch");
  if (P.maxlsiters < 1) return fail(b, CLP_ERR_INVALID, "maxlsiters must be >= 1");
  const auto t_begin = std::chrono::steady_clock::now();
  CLP_CUDA(b, cudaSetDevice(b->device));
  // every problem's u0 / u slot starts on a 128-byte line of its own: the CTAs stage u0 and read u back themselves
  const long long ustride = round_up(max_m, 16);
  const long long nu = (long long)nprob * ustride;
  std::vector<BatchMatProblem> probs((size_t)nprob);
  for (int p = 0; p < nprob; ++p) { probs[(size_t)p].m = (int)m[p]; probs[(size_t)p].u_off = p * ustride; }
  const size_t bytes_in = (size_t)nprob * sizeof(BatchMatProblem);
  const size_t bytes_out = (size_t)nu * 8 + (size_t)nprob * (sizeof(SolverOut) + 4);
  CLP_CUDA(b, b->pinned.ensure(std::max(bytes_in, bytes_out) + 4096));
  std::memcpy(b->pinned.p, probs.data(), bytes_in);
  CLP_CUDA(b, b->probs.ensure(bytes_in));
  CLP_CUDA(b, b->in_u0.ensure((size_t)nu * 8 + 16));
  CLP_CUDA(b, b->out_u.ensure((size_t)nu * 8 + 16));
  CLP_CUDA(b, b->outs.ensure((size_t)nprob * sizeof(SolverOut)));
  CLP_CUDA(b, b->nnz.ensure((size_t)nprob * 4 + 16));
  CLP_CUDA(b, cudaEventRecord(b->ev_up, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(b->probs.p, b->pinned.p, bytes_in, cudaMemcpyHostToDevice, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->nnz.p, 0, (size_t)nprob * 4 + 16, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->outs.p, 0, (size_t)nprob * sizeof(SolverOut), b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->sync.p, 0, sizeof(SyncBlock), b->stream));
  const BatchSmem bs = batch_smem_plan(max_m);
  if ((long long)bs.total > (long long)b->smem_optin) return fail(b, CLP_ERR_UNSUPPORTED, "batch: shared memory plan exceeds the device limit");
  const BatchLayout L = batch_layout(max_m, 0, /*points*/ false);
  SyncBlock* sb = b->sync.as<SyncBlock>();
  BatchDenseArgs ba;
  std::memset(&ba, 0, sizeof(ba));
  ba.prob = b->probs.as<BatchMatProblem>(); ba.nprob = nprob;
  ba.M = M; ba.C = Cm; ba.bstride = bstride; ba.rs = rs; ba.cs = cs;
  ba.u0_in = u0; ba.u0_stride = u0_stride; ba.u0 = b->in_u0.as<double>();
  ba.u_out = b->out_u.as<double>(); ba.u_out_dev = u_out_dev; ba.u_out_stride = u_out_stride;
  ba.out = b->outs.as<SolverOut>(); ba.nnz_out = b->nnz.as<unsigned int>();
  ba.next = reinterpret_cast<int*>(&sb->counts[0]); ba.bad = &sb->counts[1];
  ba.scratch_stride = L.total;
  ba.max_m = max_m;
  ba.prm = solver_params(P);
  ba.sb = sb; ba.spin_limit = 4LL * 1900000000LL;
  if (b->prof_on) { CLP_CUDA(b, b->prof.ensure((size_t)nprob * 4 * sizeof(unsigned long long))); ba.prof = b->prof.as<unsigned long long>(); }
  int grid = 0;
  const int rc = dtype == CLP_IN_F32 ? batch_launch_dense<float>(b, ba, bs.total, nprob, L.total, &grid)
                                     : batch_launch_dense<double>(b, ba, bs.total, nprob, L.total, &grid);
  if (rc) return rc;
  return batch_finish(b, "batch dense", "load", probs, nu, max_m, grid, L.total, bytes_in, t_begin, sols, nullptr, nodes_out);
}

// ---- batched maximum clique (clp_batch_clique.cuh) ----------------------------------------------------------------
// kind 0 / 1: scored problems (EuclideanDistance d = 2, 3 / PointNormalDistance); kind 2: graphs given as strictly-upper
// CSC patterns; kBatchKindCustom: scored with a caller's invariant, phase A in rounds (gather and score, then the
// prepare kernel on the stored matrices).  Phase A, then for EXACT with a positive time limit phases B and C: two host
// synchronisations.
const void* mcb_prepare_fn(int kind, int dd) {
  if (kind == kMcbKindGraph) return (const void*)mc_batch_prepare_kernel<kMcbKindGraph, 1>;
  if (kind == kMcbKindStored) return (const void*)mc_batch_prepare_kernel<kMcbKindStored, 1>;
  if (kind == 1) return (const void*)mc_batch_prepare_kernel<1, 6>;
  return dd == 3 ? (const void*)mc_batch_prepare_kernel<0, 3> : (const void*)mc_batch_prepare_kernel<0, 2>;
}

int batch_max_clique(clp_batch b, int kind, int dd, int32_t nprob, const BatchInput& in, int method, double time_limit_s,
                     clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out) {
  if (!b) return CLP_ERR_INVALID;
  const auto t_begin = std::chrono::steady_clock::now();
  if (nprob <= 0 || !infos || !in.m) return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  if (method < CLP_MC_EXACT || method > CLP_MC_KCORE) return fail(b, CLP_ERR_INVALID, "unknown maximum-clique method");
  const bool graph = kind == kMcbKindGraph, custom = kind == kBatchKindCustom;
  if (graph ? (!in.colptr || !in.rowidx) : ((!in.dev && (!in.D1 || !in.D2)) || !in.n1 || !in.n2))
    return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  if (custom) {
    if (int rc = custom_check(b, *in.inv, nprob, dd, in)) return rc;
  } else if (!graph && !((kind == 0 && (dd == 2 || dd == 3)) || (kind == 1 && dd == 6))) {
    return fail(b, CLP_ERR_UNSUPPORTED, "batched scoring supports EuclideanDistance with d = 2, 3 and PointNormalDistance");
  }
  const bool search = method == CLP_MC_EXACT && time_limit_s > 0;
  CLP_CUDA(b, cudaSetDevice(b->device));
  CustomRounds cr;
  if (custom)
    if (int rc = custom_compile(b, *in.inv, dd, &cr)) return rc;
  // ---- problem table and per-problem regions; scored inputs are checked by plan_points and staged by fill_points
  // once the table is on the device, graphs are checked here
  std::vector<McBatchProblem> probs((size_t)nprob);
  PointsPlan pl;
  const std::vector<BatchProblem>& pts = pl.probs;
  if (!graph) {
    if (int rc = plan_points(b, dd, nprob, in, &pl)) return rc;
    for (int p = 0; p < nprob; ++p) probs[(size_t)p].sp = pts[(size_t)p];
  }
  long long ne = 0, nadj = 0, nv = 0, nt = 0;
  int max_m = 1;
  for (int p = 0; p < nprob; ++p) {
    McBatchProblem& q = probs[(size_t)p];
    if (graph) {
      const long long mp = (long long)in.m[p];
      if (mp <= 0 || mp > kBatchMaxM) return fail(b, CLP_ERR_INVALID, "batched problems need 1 <= m <= 4096 vertices");
      const int64_t* cp = in.colptr[p];
      const int32_t* ri = in.rowidx[p];
      if (!cp || cp[0] != 0) return fail(b, CLP_ERR_INVALID, "graph " + std::to_string(p) + ": colptr must start at 0");
      for (long long c = 0; c < mp; ++c) {
        if (cp[c + 1] < cp[c]) return fail(b, CLP_ERR_INVALID, "graph " + std::to_string(p) + ": colptr decreases");
        for (int64_t k = cp[c]; k < cp[c + 1]; ++k)
          if (!ri || ri[k] < 0 || ri[k] >= c)
            return fail(b, CLP_ERR_INVALID, "graph " + std::to_string(p) + ": entry (" + std::to_string(ri ? ri[k] : -1) + ", " +
                                                std::to_string(c) + ") is not strictly upper (row < column)");
      }
      q.e_off = ne; q.ne = cp[mp];
      ne += cp[mp];
      q.sp.m = (int)mp;
    }
    const long long mp = q.sp.m;
    const long long W = (mp + 31) / 32;
    q.adj_off = nadj; nadj += mp * W;
    q.v_off = nv; nv += (4 * mp + 1 + 3) & ~3LL;
    q.t_off = nt; nt += mp + 1;
    max_m = std::max(max_m, (int)mp);
  }
  // ---- edges and the problem table through the pinned staging buffer
  const size_t bytes_in = (size_t)(2 * ne) * 4 + (size_t)nprob * sizeof(McBatchProblem) + 64;
  const size_t bytes_out = (size_t)nv * 4 + (size_t)nprob * (sizeof(McBatchOut) + 3 * 8 + 2 * 4) + 64;
  CLP_CUDA(b, b->pinned.ensure(std::max(bytes_in, bytes_out) + 4096));
  char* hp = b->pinned.as<char>();
  int32_t* h_e = reinterpret_cast<int32_t*>(hp);
  McBatchProblem* h_pr = reinterpret_cast<McBatchProblem*>(hp + (((size_t)(2 * ne) * 4 + 15) & ~(size_t)15));
  if (graph)
    for (int p = 0; p < nprob; ++p) {
      const McBatchProblem& q = probs[(size_t)p];
      const int64_t* cp = in.colptr[p];
      int32_t* e = h_e + 2 * q.e_off;
      for (int c = 0; c < q.sp.m; ++c)
        for (int64_t k = cp[c]; k < cp[c + 1]; ++k) { *e++ = in.rowidx[p][k]; *e++ = c; }
    }
  std::memcpy(h_pr, probs.data(), (size_t)nprob * sizeof(McBatchProblem));
  CLP_CUDA(b, b->mc_edges.ensure((size_t)ne * 8 + 16));
  CLP_CUDA(b, b->mc_probs.ensure((size_t)nprob * sizeof(McBatchProblem)));
  CLP_CUDA(b, b->mc_adj.ensure((size_t)nadj * 4 + 16));
  CLP_CUDA(b, b->mc_vint.ensure((size_t)nv * 4 + 16));
  CLP_CUDA(b, b->mc_tpre.ensure((size_t)nt * 8 + 16));
  CLP_CUDA(b, b->mc_out.ensure((size_t)nprob * sizeof(McBatchOut)));
  if (ne) CLP_CUDA(b, cudaMemcpyAsync(b->mc_edges.p, h_e, (size_t)ne * 8, cudaMemcpyHostToDevice, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(b->mc_probs.p, h_pr, (size_t)nprob * sizeof(McBatchProblem), cudaMemcpyHostToDevice, b->stream));
  if (graph) CLP_CUDA(b, cudaMemsetAsync(b->mc_adj.p, 0, (size_t)nadj * 4, b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->mc_out.p, 0, (size_t)nprob * sizeof(McBatchOut), b->stream));
  CLP_CUDA(b, cudaMemsetAsync(b->sync.p, 0, sizeof(SyncBlock), b->stream));
  if (!graph) {
    size_t bytes_pts = 0;
    const void* table = b->mc_probs.as<unsigned char>() + offsetof(McBatchProblem, sp);
    if (int rc = fill_points(b, dd, in, pl, table, sizeof(McBatchProblem), &bytes_pts)) return rc;
  }

  // ---- phase A: one CTA per problem, as many CTAs as are co-resident and, for scored problems, fit their scratch
  const McbSmem sm = mcb_smem_plan(max_m);
  if ((long long)sm.total > (long long)b->smem_optin) return fail(b, CLP_ERR_UNSUPPORTED, "batched maximum clique: shared memory plan exceeds the device limit");
  const void* fn = mcb_prepare_fn(kind, dd);
  CLP_CUDA(b, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm.total));
  int occ = 0;
  CLP_CUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kBatchThreads, sm.total));
  if (occ < 1) return fail(b, CLP_ERR_CUDA, "batched maximum-clique kernel does not fit an SM");
  const McbLayout ML = mcb_layout(max_m, dd);
  const size_t pstride = graph ? 0 : ML.total;
  int grid = 0;
  if (int rc = batch_grid(b, occ, nprob, pstride, b->mc_pscratch,
                          "batched maximum clique: not enough device memory for one problem's scoring scratch", &grid))
    return rc;
  McBatchArgs ba;
  std::memset(&ba, 0, sizeof(ba));
  ba.prob = b->mc_probs.as<McBatchProblem>(); ba.nprob = nprob; ba.run_heu = method != CLP_MC_KCORE ? 1 : 0; ba.build_tasks = search ? 1 : 0;
  ba.next = reinterpret_cast<int*>(&b->sync.as<SyncBlock>()->counts[0]);
  ba.adj = b->mc_adj.as<unsigned>(); ba.vint = b->mc_vint.as<int>(); ba.tpre = b->mc_tpre.as<long long>();
  ba.out = b->mc_out.as<McBatchOut>(); ba.edges = b->mc_edges.as<int>();
  ba.D1 = b->in_d1.as<double>(); ba.D2 = b->in_d2.as<double>(); ba.A = b->in_a.as<int>();
  ba.p0 = in.p[0]; ba.p1 = in.p[1]; ba.p2 = in.p[2]; ba.p3 = in.p[3]; ba.affinityeps = b->prm.affinityeps;
  ba.error = &b->sync.as<SyncBlock>()->error;
  ba.scratch = b->mc_pscratch.as<unsigned char>(); ba.scratch_stride = pstride; ba.max_m = max_m;
  if (custom)
    if (int rc = custom_stage(b, *in.inv, dd, pts, ba.scratch, pstride, ML.E1, ML.E2, ML.A, ML.M, &cr)) return rc;
  McEvents ev;
  for (cudaEvent_t& x : ev.e) CLP_CUDA(b, cudaEventCreate(&x));
  CLP_CUDA(b, cudaEventRecord(ev.e[0], b->stream));
  if (custom) {  // rounds: problem first + k in slot k; the prepare kernel sees the round's problems as 0 .. count - 1
    ba.scratch += ML.M;
    for (int first = 0; first < nprob; first += grid) {
      const int count = std::min(grid, nprob - first);
      if (int rc = custom_score_round(b, cr, first, count)) return rc;
      McBatchArgs ra = ba;
      ra.prob = ba.prob + first; ra.out = ba.out + first; ra.nprob = count;
      CLP_CUDA(b, cudaMemsetAsync(ba.next, 0, sizeof(int), b->stream));
      void* args[] = {&ra};
      CLP_CUDA(b, cudaLaunchKernel(fn, dim3((unsigned)count), dim3(kBatchThreads), args, sm.total, b->stream));
    }
  } else {
    void* args[] = {&ba};
    CLP_CUDA(b, cudaLaunchKernel(fn, dim3((unsigned)grid), dim3(kBatchThreads), args, sm.total, b->stream));
  }
  CLP_CUDA(b, cudaEventRecord(ev.e[1], b->stream));
  std::vector<McBatchOut> outs((size_t)nprob);
  SyncBlock h_sb;
  CLP_CUDA(b, cudaMemcpyAsync(outs.data(), b->mc_out.p, (size_t)nprob * sizeof(McBatchOut), cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaMemcpyAsync(&h_sb, b->sync.p, sizeof(SyncBlock), cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaStreamSynchronize(b->stream));
  if (int rc = bad_problem(b, h_sb.counts[1])) return rc;
  if (h_sb.error == 2) return fail(b, CLP_ERR_INVALID, "association index out of range of D1/D2 in a batched problem");
  b->last_ctas = grid;
  b->last_scratch = (long long)grid * (long long)pstride;

  // ---- phases B and C: the search over the tasks of every problem, then the replays
  int* h_v = reinterpret_cast<int*>(hp);
  unsigned long long* h_best = reinterpret_cast<unsigned long long*>(hp + (((size_t)nv * 4 + 15) & ~(size_t)15));
  unsigned long long* h_br = h_best + nprob;
  unsigned long long* h_done = h_br + nprob;
  int* h_flags = reinterpret_cast<int*>(h_done + nprob);
  float search_ms = 0.f;
  long long total = 0;
  if (search) {
    std::vector<int> porder;
    for (int p = 0; p < nprob; ++p) if (outs[(size_t)p].ntasks > 0) porder.push_back(p);
    std::stable_sort(porder.begin(), porder.end(), [&](int x, int y) { return outs[(size_t)x].ntasks > outs[(size_t)y].ntasks; });
    // rounds: round k holds task k of the first w problems of porder (those with more than k tasks); equal widths
    // form one segment
    std::vector<long long> seg_start, seg_k0;
    std::vector<int> seg_width;
    long long k0 = 0;
    for (int i = (int)porder.size() - 1; i >= 0; --i) {
      const long long kend = outs[(size_t)porder[(size_t)i]].ntasks;
      if (kend <= k0) continue;
      seg_start.push_back(total); seg_k0.push_back(k0); seg_width.push_back(i + 1);
      total += (kend - k0) * (i + 1);
      k0 = kend;
    }
    seg_start.push_back(total);
    if (total > 0) {
      int K = 1;
      for (int p : porder) K = std::max(K, outs[(size_t)p].K);
      size_t free_b = 0, total_b = 0;
      CLP_CUDA(b, cudaMemGetInfo(&free_b, &total_b));
      const McSearchSetup ss = mc_search_setup(K, free_b + b->mc_sscratch.cap, b->sm_count, time_limit_s, t_begin);
      if (ss.nworkers < kMcSearchWarps) return fail(b, CLP_ERR_ALLOC, "batched maximum clique EXACT: not enough device memory for the search scratch");
      CLP_CUDA(b, b->mc_sscratch.ensure((size_t)ss.nworkers * ss.stride));
      const int nseg = (int)seg_width.size();
      // device state: best | branches | done [nprob] 8-byte, next, deadline, flags [2 nprob]; rounds: porder, segments
      CLP_CUDA(b, b->mc_state.ensure((size_t)nprob * 3 * 8 + 16 + (size_t)nprob * 8 + 16));
      CLP_CUDA(b, b->mc_rounds.ensure((size_t)(nprob + 1) * 4 + (size_t)(2 * nseg + 1) * 8 + (size_t)nseg * 4 + 64));
      unsigned long long* d_best = b->mc_state.as<unsigned long long>();
      unsigned long long* d_br = d_best + nprob;
      unsigned long long* d_done = d_br + nprob;
      unsigned long long* d_next = d_done + nprob;
      unsigned long long* d_deadline = d_next + 1;
      int* d_flags = reinterpret_cast<int*>(d_deadline + 1);
      long long* d_seg_start = b->mc_rounds.as<long long>();
      long long* d_seg_k0 = d_seg_start + nseg + 1;
      int* d_seg_width = reinterpret_cast<int*>(d_seg_k0 + nseg);
      int* d_porder = d_seg_width + nseg;
      std::vector<unsigned long long> best0((size_t)nprob);
      for (int p = 0; p < nprob; ++p) best0[(size_t)p] = mc_key((unsigned)outs[(size_t)p].lb, 0u);
      CLP_CUDA(b, cudaMemcpyAsync(d_best, best0.data(), (size_t)nprob * 8, cudaMemcpyHostToDevice, b->stream));
      CLP_CUDA(b, cudaMemsetAsync(d_br, 0, (size_t)nprob * 2 * 8 + 16 + (size_t)nprob * 8, b->stream));
      CLP_CUDA(b, cudaMemcpyAsync(d_seg_start, seg_start.data(), seg_start.size() * 8, cudaMemcpyHostToDevice, b->stream));
      CLP_CUDA(b, cudaMemcpyAsync(d_seg_k0, seg_k0.data(), seg_k0.size() * 8, cudaMemcpyHostToDevice, b->stream));
      CLP_CUDA(b, cudaMemcpyAsync(d_seg_width, seg_width.data(), seg_width.size() * 4, cudaMemcpyHostToDevice, b->stream));
      CLP_CUDA(b, cudaMemcpyAsync(d_porder, porder.data(), porder.size() * 4, cudaMemcpyHostToDevice, b->stream));
      McBatchSearchArgs sa;
      sa.prob = b->mc_probs.as<McBatchProblem>(); sa.out = b->mc_out.as<McBatchOut>();
      sa.adj = b->mc_adj.as<unsigned>(); sa.vint = b->mc_vint.as<int>(); sa.tpre = b->mc_tpre.as<long long>();
      sa.porder = d_porder; sa.seg_start = d_seg_start; sa.seg_k0 = d_seg_k0; sa.seg_width = d_seg_width; sa.nseg = nseg;
      sa.total = total; sa.K = K; sa.KW = ss.KW; sa.arena_cap = ss.arena_cap;
      sa.scratch = b->mc_sscratch.as<unsigned char>(); sa.stride = ss.stride;
      sa.best = d_best; sa.branches = d_br; sa.done = d_done; sa.flags = d_flags; sa.next = d_next; sa.deadline = d_deadline;
      const size_t ssmem = (size_t)kMcSearchWarps * 2 * ss.KW * sizeof(unsigned);
      CLP_CUDA(b, cudaFuncSetAttribute(mc_batch_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssmem));
      CLP_CUDA(b, cudaFuncSetAttribute(mc_batch_replay_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssmem));
      CLP_CUDA(b, cudaEventRecord(ev.e[2], b->stream));
      mc_deadline_kernel<<<1, 1, 0, b->stream>>>(d_deadline, ss.limit_ns);
      mc_batch_search_kernel<<<(unsigned)(ss.nworkers / kMcSearchWarps), kMcSearchWarps * 32, ssmem, b->stream>>>(sa);
      CLP_CUDA(b, cudaGetLastError());
      const long long rgrid = std::min<long long>(ss.nworkers / kMcSearchWarps, (nprob + kMcSearchWarps - 1) / kMcSearchWarps);
      mc_batch_replay_kernel<<<(unsigned)rgrid, kMcSearchWarps * 32, ssmem, b->stream>>>(sa, nprob);
      CLP_CUDA(b, cudaGetLastError());
      CLP_CUDA(b, cudaEventRecord(ev.e[3], b->stream));
      CLP_CUDA(b, cudaMemcpyAsync(h_best, d_best, (size_t)nprob * 3 * 8, cudaMemcpyDeviceToHost, b->stream));
      CLP_CUDA(b, cudaMemcpyAsync(h_flags, d_flags, (size_t)nprob * 8, cudaMemcpyDeviceToHost, b->stream));
      b->last_scratch += (long long)ss.nworkers * (long long)ss.stride;
    }
  }
  CLP_CUDA(b, cudaMemcpyAsync(h_v, b->mc_vint.p, (size_t)nv * 4, cudaMemcpyDeviceToHost, b->stream));
  CLP_CUDA(b, cudaStreamSynchronize(b->stream));
  if (total > 0) search_ms = mc_elapsed(ev.e[2], ev.e[3]);

  // ---- results per problem
  const float phase_a_ms = mc_elapsed(ev.e[0], ev.e[1]);
  double ns_sum[3] = {0.0, 0.0, 0.0};
  for (const McBatchOut& o : outs) for (int q = 0; q < 3; ++q) ns_sum[q] += (double)o.ns[q];
  const double ns_all = ns_sum[0] + ns_sum[1] + ns_sum[2];
  double split[3] = {0.0, 0.0, 0.0};
  for (int q = 0; q < 3; ++q) split[q] = ns_all > 0 ? phase_a_ms * ns_sum[q] / ns_all : 0.0;
  std::vector<int32_t> nodes;
  for (int p = 0; p < nprob; ++p) {
    const McBatchProblem& q = probs[(size_t)p];
    const McBatchOut& o = outs[(size_t)p];
    const int m = q.sp.m;
    const int* core = h_v + q.v_off;
    const int* vnodes = core + 3 * m;
    int lb = 0, proven = 0, timed_out = 0;
    long long branches = 0;
    nodes.clear();
    if (method == CLP_MC_KCORE) {
      for (int v = 0; v < m; ++v) if (core[v] >= o.max_core) nodes.push_back(v);
    } else {
      lb = o.lb;
      int size = vnodes[m];  // the heuristic's replay, or the search's when it beat the heuristic
      proven = (lb == o.max_core + 1) ? 1 : 0;
      if (search && lb < o.max_core + 1) {
        proven = 1;
        if (o.ntasks > 0) {
          const int s = (int)(h_best[p] >> 32);
          branches = (long long)h_br[p];
          timed_out = h_done[p] < (unsigned long long)o.ntasks ? 1 : 0;
          proven = (!timed_out && h_flags[2 * p + 1] == 0) ? 1 : 0;
          if (s > lb && (size < s || size > m))
            return fail(b, CLP_ERR_CUDA, "batched maximum clique: search replay did not reproduce its clique (problem " + std::to_string(p) + ")");
          if (s <= lb && size != lb) return fail(b, CLP_ERR_CUDA, "batched maximum clique: heuristic replay disagrees with its winner");
        } else if (size != lb) {
          return fail(b, CLP_ERR_CUDA, "batched maximum clique: heuristic replay disagrees with its winner");
        }
      } else if (size != lb) {
        return fail(b, CLP_ERR_CUDA, "batched maximum clique: heuristic replay disagrees with its winner");
      }
      nodes.assign(vnodes, vnodes + size);
      std::sort(nodes.begin(), nodes.end());
    }
    if (nodes_out && nodes_out[p] && !nodes.empty()) std::memcpy(nodes_out[p], nodes.data(), nodes.size() * sizeof(int32_t));
    if (core_out && core_out[p]) std::memcpy(core_out[p], core, (size_t)m * sizeof(int32_t));
    clp_mc_info& info = infos[p];
    std::memset(&info, 0, sizeof(info));
    info.n_nodes = (int32_t)nodes.size();
    info.max_core = o.max_core;
    info.lower_bound = lb;
    info.upper_bound = o.max_core + 1;
    info.proven = proven;
    info.timed_out = timed_out;
    info.n_edges = (int64_t)o.n_edges;
    info.n_branches = branches;
    info.adjacency_ms = split[0]; info.peel_ms = split[1]; info.heuristic_ms = split[2]; info.search_ms = search_ms;
    info.kernel_ms = phase_a_ms + search_ms;
  }
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  for (int p = 0; p < nprob; ++p) infos[p].t = wall / nprob;
  return CLP_OK;
}

// ---- points and associations on the device (clp_batch_*_dev) -----------------------------------------------------
// The checks these calls make before those of their host twins (CLP_ERR_INVALID): pointers, strides and sizes of pts,
// every problem's association count (*max_m: the largest).  Then in is set up for batch_solve / batch_max_clique.
int points_dev_check(clp_batch b, int32_t nprob, const clp_points_dev* pts, BatchInput& in, long long* max_m) {
  if (!b) return CLP_ERR_INVALID;
  if (nprob <= 0 || !pts || !pts->D1 || !pts->D2 || !pts->n1 || !pts->n2 || !pts->m) return fail(b, CLP_ERR_INVALID, "bad batch arguments");
  auto strides_ok = [](const int64_t* s) { return s[0] >= 0 && s[1] >= 1 && s[2] >= 1; };
  if (!strides_ok(pts->d1_strides) || !strides_ok(pts->d2_strides) || (pts->A && !strides_ok(pts->a_strides)))
    return fail(b, CLP_ERR_INVALID, "bad strides (coordinate, point, row and column strides must be >= 1, batch strides >= 0)");
  *max_m = 1;
  for (int p = 0; p < nprob; ++p) {
    const std::string tag = "problem " + std::to_string(p) + ": ";
    const int64_t n1 = pts->n1[p], n2 = pts->n2[p], m = pts->m[p];
    if (n1 < 1 || n2 < 1 || n1 > INT32_MAX || n2 > INT32_MAX || m < 0)
      return fail(b, CLP_ERR_INVALID, tag + "bad sizes (n1, n2 >= 1, m >= 0)");
    const long long mp = (!pts->A || m == 0) ? (long long)n1 * n2 : (long long)m;
    if (mp > kBatchMaxM) return fail(b, CLP_ERR_INVALID, tag + "batched problems need 1 <= m <= 4096 associations");
    *max_m = std::max(*max_m, mp);
  }
  in.dev = pts; in.n1 = pts->n1; in.n2 = pts->n2; in.m = pts->m;
  return CLP_OK;
}

// the solves' device u0 and u: u0_dev + p u0_stride (u0_stride >= 1), u_out_dev + p u_out_stride (nullable,
// u_out_stride >= the largest m)
int solve_dev_check(clp_batch b, int32_t nprob, const clp_points_dev* pts, const double* u0_dev, int64_t u0_stride,
                    double* u_out_dev, int64_t u_out_stride, BatchInput& in) {
  long long max_m = 0;
  if (int rc = points_dev_check(b, nprob, pts, in, &max_m)) return rc;
  if (!u0_dev) return fail(b, CLP_ERR_INVALID, "null u0");
  if (u0_stride < 1 || (u_out_dev && u_out_stride < max_m))
    return fail(b, CLP_ERR_INVALID, "bad strides (u0_stride >= 1; u_out_stride >= the largest m)");
  in.u0_dev = u0_dev; in.u0_stride = u0_stride; in.u_out_dev = u_out_dev; in.u_out_stride = u_out_stride;
  return CLP_OK;
}

// ---- putative associations for a batch of cloud pairs (clp_knn.cuh) -------------------------------------------------
template <int D, int K>
cudaError_t knn_batch_partial(dim3 grid, size_t smem, cudaStream_t s, const KnnBatchArgs& a) {
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(knn_batch_partial_kernel<D, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  knn_batch_partial_kernel<D, K><<<grid, kKnnThreads, smem, s>>>(a);
  return cudaGetLastError();
}

template <int D>
cudaError_t knn_batch_partial_k(int K, dim3 grid, size_t smem, cudaStream_t s, const KnnBatchArgs& a) {
  switch (K) {
    case 1: return knn_batch_partial<D, 1>(grid, smem, s, a);
    case 2: return knn_batch_partial<D, 2>(grid, smem, s, a);
    case 4: return knn_batch_partial<D, 4>(grid, smem, s, a);
    case 8: return knn_batch_partial<D, 8>(grid, smem, s, a);
    case 16: return knn_batch_partial<D, 16>(grid, smem, s, a);
    default: return knn_batch_partial<D, 32>(grid, smem, s, a);
  }
}

cudaError_t knn_batch_merge(int K, unsigned blocks, cudaStream_t s, const KnnBatchArgs& a) {
  switch (K) {
    case 1: knn_batch_merge_kernel<1><<<blocks, kKnnThreads, 0, s>>>(a); break;
    case 2: knn_batch_merge_kernel<2><<<blocks, kKnnThreads, 0, s>>>(a); break;
    case 4: knn_batch_merge_kernel<4><<<blocks, kKnnThreads, 0, s>>>(a); break;
    case 8: knn_batch_merge_kernel<8><<<blocks, kKnnThreads, 0, s>>>(a); break;
    case 16: knn_batch_merge_kernel<16><<<blocks, kKnnThreads, 0, s>>>(a); break;
    default: knn_batch_merge_kernel<32><<<blocks, kKnnThreads, 0, s>>>(a); break;
  }
  return cudaGetLastError();
}

// The clouds and outputs of clp_batch_correspondences(_dev): host arrays of nprob pointers (D1h, D2h, A_out; A_out[p]
// filled with leading dimension m[p]) or device tensors in element strides (D1, D2, A_dev).
struct KnnBatchIn {
  const double* const* D1h = nullptr; const double* const* D2h = nullptr; int32_t* const* A_out = nullptr;
  const double* D1 = nullptr; const int64_t* s1 = nullptr;
  const double* D2 = nullptr; const int64_t* s2 = nullptr;
  int32_t* A_dev = nullptr; const int64_t* sa = nullptr;
};

// clp_batch_correspondences(_dev).  Everything is checked on the host first; the device work is one upload (the table,
// and the clouds of the host call), one staging launch (device call), the launches of clp_knn.cuh's batch section and
// one readback of the counts.  Nothing of the batch but knn_buf, knn_pinned, its stream and its error string is touched.
int batch_correspondences(clp_batch b, bool on_device, int32_t nprob, int32_t d, const KnnBatchIn& in, const int64_t* n1,
                          const int64_t* n2, int32_t knn, double radius, int enforce_1to1, int64_t capacity, int64_t* m_out) {
  if (!b) return CLP_ERR_INVALID;
  const std::string who = "batch correspondences: ";
  auto tag = [&](int p) { return who + "problem " + std::to_string(p) + ": "; };
  if (!m_out || !n1 || !n2) return fail(b, CLP_ERR_INVALID, who + "n1, n2 and m are required");
  if (nprob < 1) return fail(b, CLP_ERR_INVALID, who + "nprob must be >= 1");
  std::fill(m_out, m_out + nprob, (int64_t)0);
  if (on_device ? (!in.s1 || !in.s2 || !in.sa) : (!in.D1h || !in.D2h || !in.A_out))
    return fail(b, CLP_ERR_INVALID, who + "NULL pointer arrays or strides");
  if (knn < 1) return fail(b, CLP_ERR_INVALID, who + "knn must be >= 1");
  if (d < 1) return fail(b, CLP_ERR_INVALID, who + "d must be >= 1");
  for (int p = 0; p < nprob; ++p) {
    if (n1[p] < 0 || n2[p] < 0) return fail(b, CLP_ERR_INVALID, tag(p) + "negative n1 or n2");
    if ((n1[p] > 0 && !(on_device ? in.D1 : in.D1h[p])) || (n2[p] > 0 && !(on_device ? in.D2 : in.D2h[p])))
      return fail(b, CLP_ERR_INVALID, tag(p) + "NULL point cloud");
  }
  if (on_device) {
    auto ok = [](const int64_t* s) { return s[0] >= 0 && s[1] >= 1 && s[2] >= 1; };
    if (!ok(in.s1) || !ok(in.s2) || !ok(in.sa))
      return fail(b, CLP_ERR_INVALID, who + "bad strides (coordinate, point, row and column strides must be >= 1, batch "
                                            "strides >= 0)");
  }
  if (knn > kKnnMaxK)
    return fail(b, CLP_ERR_UNSUPPORTED, who + "knn = " + std::to_string(knn) + " exceeds CLP_KNN_MAX_K = " + std::to_string(kKnnMaxK));
  if (d > kKnnMaxD)
    return fail(b, CLP_ERR_UNSUPPORTED, who + "d = " + std::to_string(d) + " exceeds CLP_KNN_MAX_D = " + std::to_string(kKnnMaxD));
  for (int p = 0; p < nprob; ++p)
    if (n1[p] >= kKnnNone || n2[p] >= kKnnNone)
      return fail(b, CLP_ERR_UNSUPPORTED, tag(p) + "n1 and n2 must be below 2^31 - 1 (int32 indices)");
  for (int p = 0; p < nprob; ++p) {
    const long long rows = (long long)n1[p] * std::min<int64_t>(knn, n2[p]);
    if (capacity < rows || (rows > 0 && (on_device ? !in.A_dev : !in.A_out[p])))
      return fail(b, CLP_ERR_INVALID, tag(p) + "A holds " + std::to_string(capacity) + " rows, n1 * min(knn, n2) = " +
                                          std::to_string(rows) + " are required");
  }
  // the plan: a problem without rows (n1 = 0 or n2 = 0) takes no queries and no candidates
  const int D = d <= 3 ? d : 0;
  const int T = D > 0 ? kKnnTileReg : kKnnTileGen;
  std::vector<KnnProb> tab((size_t)nprob);
  long long nq = 0, nc = 0, ctas = 0, lsz = 0, rows_all = 0, max_nc = 0, most = 1;
  int kmax = 1;
  for (int p = 0; p < nprob; ++p) {
    KnnProb& P = tab[(size_t)p];
    std::memset(&P, 0, sizeof(P));
    const int kk = (int)std::min<int64_t>(knn, n2[p]);
    const bool live = (long long)n1[p] * kk > 0;
    P.bp.n1 = live ? (int)n1[p] : 0; P.bp.n2 = live ? (int)n2[p] : 0; P.kk = live ? kk : 0;
    P.bp.d1_off = (long long)d * nq; P.bp.d2_off = (long long)d * nc; P.bp.a_off = -1;
    P.q_off = nq; P.c_off = nc; P.cta0 = ctas; P.m_off = lsz;
    nq += P.bp.n1; nc += P.bp.n2; ctas += (P.bp.n1 + kKnnThreads - 1) / kKnnThreads; lsz += (long long)P.kk * P.bp.n1;
    rows_all += (long long)P.kk * P.bp.n1;
    max_nc = std::max<long long>(max_nc, P.bp.n2);
    most = std::max<long long>(most, (long long)d * std::max(P.bp.n1, P.bp.n2));
    kmax = std::max(kmax, P.kk);
  }
  if (rows_all == 0) return CLP_OK;
  // candidate slices, as the single call cuts them but for the whole batch's query CTAs; bounds relative to each n2
  const long long want = (4LL * b->sm_count + ctas - 1) / ctas;
  const int nsplit = (int)std::max<long long>(1, std::min<long long>({want, (max_nc + 1023) / 1024, 1024}));
  for (KnnProb& P : tab) {
    P.chunk = round_up((P.bp.n2 + nsplit - 1) / nsplit, T);
    P.l_off = (long long)nsplit * P.m_off;
  }
  int K = 1;
  while (K < kmax) K *= 2;
  // scratch layout, every region 256-byte aligned; the prefix table | d1 | d2 is uploaded from knn_pinned as it lies
  const long long nscan = std::max(nq, nc), nb = (nscan + kKnnScanItems - 1) / kKnnScanItems;
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t o = at; at = (at + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_tab = take((size_t)nprob * sizeof(KnnProb));
  const size_t o_d1 = take((size_t)d * nq * 8), o_d2 = take((size_t)d * nc * 8);
  const size_t up = on_device ? (size_t)nprob * sizeof(KnnProb) : o_d2 + (size_t)d * nc * 8;
  const size_t o_psd = take((size_t)nsplit * lsz * 8), o_pj = take((size_t)nsplit * lsz * 4);
  const size_t o_lsd = nsplit > 1 ? take((size_t)lsz * 8) : o_psd, o_lj = nsplit > 1 ? take((size_t)lsz * 4) : o_pj;
  const size_t o_cnt = take((size_t)nscan * 4), o_off = take((size_t)nscan * 8), o_bsum = take((size_t)nb * 8), o_tot = take(8);
  const size_t o_m = take((size_t)nprob * 8), o_rb = take((size_t)nprob * 8);
  const size_t o_best = enforce_1to1 ? take((size_t)nc * 8) : 0, o_c0 = enforce_1to1 ? take((size_t)nc * 4) : 0;
  const size_t o_a = on_device ? 0 : take((size_t)2 * rows_all * 4);
  CLP_CUDA(b, cudaSetDevice(b->device));
  if (at > b->knn_buf.cap) {
    size_t free_b = 0, total_b = 0;
    CLP_CUDA(b, cudaMemGetInfo(&free_b, &total_b));
    if (at > free_b + b->knn_buf.cap)
      return fail(b, CLP_ERR_ALLOC, who + "the scratch (" + std::to_string(at) + " bytes) does not fit the free device memory (" +
                                        std::to_string(free_b + b->knn_buf.cap) + " bytes)");
  }
  CLP_CUDA(b, b->knn_buf.ensure(at));
  const size_t o_hm = (up + 255) & ~(size_t)255;  // the counts come back here
  CLP_CUDA(b, b->knn_pinned.ensure(o_hm + (size_t)nprob * 8));
  char* hp = b->knn_pinned.as<char>();
  std::memcpy(hp + o_tab, tab.data(), (size_t)nprob * sizeof(KnnProb));
  if (!on_device)
    for (int p = 0; p < nprob; ++p) {
      const KnnProb& P = tab[(size_t)p];
      if (P.bp.n1) std::memcpy(hp + o_d1 + (size_t)P.bp.d1_off * 8, in.D1h[p], (size_t)d * P.bp.n1 * 8);
      if (P.bp.n2) std::memcpy(hp + o_d2 + (size_t)P.bp.d2_off * 8, in.D2h[p], (size_t)d * P.bp.n2 * 8);
    }
  const cudaStream_t st = b->stream;
  char* base = b->knn_buf.as<char>();
  CLP_CUDA(b, cudaMemcpyAsync(base, hp, up, cudaMemcpyHostToDevice, st));
  KnnBatchArgs a;
  std::memset(&a, 0, sizeof(a));
  a.prob = reinterpret_cast<const KnnProb*>(base + o_tab); a.nprob = nprob; a.d = d; a.nsplit = nsplit;
  a.D1 = reinterpret_cast<const double*>(base + o_d1); a.D2 = reinterpret_cast<const double*>(base + o_d2);
  a.part_sd = reinterpret_cast<double*>(base + o_psd); a.part_j = reinterpret_cast<int*>(base + o_pj);
  a.lsd = reinterpret_cast<double*>(base + o_lsd); a.lj = reinterpret_cast<int*>(base + o_lj);
  a.r2 = radius * radius;  // bm_utils.cpp:192: NaN keeps nothing, inf keeps every neighbour
  a.cnt = reinterpret_cast<int*>(base + o_cnt); a.off = reinterpret_cast<long long*>(base + o_off);
  a.bsum = reinterpret_cast<long long*>(base + o_bsum); a.total = reinterpret_cast<long long*>(base + o_tot);
  a.mcount = reinterpret_cast<long long*>(base + o_m); a.rbase = reinterpret_cast<long long*>(base + o_rb);
  a.best = reinterpret_cast<unsigned long long*>(base + o_best); a.c0best = reinterpret_cast<unsigned int*>(base + o_c0);
  if (on_device) {
    a.A = in.A_dev;
    for (int k = 0; k < 3; ++k) a.as[k] = in.sa[k];
    BatchStageArgs g;
    std::memset(&g, 0, sizeof(g));
    g.prob = reinterpret_cast<const unsigned char*>(base + o_tab); g.prob_stride = sizeof(KnnProb);
    g.nprob = nprob; g.dd = d;
    g.D1 = in.D1; g.D2 = in.D2;
    for (int k = 0; k < 3; ++k) { g.s1[k] = in.s1[k]; g.s2[k] = in.s2[k]; }
    g.d1 = reinterpret_cast<double*>(base + o_d1); g.d2 = reinterpret_cast<double*>(base + o_d2);
    g.bad = &b->sync.as<SyncBlock>()->counts[1];  // never written: the table holds no associations
    const dim3 grid((unsigned)std::min<long long>(64, (most + kBatchThreads - 1) / kBatchThreads), (unsigned)std::min(nprob, 65535));
    batch_stage_points_kernel<<<grid, kBatchThreads, 0, st>>>(g);
    CLP_CUDA(b, cudaGetLastError());
  } else {
    a.A = reinterpret_cast<int*>(base + o_a);
    a.packed = 1;
  }
  const dim3 pgrid((unsigned)ctas, (unsigned)nsplit);
  const size_t smem = knn_partial_smem(D, d);
  cudaError_t e;
  switch (D) {
    case 1: e = knn_batch_partial_k<1>(K, pgrid, smem, st, a); break;
    case 2: e = knn_batch_partial_k<2>(K, pgrid, smem, st, a); break;
    case 3: e = knn_batch_partial_k<3>(K, pgrid, smem, st, a); break;
    default: e = knn_batch_partial_k<0>(K, pgrid, smem, st, a); break;
  }
  CLP_CUDA(b, e);
  CLP_CUDA(b, knn_batch_merge(K, (unsigned)ctas, st, a));
  const unsigned bp = (unsigned)((nprob + 255) / 256);
  if (!enforce_1to1) {
    a.nscan = nq;
    knn_scan_blocks_kernel<<<(unsigned)((nq + kKnnScanItems - 1) / kKnnScanItems), 256, 0, st>>>(a.cnt, nq, a.off, a.bsum);
    knn_scan_top_kernel<<<1, 1024, 0, st>>>(a.bsum, (nq + kKnnScanItems - 1) / kKnnScanItems, a.total);
    knn_batch_rows_kernel<<<bp, 256, 0, st>>>(a, 0);
    knn_batch_write_kernel<<<(unsigned)ctas, kKnnThreads, 0, st>>>(a);
  } else {
    CLP_CUDA(b, cudaMemsetAsync(a.best, 0xff, (size_t)nc * 8, st));
    CLP_CUDA(b, cudaMemsetAsync(a.c0best, 0xff, (size_t)nc * 4, st));
    knn_batch_best_sd_kernel<<<(unsigned)ctas, kKnnThreads, 0, st>>>(a);
    knn_batch_best_c0_kernel<<<(unsigned)ctas, kKnnThreads, 0, st>>>(a);
    const unsigned b2 = (unsigned)((nc + 255) / 256);
    knn_flag_kernel<<<b2, 256, 0, st>>>(a.c0best, nc, a.cnt);
    a.nscan = nc;
    knn_scan_blocks_kernel<<<(unsigned)((nc + kKnnScanItems - 1) / kKnnScanItems), 256, 0, st>>>(a.cnt, nc, a.off, a.bsum);
    knn_scan_top_kernel<<<1, 1024, 0, st>>>(a.bsum, (nc + kKnnScanItems - 1) / kKnnScanItems, a.total);
    knn_batch_rows_kernel<<<bp, 256, 0, st>>>(a, 1);
    knn_batch_write_1to1_kernel<<<b2, 256, 0, st>>>(a);
  }
  CLP_CUDA(b, cudaGetLastError());
  long long* h_m = reinterpret_cast<long long*>(hp + o_hm);
  CLP_CUDA(b, cudaMemcpyAsync(h_m, a.mcount, (size_t)nprob * 8, cudaMemcpyDeviceToHost, st));
  CLP_CUDA(b, cudaStreamSynchronize(st));
  const std::vector<long long> ms(h_m, h_m + nprob);
  long long M = 0;
  for (long long x : ms) M += x;
  if (!on_device && M > 0) {  // the staged rows of problem p start at 2 (m[0] + .. + m[p - 1])
    CLP_CUDA(b, b->knn_pinned.ensure((size_t)2 * M * 4));
    int32_t* h_a = b->knn_pinned.as<int32_t>();
    CLP_CUDA(b, cudaMemcpyAsync(h_a, a.A, (size_t)2 * M * 4, cudaMemcpyDeviceToHost, st));
    CLP_CUDA(b, cudaStreamSynchronize(st));
    long long r0 = 0;
    for (int p = 0; p < nprob; ++p) {
      if (ms[(size_t)p] > 0) std::memcpy(in.A_out[p], h_a + 2 * r0, (size_t)2 * ms[(size_t)p] * 4);
      r0 += ms[(size_t)p];
    }
  }
  std::copy(ms.begin(), ms.end(), m_out);
  return CLP_OK;
}

// ---- rigid transform of selected associations (clp_transform.cuh) -------------------------------------------------
// The inputs of the four clp_*estimate_transform* entries; a single call is a batch of one.  Host inputs: D1h, D2h, Ah
// (column-major m x 2, NULL or m = 0: all-to-all) per problem; device inputs: pts (clp_points_dev).  rows and k are
// host arrays.  Outputs: T_out[p] on the host (column-major), or T_dev at element strides ts.
struct TfIn {
  const double* const* D1h = nullptr; const double* const* D2h = nullptr; const int32_t* const* Ah = nullptr;
  const int64_t* n1 = nullptr; const int64_t* n2 = nullptr; const int64_t* m = nullptr;
  const clp_points_dev* pts = nullptr;
  const int32_t* const* rows = nullptr; const int64_t* k = nullptr;
  double* const* T_out = nullptr;
  double* T_dev = nullptr; const int64_t* ts = nullptr;
};

// One host path for the handle (H = clp_handle_s) and the batch (clp_batch_s): only o's device, stream, events and error
// string are used, and the transform's own scratch (buf, pin).  Everything is checked on the host first; the device
// work is one upload (the pairs gathered on the host, or the rows for the device gather), a gather launch (device
// inputs), the estimate launch and one readback.
template <typename H>
int estimate_transform(H* o, DevBuf& buf, PinnedBuf& pin, int32_t nprob, int32_t d, const TfIn& in, clp_tf_info* infos) {
  const auto t_begin = std::chrono::steady_clock::now();
  const bool dev = in.pts != nullptr;
  const std::string who = "estimate transform: ";
  auto tag = [&](int p) { return who + "problem " + std::to_string(p) + ": "; };
  if (!infos || !in.n1 || !in.n2 || !in.k || nprob < 1)
    return fail(o, CLP_ERR_INVALID, who + "n1, n2, k and infos are required, and nprob >= 1");
  if (dev ? (!in.T_dev || !in.ts) : (!in.D1h || !in.D2h || !in.T_out))
    return fail(o, CLP_ERR_INVALID, who + "NULL pointer arrays or output");
  if (d < 1) return fail(o, CLP_ERR_INVALID, who + "d must be >= 1");
  if (dev) {
    auto ok = [](const int64_t* s) { return s[0] >= 0 && s[1] >= 1 && s[2] >= 1; };
    if (!ok(in.pts->d1_strides) || !ok(in.pts->d2_strides) || (in.pts->A && !ok(in.pts->a_strides)) || !ok(in.ts))
      return fail(o, CLP_ERR_INVALID, who + "bad strides (coordinate, point, row and column strides must be >= 1, batch "
                                            "strides >= 0)");
  }
  // the problem table: sizes, rows and, for host inputs, every used association index
  std::vector<TfProb> tab((size_t)nprob);
  long long npairs = 0, nrows = 0, most = 1;
  for (int p = 0; p < nprob; ++p) {
    TfProb& P = tab[(size_t)p];
    const int64_t n1 = in.n1[p], n2 = in.n2[p], m = in.m ? in.m[p] : 0;
    if (n1 < 0 || n2 < 0 || m < 0) return fail(o, CLP_ERR_INVALID, tag(p) + "negative n1, n2 or m");
    const double* D1 = dev ? in.pts->D1 : in.D1h[p];
    const double* D2 = dev ? in.pts->D2 : in.D2h[p];
    if ((n1 > 0 && !D1) || (n2 > 0 && !D2)) return fail(o, CLP_ERR_INVALID, tag(p) + "NULL point cloud");
    if (!dev && !in.T_out[p]) return fail(o, CLP_ERR_INVALID, tag(p) + "NULL T_out");
    const int32_t* A = dev ? in.pts->A : (in.Ah ? in.Ah[p] : nullptr);
    const bool a2a = !A || m == 0;
    const long long rows_of = a2a ? (long long)n1 * n2 : (long long)m;
    const int32_t* rows = in.rows ? in.rows[p] : nullptr;
    if (rows && in.k[p] < 0) return fail(o, CLP_ERR_INVALID, tag(p) + "k must be >= 0");
    const long long k = rows ? (long long)in.k[p] : rows_of;
    for (long long i = 0; i < ((rows || (!a2a && !dev)) ? k : 0); ++i) {  // every row 0 .. k-1 is in range
      const long long r = rows ? (long long)rows[i] : i;
      if (r < 0 || r >= rows_of)
        return fail(o, CLP_ERR_INVALID, tag(p) + "row " + std::to_string(r) + " outside [0, " + std::to_string(rows_of) + ")");
      if (!a2a && !dev && (A[r] < 0 || A[r] >= n1 || A[m + r] < 0 || A[m + r] >= n2))
        return fail(o, CLP_ERR_INVALID, tag(p) + "association index out of range of D1/D2");
    }
    P.off = npairs; P.k = k; P.rows_off = (dev && rows) ? nrows : -1;
    P.n1 = n1; P.n2 = n2; P.m = a2a ? 0 : m;
    npairs += 2LL * d * k;
    if (dev && rows) nrows += k;
    most = std::max(most, k);
  }
  if (d != 2 && d != 3) return fail(o, CLP_ERR_UNSUPPORTED, who + "d = " + std::to_string(d) + ", only 2 and 3 are supported");
  // scratch, every region 256-byte aligned; bad key | table | rows | pairs (host inputs) go up from pin as they lie
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t q = at; at = (at + bytes + 255) & ~(size_t)255; return q; };
  const size_t o_bad = take(8), o_tab = take((size_t)nprob * sizeof(TfProb)), o_rows = take((size_t)nrows * 4);
  const size_t o_pairs = take((size_t)npairs * 8);
  const size_t up = dev ? o_pairs : at;
  const size_t o_out = take((size_t)nprob * sizeof(TfOut));
  CLP_CUDA(o, cudaSetDevice(o->device));
  if (at > buf.cap) {
    size_t free_b = 0, total_b = 0;
    CLP_CUDA(o, cudaMemGetInfo(&free_b, &total_b));
    if (at > free_b + buf.cap)
      return fail(o, CLP_ERR_ALLOC, who + "the scratch (" + std::to_string(at) + " bytes) does not fit the free device memory (" +
                                        std::to_string(free_b + buf.cap) + " bytes)");
  }
  CLP_CUDA(o, buf.ensure(at));
  CLP_CUDA(o, pin.ensure(std::max(up, (size_t)nprob * sizeof(TfOut) + 256)));
  char* hp = pin.as<char>();
  std::memset(hp + o_bad, 0, 8);
  std::memcpy(hp + o_tab, tab.data(), (size_t)nprob * sizeof(TfProb));
  for (int p = 0; p < nprob; ++p) {
    const TfProb& P = tab[(size_t)p];
    const int32_t* rows = in.rows ? in.rows[p] : nullptr;
    if (dev) {
      if (P.rows_off >= 0 && P.k > 0) std::memcpy(hp + o_rows + (size_t)P.rows_off * 4, rows, (size_t)P.k * 4);
      continue;
    }
    double* q = reinterpret_cast<double*>(hp + o_pairs) + P.off;
    const double* D1 = in.D1h[p];
    const double* D2 = in.D2h[p];
    const int32_t* A = in.Ah ? in.Ah[p] : nullptr;
    for (long long i = 0; i < P.k; ++i) {
      const long long r = rows ? (long long)rows[i] : i;
      const long long i1 = P.m == 0 ? r / P.n2 : A[r], i2 = P.m == 0 ? r % P.n2 : A[P.m + r];
      for (int c = 0; c < d; ++c) {
        q[c * P.k + i] = D1[i1 * d + c];
        q[(d + c) * P.k + i] = D2[i2 * d + c];
      }
    }
  }
  const cudaStream_t st = o->stream;
  char* base = buf.as<char>();
  CLP_CUDA(o, cudaMemcpyAsync(base, hp, up, cudaMemcpyHostToDevice, st));
  unsigned long long* bad = reinterpret_cast<unsigned long long*>(base + o_bad);
  const TfProb* dtab = reinterpret_cast<const TfProb*>(base + o_tab);
  double* pairs = reinterpret_cast<double*>(base + o_pairs);
  TfOut* outs = reinterpret_cast<TfOut*>(base + o_out);
  CLP_CUDA(o, cudaEventRecord(o->ev0, st));
  if (dev) {
    const clp_points_dev& s = *in.pts;
    TfGatherArgs g;
    std::memset(&g, 0, sizeof(g));
    g.prob = dtab; g.nprob = nprob; g.d = d;
    g.D1 = s.D1; g.D2 = s.D2; g.A = s.A;
    for (int c = 0; c < 3; ++c) { g.s1[c] = s.d1_strides[c]; g.s2[c] = s.d2_strides[c]; g.sa[c] = s.a_strides[c]; }
    g.rows = reinterpret_cast<const int*>(base + o_rows); g.pairs = pairs; g.bad = bad;
    const dim3 grid((unsigned)std::min<long long>(64, (most + kTfThreads - 1) / kTfThreads), (unsigned)std::min(nprob, 65535));
    tf_gather_kernel<<<grid, kTfThreads, 0, st>>>(g);
    CLP_CUDA(o, cudaGetLastError());
  }
  TfEstimateArgs e;
  std::memset(&e, 0, sizeof(e));
  e.prob = dtab; e.nprob = nprob; e.pairs = pairs; e.out = outs; e.bad = bad;
  if (dev) { e.T_dev = in.T_dev; for (int c = 0; c < 3; ++c) e.ts[c] = in.ts[c]; }
  const unsigned grid = (unsigned)std::min(nprob, 1 << 20);
  if (d == 2) tf_estimate_kernel<2><<<grid, kTfThreads, 0, st>>>(e);
  else tf_estimate_kernel<3><<<grid, kTfThreads, 0, st>>>(e);
  CLP_CUDA(o, cudaGetLastError());
  CLP_CUDA(o, cudaEventRecord(o->ev1, st));
  unsigned long long* h_bad = reinterpret_cast<unsigned long long*>(hp);
  TfOut* h_out = reinterpret_cast<TfOut*>(hp + 256);
  CLP_CUDA(o, cudaMemcpyAsync(h_bad, bad, 8, cudaMemcpyDeviceToHost, st));
  CLP_CUDA(o, cudaMemcpyAsync(h_out, outs, (size_t)nprob * sizeof(TfOut), cudaMemcpyDeviceToHost, st));
  CLP_CUDA(o, cudaStreamSynchronize(st));
  if (const unsigned long long key = *h_bad)
    return fail(o, CLP_ERR_INVALID, tag((int)(0xffffffffu - (unsigned int)(key & 0xffffffffu))) +
                                        "association index out of range of D1/D2");
  float ms = 0.f;
  CLP_CUDA(o, cudaEventElapsedTime(&ms, o->ev0, o->ev1));
  const double t = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count() / nprob;
  const int E = d + 1;
  for (int p = 0; p < nprob; ++p) {
    const TfOut& r = h_out[p];
    clp_tf_info& f = infos[p];
    std::memset(&f, 0, sizeof(f));
    f.status = r.status; f.k = tab[(size_t)p].k; f.rmse = r.rmse;
    f.sv[0] = r.sv[0]; f.sv[1] = r.sv[1]; f.sv[2] = r.sv[2]; f.gap = r.gap;
    f.t = t; f.kernel_ms = ms;
    if (!dev) std::memcpy(in.T_out[p], r.T, (size_t)E * E * 8);
  }
  return CLP_OK;
}
}  // namespace

extern "C" {

int clp_batch_create(int device, clp_batch* out) {
  if (!out) return CLP_ERR_INVALID;
  *out = nullptr;
  cudaDeviceProp prop;
  if (int rc = probe_device<clp_batch_s>(device, &prop)) return rc;
  clp_batch b = new (std::nothrow) clp_batch_s();
  if (!b) return fail<clp_batch_s>(nullptr, CLP_ERR_ALLOC, "host allocation failed");
  b->device = device; b->sm_count = prop.multiProcessorCount;
  clp_default_params(&b->prm);
  auto bail = [&](const char* what, cudaError_t ce) {
    clp_batch_destroy(b);
    return fail<clp_batch_s>(nullptr, CLP_ERR_CUDA, std::string(what) + ": " + cudaGetErrorString(ce));
  };
  cudaError_t e;
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  if ((e = cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaEventCreate(&b->ev0)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaEventCreate(&b->ev1)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaEventCreate(&b->ev_up)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = b->sync.ensure(sizeof(SyncBlock))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaDeviceGetAttribute(&b->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device)) != cudaSuccess) return bail("cudaDeviceGetAttribute", e);
  *out = b;
  return CLP_OK;
}

int clp_batch_destroy(clp_batch b) {
  if (!b) return CLP_OK;
  cudaSetDevice(b->device);
  for (DevBuf* d : {&b->in_d1, &b->in_d2, &b->in_a, &b->in_u0, &b->out_u, &b->probs, &b->outs, &b->nnz, &b->sync, &b->scratch, &b->prof, &b->mat_in, &b->custom_in,
                    &b->mc_probs, &b->mc_edges, &b->mc_adj, &b->mc_vint, &b->mc_tpre, &b->mc_out, &b->mc_state, &b->mc_rounds,
                    &b->mc_pscratch, &b->mc_sscratch, &b->sdp_out, &b->knn_buf, &b->tf_buf})
    d->release();
  b->pinned.release();
  b->tf_pinned.release();
  b->knn_pinned.release();
  b->pinned_points.release();
  if (b->ev0) cudaEventDestroy(b->ev0);
  if (b->ev1) cudaEventDestroy(b->ev1);
  if (b->ev_up) cudaEventDestroy(b->ev_up);
  if (b->stream && b->own_stream) cudaStreamDestroy(b->stream);
  delete b;
  return CLP_OK;
}

const char* clp_batch_last_error(clp_batch b) { return b ? b->err.c_str() : create_error<clp_batch_s>().c_str(); }

int clp_batch_set_params(clp_batch b, const clp_params* p) {
  if (!b || !p) return CLP_ERR_INVALID;
  if (p->rounding < 0 || p->rounding > 2) return fail(b, CLP_ERR_INVALID, "unknown rounding mode");
  b->prm = *p;
  return CLP_OK;
}

int clp_batch_solve_euclidean(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                              const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                              const double* const* u0, double sigma, double epsilon, double mindist,
                              clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  BatchInput in;
  in.D1 = D1; in.n1 = n1; in.D2 = D2; in.n2 = n2; in.A = A; in.m = m;
  in.p[0] = sigma; in.p[1] = epsilon; in.p[2] = mindist;
  return guarded(b, [&] { return batch_solve(b, 0, d, nprob, in, u0, sols, u_out, nodes_out); });
}

int clp_batch_solve_pointnormal(clp_batch b, int32_t nprob, const double* const* D1, const int64_t* n1,
                                const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                const double* const* u0, double sigp, double epsp, double sign, double epsn,
                                clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  BatchInput in;
  in.D1 = D1; in.n1 = n1; in.D2 = D2; in.n2 = n2; in.A = A; in.m = m;
  in.p[0] = sigp; in.p[1] = epsp; in.p[2] = sign; in.p[3] = epsn;
  return guarded(b, [&] { return batch_solve(b, 1, 6, nprob, in, u0, sols, u_out, nodes_out); });
}

int clp_batch_solve_matrices(clp_batch b, int32_t nprob, const int64_t* m,
                             const int64_t* const* colptrM, const int32_t* const* rowidxM, const double* const* valM,
                             const int64_t* const* colptrC, const int32_t* const* rowidxC, const double* const* valC,
                             const double* const* u0, clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  return guarded(b, [&] {
    return batch_solve_matrices(b, nprob, m, colptrM, rowidxM, valM, colptrC, rowidxC, valC, u0, sols, u_out, nodes_out);
  });
}

int clp_batch_sdp_matrices(clp_batch b, int32_t nprob, const int64_t* m,
                           const int64_t* const* colptrM, const int32_t* const* rowidxM, const double* const* valM,
                           const int64_t* const* colptrC, const int32_t* const* rowidxC, const double* const* valC,
                           const clp_sdp_params* p, clp_sdp_info* infos, int32_t* const* nodes_out,
                           double* const* X_out, double* const* lambdas_out, double* const* evec1_out) {
  return guarded(b, [&] {
    return batch_sdp_matrices(b, nprob, m, colptrM, rowidxM, valM, colptrC, rowidxC, valC, p, infos, nodes_out, X_out,
                              lambdas_out, evec1_out);
  });
}

int clp_batch_set_stream(clp_batch b, void* cuda_stream) {
  if (!b) return CLP_ERR_INVALID;
  CLP_CUDA(b, cudaSetDevice(b->device));
  if (b->stream && b->own_stream) { cudaStreamSynchronize(b->stream); cudaStreamDestroy(b->stream); }
  if (cuda_stream) { b->stream = reinterpret_cast<cudaStream_t>(cuda_stream); b->own_stream = false; }
  else { CLP_CUDA(b, cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking)); b->own_stream = true; }
  return CLP_OK;
}

int clp_batch_solve_dense_dev(clp_batch b, int32_t nprob, const int64_t* m, int dtype, const void* M_dev, const void* C_dev,
                              int64_t batch_stride, int64_t row_stride, int64_t col_stride, const double* u0_dev,
                              int64_t u0_stride, clp_solution* sols, double* u_out_dev, int64_t u_out_stride,
                              int32_t* const* nodes_out) {
  return guarded(b, [&] {
    return batch_solve_dense_dev(b, nprob, m, dtype, M_dev, C_dev, batch_stride, row_stride, col_stride, u0_dev, u0_stride,
                                 sols, u_out_dev, u_out_stride, nodes_out);
  });
}

int clp_batch_info(clp_batch b, int32_t* n_ctas, int64_t* scratch_bytes, int64_t* nnz_upper_total) {
  if (!b) return CLP_ERR_INVALID;
  if (n_ctas) *n_ctas = b->last_ctas;
  if (scratch_bytes) *scratch_bytes = b->last_scratch;
  if (nnz_upper_total) *nnz_upper_total = b->last_nnz;
  return CLP_OK;
}

int clp_batch_max_clique_euclidean(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                                   const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                   double sigma, double epsilon, double mindist, int method, double time_limit_s,
                                   clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out) {
  BatchInput in;
  in.D1 = D1; in.n1 = n1; in.D2 = D2; in.n2 = n2; in.A = A; in.m = m;
  in.p[0] = sigma; in.p[1] = epsilon; in.p[2] = mindist;
  return guarded(b, [&] { return batch_max_clique(b, 0, d, nprob, in, method, time_limit_s, infos, nodes_out, core_out); });
}

int clp_batch_max_clique_pointnormal(clp_batch b, int32_t nprob, const double* const* D1, const int64_t* n1,
                                     const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                     double sigp, double epsp, double sign, double epsn, int method, double time_limit_s,
                                     clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out) {
  BatchInput in;
  in.D1 = D1; in.n1 = n1; in.D2 = D2; in.n2 = n2; in.A = A; in.m = m;
  in.p[0] = sigp; in.p[1] = epsp; in.p[2] = sign; in.p[3] = epsn;
  return guarded(b, [&] { return batch_max_clique(b, 1, 6, nprob, in, method, time_limit_s, infos, nodes_out, core_out); });
}

int clp_batch_max_clique_graphs(clp_batch b, int32_t nprob, const int64_t* m, const int64_t* const* colptr,
                                const int32_t* const* rowidx, int method, double time_limit_s, clp_mc_info* infos,
                                int32_t* const* nodes_out, int32_t* const* core_out) {
  BatchInput in;
  in.m = m; in.colptr = colptr; in.rowidx = rowidx;
  return guarded(b, [&] { return batch_max_clique(b, kMcbKindGraph, 0, nprob, in, method, time_limit_s, infos, nodes_out, core_out); });
}

int clp_batch_solve_custom(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob, int32_t d,
                           const double* const* D1, const int64_t* n1, const double* const* D2, const int64_t* n2,
                           const int32_t* const* A, const int64_t* m, const double* const* u0,
                           clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  const CustomInvariant inv{source, prm, nprm};
  BatchInput in;
  in.D1 = D1; in.n1 = n1; in.D2 = D2; in.n2 = n2; in.A = A; in.m = m; in.inv = &inv;
  return guarded(b, [&] { return batch_solve(b, kBatchKindCustom, d, nprob, in, u0, sols, u_out, nodes_out); });
}

int clp_batch_max_clique_custom(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob, int32_t d,
                                const double* const* D1, const int64_t* n1, const double* const* D2, const int64_t* n2,
                                const int32_t* const* A, const int64_t* m, int method, double time_limit_s,
                                clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out) {
  const CustomInvariant inv{source, prm, nprm};
  BatchInput in;
  in.D1 = D1; in.n1 = n1; in.D2 = D2; in.n2 = n2; in.A = A; in.m = m; in.inv = &inv;
  return guarded(b, [&] { return batch_max_clique(b, kBatchKindCustom, d, nprob, in, method, time_limit_s, infos, nodes_out, core_out); });
}

int clp_batch_solve_euclidean_dev(clp_batch b, int32_t nprob, int32_t d, const clp_points_dev* pts, const double* u0_dev,
                                  int64_t u0_stride, double sigma, double epsilon, double mindist, clp_solution* sols,
                                  double* u_out_dev, int64_t u_out_stride, int32_t* const* nodes_out) {
  return guarded(b, [&] {
    BatchInput in;
    if (int rc = solve_dev_check(b, nprob, pts, u0_dev, u0_stride, u_out_dev, u_out_stride, in)) return rc;
    in.p[0] = sigma; in.p[1] = epsilon; in.p[2] = mindist;
    return batch_solve(b, 0, d, nprob, in, nullptr, sols, nullptr, nodes_out);
  });
}

int clp_batch_solve_pointnormal_dev(clp_batch b, int32_t nprob, const clp_points_dev* pts, const double* u0_dev,
                                    int64_t u0_stride, double sigp, double epsp, double sign, double epsn,
                                    clp_solution* sols, double* u_out_dev, int64_t u_out_stride, int32_t* const* nodes_out) {
  return guarded(b, [&] {
    BatchInput in;
    if (int rc = solve_dev_check(b, nprob, pts, u0_dev, u0_stride, u_out_dev, u_out_stride, in)) return rc;
    in.p[0] = sigp; in.p[1] = epsp; in.p[2] = sign; in.p[3] = epsn;
    return batch_solve(b, 1, 6, nprob, in, nullptr, sols, nullptr, nodes_out);
  });
}

int clp_batch_solve_custom_dev(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob, int32_t d,
                               const clp_points_dev* pts, const double* u0_dev, int64_t u0_stride, clp_solution* sols,
                               double* u_out_dev, int64_t u_out_stride, int32_t* const* nodes_out) {
  const CustomInvariant inv{source, prm, nprm};
  return guarded(b, [&] {
    BatchInput in;
    if (int rc = solve_dev_check(b, nprob, pts, u0_dev, u0_stride, u_out_dev, u_out_stride, in)) return rc;
    in.inv = &inv;
    return batch_solve(b, kBatchKindCustom, d, nprob, in, nullptr, sols, nullptr, nodes_out);
  });
}

int clp_batch_max_clique_euclidean_dev(clp_batch b, int32_t nprob, int32_t d, const clp_points_dev* pts, double sigma,
                                       double epsilon, double mindist, int method, double time_limit_s,
                                       clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out) {
  return guarded(b, [&] {
    BatchInput in;
    long long max_m = 0;
    if (int rc = points_dev_check(b, nprob, pts, in, &max_m)) return rc;
    in.p[0] = sigma; in.p[1] = epsilon; in.p[2] = mindist;
    return batch_max_clique(b, 0, d, nprob, in, method, time_limit_s, infos, nodes_out, core_out);
  });
}

int clp_batch_max_clique_pointnormal_dev(clp_batch b, int32_t nprob, const clp_points_dev* pts, double sigp, double epsp,
                                         double sign, double epsn, int method, double time_limit_s, clp_mc_info* infos,
                                         int32_t* const* nodes_out, int32_t* const* core_out) {
  return guarded(b, [&] {
    BatchInput in;
    long long max_m = 0;
    if (int rc = points_dev_check(b, nprob, pts, in, &max_m)) return rc;
    in.p[0] = sigp; in.p[1] = epsp; in.p[2] = sign; in.p[3] = epsn;
    return batch_max_clique(b, 1, 6, nprob, in, method, time_limit_s, infos, nodes_out, core_out);
  });
}

int clp_batch_max_clique_custom_dev(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob,
                                    int32_t d, const clp_points_dev* pts, int method, double time_limit_s,
                                    clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out) {
  const CustomInvariant inv{source, prm, nprm};
  return guarded(b, [&] {
    BatchInput in;
    long long max_m = 0;
    if (int rc = points_dev_check(b, nprob, pts, in, &max_m)) return rc;
    in.inv = &inv;
    return batch_max_clique(b, kBatchKindCustom, d, nprob, in, method, time_limit_s, infos, nodes_out, core_out);
  });
}

int clp_batch_correspondences(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                              const double* const* D2, const int64_t* n2, int32_t knn, double radius, int enforce_1to1,
                              int32_t* const* A_out, int64_t capacity, int64_t* m) {
  KnnBatchIn in;
  in.D1h = D1; in.D2h = D2; in.A_out = A_out;
  return guarded(b, [&] { return batch_correspondences(b, false, nprob, d, in, n1, n2, knn, radius, enforce_1to1, capacity, m); });
}

int clp_batch_correspondences_dev(clp_batch b, int32_t nprob, int32_t d, const double* D1_dev, const int64_t d1_strides[3],
                                  const int64_t* n1, const double* D2_dev, const int64_t d2_strides[3], const int64_t* n2,
                                  int32_t knn, double radius, int enforce_1to1, int32_t* A_dev, const int64_t a_strides[3],
                                  int64_t capacity, int64_t* m) {
  KnnBatchIn in;
  in.D1 = D1_dev; in.s1 = d1_strides; in.D2 = D2_dev; in.s2 = d2_strides; in.A_dev = A_dev; in.sa = a_strides;
  return guarded(b, [&] { return batch_correspondences(b, true, nprob, d, in, n1, n2, knn, radius, enforce_1to1, capacity, m); });
}

// a single call is a batch of one: the clp_score_*_dev layouts are the strides (0, 1, d) of the clouds, (0, 1, m) of A
// and (0, 1, d + 1) of T
int clp_estimate_transform(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2,
                           const int32_t* A, int64_t m, const int32_t* rows, int64_t k, double* T_out, clp_tf_info* info) {
  if (!h) return CLP_ERR_INVALID;
  TfIn in;
  in.D1h = &D1; in.D2h = &D2; in.Ah = &A; in.n1 = &n1; in.n2 = &n2; in.m = &m; in.rows = &rows; in.k = &k;
  in.T_out = &T_out;
  return guarded(h, [&] { return estimate_transform(h, h->tf_buf, h->tf_pinned, 1, d, in, info); });
}

int clp_estimate_transform_dev(clp_handle h, const double* D1_dev, int32_t d, int64_t n1, const double* D2_dev, int64_t n2,
                               const int32_t* A_dev, int64_t m, const int32_t* rows, int64_t k, double* T_dev,
                               clp_tf_info* info) {
  if (!h) return CLP_ERR_INVALID;
  clp_points_dev pts;
  std::memset(&pts, 0, sizeof(pts));
  pts.D1 = D1_dev; pts.D2 = D2_dev; pts.A = A_dev;
  const int64_t dd = std::max<int64_t>(d, 1), ts[3] = {0, 1, dd + 1};
  pts.d1_strides[1] = pts.d2_strides[1] = 1; pts.d1_strides[2] = pts.d2_strides[2] = dd;
  pts.a_strides[1] = 1; pts.a_strides[2] = std::max<int64_t>(m, 1);
  TfIn in;
  in.pts = &pts; in.n1 = &n1; in.n2 = &n2; in.m = &m; in.rows = &rows; in.k = &k; in.T_dev = T_dev; in.ts = ts;
  return guarded(h, [&] { return estimate_transform(h, h->tf_buf, h->tf_pinned, 1, d, in, info); });
}

int clp_batch_estimate_transform(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                                 const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                 const int32_t* const* rows, const int64_t* k, double* const* T_out, clp_tf_info* infos) {
  if (!b) return CLP_ERR_INVALID;
  TfIn in;
  in.D1h = D1; in.D2h = D2; in.Ah = A; in.n1 = n1; in.n2 = n2; in.m = m; in.rows = rows; in.k = k; in.T_out = T_out;
  return guarded(b, [&] { return estimate_transform(b, b->tf_buf, b->tf_pinned, nprob, d, in, infos); });
}

int clp_batch_estimate_transform_dev(clp_batch b, int32_t nprob, int32_t d, const clp_points_dev* pts,
                                     const int32_t* const* rows, const int64_t* k, double* T_dev, const int64_t t_strides[3],
                                     clp_tf_info* infos) {
  if (!b) return CLP_ERR_INVALID;
  if (!pts) return fail(b, CLP_ERR_INVALID, "estimate transform: pts is required");
  TfIn in;
  in.pts = pts; in.n1 = pts->n1; in.n2 = pts->n2; in.m = pts->m; in.rows = rows; in.k = k; in.T_dev = T_dev;
  in.ts = t_strides;
  return guarded(b, [&] { return estimate_transform(b, b->tf_buf, b->tf_pinned, nprob, d, in, infos); });
}

}  // extern "C"
