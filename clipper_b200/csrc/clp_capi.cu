// clp_capi.cu -- host side of the C-ABI declared in include/clipper_b200.h.
//
// One handle = one CUDA device + one stream + the dense M store + the solver workspace.
// There is NO CPU implementation of the hot path in this library: every scoring / mat-vec /
// solve call launches the sm_90a kernels of clp_kernels.cuh or fails with an error code.
#include "clp_kernels.cuh"
#include "clp_host_utils.h"
#include "../../include/clipper_b200.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include <unistd.h>

#ifndef CLP_VERSION
#define CLP_VERSION "0.1.0"
#endif

using namespace clp;

namespace {

thread_local std::string g_create_error;

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

}  // namespace

static int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return (v && *v) ? std::atoi(v) : dflt;
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
  int prof_ctas = env_int("CLP_PROF_CTAS", 0);      // print the per-CTA phase times of every resident solve (stderr)
  int prof_host = env_int("CLP_PROF_HOST", 0);      // print wall-clock marks of the scoring / solve calls (stderr)
  int prof_laps = env_int("CLP_PROF_LAPS", 1);      // in-kernel phase timers (the split reported in clp_solution.prof_*)
  DevBuf prof_buf;
  // resident-vector solver (clp_resident.cuh): the default whenever the whole trial vector fits shared memory
  int res_G = 0;                                    // CTAs of the resident kernels for the current matrix
  int res_NI = 0;
  bool compact_resident = false;                    // layout of the current compact copy: full rows + column indices
  int smem_optin = 0;                               // cudaDevAttrMaxSharedMemoryPerBlockOptin
  bool score_pending = false;                       // a scoring launch's error flag has not been read back yet
  bool counts_fused = false;                        // sp_ptr4 already holds the counts of the current matrix
  long long counts_m = 0; int counts_rows_pad = 0, counts_nseg = 0, counts_W = 0;  // ... which was this one
  int pack = env_int("CLP_PACK", 1);              // resident layout of plain fp32 matrices with 4-byte entries (0: always 6 bytes)
  bool counts_win = false;                          // the fused counts came with the occupied-window bitmap (sp_win)

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
  void* pinned = nullptr;
  size_t pinned_cap = 0;
  Plan plan{};
  long long mpad = 0;
  // stripe decomposition (clp_dense2.cuh)
  int dense_mode = 4;     // requested: 0 segments, 2 stripes/upper-triangle two-sided (one GPU),
                          //            3 compact rows (segmented), 6 compact rows + resident vector,
                          //            4 auto (6 if the vector fits shared memory, else 3, when the graph is sparse enough; else 2 / 0)
  int dense_mode_eff = 2; // effective, decided when the matrix is finalised
  // compact-row copy (clp_sparse.cuh)
  DevBuf sp_val, sp_col, sp_ptr4, sp_part, sp_item, sp_rowid;  // sp_ptr4: kept entries per (segment, row)
  DevBuf sp_win, res_wcol;  // packed layout: occupied 16-column windows per row | members' columns where every warp starts
  unsigned long long sp_nnz = 0, sp_nnz_real = 0;
  SparseView sp{};
  Plan2 plan2{};
  Dense2Buffers d2{};
  DevBuf d2buf, plan2buf;

  size_t esize() const { return storage == CLP_STORE_F64 ? 8 : 4; }
  int entry_bytes() const { return sp.packed ? 4 : (int)esize() + 2; }  // compact copy: bytes per stored entry
  int wwords() const { return (int)((ld + 511) / 512); }  // 32-bit words of a row's window bitmap
  // the packed layout may be built: whole rows, fp32, one GPU, not switched off
  bool pack_candidate() const { return pack && storage == CLP_STORE_F32 && world == 1; }
};

namespace {

int fail(clp_handle h, int code, const std::string& msg) {
  if (h) h->err = msg; else g_create_error = msg;
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
int reset_sync(clp_handle h);

// nothing may propagate out of an extern "C" entry point (the library is loaded into Python and into C callers)
template <typename F>
int guarded(clp_handle h, F&& f) {
  try { return f(); }
  catch (const std::bad_alloc&) { return fail(h, CLP_ERR_ALLOC, "host allocation failed"); }
  catch (const std::exception& e) { return fail(h, CLP_ERR_INVALID, std::string("internal error: ") + e.what()); }
  catch (...) { return fail(h, CLP_ERR_INVALID, "internal error"); }
}

int ensure_pinned(clp_handle h, size_t bytes) {
  if (bytes <= h->pinned_cap) return CLP_OK;
  if (h->pinned) { cudaFreeHost(h->pinned); h->pinned = nullptr; h->pinned_cap = 0; }
  CLP_CUDA(h, cudaMallocHost(&h->pinned, bytes));
  h->pinned_cap = bytes;
  return CLP_OK;
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
      return {(const void*)solver_resident_kernel<T, false, true>, (const void*)matvec_resident_kernel<T, S, true>, S::NT};
  return {(const void*)solver_resident_kernel<T, false>, (const void*)matvec_resident_kernel<T, S>, S::NT};
}
int res_warps(clp_handle h) {
  return (h->storage == CLP_STORE_F64 ? res_kernels<double>(h) : res_kernels<float>(h)).NT / 32;
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

// can the resident solver take a problem of this size on this handle?
bool resident_possible(clp_handle h, long long m) {
  if (m > kResMaxM || m > 65535) return false;
  if (!(h->dense_mode == 4 || h->dense_mode == 6)) return false;
  return (long long)res_smem_plan((int)m, kResThreads / 32).total <= (long long)h->smem_optin;
}

template <typename T>
cudaError_t res_set_attrs(clp_handle h) {
  // [storage][sharded][packed][device]: set once per process (handles may live on different host threads)
  static std::atomic<bool> done[2][2][2][8];
  std::atomic<bool>& flag = done[sizeof(T) == 8 ? 1 : 0][h->world > 1 ? 1 : 0][h->sp.packed ? 1 : 0][h->device & 7];
  if (flag.load(std::memory_order_acquire)) return cudaSuccess;
  // the attribute is a per-function PERMISSION shared by every handle of the process (two shards in one process ask
  // for different sizes): always the device maximum; the carve-out follows what each launch actually requests
  const ResKernels k = res_kernels<T>(h);
  cudaError_t rc = cudaFuncSetAttribute(k.matvec, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin);
  if (rc == cudaSuccess) rc = cudaFuncSetAttribute(k.solver, cudaFuncAttributeMaxDynamicSharedMemorySize, h->smem_optin);
  if (rc == cudaSuccess) flag.store(true, std::memory_order_release);
  return rc;
}

ResArgs res_args(clp_handle h) {
  ResArgs a;
  std::memset(&a, 0, sizeof(a));
  a.sp = h->sp;
  a.m = (int)h->m; a.row0 = h->row0; a.rows = h->rows; a.rows_pad = h->rows_pad; a.NI = h->res_NI; a.G = h->res_G;
  const clp_params& P = h->prm;
  a.prm.tol_u = P.tol_u; a.prm.tol_F = P.tol_F; a.prm.beta = P.beta; a.prm.eps = P.eps;
  a.prm.maxiniters = P.maxiniters; a.prm.maxoliters = P.maxoliters; a.prm.maxlsiters = P.maxlsiters;
  a.prm.rescale_u0 = P.rescale_u0 ? 1 : 0;
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

// Called once the dense store holds the new matrix: pick the sweep (dense mode) and build what it needs.
template <typename T>
int build_sparse(clp_handle h, bool force, bool resident) {
  // layout of the compact copy: the column segments of the Plan (segmented sweep, byte offsets), or one segment =
  // the whole row (resident sweep, column indices; padding entries point at column m of the staged vector)
  Plan p = h->plan;
  if (resident) { p.NSEG = 1; p.W = (int)h->ld; }
  const int nseg = p.NSEG;
  const long long nptr = (long long)nseg * (h->rows_pad + 1);
  // counts produced by the scoring kernel (scored matrices are "plain"): only trusted for the very matrix and
  // segmentation they were counted for
  const bool fused = h->counts_fused && h->counts_m == h->m && h->counts_rows_pad == h->rows_pad &&
                     h->counts_nseg == nseg && h->counts_W == p.W;
  const bool fused_win = fused && h->counts_win;
  h->counts_fused = false; h->counts_win = false;
  // right after a scoring launch the sync block still carries that launch's error flag (checked below, with the
  // totals: one host synchronisation per scoring call) and zeroed counters; otherwise start from a clean block
  const bool after_score = h->score_pending;
  h->score_pending = false;
  if (!after_score) { if (int rc = reset_sync(h)) return rc; }
  SyncBlock* sb = h->sync.as<SyncBlock>();
  const T* M = h->Mbuf.as<T>();
  const unsigned blocks = (unsigned)(((size_t)h->rows_pad * 32 + 255) / 256);
  // packed layout (whole rows, fp32): the counts also describe the occupied 16-column windows and the exponent range;
  // the sort and the item lengths then decide on the device whether the fillers count (PackCount::on), the host reads
  // the same decision back with the totals
  const bool want_pack = resident && h->pack_candidate() && (!fused || fused_win);
  const int wwords = h->wwords();
  if (!fused) {
    CLP_CUDA(h, h->sp_ptr4.ensure((size_t)nptr * sizeof(unsigned int)));
    CLP_CUDA(h, cudaMemsetAsync(h->sp_ptr4.p, 0, (size_t)nptr * sizeof(unsigned int), h->stream));
    if (want_pack) {
      CLP_CUDA(h, h->sp_win.ensure((size_t)h->rows_pad * wwords * sizeof(unsigned int)));
      CLP_CUDA(h, cudaMemsetAsync(h->sp_win.p, 0, (size_t)h->rows_pad * wwords * sizeof(unsigned int), h->stream));
    }
    sparse_count_kernel<T><<<blocks, 256, 0, h->stream>>>(M, h->ld, (int)h->m, h->rows, h->rows_pad, p.W, nseg,
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
  const int nb = p.W / 4 + 2;  // possible slice lengths in chunks
  sell_sort_kernel<<<nseg, 1024, (size_t)(nb + 1) * sizeof(unsigned int), h->stream>>>(
      h->sp_ptr4.as<unsigned int>(), h->rows_pad, nb, h->sp_rowid.as<unsigned int>(), fused ? &sb->counts[0] : nullptr, pc);
  CLP_CUDA(h, cudaGetLastError());
  sell_itemlen_kernel<<<(unsigned)((nitem + 255) / 256), 256, 0, h->stream>>>(h->sp_ptr4.as<unsigned int>(), h->sp_rowid.as<unsigned int>(),
                                                                              h->rows_pad, nseg, h->sp_item.as<unsigned int>(), pc);
  CLP_CUDA(h, cudaGetLastError());
  unsigned long long* total4_d = reinterpret_cast<unsigned long long*>(&sb->leaf[0][0]);  // scratch words of the sync block
  unsigned long long* segtot_d = reinterpret_cast<unsigned long long*>(&sb->leaf[1][0]);  // [<= 64] (leaf[1..4])
  sparse_scan_seg_kernel<<<nseg, 1024, 0, h->stream>>>(h->sp_item.as<unsigned int>(), NI + 1, segtot_d);
  CLP_CUDA(h, cudaGetLastError());
  sparse_scan_fix_kernel<<<nseg, 1024, 0, h->stream>>>(h->sp_item.as<unsigned int>(), NI + 1, nseg, segtot_d, total4_d);
  CLP_CUDA(h, cudaGetLastError());
  unsigned long long host[3] = {0, 0, 0};
  unsigned int hexpo[2] = {0u, 0u};
  int host_err = 0;
  CLP_CUDA(h, cudaMemcpyAsync(&host[0], total4_d, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(&host[1], &sb->counts[0], 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  if (want_pack) CLP_CUDA(h, cudaMemcpyAsync(hexpo, &sb->expo[0], sizeof(hexpo), cudaMemcpyDeviceToHost, h->stream));
  if (after_score) CLP_CUDA(h, cudaMemcpyAsync(&host_err, &sb->error, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
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
  if (h->sp.packed) {  // whole rows (nseg = 1), fp32 only
    if constexpr (sizeof(T) == 4)
      sparse_fill_items_kernel<T, true><<<(unsigned)((NI + kFillWarps - 1) / kFillWarps), kFillWarps * 32, 0, h->stream>>>(
          M, h->ld, (int)h->m, h->rows, h->rows_pad, p.W, nseg, h->sp_item.as<unsigned int>(), h->sp_rowid.as<unsigned int>(),
          h->sp_val.as<T>(), nullptr, 0, 0u, bias);
  } else {
    const long long nwarp = (long long)nseg * NI;
    sparse_fill_items_kernel<T><<<(unsigned)((nwarp + kFillWarps - 1) / kFillWarps), kFillWarps * 32, 0, h->stream>>>(
        M, h->ld, (int)h->m, h->rows, h->rows_pad, p.W, nseg, h->sp_item.as<unsigned int>(), h->sp_rowid.as<unsigned int>(),
        h->sp_val.as<T>(), h->sp_col.as<unsigned short>(), resident ? 0 : 3, resident ? (unsigned int)h->m : kZeroSlot);
  }
  CLP_CUDA(h, cudaGetLastError());
  h->sp.val = h->sp_val.p; h->sp.off16 = h->sp.packed ? nullptr : h->sp_col.as<unsigned short>();
  h->sp.itemptr = h->sp_item.as<unsigned int>(); h->sp.rowid = h->sp_rowid.as<unsigned int>(); h->sp.rows_pad = h->rows_pad;
  // byte-balanced contiguous item range of every CTA (depends on the grid size: rebuilt with the plan)
  int G = p.G;
  if (resident) {
    // one fat CTA per SM; small problems use fewer CTAs -- every CTA should stream at least ~32 KB per sweep, since
    // with more CTAs the per-evaluation exchange costs more than the sweep saves; shards sharing a GPU honour the cap
    h->res_NI = NI;
    const long long by_bytes = (long long)((double)h->sp_nnz * h->entry_bytes() / (32.0 * 1024.0));
    G = (int)std::max<long long>(1, std::min<long long>(std::min<long long>(h->grid_cap > 0 ? std::min(h->grid_cap, h->sm_count) : h->sm_count, NI / 2),
                                                        std::max<long long>(1, by_bytes)));
    h->res_G = G;
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
  h->compact_resident = resident;
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

int finalize_matrix_impl(clp_handle h) {
  int eff = h->dense_mode;
  if (eff == 3 || eff == 4 || eff == 6) {
    h->sp.plain = 0; h->sp.packed = 0;
    if (int rc = set_plan_for(h, 3)) return rc;  // column segmentation (NSEG, W) depends on m only
    const bool resident = (eff != 3) && resident_possible(h, h->m);
    const bool force = (eff == 3) || (eff == 6);
    const int rc = (h->storage == CLP_STORE_F64) ? build_sparse<double>(h, force, resident) : build_sparse<float>(h, force, resident);
    if (rc == CLP_OK) eff = resident ? 6 : 3;
    else if (rc == kKeepDense) eff = (h->world > 1) ? 0 : 2;
    else return rc;
  }
  if (eff == 2 && h->world > 1) eff = 0;  // a shard holds row blocks, not the whole upper triangle
  if (eff != 3 && eff != 6) { if (int rc = set_plan_for(h, eff)) return rc; }
  h->dense_mode_eff = eff;
  if (eff == 2) { if (int rc = build_plan2(h)) return rc; }
  return CLP_OK;
}

int finalize_matrix(clp_handle h) { return guarded(h, [&] { return finalize_matrix_impl(h); }); }

// (re)allocate the matrix store for problem size m under the current shard config
int ensure_matrix(clp_handle h, long long m) {
  if (m <= 0) return fail(h, CLP_ERR_INVALID, "number of associations must be positive");
  if (m > (long long)kMaxSeg * kSegMax) return fail(h, CLP_ERR_INVALID, "m exceeds the supported maximum (262144)");
  CLP_CUDA(h, cudaSetDevice(h->device));
  h->m = m;
  shard_rows(m, h->rank, h->world, &h->row0, &h->rows);
  h->rows_pad = (int)round_up(std::max(h->rows, 1), kRowTile);
  h->ld = round_up(m, 128);
  h->mpad = round_up(m, 128);
  CLP_CUDA(h, h->Mbuf.ensure((size_t)h->rows_pad * (size_t)h->ld * h->esize()));
  h->plan = make_plan(m, h->rows_pad, h->grid_for(h->ctas_for(h->dense_mode == 3 || h->dense_mode == 4 ? 3 : h->dense_mode)));
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
  CLP_CUDA(h, h->parts.ensure((size_t)2 * h->plan.NSEG * h->rows_pad * sizeof(double)));
  CLP_CUDA(h, h->small.ensure(((size_t)kMaxSeg + (size_t)2 * h->plan.G * kRedVals) * sizeof(double)));
  CLP_CUDA(h, h->result.ensure(256 + (size_t)h->mpad * sizeof(double)));
  CLP_CUDA(h, h->u0dev.ensure((size_t)h->mpad * sizeof(double)));
  CLP_CUDA(h, h->ybuf.ensure((size_t)4 * h->mpad * sizeof(double)));
  if (int rc = ensure_pinned(h, 256 + (size_t)h->mpad * sizeof(double))) return rc;
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
  return h->storage == CLP_STORE_F32 && (kind == 1 || d == 2 || d == 3);
}

template <typename T, bool MIRROR>
int launch_score_m(clp_handle h, int kind, int d, const ScoreArgs& a) {
  dim3 grid((unsigned)(h->ld / 128), (unsigned)(h->rows_pad / kRowTile));
  if constexpr (sizeof(T) == 4) {
    if (!screened_scoring(h, kind, d)) score_tile_kernel<T, 0, 0, MIRROR, false><<<grid, kThreads, 0, h->stream>>>(a);
    else if (kind == 1) score_tile_kernel<T, 1, 6, MIRROR, true><<<grid, kThreads, 0, h->stream>>>(a);
    else if (d == 3) score_tile_kernel<T, 0, 3, MIRROR, true><<<grid, kThreads, 0, h->stream>>>(a);
    else score_tile_kernel<T, 0, 2, MIRROR, true><<<grid, kThreads, 0, h->stream>>>(a);
  } else {
    if (kind == 1) score_tile_kernel<T, 1, 6, MIRROR, false><<<grid, kThreads, 0, h->stream>>>(a);
    else if (d == 3) score_tile_kernel<T, 0, 3, MIRROR, false><<<grid, kThreads, 0, h->stream>>>(a);
    else if (d == 2) score_tile_kernel<T, 0, 2, MIRROR, false><<<grid, kThreads, 0, h->stream>>>(a);
    else score_tile_kernel<T, 0, 0, MIRROR, false><<<grid, kThreads, 0, h->stream>>>(a);
  }
  CLP_CUDA(h, cudaGetLastError());
  return CLP_OK;
}
template <typename T>
int launch_score(clp_handle h, int kind, int d, const ScoreArgs& a) {
  // an unsharded handle holds the whole symmetric matrix: compute the upper triangle, mirror the rest
  return (h->world == 1) ? launch_score_m<T, true>(h, kind, d, a) : launch_score_m<T, false>(h, kind, d, a);
}

// common tail of the four scoring entry points: D1/D2/A already on the device
int score_on_device(clp_handle h, int kind, const double* D1d, int d, long long n1, const double* D2d,
                    long long n2, const int32_t* Ad, long long m, double p0, double p1, double p2, double p3) {
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
  const bool res_layout = resident_possible(h, m);  // the compact copy will use one segment = the whole row
  const int cnt_nseg = res_layout ? 1 : h->plan.NSEG, cnt_W = res_layout ? (int)h->ld : h->plan.W;
  a.cnt = nullptr; a.W = cnt_W; a.win = nullptr; a.wwords = 0; a.expo = nullptr;
  h->counts_fused = false;
  const bool compact_next = (h->dense_mode == 3 || h->dense_mode == 4 || h->dense_mode == 6);
  if (compact_next && screened_scoring(h, kind, d)) {
    // the screened scoring kernel also counts the kept entries per (segment, row): first pass of the compact build
    const size_t nptr = (size_t)cnt_nseg * (h->rows_pad + 1);
    CLP_CUDA(h, h->sp_ptr4.ensure(nptr * sizeof(unsigned int)));
    CLP_CUDA(h, cudaMemsetAsync(h->sp_ptr4.p, 0, nptr * sizeof(unsigned int), h->stream));
    a.cnt = h->sp_ptr4.as<unsigned int>();
    if (res_layout && h->pack_candidate()) {  // and what the packed layout needs (occupied windows, exponent range)
      const size_t nw = (size_t)h->rows_pad * h->wwords();
      CLP_CUDA(h, h->sp_win.ensure(nw * sizeof(unsigned int)));
      CLP_CUDA(h, cudaMemsetAsync(h->sp_win.p, 0, nw * sizeof(unsigned int), h->stream));
      a.win = h->sp_win.as<unsigned int>(); a.wwords = h->wwords(); a.expo = &sb->expo[0];
    }
  }
  a.d = d; a.p0 = p0; a.p1 = p1; a.p2 = p2; a.p3 = p3; a.affinityeps = h->prm.affinityeps;
  int rc = (h->storage == CLP_STORE_F64) ? launch_score<double>(h, kind, d, a) : launch_score<float>(h, kind, d, a);
  if (rc) return rc;
  if (!compact_next) {  // dense sweeps: nothing else synchronises with the scoring launch
    SyncBlock host;
    if ((rc = read_sync(h, &host))) return rc;
    if (host.error == 2) return fail(h, CLP_ERR_INVALID, "association index out of range of D1/D2");
  } else {
    h->score_pending = true;  // the compact build reads the flag back together with its totals
  }
  const auto tp1 = std::chrono::steady_clock::now();
  if (a.cnt) {  // counts produced by this launch describe this matrix (a failed launch / bad index aborts the build)
    h->counts_fused = true; h->counts_win = a.win != nullptr;
    h->counts_m = m; h->counts_rows_pad = h->rows_pad; h->counts_nseg = cnt_nseg; h->counts_W = cnt_W;
  }
  rc = finalize_matrix(h);
  h->score_pending = false;
  if (rc) { h->counts_fused = false; return rc; }
  h->has_matrix = true;
  h->has_A = true;
  if (h->prof_host) {
    const auto tp2 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[clp host] score call: scoring kernel done after %.3f ms, build enqueued after %.3f ms (total)\n",
                 1e3 * std::chrono::duration<double>(tp1 - tp0).count(), 1e3 * std::chrono::duration<double>(tp2 - tp0).count());
  }
  return CLP_OK;
}

int score_from_host(clp_handle h, int kind, const double* D1, int d, long long n1, const double* D2,
                    long long n2, const int32_t* A, long long m, double p0, double p1, double p2, double p3) {
  if (!h) return CLP_ERR_INVALID;
  if (!D1 || !D2 || d <= 0 || n1 <= 0 || n2 <= 0) return fail(h, CLP_ERR_INVALID, "bad data set arguments");
  CLP_CUDA(h, cudaSetDevice(h->device));
  const bool all_to_all = (A == nullptr || m == 0);  // all-to-all hypothesis (ref clipper.cpp:24, utils.h:61-71)
  if (all_to_all) {
    m = n1 * n2;
    if (m > (long long)kMaxSeg * kSegMax) return fail(h, CLP_ERR_INVALID, "all-to-all hypothesis too large");
  } else if (m < 0) return fail(h, CLP_ERR_INVALID, "negative m");
  CLP_CUDA(h, h->A_dev.ensure((size_t)2 * m * sizeof(int32_t)));
  CLP_CUDA(h, h->D1dev.ensure((size_t)d * n1 * sizeof(double)));
  CLP_CUDA(h, h->D2dev.ensure((size_t)d * n2 * sizeof(double)));
  if (all_to_all) {  // generated on the device: A never crosses PCIe; the host copy is fetched only if asked for
    all_to_all_kernel<<<(unsigned)std::min<long long>((m + 255) / 256, 4096), 256, 0, h->stream>>>(n1, n2, h->A_dev.as<int32_t>());
    CLP_CUDA(h, cudaGetLastError());
    h->A_host_valid = false;
  } else {
    h->A_host.assign(A, A + (size_t)2 * m);
    h->A_host_valid = true;
    CLP_CUDA(h, cudaMemcpyAsync(h->A_dev.p, h->A_host.data(), (size_t)2 * m * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
  }
  CLP_CUDA(h, cudaMemcpyAsync(h->D1dev.p, D1, (size_t)d * n1 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CLP_CUDA(h, cudaMemcpyAsync(h->D2dev.p, D2, (size_t)d * n2 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  return score_on_device(h, kind, h->D1dev.as<double>(), d, n1, h->D2dev.as<double>(), n2,
                         h->A_dev.as<int32_t>(), m, p0, p1, p2, p3);
}

int score_from_device(clp_handle h, int kind, const double* D1d, int d, long long n1, const double* D2d,
                      long long n2, const int32_t* Ad, long long m, double p0, double p1, double p2, double p3) {
  if (!h) return CLP_ERR_INVALID;
  if (!D1d || !D2d || d <= 0 || n1 <= 0 || n2 <= 0 || m < 0 || (Ad && m == 0))
    return fail(h, CLP_ERR_INVALID, "bad device arguments");
  CLP_CUDA(h, cudaSetDevice(h->device));
  if (!Ad) {  // all-to-all hypothesis, generated on the device
    m = n1 * n2;
    if (m > (long long)kMaxSeg * kSegMax) return fail(h, CLP_ERR_INVALID, "all-to-all hypothesis too large");
  }
  CLP_CUDA(h, h->A_dev.ensure((size_t)2 * m * sizeof(int32_t)));
  if (Ad) CLP_CUDA(h, cudaMemcpyAsync(h->A_dev.p, Ad, (size_t)2 * m * sizeof(int32_t), cudaMemcpyDeviceToDevice, h->stream));
  else {
    all_to_all_kernel<<<(unsigned)std::min<long long>((m + 255) / 256, 4096), 256, 0, h->stream>>>(n1, n2, h->A_dev.as<int32_t>());
    CLP_CUDA(h, cudaGetLastError());
  }
  h->A_host_valid = false;
  return score_on_device(h, kind, D1d, d, n1, D2d, n2, h->A_dev.as<int32_t>(), m, p0, p1, p2, p3);
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
  return (h->storage == CLP_STORE_F64) ? launch_matvec<double>(h, st, v_dev, d, y_dev, Mv_dev, Cv_dev)
                                       : launch_matvec<float>(h, st, v_dev, d, y_dev, Mv_dev, Cv_dev);
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
  a.prm.tol_u = P.tol_u; a.prm.tol_F = P.tol_F; a.prm.beta = P.beta; a.prm.eps = P.eps;
  a.prm.maxiniters = P.maxiniters; a.prm.maxoliters = P.maxoliters; a.prm.maxlsiters = P.maxlsiters;
  a.prm.rescale_u0 = P.rescale_u0 ? 1 : 0;
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
    ResArgs ra = res_args(h);
    le = (h->storage == CLP_STORE_F64) ? launch_resident_solver<double>(h, ra) : launch_resident_solver<float>(h, ra);
  } else {
    le = (h->storage == CLP_STORE_F64) ? launch_solver<double>(h, a) : launch_solver<float>(h, a);
  }
  CLP_CUDA(h, le);
  CLP_CUDA(h, cudaEventRecord(h->ev1, h->stream));
  const size_t rbytes = 256 + (size_t)h->m * sizeof(double);
  CLP_CUDA(h, cudaMemcpyAsync(h->pinned, h->result.p, rbytes, cudaMemcpyDeviceToHost, h->stream));
  if (u_out_dev)
    CLP_CUDA(h, cudaMemcpyAsync(u_out_dev, a.u_final, (size_t)h->m * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  const auto tp_sync = std::chrono::steady_clock::now();
  float ms = 0.f;
  CLP_CUDA(h, cudaEventElapsedTime(&ms, h->ev0, h->ev1));

  const SolverOut so = *reinterpret_cast<const SolverOut*>(h->pinned);
  h->seq = so.seq_end;
  if (h->prof_ctas && h->dense_mode_eff == 6) {  // diagnostics: spread of the per-CTA phase times
    std::vector<double> pc((size_t)h->res_G * 8);
    CLP_CUDA(h, cudaMemcpy(pc.data(), h->prof_buf.p, pc.size() * sizeof(double), cudaMemcpyDeviceToHost));
    if (h->prof_ctas >= 2) {  // one line per CTA: index, ms in sweeps / epilogues / exchanges / staging, items, chunks
      for (int b = 0; b < h->res_G; ++b)
        std::fprintf(stderr, "[clp cta] %d %.4f %.4f %.4f %.4f %.0f %.0f\n", b, 1e-6 * pc[(size_t)b * 8], 1e-6 * pc[(size_t)b * 8 + 1],
                     1e-6 * pc[(size_t)b * 8 + 2], 1e-6 * pc[(size_t)b * 8 + 3], pc[(size_t)b * 8 + 4], pc[(size_t)b * 8 + 5]);
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
  const double* u = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->pinned) + 256);

  // rounding (ref clipper.cpp:287-310) on the device-produced u
  std::vector<int32_t> nodes;
  if (P.rounding == CLP_ROUND_NONZERO) {
    nodes.resize((size_t)h->m);
    nodes.resize((size_t)clp_find_above(u, h->m, 0.0, nodes.data()));
  } else if (P.rounding == CLP_ROUND_DSD_HEU) {
    const int omega = (int)std::round(so.F);
    if (omega >= 1) {
      nodes.resize((size_t)std::min<long long>(omega, h->m));
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
      if (h->storage == CLP_STORE_F64) gather_subblock_kernel<double><<<g, 128, 0, h->stream>>>(h->Mbuf.as<double>(), h->ld, S_d, k, sub_d);
      else gather_subblock_kernel<float><<<g, 128, 0, h->stream>>>(h->Mbuf.as<float>(), h->ld, S_d, k, sub_d);
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
  if (storage != CLP_STORE_F32 && storage != CLP_STORE_F64) return fail(nullptr, CLP_ERR_INVALID, "unknown storage type");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return fail(nullptr, CLP_ERR_CUDA, std::string("no usable CUDA device: ") + cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return fail(nullptr, CLP_ERR_INVALID, "device ordinal out of range");
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return fail(nullptr, CLP_ERR_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, CLP_ERR_CUDA, "clipper_b200 is built for sm_90a only; device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
  if (!prop.cooperativeLaunch) return fail(nullptr, CLP_ERR_CUDA, "device lacks cooperative launch");
  clp_handle h = new (std::nothrow) clp_handle_s();
  if (!h) return fail(nullptr, CLP_ERR_ALLOC, "host allocation failed");
  h->device = device; h->storage = storage; h->sm_count = prop.multiProcessorCount;
  clp_default_params(&h->prm);
  auto bail = [&](const char* what, cudaError_t ce) {
    g_create_error = std::string(what) + ": " + cudaGetErrorString(ce);
    clp_destroy(h);
    return CLP_ERR_CUDA;
  };
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
  for (DevBuf* b : {&h->Mbuf, &h->A_dev, &h->E1, &h->E2, &h->F12, &h->D1dev, &h->D2dev, &h->vecs, &h->llbuf, &h->d2buf, &h->plan2buf, &h->sp_val, &h->sp_col, &h->sp_ptr4, &h->sp_part, &h->sp_item, &h->sp_rowid, &h->parts, &h->small,
                    &h->result, &h->u0dev, &h->ybuf, &h->sync, &h->panel, &h->cscbuf, &h->res_vecs, &h->res_cand, &h->res_pieces, &h->res_redll, &h->prof_buf})
    b->release();
  if (h->pinned) cudaFreeHost(h->pinned);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->stream && h->own_stream) cudaStreamDestroy(h->stream);
  delete h;
  return CLP_OK;
}

const char* clp_last_error(clp_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

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
  return guarded(h, [&] { return score_from_host(h, 0, D1, d, n1, D2, n2, A, m, sigma, epsilon, mindist, 0.0); });
}
int clp_score_pointnormal(clp_handle h, const double* D1, int64_t n1, const double* D2, int64_t n2,
                          const int32_t* A, int64_t m, double sigp, double epsp, double sign, double epsn) {
  return guarded(h, [&] { return score_from_host(h, 1, D1, 6, n1, D2, n2, A, m, sigp, epsp, sign, epsn); });
}
int clp_score_euclidean_dev(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2,
                            const int32_t* A, int64_t m, double sigma, double epsilon, double mindist) {
  return guarded(h, [&] { return score_from_device(h, 0, D1, d, n1, D2, n2, A, m, sigma, epsilon, mindist, 0.0); });
}
int clp_score_pointnormal_dev(clp_handle h, const double* D1, int64_t n1, const double* D2, int64_t n2,
                              const int32_t* A, int64_t m, double sigp, double epsp, double sign, double epsn) {
  return guarded(h, [&] { return score_from_device(h, 1, D1, 6, n1, D2, n2, A, m, sigp, epsp, sign, epsn); });
}

// ---- get / set ----------------------------------------------------------------------------
int clp_set_dense(clp_handle h, const double* M, const double* C, int64_t m) {
  if (!h || !M || !C) return CLP_ERR_INVALID;
  h->counts_fused = false;
  if (int rc = ensure_matrix(h, m)) return rc;
  h->has_A = false; h->A_host_valid = false;
  if (int rc = reset_sync(h)) return rc;
  SyncBlock* sb = h->sync.as<SyncBlock>();
  const size_t total = (size_t)h->rows_pad * (size_t)h->ld;
  if (h->storage == CLP_STORE_F64) fill_neutral_kernel<double><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<double>(), total);
  else fill_neutral_kernel<float><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<float>(), total);
  CLP_CUDA(h, cudaGetLastError());
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
    if (h->storage == CLP_STORE_F64)
      encode_dense_panel_kernel<double><<<grid, 256, 0, h->stream>>>(Mp, Cp, (int)m, (int)j0, (int)j1, h->Mbuf.as<double>(), h->ld, h->row0, h->rows, &sb->flags);
    else
      encode_dense_panel_kernel<float><<<grid, 256, 0, h->stream>>>(Mp, Cp, (int)m, (int)j0, (int)j1, h->Mbuf.as<float>(), h->ld, h->row0, h->rows, &sb->flags);
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));  // the panel buffer is reused
  }
  SyncBlock host;
  if (int rc = read_sync(h, &host)) return rc;
  if (host.flags & 1) return fail(h, CLP_ERR_UNSUPPORTED, "affinity matrix has negative entries (contract: M in [0,1], ref clipper.h:166-171)");
  if (host.flags & 2) return fail(h, CLP_ERR_UNSUPPORTED, "constraint matrix is not binary (contract: ref clipper.h:176)");
  if (int rc = finalize_matrix(h)) return rc;
  h->has_matrix = true;
  return CLP_OK;
}

int clp_set_sparse_upper(clp_handle h, int64_t m, const int64_t* cpM, const int32_t* riM, const double* vM,
                         const int64_t* cpC, const int32_t* riC, const double* vC) {
  if (!h || !cpM || !cpC) return CLP_ERR_INVALID;
  h->counts_fused = false;
  if (int rc = ensure_matrix(h, m)) return rc;
  h->has_A = false; h->A_host_valid = false;
  if (int rc = reset_sync(h)) return rc;
  SyncBlock* sb = h->sync.as<SyncBlock>();
  const size_t total = (size_t)h->rows_pad * (size_t)h->ld;
  if (h->storage == CLP_STORE_F64) fill_neutral_kernel<double><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<double>(), total);
  else fill_neutral_kernel<float><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<float>(), total);
  CLP_CUDA(h, cudaGetLastError());
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
    if (h->storage == CLP_STORE_F64) {
      if (which == 0) scatter_csc_M_kernel<double><<<(unsigned)m, 128, 0, h->stream>>>(cp_d, ri_d, v_d, (int)m, h->Mbuf.as<double>(), h->ld, h->row0, h->rows, &sb->flags);
      else scatter_csc_C_kernel<double><<<(unsigned)m, 128, 0, h->stream>>>(cp_d, ri_d, v_d, (int)m, h->Mbuf.as<double>(), h->ld, h->row0, h->rows, &sb->flags);
    } else {
      if (which == 0) scatter_csc_M_kernel<float><<<(unsigned)m, 128, 0, h->stream>>>(cp_d, ri_d, v_d, (int)m, h->Mbuf.as<float>(), h->ld, h->row0, h->rows, &sb->flags);
      else scatter_csc_C_kernel<float><<<(unsigned)m, 128, 0, h->stream>>>(cp_d, ri_d, v_d, (int)m, h->Mbuf.as<float>(), h->ld, h->row0, h->rows, &sb->flags);
    }
    CLP_CUDA(h, cudaGetLastError());
    CLP_CUDA(h, cudaStreamSynchronize(h->stream));
  }
  SyncBlock host;
  if (int rc = read_sync(h, &host)) return rc;
  if (host.flags & 4) return fail(h, CLP_ERR_INVALID, "sparse input is not strictly upper triangular (ref clipper.h:137-138)");
  if (host.flags & 1) return fail(h, CLP_ERR_UNSUPPORTED, "affinity matrix has negative entries");
  if (host.flags & 2) return fail(h, CLP_ERR_UNSUPPORTED, "constraint matrix is not binary");
  if (int rc = finalize_matrix(h)) return rc;
  h->has_matrix = true;
  return CLP_OK;
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
    if (h->storage == CLP_STORE_F64) decode_dense_panel_kernel<double><<<grid, 256, 0, h->stream>>>(h->Mbuf.as<double>(), h->ld, (int)m, (int)j0, (int)j1, which, P);
    else decode_dense_panel_kernel<float><<<grid, 256, 0, h->stream>>>(h->Mbuf.as<float>(), h->ld, (int)m, (int)j0, (int)j1, which, P);
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
  if (h->storage == CLP_STORE_F64) count_upper_kernel<double><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<double>(), h->ld, (int)h->m, h->row0, h->rows, sb->counts);
  else count_upper_kernel<float><<<h->sm_count * 8, 256, 0, h->stream>>>(h->Mbuf.as<float>(), h->ld, (int)h->m, h->row0, h->rows, sb->counts);
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
  double* stage = reinterpret_cast<double*>(reinterpret_cast<char*>(h->pinned) + 256);
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
  if (h->m > 0) {
    CLP_CUDA(h, cudaSetDevice(h->device));
    if (h->has_matrix) { if (int rc = finalize_matrix(h)) return rc; }
    else { if (int rc = set_plan_for(h, h->dense_mode == 3 || h->dense_mode == 4 ? 3 : h->dense_mode)) return rc; }
  }
  return CLP_OK;
}

int clp_set_ctas_per_sm(clp_handle h, int n) {
  if (!h || n < 1 || n > 3) return fail(h, CLP_ERR_INVALID, "ctas_per_sm must be 1, 2 or 3");
  h->ctas_cap = n;
  if (h->m > 0) {
    CLP_CUDA(h, cudaSetDevice(h->device));
    if (h->has_matrix) { if (int rc = finalize_matrix(h)) return rc; }
    else { if (int rc = set_plan_for(h, h->dense_mode == 3 || h->dense_mode == 4 ? 3 : h->dense_mode)) return rc; }
  }
  return CLP_OK;
}

int clp_sparse_info(clp_handle h, int64_t* nnz_kept, int64_t* bytes_per_pass) {
  if (!h) return CLP_ERR_INVALID;
  if (nnz_kept) *nnz_kept = (int64_t)h->sp_nnz_real;
  if (bytes_per_pass)
    *bytes_per_pass = (int64_t)(h->sp_nnz * h->entry_bytes() +
                                (unsigned long long)(h->rows_pad / 4) * (h->compact_resident ? 1 : h->plan.NSEG) * 20);
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
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  clp_params prm;
  std::string err;
  int sm_count = 0, smem_optin = 0;
  DevBuf in_d1, in_d2, in_a, in_u0, out_u, probs, outs, nnz, sync, scratch, prof;
  int prof_on = env_int("CLP_PROF_BATCH", 0);
  void* pinned = nullptr; size_t pinned_cap = 0;
  int last_ctas = 0; long long last_scratch = 0, last_nnz = 0;
};

namespace {
thread_local std::string g_batch_create_error;
int bfail(clp_batch b, int code, const std::string& msg) {
  if (b) b->err = msg; else g_batch_create_error = msg;
  return code;
}
#define CLP_BCUDA(b, call)                                                                 \
  do {                                                                                     \
    cudaError_t e__ = (call);                                                              \
    if (e__ != cudaSuccess)                                                                \
      return bfail(b, e__ == cudaErrorMemoryAllocation ? CLP_ERR_ALLOC : CLP_ERR_CUDA,     \
                   std::string(#call) + ": " + cudaGetErrorString(e__));                   \
  } while (0)

template <int KIND, int DD>
int batch_launch(clp_batch b, BatchArgs& ba, int grid, size_t smem) {
  CLP_BCUDA(b, cudaFuncSetAttribute(batch_solve_kernel<KIND, DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  batch_solve_kernel<KIND, DD><<<grid, kBatchThreads, smem, b->stream>>>(ba);
  CLP_BCUDA(b, cudaGetLastError());
  return CLP_OK;
}
template <int KIND, int DD>
int batch_occupancy(clp_batch b, size_t smem, int* occ) {
  CLP_BCUDA(b, cudaFuncSetAttribute(batch_solve_kernel<KIND, DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CLP_BCUDA(b, cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, batch_solve_kernel<KIND, DD>, kBatchThreads, smem));
  return CLP_OK;
}

int batch_solve(clp_batch b, int kind, int dd, int32_t nprob, const double* const* D1, const int64_t* n1,
                const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                const double* const* u0, double p0, double p1, double p2, double p3, clp_solution* sols,
                double* const* u_out, int32_t* const* nodes_out) {
  if (!b) return CLP_ERR_INVALID;
  if (nprob <= 0 || !D1 || !n1 || !D2 || !n2 || !m || !u0 || !sols) return bfail(b, CLP_ERR_INVALID, "bad batch arguments");
  if (!((kind == 0 && (dd == 2 || dd == 3)) || (kind == 1 && dd == 6)))
    return bfail(b, CLP_ERR_UNSUPPORTED, "batched scoring supports EuclideanDistance with d = 2, 3 and PointNormalDistance");
  const clp_params& P = b->prm;
  if (P.rounding == CLP_ROUND_DSD) return bfail(b, CLP_ERR_UNSUPPORTED, "Rounding::DSD is not available in a batch");
  if (P.maxlsiters < 1) return bfail(b, CLP_ERR_INVALID, "maxlsiters must be >= 1");
  const auto t_begin = std::chrono::steady_clock::now();
  CLP_BCUDA(b, cudaSetDevice(b->device));
  // ---- problem table and concatenated inputs
  std::vector<BatchProblem> probs((size_t)nprob);
  long long nd1 = 0, nd2 = 0, na = 0, nu = 0;
  int max_m = 1;
  for (int p = 0; p < nprob; ++p) {
    BatchProblem& q = probs[(size_t)p];
    if (!D1[p] || !D2[p] || !u0[p] || n1[p] <= 0 || n2[p] <= 0) return bfail(b, CLP_ERR_INVALID, "bad problem in the batch (null data or u0)");
    const bool a2a = (A == nullptr || A[p] == nullptr || m[p] == 0);
    const long long mp = a2a ? (long long)n1[p] * n2[p] : (long long)m[p];
    if (mp <= 0 || mp > kBatchMaxM) return bfail(b, CLP_ERR_INVALID, "batched problems need 1 <= m <= 4096 associations");
    q.d1_off = nd1; q.d2_off = nd2; q.a_off = a2a ? -1 : na; q.u_off = nu;
    q.n1 = (int)n1[p]; q.n2 = (int)n2[p]; q.m = (int)mp; q.pad_ = 0;
    nd1 += (long long)dd * n1[p]; nd2 += (long long)dd * n2[p]; if (!a2a) na += 2 * mp;
    nu += (mp + 1) & ~1LL;  // every problem's u0 / u slot starts on a 16-byte boundary (the kernels use 16-byte loads)
    max_m = std::max(max_m, (int)mp);
  }
  const size_t bytes_in = (size_t)(nd1 + nd2 + nu) * 8 + (size_t)na * 4 + (size_t)nprob * sizeof(BatchProblem);
  const size_t bytes_out = (size_t)nu * 8 + (size_t)nprob * (sizeof(SolverOut) + 4);
  const size_t need = std::max(bytes_in, bytes_out) + 4096;
  if (need > b->pinned_cap) {
    if (b->pinned) { cudaFreeHost(b->pinned); b->pinned = nullptr; b->pinned_cap = 0; }
    CLP_BCUDA(b, cudaMallocHost(&b->pinned, need));
    b->pinned_cap = need;
  }
  char* hp = reinterpret_cast<char*>(b->pinned);
  double* h_d1 = reinterpret_cast<double*>(hp);
  double* h_d2 = h_d1 + nd1;
  double* h_u0 = h_d2 + nd2;
  int32_t* h_a = reinterpret_cast<int32_t*>(h_u0 + nu);
  BatchProblem* h_pr = reinterpret_cast<BatchProblem*>(reinterpret_cast<char*>(h_a) + (((size_t)na * 4 + 15) & ~(size_t)15));
  for (int p = 0; p < nprob; ++p) {
    const BatchProblem& q = probs[(size_t)p];
    std::memcpy(h_d1 + q.d1_off, D1[p], (size_t)dd * q.n1 * 8);
    std::memcpy(h_d2 + q.d2_off, D2[p], (size_t)dd * q.n2 * 8);
    std::memcpy(h_u0 + q.u_off, u0[p], (size_t)q.m * 8);
    if (q.a_off >= 0) std::memcpy(h_a + q.a_off, A[p], (size_t)2 * q.m * 4);
  }
  std::memcpy(h_pr, probs.data(), (size_t)nprob * sizeof(BatchProblem));
  CLP_BCUDA(b, b->in_d1.ensure((size_t)nd1 * 8 + 16));
  CLP_BCUDA(b, b->in_d2.ensure((size_t)nd2 * 8 + 16));
  CLP_BCUDA(b, b->in_u0.ensure((size_t)nu * 8 + 16));
  CLP_BCUDA(b, b->in_a.ensure((size_t)na * 4 + 16));
  CLP_BCUDA(b, b->out_u.ensure((size_t)nu * 8 + 16));
  CLP_BCUDA(b, b->probs.ensure((size_t)nprob * sizeof(BatchProblem)));
  CLP_BCUDA(b, b->outs.ensure((size_t)nprob * sizeof(SolverOut)));
  CLP_BCUDA(b, b->nnz.ensure((size_t)nprob * 4 + 16));
  CLP_BCUDA(b, cudaMemcpyAsync(b->in_d1.p, h_d1, (size_t)nd1 * 8, cudaMemcpyHostToDevice, b->stream));
  CLP_BCUDA(b, cudaMemcpyAsync(b->in_d2.p, h_d2, (size_t)nd2 * 8, cudaMemcpyHostToDevice, b->stream));
  CLP_BCUDA(b, cudaMemcpyAsync(b->in_u0.p, h_u0, (size_t)nu * 8, cudaMemcpyHostToDevice, b->stream));
  if (na) CLP_BCUDA(b, cudaMemcpyAsync(b->in_a.p, h_a, (size_t)na * 4, cudaMemcpyHostToDevice, b->stream));
  CLP_BCUDA(b, cudaMemcpyAsync(b->probs.p, h_pr, (size_t)nprob * sizeof(BatchProblem), cudaMemcpyHostToDevice, b->stream));
  CLP_BCUDA(b, cudaMemsetAsync(b->nnz.p, 0, (size_t)nprob * 4 + 16, b->stream));
  CLP_BCUDA(b, cudaMemsetAsync(b->outs.p, 0, (size_t)nprob * sizeof(SolverOut), b->stream));
  CLP_BCUDA(b, cudaMemsetAsync(b->sync.p, 0, sizeof(SyncBlock), b->stream));
  // ---- grid: as many CTAs as are co-resident (and as there are problems), each with its own scratch slot
  const BatchSmem bs = batch_smem_plan(max_m);
  if ((long long)bs.total > (long long)b->smem_optin) return bfail(b, CLP_ERR_UNSUPPORTED, "batch: shared memory plan exceeds the device limit");
  int occ = 0;
  int rc = (kind == 1) ? batch_occupancy<1, 6>(b, bs.total, &occ) : (dd == 3 ? batch_occupancy<0, 3>(b, bs.total, &occ) : batch_occupancy<0, 2>(b, bs.total, &occ));
  if (rc) return rc;
  if (occ < 1) return bfail(b, CLP_ERR_CUDA, "batch kernel does not fit an SM");
  const BatchLayout L = batch_layout(max_m, dd);
  size_t free_b = 0, total_b = 0;
  CLP_BCUDA(b, cudaMemGetInfo(&free_b, &total_b));
  const long long by_mem = (long long)((double)(free_b + b->scratch.cap) * 0.8 / (double)L.total);
  int grid = (int)std::max<long long>(1, std::min<long long>(std::min<long long>(nprob, (long long)occ * b->sm_count), by_mem));
  CLP_BCUDA(b, b->scratch.ensure((size_t)grid * L.total));
  BatchArgs ba;
  std::memset(&ba, 0, sizeof(ba));
  ba.prob = b->probs.as<BatchProblem>(); ba.nprob = nprob;
  ba.D1 = b->in_d1.as<double>(); ba.D2 = b->in_d2.as<double>(); ba.A = b->in_a.as<int>(); ba.u0 = b->in_u0.as<double>();
  ba.u_out = b->out_u.as<double>(); ba.out = b->outs.as<SolverOut>(); ba.nnz_out = b->nnz.as<unsigned int>();
  ba.next = reinterpret_cast<int*>(&b->sync.as<SyncBlock>()->counts[0]);
  ba.scratch = b->scratch.as<unsigned char>(); ba.scratch_stride = L.total;
  ba.max_m = max_m; ba.kind = kind; ba.dd = dd;
  ba.prm.tol_u = P.tol_u; ba.prm.tol_F = P.tol_F; ba.prm.beta = P.beta; ba.prm.eps = P.eps;
  ba.prm.maxiniters = P.maxiniters; ba.prm.maxoliters = P.maxoliters; ba.prm.maxlsiters = P.maxlsiters;
  ba.prm.rescale_u0 = P.rescale_u0 ? 1 : 0;
  ba.p0 = p0; ba.p1 = p1; ba.p2 = p2; ba.p3 = p3; ba.affinityeps = P.affinityeps;
  ba.sb = b->sync.as<SyncBlock>(); ba.spin_limit = 4LL * 1900000000LL;
  if (b->prof_on) { CLP_BCUDA(b, b->prof.ensure((size_t)nprob * 4 * sizeof(unsigned long long))); ba.prof = b->prof.as<unsigned long long>(); }
  CLP_BCUDA(b, cudaEventRecord(b->ev0, b->stream));
  rc = (kind == 1) ? batch_launch<1, 6>(b, ba, grid, bs.total) : (dd == 3 ? batch_launch<0, 3>(b, ba, grid, bs.total) : batch_launch<0, 2>(b, ba, grid, bs.total));
  if (rc) return rc;
  CLP_BCUDA(b, cudaEventRecord(b->ev1, b->stream));
  // ---- results
  double* h_u = reinterpret_cast<double*>(hp);
  SolverOut* h_out = reinterpret_cast<SolverOut*>(h_u + nu);
  unsigned int* h_nnz = reinterpret_cast<unsigned int*>(h_out + nprob);
  SyncBlock h_sb;
  CLP_BCUDA(b, cudaMemcpyAsync(h_u, b->out_u.p, (size_t)nu * 8, cudaMemcpyDeviceToHost, b->stream));
  CLP_BCUDA(b, cudaMemcpyAsync(h_out, b->outs.p, (size_t)nprob * sizeof(SolverOut), cudaMemcpyDeviceToHost, b->stream));
  CLP_BCUDA(b, cudaMemcpyAsync(h_nnz, b->nnz.p, (size_t)nprob * 4, cudaMemcpyDeviceToHost, b->stream));
  CLP_BCUDA(b, cudaMemcpyAsync(&h_sb, b->sync.p, sizeof(SyncBlock), cudaMemcpyDeviceToHost, b->stream));
  CLP_BCUDA(b, cudaStreamSynchronize(b->stream));
  float ms = 0.f;
  CLP_BCUDA(b, cudaEventElapsedTime(&ms, b->ev0, b->ev1));
  if (b->prof_on) {
    std::vector<unsigned long long> pr((size_t)nprob * 4);
    CLP_BCUDA(b, cudaMemcpy(pr.data(), b->prof.p, pr.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    double acc[4] = {0, 0, 0, 0};
    for (int p = 0; p < nprob; ++p) for (int q = 0; q < 4; ++q) acc[q] += 1e-6 * (double)pr[(size_t)p * 4 + q];
    std::fprintf(stderr, "[clp batch prof] %d problems (max m %d), %d CTAs, kernel %.3f ms; mean per problem: score %.3f  build %.3f  solve %.3f  total %.3f ms\n",
                 nprob, max_m, grid, ms, acc[0] / nprob, acc[1] / nprob, acc[2] / nprob, acc[3] / nprob);
  }
  if (h_sb.error == 2) return bfail(b, CLP_ERR_INVALID, "association index out of range of D1/D2 in a batched problem");
  if (h_sb.error != 0) return bfail(b, CLP_ERR_TIMEOUT, "batch kernel: an in-kernel wait timed out");
  b->last_ctas = grid; b->last_scratch = (long long)grid * (long long)L.total; b->last_nnz = 0;
  std::vector<int32_t> nodes;
  for (int p = 0; p < nprob; ++p) {
    const BatchProblem& q = probs[(size_t)p];
    const SolverOut& so = h_out[p];
    const double* u = h_u + q.u_off;
    b->last_nnz += h_nnz[p] / 2;
    nodes.clear();
    if (P.rounding == CLP_ROUND_NONZERO) {
      nodes.resize((size_t)q.m);
      nodes.resize((size_t)clp_find_above(u, q.m, 0.0, nodes.data()));
    } else {  // DSD_HEU, ref clipper.cpp:302-308
      const int omega = (int)std::round(so.F);
      if (omega >= 1) {
        nodes.resize((size_t)std::min<long long>(omega, q.m));
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
  const double wall = std::chrono::duration<double>(std::chrono::steady_clock::now() - t_begin).count();
  for (int p = 0; p < nprob; ++p) sols[p].t = wall / nprob;
  return CLP_OK;
}
}  // namespace

extern "C" {

int clp_batch_create(int device, clp_batch* out) {
  if (!out) return CLP_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) return bfail(nullptr, CLP_ERR_CUDA, std::string("no usable CUDA device: ") + cudaGetErrorString(e));
  if (device < 0 || device >= ndev) return bfail(nullptr, CLP_ERR_INVALID, "device ordinal out of range");
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bfail(nullptr, CLP_ERR_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0) return bfail(nullptr, CLP_ERR_CUDA, "clipper_b200 is built for sm_90a only");
  clp_batch b = new (std::nothrow) clp_batch_s();
  if (!b) return bfail(nullptr, CLP_ERR_ALLOC, "host allocation failed");
  b->device = device; b->sm_count = prop.multiProcessorCount;
  clp_default_params(&b->prm);
  auto bail = [&](const char* what, cudaError_t ce) {
    g_batch_create_error = std::string(what) + ": " + cudaGetErrorString(ce);
    clp_batch_destroy(b);
    return CLP_ERR_CUDA;
  };
  if ((e = cudaSetDevice(device)) != cudaSuccess) return bail("cudaSetDevice", e);
  if ((e = cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
  if ((e = cudaEventCreate(&b->ev0)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = cudaEventCreate(&b->ev1)) != cudaSuccess) return bail("cudaEventCreate", e);
  if ((e = b->sync.ensure(sizeof(SyncBlock))) != cudaSuccess) return bail("cudaMalloc", e);
  if ((e = cudaDeviceGetAttribute(&b->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device)) != cudaSuccess) return bail("cudaDeviceGetAttribute", e);
  *out = b;
  return CLP_OK;
}

int clp_batch_destroy(clp_batch b) {
  if (!b) return CLP_OK;
  cudaSetDevice(b->device);
  for (DevBuf* d : {&b->in_d1, &b->in_d2, &b->in_a, &b->in_u0, &b->out_u, &b->probs, &b->outs, &b->nnz, &b->sync, &b->scratch, &b->prof}) d->release();
  if (b->pinned) cudaFreeHost(b->pinned);
  if (b->ev0) cudaEventDestroy(b->ev0);
  if (b->ev1) cudaEventDestroy(b->ev1);
  if (b->stream) cudaStreamDestroy(b->stream);
  delete b;
  return CLP_OK;
}

const char* clp_batch_last_error(clp_batch b) { return b ? b->err.c_str() : g_batch_create_error.c_str(); }

int clp_batch_set_params(clp_batch b, const clp_params* p) {
  if (!b || !p) return CLP_ERR_INVALID;
  if (p->rounding < 0 || p->rounding > 2) return bfail(b, CLP_ERR_INVALID, "unknown rounding mode");
  b->prm = *p;
  return CLP_OK;
}

int clp_batch_solve_euclidean(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                              const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                              const double* const* u0, double sigma, double epsilon, double mindist,
                              clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  try { return batch_solve(b, 0, d, nprob, D1, n1, D2, n2, A, m, u0, sigma, epsilon, mindist, 0.0, sols, u_out, nodes_out); }
  catch (const std::bad_alloc&) { return bfail(b, CLP_ERR_ALLOC, "host allocation failed"); }
  catch (...) { return bfail(b, CLP_ERR_INVALID, "internal error"); }
}

int clp_batch_solve_pointnormal(clp_batch b, int32_t nprob, const double* const* D1, const int64_t* n1,
                                const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                const double* const* u0, double sigp, double epsp, double sign, double epsn,
                                clp_solution* sols, double* const* u_out, int32_t* const* nodes_out) {
  try { return batch_solve(b, 1, 6, nprob, D1, n1, D2, n2, A, m, u0, sigp, epsp, sign, epsn, sols, u_out, nodes_out); }
  catch (const std::bad_alloc&) { return bfail(b, CLP_ERR_ALLOC, "host allocation failed"); }
  catch (...) { return bfail(b, CLP_ERR_INVALID, "internal error"); }
}

int clp_batch_info(clp_batch b, int32_t* n_ctas, int64_t* scratch_bytes, int64_t* nnz_upper_total) {
  if (!b) return CLP_ERR_INVALID;
  if (n_ctas) *n_ctas = b->last_ctas;
  if (scratch_bytes) *scratch_bytes = b->last_scratch;
  if (nnz_upper_total) *nnz_upper_total = b->last_nnz;
  return CLP_OK;
}

}  // extern "C"
