/*
 * clipper_b200.h -- C-ABI of the H100-native (sm_90a) CLIPPER hot path.
 *
 * This is the drop-in seam: a maintainer of mit-acl/clipper binds THESE entry points from
 * the bodies of clipper::CLIPPER (see INTEGRATION.md and include/clipper/clipper.h, which is
 * exactly that shell).  Plain pointers and sizes only -- no Eigen, torch or CUDA types.
 *
 * Citations (file:line) are relative to the reference tree (mit-acl/clipper v0.2.4).
 *
 * Conventions (those of the reference, which is Eigen / column-major):
 *   D1, D2 : double, d x n, column-major  -> datum k is the d contiguous doubles at D + d*k
 *            (invariants::Data = Eigen::MatrixXd, include/clipper/invariants/abstract.h:19)
 *   A      : int32, m x 2, column-major   -> A(:,0) is m contiguous ints, then A(:,1)
 *            (Association = Eigen::Matrix<int,Dynamic,2>, include/clipper/types.h:18)
 *   M, C   : double, m x m, column-major, symmetric (Affinity/Constraint, types.h:19-20)
 *   u0, u  : double, length m
 * All functions return 0 on success and a CLP_ERR_* code otherwise; clp_last_error() gives
 * the message.  Nothing in this library aborts, exits or falls back to a CPU path: if no
 * sm_90 CUDA device (H100) is usable, clp_create() fails.
 * A handle is not thread-safe (like clipper::CLIPPER); distinct handles are independent.
 * Calls are synchronous: results are host-visible on return (the *_dev variants, which take
 * and return device pointers on the handle's stream, only enqueue work unless stated).
 */
#ifndef CLIPPER_B200_H_
#define CLIPPER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CLP_OK 0
#define CLP_ERR_INVALID 1     /* bad argument / shape / state                         */
#define CLP_ERR_CUDA 2        /* CUDA runtime error (message holds cudaGetErrorString) */
#define CLP_ERR_ALLOC 3       /* device or host allocation failed                     */
#define CLP_ERR_UNSUPPORTED 4 /* input outside the supported contract (e.g. M<0, non-binary C) */
#define CLP_ERR_TIMEOUT 5     /* an in-kernel barrier timed out (hang guard)           */
#define CLP_ERR_COMM 6        /* peer-memory / multi-GPU set-up error                  */

/* storage type of the dense affinity matrix in HBM */
#define CLP_STORE_F32 0 /* default: 4 B/entry, the only O(m^2) traffic of the solver   */
#define CLP_STORE_F64 1 /* 8 B/entry: bit-faithful fp64 affinities (strict-parity mode) */

/* Rounding, reference include/clipper/clipper.h:49-59 */
#define CLP_ROUND_NONZERO 0
#define CLP_ROUND_DSD 1
#define CLP_ROUND_DSD_HEU 2

typedef struct clp_handle_s* clp_handle;

/* POD mirror of clipper::Params, reference include/clipper/clipper.h:27-60 (same defaults) */
typedef struct clp_params {
  double tol_u;       /* 1e-8  */
  double tol_F;       /* 1e-9  */
  double tol_Fop;     /* 1e-10, declared by the reference but never read by its solver */
  int32_t maxiniters; /* 200   */
  int32_t maxoliters; /* 1000  */
  double beta;        /* 0.25  */
  int32_t maxlsiters; /* 99    */
  double eps;         /* 1e-9  */
  double affinityeps; /* 1e-4  */
  int32_t rescale_u0; /* 1     */
  int32_t rounding;   /* CLP_ROUND_DSD_HEU */
} clp_params;

/* POD mirror of clipper::Solution, reference include/clipper/clipper.h:65-73, plus counters.
 * u / u0 / nodes are returned through caller-allocated buffers of clp_solve(). */
typedef struct clp_solution {
  double t;          /* wall-clock seconds spent in the solve call (Solution::t)            */
  int32_t ifinal;    /* outer iterations before termination (Solution::ifinal)              */
  int32_t n_nodes;   /* number of selected nodes (Solution::nodes.size())                   */
  double score;      /* final objective F (Solution::score)                                 */
  double d_final;    /* final penalty d                                                      */
  int64_t n_evals;   /* line-search objective evaluations (clipper.cpp:238-242)              */
  int64_t n_matvec;  /* dense M passes executed on the device (= n_evals + 2)                */
  int64_t n_inner;   /* accepted projected-gradient steps                                    */
  double kernel_ms;  /* device time of the solver kernel, CUDA events on the handle's stream */
  /* in-kernel phase split seen by CTA 0 (globaltimer): dense passes over M (+ their barrier),
   * O(m) combine loops, partial-sum exchange (grid barrier + NVLink peer exchange if sharded) */
  double prof_matvec_ms, prof_combine_ms, prof_exchange_ms;
} clp_solution;

/* ---- lifetime ------------------------------------------------------------------------- */
/* device: CUDA ordinal.  storage: CLP_STORE_*.  Replaces the CLIPPER ctor (clipper.cpp:15-17). */
int clp_create(int device, int storage, clp_handle* out);
int clp_destroy(clp_handle h);
const char* clp_last_error(clp_handle h); /* h may be NULL: error of the last failed clp_create */
void clp_default_params(clp_params* p);
int clp_set_params(clp_handle h, const clp_params* p);
int clp_get_params(clp_handle h, clp_params* p);
/* Run on an existing cudaStream_t (e.g. torch's current stream); NULL -> handle-owned stream. */
int clp_set_stream(clp_handle h, void* cuda_stream);
/* library/compile info: "clipper_b200 <version> (sm_90a, ...)" */
const char* clp_version(void);

/* ---- K1: scorePairwiseConsistency (clipper.cpp:21-65) ----------------------------------- */
/* EuclideanDistance (src/invariants/euclidean_distance.cpp:13-31). A==NULL or m==0 ->
 * all-to-all hypothesis (utils.h:61-71), generated on the device (A never crosses PCIe; clp_get_associations
 * fetches it on demand). Host pointers; copies in, builds dense M/C in HBM. */
int clp_score_euclidean(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2,
                        int64_t n2, const int32_t* A, int64_t m, double sigma, double epsilon,
                        double mindist);
/* PointNormalDistance (src/invariants/pointnormal_distance.cpp:13-35); data are 6 x n. */
int clp_score_pointnormal(clp_handle h, const double* D1, int64_t n1, const double* D2, int64_t n2,
                          const int32_t* A, int64_t m, double sigp, double epsp, double sign,
                          double epsn);
/* Same, inputs already resident in HBM (device pointers, same layouts). A_dev == NULL: all-to-all hypothesis
 * (m is then ignored and becomes n1 * n2). */
int clp_score_euclidean_dev(clp_handle h, const double* D1_dev, int32_t d, int64_t n1,
                            const double* D2_dev, int64_t n2, const int32_t* A_dev, int64_t m,
                            double sigma, double epsilon, double mindist);
int clp_score_pointnormal_dev(clp_handle h, const double* D1_dev, int64_t n1, const double* D2_dev,
                              int64_t n2, const int32_t* A_dev, int64_t m, double sigp, double epsp,
                              double sign, double epsn);

/* A custom PairwiseInvariant (invariants/abstract.h:56-72) written in CUDA C++.  `source` defines
 *   __device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj,
 *                                   int d, const double* prm);
 * with ai = D1.col(A(i,0)), aj = D1.col(A(j,0)), bi = D2.col(A(i,1)), bj = D2.col(A(j,1)) (d doubles each) and prm
 * the nprm parameters (0 <= nprm <= CLP_INV_MAX_PARAMS; given on the host, read by the function from device memory).
 * The library calls it once per distinct pair with i < j, on every handle (sharded ones too), and stores the result
 * exactly as for the built-ins: pairs sharing an endpoint are skipped, a score is kept iff it is > affinityeps and
 * != 0 (NaN is dropped), M and C are symmetric.  Every pair takes the fp64 path (there is no fp32 screen).  The
 * function must terminate and stay in bounds; the library does not guard it (a fault is CLP_ERR_CUDA).  Kept scores
 * must be >= 0, the contract of M everywhere (clp_set_dense rejects a negative M); a kept negative score is not
 * detected, and its magnitude is stored.
 * The source is compiled at run time with NVRTC (sm_90a, -std=c++17, default precision flags) together with the
 * library's scoring kernel, once per (source, d, storage, sharded or not, device) in a process; later calls reuse the
 * kernel.  A source that does not compile returns CLP_ERR_INVALID with the compiler's log in clp_last_error, before
 * anything of the handle changes: the matrix it held stays as it was.  Other arguments as clp_score_euclidean(_dev). */
#define CLP_INV_MAX_PARAMS 16
int clp_score_custom(clp_handle h, const char* source, const double* prm, int32_t nprm, const double* D1, int32_t d,
                     int64_t n1, const double* D2, int64_t n2, const int32_t* A, int64_t m);
int clp_score_custom_dev(clp_handle h, const char* source, const double* prm, int32_t nprm, const double* D1_dev,
                         int32_t d, int64_t n1, const double* D2_dev, int64_t n2, const int32_t* A_dev, int64_t m);
/* Compiles `source` for dimension d as clp_score_custom would (no device needed, nothing loaded).  CLP_OK or
 * CLP_ERR_INVALID; the compiler's log (NUL-terminated, cut to log_bytes) goes to log, which may be NULL. */
int clp_invariant_check(const char* source, int32_t d, char* log, int64_t log_bytes);
/* run-time compilations of invariant sources in this process (clp_score_custom*, clp_batch_*_custom, clp_invariant_check)
 * and their total
 * wall-clock time in milliseconds; either pointer may be NULL */
int clp_jit_stats(int64_t* compiles, double* compile_ms);

/* ---- K7: matrix get/set (clipper.cpp:131-166) -------------------------------------------- */
/* setMatrixData: strict upper triangle of the column-major m x m inputs is used, diagonal and
 * lower triangle ignored (clipper.cpp:149-158). Contract: M >= 0, C in {0,1} (clipper.h:166-176). */
int clp_set_dense(clp_handle h, const double* M, const double* C, int64_t m);
/* setMatrixData from matrices already on the handle's device (e.g. torch tensors): entry (i, j) of M and C is
 * base[i * row_stride + j * col_stride] (element units; a torch tensor passes its own .stride(), a column-major caller
 * (1, ld)), of element type CLP_IN_F32 (float) or CLP_IN_F64 (double).  Only entries i < j are read.  An fp32 input x
 * is stored exactly as the fp64 value (double)x would be.  One stride must be 1 and the other >= 1; a bad stride, a NULL
 * pointer or an unknown dtype is CLP_ERR_INVALID.  Otherwise the call behaves as clp_set_dense: same checks, error codes
 * and messages, same compact layout, same state after a failure.  Runs on the handle's stream (clp_set_stream) and
 * returns when the load and the build are done.  A sharded handle returns CLP_ERR_UNSUPPORTED. */
#define CLP_IN_F32 0
#define CLP_IN_F64 1
int clp_set_dense_dev(clp_handle h, const void* M_dev, const void* C_dev, int64_t m, int dtype, int64_t row_stride,
                      int64_t col_stride);
/* setSparseMatrixData: strictly-upper CSC (column-major compressed) of M and of C (clipper.h:137). */
int clp_set_sparse_upper(clp_handle h, int64_t m, const int64_t* colptrM, const int32_t* rowidxM,
                         const double* valM, const int64_t* colptrC, const int32_t* rowidxC,
                         const double* valC);
/* getAffinityMatrix (which=0) / getConstraintMatrix (which=1): sym + I, column-major m x m. */
int clp_get_dense(clp_handle h, int which, double* out);
int clp_num_associations(clp_handle h, int64_t* m);
/* getInitialAssociations (clipper.cpp:117-120): column-major m x 2; error if none were scored. */
int clp_get_associations(clp_handle h, int32_t* A);
/* number of stored affinities (i<j, M_ij != 0) and constraints (C_ij = 1), for density reports */
int clp_count_nonzeros(clp_handle h, int64_t* nnzM_upper, int64_t* nnzC_upper);

/* ---- K2..K6: solve (clipper.cpp:69-78,172-323) -------------------------------------------- */
/* u0: m doubles or NULL (then U[0,1) from std::random_device like utils.cpp:22-29).
 * u_out (m doubles), u0_out (m doubles) and nodes_out (m int32) may be NULL.
 * Rounding NONZERO and DSD_HEU run on the device-produced u exactly as utils.cpp:33-68;
 * DSD pulls the support(u) sub-block of M and runs an exact densest-subgraph on the host. */
int clp_solve(clp_handle h, const double* u0, clp_solution* out, double* u_out, int32_t* nodes_out,
              double* u0_out);
/* u0 resident in HBM (device pointer, required). u_out_dev (device, m doubles) may be NULL.
 * Blocking: the solution scalars and nodes are host-visible on return. */
int clp_solve_dev(clp_handle h, const double* u0_dev, clp_solution* out, double* u_out_dev,
                  int32_t* nodes_out);

/* ---- K2 exposed: one penalised mat-vec ------------------------------------------------- */
/* y = (1+d) v - d (sum v) 1 + Mhat v + d Chat v  == Md v with Md = M - d(11' - C), unit
 * diagonals (clipper.cpp:219; matlab/clipper.m:69-70,93).  Mv/Cv (may be NULL) receive the
 * off-diagonal products Mhat v and Chat v.  Host pointers. */
int clp_matvec(clp_handle h, const double* v, double d, double* y, double* Mv, double* Cv);
/* Device pointers; enqueues reps back-to-back launches on the handle's stream and reports the
 * mean device time per launch in *ms_per_launch (CUDA events).  Used by the c5 sweep. */
int clp_matvec_dev(clp_handle h, const double* v_dev, double d, double* y_dev, double* Mv_dev,
                   double* Cv_dev, int reps, double* ms_per_launch);

/* ---- utils kept callable from the host shell (src/utils.cpp) ------------------------------ */
void clp_k2ij(uint64_t k, uint64_t n, uint64_t* i, uint64_t* j);        /* utils.cpp:87-97  */
void clp_create_all_to_all(int64_t n1, int64_t n2, int32_t* A_colmajor); /* utils.h:61-71    */
int32_t clp_find_k_largest(const double* x, int64_t n, int32_t k, int32_t* out); /* utils.cpp:33-55 */
int32_t clp_find_above(const double* x, int64_t n, double thr, int32_t* out);    /* utils.cpp:59-68 */
/* exact densest subgraph restricted to S (dsd.cpp:274-320); A is dense column-major n x n */
int32_t clp_dsd_dense(const double* A, int64_t n, const int32_t* S, int32_t nS, int32_t* out);

/* ---- putative associations by nearest-neighbour matching (ref benchmarks/bm_utils.cpp:147-232) ----------------------
 * The association set A that scoring takes, built on the device by exact brute force (clp_knn.cuh).  D1 (d x n1) and D2
 * (d x n2) are fp64 in the layout of the scoring calls.  For query i of D1 and candidate j of D2
 *   sd(i, j) = sum_k (D1[k,i] - D2[k,j])^2, accumulated for k = 0 .. d-1 in order, every subtract, multiply and add
 *   rounded on its own (no FMA).  For d = 3 this is nanoflann's L2 tail loop; the reference's own bits depend on whether
 *   its compiler contracted that loop to FMAs.
 * Neighbours of i: the min(knn, n2) candidates of least (sd, j) in lexicographic order: on equal sd the lower j wins (the
 *   reference's order among ties is that of its tree walk), and knn > n2 gives n2 neighbours (the reference reads
 *   uninitialised memory there).  A NaN sd is never a neighbour (nanoflann's strict <), so a query may have fewer.
 * Radius: the pair (i, j) is kept when sd <= radius * radius (fp64, bm_utils.cpp:192,201): radius = inf gives plain kNN,
 *   a NaN radius keeps nothing.
 * Without 1-to-1 the rows come in the order i ascending, then neighbour rank.  With enforce_1to1 != 0 the kept pairs are
 *   grouped by c1 = j: each c1 keeps the c0 = i of least sd, the smallest c0 among equal ones (the reference keeps the
 *   first pushed), and the rows come in c1 ascending order.
 * A_out receives the m rows column-major with leading dimension m (c0 in A_out[0 .. m), c1 in A_out[m .. 2m)): the layout
 * clp_score_*_dev reads.  capacity (rows) must be at least n1 * min(knn, n2); *m receives m.  n1 = 0 or n2 = 0 gives
 * m = 0 (A_out may then be NULL).  The handle's device, stream (clp_set_stream) and error string are used; its matrix and
 * state stay as they were.  The call returns when m (and, for the host call, A_out) is available.
 * Errors: CLP_ERR_INVALID for a NULL m, knn < 1, d < 1, a negative n1 or n2 or a NULL cloud; then CLP_ERR_UNSUPPORTED for
 * knn > CLP_KNN_MAX_K, d > CLP_KNN_MAX_D or n1, n2 >= 2^31 - 1; then CLP_ERR_INVALID for capacity < n1 * min(knn, n2). */
#define CLP_KNN_MAX_K 32
#define CLP_KNN_MAX_D 64
int clp_correspondences(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2, int32_t knn,
                        double radius, int enforce_1to1, int32_t* A_out, int64_t capacity, int64_t* m);
/* D1_dev, D2_dev and A_dev on the handle's device; enqueued on the handle's stream, which is synchronised to read m. */
int clp_correspondences_dev(clp_handle h, const double* D1_dev, int32_t d, int64_t n1, const double* D2_dev, int64_t n2,
                            int32_t knn, double radius, int enforce_1to1, int32_t* A_dev, int64_t capacity, int64_t* m);

/* ---- multi-GPU: row-block sharding, one process (or one handle) per GPU ------------------- */
/* SURVEY 8e.  Rank r of `world` keeps rows [row0,row0+rows) x all columns of M in its HBM
 * (clp_shard_rows gives the partition; scoring needs no communication).  clp_solve*() then runs
 * ONE persistent kernel per GPU; the single exchange step per objective evaluation happens inside
 * that kernel through NVLink peer memory (P2P stores + release/acquire flags), so every rank
 * must call clp_solve*() collectively with the same u0.  Set-up order on every rank:
 *   clp_shard_config -> first scoring/set call (allocates) -> clp_shard_export ->
 *   [caller all-gathers the 256-byte blobs, e.g. torch.distributed] -> clp_shard_import. */
int clp_shard_config(clp_handle h, int rank, int world);
void clp_shard_rows(int64_t m, int rank, int world, int64_t* row0, int64_t* rows);
int64_t clp_shard_blob_bytes(void);
int clp_shard_export(clp_handle h, void* blob, int64_t blob_bytes, int64_t* written);
/* blobs: world blobs in rank order, blob_bytes_each apart (CUDA IPC between processes, plain
 * peer access when the exporting handle lives in the calling process). */
int clp_shard_import(clp_handle h, const void* blobs, int64_t blob_bytes_each, int world);
/* Cap on the CTAs of the persistent solver per SM (1..3; default: 2 for the dense sweeps, 3 for the
 * compact-row sweep). 1 lets two shards share one GPU, which is how the sharded path is exercised on
 * a single-GPU box. */
int clp_set_ctas_per_sm(clp_handle h, int n);
/* Cap on the TOTAL number of CTAs of the persistent solver / mat-vec kernels of this handle (0 = no cap: every SM).
 * With clp_set_ctas_per_sm(h, 1) it lets the persistent kernels of several shards be co-resident on ONE GPU (the
 * resident-vector kernel takes a whole SM's shared memory per CTA): the sharded code path on a single-GPU box. */
int clp_set_grid_cap(clp_handle h, int n_ctas);
/* How the solver / mat-vec sweep the matrix (the dense store always exists; getters read it):
 *   4 (default) auto: a compact copy (6, else 3) when the graph is sparse enough for it to move fewer bytes than the
 *     best dense sweep (x0.8), else 2 on an unsharded handle / 0 on a sharded one;
 *   6: compact copy + RESIDENT trial vector (m <= 27648): the non-neutral entries are packed as (fp32 value, 16-bit
 *     column index) into a sliced-ELL layout over whole rows (rows sorted by length, four at a time, interleaved in
 *     4-entry chunks); every CTA keeps the whole trial vector in shared memory and owns complete rows, so an
 *     objective evaluation needs ONE device-wide synchronisation (clp_resident.cuh); 4 bytes per kept entry (column
 *     delta + scaled value) for plain fp32 matrices on one GPU whose values span at most 15 binades, else 6 bytes;
 *   3: compact copy cut into column segments of <= 4096 (any m <= 262144): (fp32 value, 16-bit column offset),
 *     same sliced-ELL layout per segment, two device-wide synchronisations per evaluation (SURVEY 8f #3);
 *   2: column stripes, ONLY the upper triangle is read and every element is applied two-sidedly in-tile
 *     -> ~2 m^2 bytes per objective evaluation (fp32 storage), single GPU; a sharded handle runs 0 instead;
 *   0: column-segment decomposition, full matrix (4 m^2 bytes).
 * Any other mode (1, 5, ...) is rejected with CLP_ERR_INVALID. */
int clp_set_dense_mode(clp_handle h, int mode);
int clp_get_dense_mode(clp_handle h, int* requested, int* effective);
/* entries kept by the compact copy (all local rows) and the algorithmic bytes one sparse pass reads */
int clp_sparse_info(clp_handle h, int64_t* nnz_kept, int64_t* bytes_per_pass);
/* How the line-search evaluations of the last solve read the matrix.  counts[0..5]: evaluations that swept the whole
 * compact copy, that rebuilt the restricted copy (the entries of every row in the support S' of the trial vector, once
 * |S'| <= m / 4) and swept it, that swept the restricted copy only (the support stayed inside S'); the entries and the
 * padding entries those restricted sweeps read, summed over the solve; and how many of the full sweeps came after the
 * first rebuild.  Only the resident solver on a packed copy larger than the L2 cache, on one GPU, takes restricted
 * sweeps; every other solve reports all its evaluations as full. */
int clp_last_solve_sweeps(clp_handle h, int64_t* counts);

/* ---- maximum clique of the constraint graph (solveAsMaximumClique, clipper.cpp:82-97, maxclique.cpp:89-140) --------
 * The graph is C without its diagonal: {i,j} is an edge iff C_ij = 1 (the sign bit of the stored element is clear),
 * whatever M_ij is.  Methods keep the order of clipper::maxclique::Method:
 *   CLP_MC_EXACT: a maximum clique.  lb = size of the HEU clique, ub = max core + 1; lb == ub returns the HEU clique,
 *     else a branch-and-bound on the device searches for a larger one until it is proven or time_limit_s expires
 *     (then the best clique found is returned with proven = 0, timed_out = 1).  time_limit_s <= 0 returns the HEU
 *     clique without searching.  The search sizes its scratch from the max core: a max core above 8191 is
 *     CLP_ERR_UNSUPPORTED (KCORE and HEU have no such limit).  Once proven, the clique returned does not depend on
 *     the schedule (largest clique of the first search task, in the fixed task order, that holds one).
 *   CLP_MC_HEU: greedy clique from every seed v (K = {v}, P = N(v); repeatedly add the u in P of highest core number,
 *     ties to the lowest index, P &= N(u)); the largest K, ties to the smallest seed.
 *   CLP_MC_KCORE: every vertex whose core number equals the max core (an edgeless graph returns every vertex).
 * nodes_out (m int32) receives the nodes in ascending order (info->n_nodes of them); info may be NULL.  m = 1 gives
 * {0}.  A sharded handle returns CLP_ERR_UNSUPPORTED.  The bitset adjacency (m^2/8 bytes) is built on the first call
 * and dropped when a new matrix is scored or set. */
#define CLP_MC_EXACT 0
#define CLP_MC_HEU 1
#define CLP_MC_KCORE 2
typedef struct clp_mc_info {
  int32_t n_nodes;      /* size of the returned node set                                         */
  int32_t max_core;     /* largest core number                                                    */
  int32_t lower_bound;  /* size of the HEU clique (0 for KCORE)                                   */
  int32_t upper_bound;  /* max_core + 1                                                           */
  int32_t proven;       /* 1: the nodes are known to be a maximum clique (lb == ub, or the search completed) */
  int32_t timed_out;    /* 1: the search stopped at time_limit_s                                  */
  int64_t n_edges;      /* edges of the graph                                                     */
  int64_t n_branches;   /* branch-and-bound nodes expanded                                        */
  double t;             /* wall-clock seconds of the call                                         */
  double kernel_ms;     /* device time of all kernels of the call (CUDA events)                   */
  /* phase split (CUDA events): adjacency build (0 when reused), peel, heuristic, search */
  double adjacency_ms, peel_ms, heuristic_ms, search_ms;
} clp_mc_info;
int clp_max_clique(clp_handle h, int method, double time_limit_s, int32_t* nodes_out, clp_mc_info* info);
/* core number of every vertex of the same graph (m int32) */
int clp_core_numbers(clp_handle h, int32_t* core_out);

/* ---- batches of small problems: hundreds of registrations in ONE launch (SURVEY 8f rank 4) ------------------------
 * The reference's benchmark solves its m <= 2048 problems one after the other (benchmarks/main.cpp:254-270: a fresh
 * clipper::CLIPPER, scorePairwiseConsistency, solve per trial).  A batch handle takes the whole list: ONE CTA per
 * problem scores the pairs, builds the compact copy and runs findDenseClique without any device-wide synchronisation;
 * the CTAs of a persistent grid draw problems from a counter.  Every problem gives the result the single-problem
 * path gives for it (same kernels' arithmetic).  Rounding: NONZERO and DSD_HEU (the default); Rounding::DSD is not
 * available in a batch (CLP_ERR_UNSUPPORTED).  m <= 4096 per problem.
 * Arrays of nprob host pointers / sizes; A[p] == NULL -> all-to-all hypothesis for problem p; u0[p] must be given
 * (m[p] doubles).  sols[p] receives ifinal, score, d_final, n_evals, n_matvec, n_inner, n_nodes; u_out[p] (m[p] doubles)
 * and nodes_out[p] (m[p] int32) may be NULL pointers / NULL arrays.  kernel_ms of every sols[p] is the device time of
 * the whole batch launch, t the wall-clock time of the call divided by nprob. */
typedef struct clp_batch_s* clp_batch;
int clp_batch_create(int device, clp_batch* out);
int clp_batch_destroy(clp_batch b);
const char* clp_batch_last_error(clp_batch b); /* b may be NULL: error of the last failed clp_batch_create */
int clp_batch_set_params(clp_batch b, const clp_params* p);
int clp_batch_solve_euclidean(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                              const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                              const double* const* u0, double sigma, double epsilon, double mindist,
                              clp_solution* sols, double* const* u_out, int32_t* const* nodes_out);
int clp_batch_solve_pointnormal(clp_batch b, int32_t nprob, const double* const* D1, const int64_t* n1,
                                const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                const double* const* u0, double sigp, double epsp, double sign, double epsn,
                                clp_solution* sols, double* const* u_out, int32_t* const* nodes_out);
/* Problems given as matrices (the batched form of setSparseMatrixData, ref clipper.h:132-143): problem p is two
 * strictly-upper CSC matrices M and C of m[p] columns (colptr m[p] + 1 int64 from 0, rowidx int32, val double), exactly
 * as clp_set_sparse_upper takes them, and gets the result of an fp32 handle after clp_set_sparse_upper(h, m[p], ...) +
 * clp_solve(h, u0[p], ...) with the batch's parameters (affinityeps plays no part).  The input is checked on the host
 * before anything is uploaded, with clp_set_sparse_upper's predicates: CLP_ERR_INVALID for a bad structure (m[p]
 * outside [1, 4096], colptr not starting at 0 or decreasing, a row < 0 or >= its column, rows not strictly ascending
 * within a column -- duplicates included -- or a NULL u0[p]); then CLP_ERR_UNSUPPORTED for a negative M value, then
 * for a C value other than 0 and 1 (NaN included).  The first problem with an error of the first kind found is named
 * in clp_batch_last_error; the handle stays usable.  Outputs as for clp_batch_solve_*. */
int clp_batch_solve_matrices(clp_batch b, int32_t nprob, const int64_t* m,
                             const int64_t* const* colptrM, const int32_t* const* rowidxM, const double* const* valM,
                             const int64_t* const* colptrC, const int32_t* const* rowidxC, const double* const* valC,
                             const double* const* u0, clp_solution* sols, double* const* u_out, int32_t* const* nodes_out);
/* Run the batch's work on an existing cudaStream_t (e.g. torch's current stream); NULL -> handle-owned stream. */
int clp_batch_set_stream(clp_batch b, void* cuda_stream);
/* Problems given as dense matrices already on the batch's device (e.g. a torch tensor [nprob, m_max, m_max]): problem
 * p is the leading m[p] x m[p] block (m host array, 1 <= m[p] <= 4096), entry (i, j) at
 * base[p * batch_stride + i * row_stride + j * col_stride] of M_dev and C_dev (element units, type dtype: CLP_IN_F32 or
 * CLP_IN_F64).  Only the strict upper triangle of each block is read: not the padding, the diagonal or the lower
 * triangle.  u0 of problem p: m[p] doubles at u0_dev + p * u0_stride (device).  Problem p gets exactly what
 * clp_batch_solve_matrices gives for the same values (u, score, d_final, ifinal, n_evals, n_inner, nodes and the
 * kept-entry count of clp_batch_info).  u_out_dev (device, nullable) receives u of problem p at p * u_out_stride
 * (u_out_stride >= the largest m[p]); nodes_out as for clp_batch_solve_*.  Errors, in this order: CLP_ERR_INVALID for
 * bad sizes, pointers, strides (one of row_stride, col_stride is 1 and the other >= 1; batch_stride, u0_stride >= 1) or
 * dtype; CLP_ERR_UNSUPPORTED for Rounding::DSD; then, found on the device, CLP_ERR_UNSUPPORTED naming the lowest problem
 * with a negative M value, else the lowest with a C value other than 0 and 1 (NaN included).  A problem with bad values
 * is not solved, the other outputs of a failed call are unspecified, and the handle stays usable.  Runs on the batch's
 * stream (clp_batch_set_stream) and returns when the results are host-visible. */
int clp_batch_solve_dense_dev(clp_batch b, int32_t nprob, const int64_t* m, int dtype, const void* M_dev, const void* C_dev,
                              int64_t batch_stride, int64_t row_stride, int64_t col_stride, const double* u0_dev,
                              int64_t u0_stride, clp_solution* sols, double* u_out_dev, int64_t u_out_stride,
                              int32_t* const* nodes_out);
/* diagnostics of the last batch: CTAs of the launch, HBM scratch bytes, and the kept entries i<j over all problems
 * (entries whose stored affinity is non-zero or whose C bit is set; for scored problems: the stored affinities) */
int clp_batch_info(clp_batch b, int32_t* n_ctas, int64_t* scratch_bytes, int64_t* nnz_upper_total);

/* ---- batched maximum clique: many small graphs in a constant number of launches -----------------------------------
 * Problem p gets exactly what clp_max_clique returns on an fp32 handle holding the same graph (scored from the same
 * inputs with clp_batch_set_params' affinityeps; rounding plays no part): the same core numbers, max_core, n_edges,
 * lower and upper bounds, KCORE and HEU nodes, and -- when both are proven -- the same EXACT nodes.  m <= 4096 per
 * problem; scored problems take the arguments of clp_batch_solve_* (A[p] == NULL: all-to-all).
 * clp_batch_max_clique_graphs takes problem p's graph as a strictly-upper CSC pattern of m[p] columns (colptr[p]:
 * m[p] + 1 entries from 0, rowidx[p]: row < column); every listed pair is an edge.
 * The device work: one CTA per problem builds the adjacency, peels the k-cores, runs the heuristic and lists the
 * search tasks; for EXACT one launch then searches the tasks of all problems, drawn so that task k of every problem
 * comes before task k + 1 of any; one warp per improved problem replays its winner.  time_limit_s bounds the whole call
 * from its start; <= 0 returns the HEU cliques without searching (proven = lower_bound == upper_bound).  A problem
 * whose tasks all completed is proven whatever happened to the others; one whose tasks did not comes back with its
 * best clique, proven = 0, timed_out = 1.
 * infos[p] holds the fields of clp_mc_info for problem p; kernel_ms and the phase times are those of the whole batch
 * (adjacency_ms, peel_ms and heuristic_ms split the first launch by in-kernel time, search_ms covers the search and the
 * replays), t the wall-clock time of the call divided by nprob.  nodes_out[p] (m[p] int32, ascending) and core_out[p]
 * (m[p] int32 core numbers) may be NULL arrays or NULL entries.  CLP_ERR_INVALID: m > 4096, an unknown method, a CSC
 * entry with row >= column or out of range, association indices out of range.  CLP_ERR_ALLOC: the scratch does not
 * fit the free device memory. */
int clp_batch_max_clique_euclidean(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                                   const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                   double sigma, double epsilon, double mindist, int method, double time_limit_s,
                                   clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out);
int clp_batch_max_clique_pointnormal(clp_batch b, int32_t nprob, const double* const* D1, const int64_t* n1,
                                     const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                     double sigp, double epsp, double sign, double epsn, int method, double time_limit_s,
                                     clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out);
int clp_batch_max_clique_graphs(clp_batch b, int32_t nprob, const int64_t* m, const int64_t* const* colptr,
                                const int32_t* const* rowidx, int method, double time_limit_s, clp_mc_info* infos,
                                int32_t* const* nodes_out, int32_t* const* core_out);

/* ---- batches scored with a CUDA-source invariant (the batched form of clp_score_custom) ---------------------------
 * Problem p of a batch scored with `source` and its nprm parameters prm gets exactly what an fp32 handle gives after
 * clp_score_custom(h, source, prm, nprm, D1[p], d, n1[p], D2[p], n2[p], A[p], m[p]) with clp_batch_set_params'
 * affinityeps, then clp_solve (clp_batch_solve_custom; outputs, rounding and kernel_ms as for clp_batch_solve_*) or
 * clp_max_clique (clp_batch_max_clique_custom; outputs as for clp_batch_max_clique_*).  The function is called once per
 * distinct pair with i < j, as on the handle; the storage rules are the handle's.  One source, one d >= 1 and one
 * parameter set per call; m[p] <= 4096, A[p] == NULL: all-to-all.  The source is compiled (NVRTC) before anything is
 * uploaded or launched, once per (source, d, device) in a process (clp_jit_stats counts it).
 * The device work goes in rounds of as many problems as the batch has scratch slots (clp_batch_info's CTAs): the
 * run-time compiled scoring kernel fills their fp32 matrices using the whole device, then the nvcc-built kernel of the
 * built-in batches runs one CTA per problem from the stored matrix.  Rounds are enqueued back to back; each waits for
 * its slowest problem.  For the maximum clique, adjacency_ms, peel_ms and heuristic_ms split the rounds' time,
 * scoring included, by the prepare kernel's in-kernel time.
 * Errors, in this order: CLP_ERR_INVALID for an empty source, nprm outside [0, CLP_INV_MAX_PARAMS], bad sizes or
 * pointers, d < 1, m[p] outside [1, 4096] (and, for the maximum clique, an unknown method); CLP_ERR_UNSUPPORTED for
 * Rounding::DSD (solve only); CLP_ERR_INVALID with the compiler's log for a source that does not compile; then the checks
 * of the built-in batches (association indices out of range: CLP_ERR_INVALID).  The handle stays usable after any of
 * them. */
int clp_batch_solve_custom(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob, int32_t d,
                           const double* const* D1, const int64_t* n1, const double* const* D2, const int64_t* n2,
                           const int32_t* const* A, const int64_t* m, const double* const* u0,
                           clp_solution* sols, double* const* u_out, int32_t* const* nodes_out);
int clp_batch_max_clique_custom(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob, int32_t d,
                                const double* const* D1, const int64_t* n1, const double* const* D2, const int64_t* n2,
                                const int32_t* const* A, const int64_t* m, int method, double time_limit_s,
                                clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out);

/* ---- scored batches whose point clouds and associations are already on the batch's device -------------------------
 * The device twins of clp_batch_solve_* and clp_batch_max_clique_* (custom included), e.g. for torch tensors D1
 * [nprob, d, n1_max], D2 [nprob, d, n2_max] and A [nprob, m_max, 2].  pts describes them in element units; the sizes
 * stay on the host:
 *   coordinate k of point j of problem p: D1[p * d1_strides[0] + k * d1_strides[1] + j * d1_strides[2]] (D2 alike);
 *   association i of problem p: (A[p * a_strides[0] + i * a_strides[1]], A[p * a_strides[0] + i * a_strides[1] +
 *   a_strides[2]]); A == NULL: all-to-all for every problem, m[p] == 0: all-to-all for problem p.
 * Points are fp64 only and associations int32 only.  Coordinate, point, row and column strides must be >= 1; a batch
 * stride may be 0 (every problem reads the same cloud: a torch expand).  Nothing past n1[p], n2[p] or m[p] is read.
 * The solves take u0 of problem p as m[p] doubles at u0_dev + p * u0_stride (u0_stride >= 1) and write u to u_out_dev +
 * p * u_out_stride (device, nullable; u_out_stride >= the largest m); sols, infos, nodes_out and core_out are host
 * arrays as in the host calls.  Problem p gets exactly, bit for bit, what the host-pointer call gives for the same
 * values: u, score, d_final, ifinal, n_evals, n_inner and nodes, clp_batch_info's kept-entry count, and for the clique
 * the cores, bounds, proven flag and nodes.
 * Errors, in this order: CLP_ERR_INVALID for bad sizes (n1[p], n2[p] >= 1, m[p] >= 0, every problem's association count
 * in [1, 4096]), NULL pointers or bad strides; then the host calls' checks in their order (the invariant kind and d,
 * Rounding::DSD for the solves, the method for the clique, the source compile for custom); then, found on the device,
 * CLP_ERR_INVALID naming the lowest problem with an association index out of range.  After an error the other outputs
 * are unspecified and the handle stays usable.  Runs on the batch's stream (clp_batch_set_stream) and returns when the
 * results are host-visible. */
typedef struct clp_points_dev {
  const double* D1; int64_t d1_strides[3];
  const double* D2; int64_t d2_strides[3];
  const int32_t* A; int64_t a_strides[3];
  const int64_t* n1; const int64_t* n2; const int64_t* m; /* host arrays of nprob */
} clp_points_dev;
int clp_batch_solve_euclidean_dev(clp_batch b, int32_t nprob, int32_t d, const clp_points_dev* pts, const double* u0_dev,
                                  int64_t u0_stride, double sigma, double epsilon, double mindist, clp_solution* sols,
                                  double* u_out_dev, int64_t u_out_stride, int32_t* const* nodes_out);
int clp_batch_solve_pointnormal_dev(clp_batch b, int32_t nprob, const clp_points_dev* pts, const double* u0_dev,
                                    int64_t u0_stride, double sigp, double epsp, double sign, double epsn,
                                    clp_solution* sols, double* u_out_dev, int64_t u_out_stride, int32_t* const* nodes_out);
int clp_batch_solve_custom_dev(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob, int32_t d,
                               const clp_points_dev* pts, const double* u0_dev, int64_t u0_stride, clp_solution* sols,
                               double* u_out_dev, int64_t u_out_stride, int32_t* const* nodes_out);
int clp_batch_max_clique_euclidean_dev(clp_batch b, int32_t nprob, int32_t d, const clp_points_dev* pts, double sigma,
                                       double epsilon, double mindist, int method, double time_limit_s,
                                       clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out);
int clp_batch_max_clique_pointnormal_dev(clp_batch b, int32_t nprob, const clp_points_dev* pts, double sigp, double epsp,
                                         double sign, double epsn, int method, double time_limit_s, clp_mc_info* infos,
                                         int32_t* const* nodes_out, int32_t* const* core_out);
int clp_batch_max_clique_custom_dev(clp_batch b, const char* source, const double* prm, int32_t nprm, int32_t nprob,
                                    int32_t d, const clp_points_dev* pts, int method, double time_limit_s,
                                    clp_mc_info* infos, int32_t* const* nodes_out, int32_t* const* core_out);

/* ---- putative associations for a batch of cloud pairs (the batched form of clp_correspondences) --------------------
 * Problem p gets exactly what clp_correspondences gives for (D1_p, n1[p], D2_p, n2[p]) with the call's d, knn, radius
 * and enforce_1to1: the same m[p], the same rows in the same order, bit for bit.  A problem's result depends on nothing
 * else: not on the other problems, nprob or p, and not on anything past n1[p] and n2[p] (NaN or garbage included).
 * n1[p] = 0 or n2[p] = 0 gives m[p] = 0.  n1, n2 and m are host arrays of nprob; the call returns when m is on the host.
 * clp_batch_correspondences: D1[p] (d x n1[p]) and D2[p] (d x n2[p]) are column-major host arrays; A_out[p] holds
 *   capacity rows and receives problem p's as clp_correspondences fills it (c0 in A_out[p][0 .. m[p]), c1 in
 *   A_out[p][m[p] .. 2 m[p])); A_out[p] may be NULL when n1[p] * min(knn, n2[p]) = 0.
 * clp_batch_correspondences_dev: the clouds on the batch's device in the element strides of clp_points_dev (coordinate
 *   k of point j of problem p at D1_dev[p d1_strides[0] + k d1_strides[1] + j d1_strides[2]], D2 alike; a batch stride
 *   may be 0: one cloud for every problem); entry (r, c) of problem p is written at A_dev[p a_strides[0] +
 *   r a_strides[1] + c a_strides[2]] for r < m[p] (rows m[p] .. capacity - 1 are left as they were).  With strides
 *   (2 cap, 1, cap) this is a (nprob, cap, 2) tensor that clp_batch_*_dev take as their associations.
 * The batch's device, stream (clp_batch_set_stream) and error string are used, and its own kNN scratch; its other state
 * stays as it was.  The device work is a fixed number of launches whatever nprob, and one synchronisation.
 * Errors, checked on the host before anything is uploaded, in this order, naming the first failing problem:
 *   CLP_ERR_INVALID for NULL pointers (a cloud may be NULL when every problem's size for it is 0), nprob < 1, knn < 1, d < 1, a negative size or bad strides (coordinate, point,
 *   row and column strides >= 1, batch strides >= 0); CLP_ERR_UNSUPPORTED for knn > CLP_KNN_MAX_K, d > CLP_KNN_MAX_D or
 *   a size >= 2^31 - 1; CLP_ERR_INVALID for capacity < n1[p] * min(knn, n2[p]); CLP_ERR_ALLOC when the scratch does not
 *   fit the free device memory.  m is all zero after an error; the batch stays usable.
 * Handing A and m to clp_batch_*_dev: there m[p] = 0 means the all-to-all hypothesis, so a problem without rows must be
 * left out, and m[p] > 4096 is refused. */
int clp_batch_correspondences(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                              const double* const* D2, const int64_t* n2, int32_t knn, double radius, int enforce_1to1,
                              int32_t* const* A_out, int64_t capacity, int64_t* m);
int clp_batch_correspondences_dev(clp_batch b, int32_t nprob, int32_t d, const double* D1_dev, const int64_t d1_strides[3],
                                  const int64_t* n1, const double* D2_dev, const int64_t d2_strides[3], const int64_t* n2,
                                  int32_t knn, double radius, int enforce_1to1, int32_t* A_dev, const int64_t a_strides[3],
                                  int64_t capacity, int64_t* m);

/* ---- rigid transform of selected associations (the last step of a registration) ---------------------------------------
 * The proper rigid transform that aligns the pairs a set of rows of A names, on the device (clp_transform.cuh).  D1
 * (d x n1) and D2 (d x n2) are fp64 and A (m x 2) int32 in the layouts of the scoring calls, read as they read them:
 * A == NULL or m == 0 is the all-to-all hypothesis, row r = (r / n2, r mod n2) as clp_create_all_to_all orders it, so the
 * nodes of a solve on all-to-all index the right pairs.
 * Rows: rows (host, int32) lists k row indices of A, each counted once per listing, in the given order; rows == NULL
 *   means every row 0 .. m-1 (k is then ignored).  Only the listed rows of A and the points they name are read.
 * Estimate: pair i is a_i = D1[:, A(r_i, 0)], b_i = D2[:, A(r_i, 1)].  All arithmetic is fp64 in two passes: the means
 *   mu_a, mu_b, then H = sum (b_i - mu_b)(a_i - mu_a)' on the centred points.  R is a proper rotation (det R = +1)
 *   minimising sum |R a_i + t - b_i|^2 (Umeyama's correction of the SVD solution, no scale) and t = mu_b - R mu_a, so
 *   b ~ R a + t: T maps the frame of D1 into the frame of D2.
 * Outputs: T (d+1) x (d+1), column-major, last row [0 .. 0 1].  info.rmse = sqrt(sum |r_i|^2 / k) with the residual
 *   r_i = R (a_i - mu_a) - (b_i - mu_b) (= R a_i + t - b_i).  info.sv: the singular values of H, descending (sv[2] = 0
 *   for d = 2).  info.gap = sv[d-2] + sign(det H) sv[d-1], the sign +1 when det H = 0: R is unique exactly when gap > 0,
 *   and its sensitivity to rounding is about sv[0] / gap.  info.k: the number of pairs used.
 * Status (info.status):
 *   CLP_TF_EMPTY       k = 0: T = I, rmse = 0, sv = gap = 0.
 *   CLP_TF_NONFINITE   a used coordinate is not finite (or a sum overflows): R, t, rmse, sv and gap are NaN.
 *   CLP_TF_DEGENERATE  sv[0] = 0 or gap <= 1e-12 sv[0] (one pair, collinear points in 3-D, all points equal): R is still
 *                      a proper rotation and a minimiser (R = I when H = 0), but not the only one.
 *   CLP_TF_OK          otherwise (coplanar points in 3-D included: the determinant fixes the third axis).
 * Determinism: a repeated call is bit-identical; problem p of a batch is bit for bit the single call on the same inputs,
 *   and a host call the device call; a problem's result depends on nothing it does not read (not on nprob, p or the
 *   other problems).  info.t is the wall-clock seconds of the call (batches: divided by nprob), info.kernel_ms the device
 *   time of its kernels.
 * clp_estimate_transform: host D1, D2, A; T_out host.  clp_estimate_transform_dev: D1, D2 and A on the handle's device in
 *   the clp_score_*_dev layouts (column-major, contiguous), T_out on the device.
 * clp_batch_estimate_transform: host arrays of nprob pointers (A may be NULL, or A[p] NULL: all-to-all for problem p;
 *   m may be NULL: all zero); T_out[p] host.  clp_batch_estimate_transform_dev: pts as clp_batch_*_dev take it (pts->A
 *   == NULL: all-to-all everywhere, m[p] == 0: for problem p); entry (r, c) of problem p's T goes to T_dev[p t_strides[0]
 *   + r t_strides[1] + c t_strides[2]] (element strides, so a torch (nprob, d+1, d+1) float64 tensor is written in place).
 * rows and k are host arrays of nprob (rows itself or rows[p] may be NULL: all rows).  Only the handle's or batch's
 * device, stream (clp_set_stream, clp_batch_set_stream) and error string are used, and a scratch of the transform's own:
 * its matrix, solve state and kNN scratch stay as they were.  Every call returns when infos (and host T) are on the host.
 * Errors, in this order, naming the first failing problem; the handle or batch stays usable:
 *   CLP_ERR_INVALID for NULL pointers, nprob < 1, d < 1, negative sizes, bad strides (coordinate, point, row, column and T
 *     row and column strides >= 1, batch strides >= 0), k < 0, a row outside [0, m) (m = n1 n2 for all-to-all) or a
 *     host association index out of range;
 *   CLP_ERR_UNSUPPORTED for d other than 2 and 3;
 *   CLP_ERR_ALLOC when the scratch (2 d k doubles per problem, plus the rows) does not fit the free device memory;
 *   CLP_ERR_INVALID, found on the device, for a device association index out of range, naming the lowest such problem;
 *     nothing is written to T_dev then. */
#define CLP_TF_OK 0
#define CLP_TF_EMPTY 1
#define CLP_TF_DEGENERATE 2
#define CLP_TF_NONFINITE 3
typedef struct clp_tf_info {
  int32_t status;   /* CLP_TF_*                                                                 */
  int64_t k;        /* pairs used                                                               */
  double rmse;      /* sqrt(sum |R a_i + t - b_i|^2 / k)                                        */
  double sv[3];     /* singular values of H, descending                                        */
  double gap;       /* sv[d-2] + sign(det H) sv[d-1]                                            */
  double t;         /* wall-clock seconds of the call (batches: divided by nprob)              */
  double kernel_ms; /* device time of the call's kernels (CUDA events; batches: the whole call) */
} clp_tf_info;
int clp_estimate_transform(clp_handle h, const double* D1, int32_t d, int64_t n1, const double* D2, int64_t n2,
                           const int32_t* A, int64_t m, const int32_t* rows, int64_t k, double* T_out, clp_tf_info* info);
int clp_estimate_transform_dev(clp_handle h, const double* D1_dev, int32_t d, int64_t n1, const double* D2_dev, int64_t n2,
                               const int32_t* A_dev, int64_t m, const int32_t* rows, int64_t k, double* T_dev,
                               clp_tf_info* info);
int clp_batch_estimate_transform(clp_batch b, int32_t nprob, int32_t d, const double* const* D1, const int64_t* n1,
                                 const double* const* D2, const int64_t* n2, const int32_t* const* A, const int64_t* m,
                                 const int32_t* const* rows, const int64_t* k, double* const* T_out, clp_tf_info* infos);
int clp_batch_estimate_transform_dev(clp_batch b, int32_t nprob, int32_t d, const clp_points_dev* pts,
                                     const int32_t* const* rows, const int64_t* k, double* T_dev, const int64_t t_strides[3],
                                     clp_tf_info* infos);

/* ---- semidefinite relaxation (solveAsMSRCSDR / sdp::solve, ref clipper.cpp:101-113, sdp.cpp:88-296) ---------------
 * Solves  maximise <M, X>  subject to  X PSD, tr X = 1, X_ij = 0 where C_ij = 0, X_ij >= 0 where C_ij != 0  on the
 * device by two-block ADMM (X in the spectraplex, Z in the polyhedral set), with a Jacobi eigensolver in shared memory
 * and the whole iteration inside one kernel (DESIGN §3 "SDR" states every step).  It is not SCS: the iterates and the
 * iteration counts differ from the reference's; the problem and the read-out of the answer are the reference's.
 * The relaxation is always feasible and bounded (X = e_i e_i' is feasible, C has a unit diagonal), so there is no
 * infeasibility detection.  Stopping: the primal and dual residuals (max norm) within eps_abs + eps_rel * scale, and
 * |value - bound| within eps_abs + eps_rel * max(|value|, |bound|), where bound is a dual upper bound on the optimum.
 * Outputs of the last iterate: X (m x m, PSD with trace 1; the polyhedral constraints hold to res_pri), lambdas = the
 * eigenvalues of X ascending, evec1 = the eigenvector of the largest one (its largest-magnitude entry, lowest index
 * among equals, made positive), thr = max|evec1| / 2 and the nodes {i : |evec1_i| > thr} ascending (sdp.cpp:249-262).
 * m <= CLP_SDP_MAX_M.  A repeated call gives bit-identical outputs. */
#define CLP_SDP_MAX_M 128
typedef struct clp_sdp_params {
  int32_t max_iters;   /* 2000 (reference sdp.h defaults) */
  double eps_abs;      /* 1e-3 */
  double eps_rel;      /* 1e-3 */
  double time_limit_s; /* 0: none; else the call returns its last iterate with timed_out = 1 once this has passed */
} clp_sdp_params;
void clp_sdp_default_params(clp_sdp_params* p);
typedef struct clp_sdp_info {
  int32_t iters, converged, timed_out, n_nodes;
  double value;     /* <M, X>                                                                  */
  double bound;     /* dual upper bound on the optimum                                         */
  double res_pri;   /* max |X - Z|                                                             */
  double res_dual;  /* rho * max |Z - Z_previous|                                              */
  double rho;       /* final ADMM penalty                                                      */
  double thr;       /* node threshold max|evec1| / 2                                           */
  int64_t n_sweeps; /* Jacobi sweeps, all iterations and bound evaluations                     */
  double t;         /* wall-clock seconds of the call (batches: divided by nprob)              */
  double kernel_ms; /* device time of the launch (CUDA events; batches: the whole launch)      */
  double proj_ms;   /* in-kernel time in the eigendecompositions and simplex projections       */
} clp_sdp_info;
/* The handle's M and C, exactly as clp_get_dense(h, 0 / 1) returns them, gathered on the device; the handle's matrix is
 * left as it was.  nodes_out (m int32), X_out (m * m, column-major), lambdas_out (m) and evec1_out (m) may be NULL.
 * CLP_ERR_INVALID: no matrix, NULL p or info, max_iters < 1, a negative or NaN eps or time limit.
 * CLP_ERR_UNSUPPORTED: m > CLP_SDP_MAX_M, a sharded handle.  m = 1 gives X = [1] and nodes {0}. */
int clp_sdp_solve(clp_handle h, const clp_sdp_params* p, clp_sdp_info* info, int32_t* nodes_out, double* X_out,
                  double* lambdas_out, double* evec1_out);
/* Many relaxations in one launch (one CTA per problem, problems drawn from a counter).  Problems as
 * clp_batch_solve_matrices takes them (strictly-upper CSC M and C), checked in the same order with the same messages,
 * and then CLP_ERR_UNSUPPORTED for m[p] > CLP_SDP_MAX_M naming the problem.  Problem p gets bit for bit what an fp32
 * handle gives after clp_set_sparse_upper and clp_sdp_solve with the same parameters.  time_limit_s bounds the whole
 * call: a problem cut off returns its last iterate with timed_out = 1.  infos[p].kernel_ms is the whole launch, t the
 * wall-clock time divided by nprob.  Output arrays and their entries may be NULL. */
int clp_batch_sdp_matrices(clp_batch b, int32_t nprob, const int64_t* m,
                           const int64_t* const* colptrM, const int32_t* const* rowidxM, const double* const* valM,
                           const int64_t* const* colptrC, const int32_t* const* rowidxC, const double* const* valC,
                           const clp_sdp_params* p, clp_sdp_info* infos, int32_t* const* nodes_out,
                           double* const* X_out, double* const* lambdas_out, double* const* evec1_out);

#ifdef __cplusplus
}
#endif
#endif /* CLIPPER_B200_H_ */
