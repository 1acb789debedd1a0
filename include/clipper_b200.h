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

/* ---- K7: matrix get/set (clipper.cpp:131-166) -------------------------------------------- */
/* setMatrixData: strict upper triangle of the column-major m x m inputs is used, diagonal and
 * lower triangle ignored (clipper.cpp:149-158). Contract: M >= 0, C in {0,1} (clipper.h:166-176). */
int clp_set_dense(clp_handle h, const double* M, const double* C, int64_t m);
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
/* diagnostics of the last batch: CTAs of the launch, HBM scratch bytes, stored affinities (i<j) over all problems */
int clp_batch_info(clp_batch b, int32_t* n_ctas, int64_t* scratch_bytes, int64_t* nnz_upper_total);

#ifdef __cplusplus
}
#endif
#endif /* CLIPPER_B200_H_ */
