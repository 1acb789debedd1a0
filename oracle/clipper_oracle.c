/*
 * clipper_oracle.c -- CPU restatement of the CLIPPER hot path (TEST INFRASTRUCTURE ONLY).
 *
 * This file is the parity ORACLE for the H100 build. It is NOT part of the product:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs may load it. The product (clipper_b200/) never links or calls it.
 *
 * It restates, in plain C99 / fp64, the algorithm of mit-acl/clipper v0.2.4:
 *   - scorePairwiseConsistency      reference src/clipper.cpp:21-65
 *   - EuclideanDistance::operator() reference src/invariants/euclidean_distance.cpp:13-31
 *   - PointNormalDistance::op()     reference src/invariants/pointnormal_distance.cpp:13-35
 *   - findDenseClique (solve)       reference src/clipper.cpp:172-323
 *   - k2ij / createAllToAll / findIndicesOfkLargest / findIndicesWhereAboveThreshold /
 *     selectFromIndicator           reference src/utils.cpp:33-97, include/clipper/utils.h:61-71
 *   - get/setMatrixData             reference src/clipper.cpp:131-166
 *   - Rounding::DSD (Goldberg)      reference src/dsd.cpp:17-320
 *
 * Storage follows the reference: M_ and C_ are strictly-upper-triangular column-major
 * sparse matrices (CSC) with no diagonal; the identity on the diagonal is applied
 * analytically inside the solver (reference src/clipper.cpp:58,194,238).
 *
 * PARITY STATUS.  The reference itself cannot be built in this environment (it needs
 * Eigen3, which is not installed and cannot be fetched), so the linear algebra the
 * reference delegates to Eigen (sparse self-adjoint product, norm, dot, sum, mean) is
 * restated here with plain left-to-right loops, compiled with -ffp-contract=off.
 * What IS pinned against the reference's own fixtures (tests/test_oracle_golden.py):
 *   - the 12x12 Mtrue literal and M==C, diag==1, symmetry   (test/affinity_test.cpp:83-107)
 *   - the inlier set {(0,0),(1,1),(2,2)} of the m=12 toy     (test/clipper_test.cpp:63-66)
 *   - the dense cluster {3,5,12,14,15} of the 20x20 matrix   (test/dsd_test.cpp:15, sdp_test.cpp:17-40)
 *   - the plane-cloud associations Agt=[1 4;2 3;3 2]         (examples/matlab/ex3_planecloud.m:18-33,79-86)
 * What is NOT pinned by any reference fixture: intermediates of findDenseClique (u, F, d,
 * ifinal, matvec values).  For those: "parity unpinned" -- this restatement is the pin.
 * Summation order inside Eigen reductions is an Eigen implementation detail; differences
 * are O(1e-16) relative and no reference test observes them.
 */
#define _POSIX_C_SOURCE 200809L
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#ifdef _OPENMP
#include <omp.h>
#endif

typedef struct {
  int64_t m;
  int64_t *colptr; /* m+1 */
  int32_t *rowidx; /* nnz, strictly < column, ascending within a column */
  double *val;     /* nnz */
} orc_csc;

typedef struct orc_problem {
  int64_t m;
  orc_csc M, C;
  int32_t *A; /* column-major m x 2 (A(:,0) then A(:,1)), reference types.h:18 */
} orc_problem;

/* reference include/clipper/clipper.h:27-60 */
typedef struct {
  double tol_u, tol_F, tol_Fop;
  int32_t maxiniters, maxoliters;
  double beta;
  int32_t maxlsiters;
  double eps, affinityeps;
  int32_t rescale_u0;
  int32_t rounding; /* 0 NONZERO, 1 DSD, 2 DSD_HEU */
} orc_params;

/* reference include/clipper/clipper.h:65-73, plus counters used by the tests/bench */
typedef struct {
  double t;
  int32_t ifinal;
  int32_t n_nodes;
  double score;
  double d_final;
  int64_t n_evals;   /* objective evaluations inside the line search (clipper.cpp:238-242) */
  int64_t n_spmv;    /* sparse self-adjoint products executed (M and C counted separately) */
  int64_t n_inner;   /* accepted gradient steps */
} orc_solution;

void orc_default_params(orc_params *p) {
  p->tol_u = 1e-8; p->tol_F = 1e-9; p->tol_Fop = 1e-10;
  p->maxiniters = 200; p->maxoliters = 1000;
  p->beta = 0.25; p->maxlsiters = 99;
  p->eps = 1e-9; p->affinityeps = 1e-4;
  p->rescale_u0 = 1; p->rounding = 2;
}

static void csc_free(orc_csc *s) {
  free(s->colptr); free(s->rowidx); free(s->val);
  memset(s, 0, sizeof(*s));
}

orc_problem *orc_create(void) { return (orc_problem *)calloc(1, sizeof(orc_problem)); }

void orc_destroy(orc_problem *p) {
  if (!p) return;
  csc_free(&p->M); csc_free(&p->C); free(p->A); free(p);
}

int64_t orc_m(const orc_problem *p) { return p->m; }
int64_t orc_nnz(const orc_problem *p, int which) {
  const orc_csc *s = which ? &p->C : &p->M;
  return s->colptr ? s->colptr[s->m] : 0;
}

/* ---- utils ------------------------------------------------------------------------- */

/* reference src/utils.cpp:87-97 (size_t arithmetic, one double sqrt) */
void orc_k2ij(uint64_t k, uint64_t n, uint64_t *i_out, uint64_t *j_out) {
  k += 1;
  const uint64_t l = n * (n - 1) / 2 - k;
  const uint64_t o = (uint64_t)floor((sqrt((double)(1 + 8 * l)) - 1) / 2.);
  const uint64_t p = l - o * (o + 1) / 2;
  const uint64_t i = n - (o + 1);
  const uint64_t j = n - p;
  *i_out = i - 1; *j_out = j - 1;
}

/* reference include/clipper/utils.h:61-71; A is column-major (n1*n2) x 2 */
void orc_create_all_to_all(int64_t n1, int64_t n2, int32_t *A) {
  const int64_t m = n1 * n2;
  for (int64_t i = 0; i < n1; ++i)
    for (int64_t j = 0; j < n2; ++j) {
      A[j + i * n2] = (int32_t)i;
      A[m + j + i * n2] = (int32_t)j;
    }
}

/* reference src/utils.cpp:59-68 */
int32_t orc_find_above(const double *x, int64_t n, double thr, int32_t *out) {
  int32_t c = 0;
  for (int64_t i = 0; i < n; ++i) if (x[i] > thr) out[c++] = (int32_t)i;
  return c;
}

/* (value,index) lexicographic "a < b" */
static int pair_less(double va, int32_t ia, double vb, int32_t ib) {
  return (va < vb) || (!(vb < va) && ia < ib);
}

/* reference src/utils.cpp:33-55.  A bounded min-heap of (value,index) pairs ordered
 * lexicographically: fill with the first k elements, afterwards an element replaces the
 * heap minimum only if its VALUE is strictly larger than the minimum's value.  The result
 * is emitted in descending (value,index) order.  k<1 -> nothing.  The reference has UB for
 * k>n (pops an empty heap); here k is clamped to n. */
int32_t orc_find_k_largest(const double *x, int64_t n, int32_t k, int32_t *out) {
  if (k < 1) return 0;
  if ((int64_t)k > n) k = (int32_t)n;
  double *hv = (double *)malloc(sizeof(double) * (size_t)k);
  int32_t *hi = (int32_t *)malloc(sizeof(int32_t) * (size_t)k);
  int32_t sz = 0;
  for (int64_t t = 0; t < n; ++t) {
    if (sz < k) { /* sift up */
      int32_t c = sz++;
      hv[c] = x[t]; hi[c] = (int32_t)t;
      while (c > 0) {
        int32_t par = (c - 1) / 2;
        if (pair_less(hv[c], hi[c], hv[par], hi[par])) {
          double tv = hv[c]; hv[c] = hv[par]; hv[par] = tv;
          int32_t ti = hi[c]; hi[c] = hi[par]; hi[par] = ti;
          c = par;
        } else break;
      }
    } else if (hv[0] < x[t]) { /* replace min, sift down */
      hv[0] = x[t]; hi[0] = (int32_t)t;
      int32_t c = 0;
      for (;;) {
        int32_t l = 2 * c + 1, r = l + 1, s = c;
        if (l < sz && pair_less(hv[l], hi[l], hv[s], hi[s])) s = l;
        if (r < sz && pair_less(hv[r], hi[r], hv[s], hi[s])) s = r;
        if (s == c) break;
        double tv = hv[c]; hv[c] = hv[s]; hv[s] = tv;
        int32_t ti = hi[c]; hi[c] = hi[s]; hi[s] = ti;
        c = s;
      }
    }
  }
  /* pop ascending, write back to front */
  for (int32_t e = 0; e < k; ++e) {
    out[k - e - 1] = hi[0];
    --sz;
    if (sz > 0) {
      hv[0] = hv[sz]; hi[0] = hi[sz];
      int32_t c = 0;
      for (;;) {
        int32_t l = 2 * c + 1, r = l + 1, s = c;
        if (l < sz && pair_less(hv[l], hi[l], hv[s], hi[s])) s = l;
        if (r < sz && pair_less(hv[r], hi[r], hv[s], hi[s])) s = r;
        if (s == c) break;
        double tv = hv[c]; hv[c] = hv[s]; hv[s] = tv;
        int32_t ti = hi[c]; hi[c] = hi[s]; hi[s] = ti;
        c = s;
      }
    }
  }
  free(hv); free(hi);
  return k;
}

/* ---- invariants -------------------------------------------------------------------- */

static double vec_dist(const double *a, const double *b, int d) {
  double s = 0.0;
  for (int q = 0; q < d; ++q) { const double t = a[q] - b[q]; s = s + t * t; }
  return sqrt(s);
}

/* reference src/invariants/euclidean_distance.cpp:13-31 */
double orc_euclidean(const double *ai, const double *aj, const double *bi, const double *bj,
                     int d, double sigma, double epsilon, double mindist) {
  const double l1 = vec_dist(ai, aj, d);
  const double l2 = vec_dist(bi, bj, d);
  if (mindist > 0 && (l1 < mindist || l2 < mindist)) return 0.0;
  const double c = fabs(l1 - l2);
  return (c < epsilon) ? exp(-0.5 * c * c / (sigma * sigma)) : 0.0;
}

/* reference src/invariants/pointnormal_distance.cpp:13-35; datum = [point(3); normal(3)].
 * acos is NOT clamped: |dot|>1 -> NaN -> the comparisons are false -> 0 (SURVEY H3). */
double orc_pointnormal(const double *ai, const double *aj, const double *bi, const double *bj,
                       double sigp, double epsp, double sign, double epsn) {
  const double l1 = vec_dist(ai, aj, 3);
  const double l2 = vec_dist(bi, bj, 3);
  const double dot1 = (ai[3] * aj[3] + ai[4] * aj[4]) + ai[5] * aj[5];
  const double dot2 = (bi[3] * bj[3] + bi[4] * bj[4]) + bi[5] * bj[5];
  const double alpha1 = acos(dot1);
  const double alpha2 = acos(dot2);
  const double dp = fabs(l1 - l2);
  const double dn = fabs(alpha1 - alpha2);
  if (dp < epsp && dn < epsn) {
    const double sp = exp(-0.5 * dp * dp / (sigp * sigp));
    const double sn = exp(-0.5 * dn * dn / (sign * sign));
    return sp * sn;
  }
  return 0.0;
}

/* ---- scoring ----------------------------------------------------------------------- */

typedef struct {
  int kind; /* 0 euclidean, 1 pointnormal */
  int d;
  double p0, p1, p2, p3; /* sigma,epsilon,mindist | sigp,epsp,sign,epsn */
} inv_cfg;

/* reference src/clipper.cpp:21-65.  The reference fills a dense m x m scratch and calls
 * sparseView(); here the strictly-upper CSC is built directly, column by column (identical
 * result, SURVEY H8).  Entry (i,j), i<j, lives in column j. */
static int score_generic(orc_problem *p, const double *D1, int64_t n1, const double *D2, int64_t n2,
                         const int32_t *A, int64_t m, const inv_cfg *cfg, double affinityeps,
                         int nthreads) {
  csc_free(&p->M); csc_free(&p->C); free(p->A); p->A = NULL;
  if (A == NULL) { /* clipper.cpp:24 */
    m = n1 * n2;
    p->A = (int32_t *)malloc(sizeof(int32_t) * 2 * (size_t)m);
    orc_create_all_to_all(n1, n2, p->A);
  } else {
    p->A = (int32_t *)malloc(sizeof(int32_t) * 2 * (size_t)m);
    memcpy(p->A, A, sizeof(int32_t) * 2 * (size_t)m);
  }
  p->m = m;
  const int32_t *A0 = p->A, *A1 = p->A + m;
  const int d = cfg->d;

  int32_t **col_idx = (int32_t **)calloc((size_t)m, sizeof(int32_t *));
  double **col_val = (double **)calloc((size_t)m, sizeof(double *));
  int64_t *cnt = (int64_t *)calloc((size_t)m + 1, sizeof(int64_t));
  (void)nthreads;
#ifdef _OPENMP
  if (nthreads <= 0) nthreads = omp_get_max_threads();
#pragma omp parallel num_threads(nthreads)
#endif
  {
    int32_t *ti = (int32_t *)malloc(sizeof(int32_t) * (size_t)(m > 0 ? m : 1));
    double *tv = (double *)malloc(sizeof(double) * (size_t)(m > 0 ? m : 1));
#ifdef _OPENMP
#pragma omp for schedule(dynamic, 16)
#endif
    for (int64_t j = 0; j < m; ++j) {
      int64_t c = 0;
      const double *d1j = D1 + (size_t)d * A0[j];
      const double *d2j = D2 + (size_t)d * A1[j];
      for (int64_t i = 0; i < j; ++i) {
        if (A0[i] == A0[j] || A1[i] == A1[j]) continue; /* clipper.cpp:35 */
        const double *d1i = D1 + (size_t)d * A0[i];
        const double *d2i = D2 + (size_t)d * A1[i];
        double scr;
        if (cfg->kind == 0) scr = orc_euclidean(d1i, d1j, d2i, d2j, d, cfg->p0, cfg->p1, cfg->p2);
        else scr = orc_pointnormal(d1i, d1j, d2i, d2j, cfg->p0, cfg->p1, cfg->p2, cfg->p3);
        /* clipper.cpp:53 keeps scr > affinityeps; sparseView() (clipper.cpp:61) then drops exact zeros */
        if (scr > affinityeps && scr != 0.0) { ti[c] = (int32_t)i; tv[c] = scr; ++c; }
      }
      cnt[j + 1] = c;
      if (c) {
        col_idx[j] = (int32_t *)malloc(sizeof(int32_t) * (size_t)c);
        col_val[j] = (double *)malloc(sizeof(double) * (size_t)c);
        memcpy(col_idx[j], ti, sizeof(int32_t) * (size_t)c);
        memcpy(col_val[j], tv, sizeof(double) * (size_t)c);
      }
    }
    free(ti); free(tv);
  }
  for (int64_t j = 0; j < m; ++j) cnt[j + 1] += cnt[j];
  const int64_t nnz = cnt[m];
  p->M.m = m; p->M.colptr = cnt;
  p->M.rowidx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  p->M.val = (double *)malloc(sizeof(double) * (size_t)(nnz > 0 ? nnz : 1));
  for (int64_t j = 0; j < m; ++j) {
    const int64_t c = cnt[j + 1] - cnt[j];
    if (c) {
      memcpy(p->M.rowidx + cnt[j], col_idx[j], sizeof(int32_t) * (size_t)c);
      memcpy(p->M.val + cnt[j], col_val[j], sizeof(double) * (size_t)c);
      free(col_idx[j]); free(col_val[j]);
    }
  }
  free(col_idx); free(col_val);
  /* C_ = M_; C_.coeffs() = 1  (clipper.cpp:63-64) */
  p->C.m = m;
  p->C.colptr = (int64_t *)malloc(sizeof(int64_t) * ((size_t)m + 1));
  memcpy(p->C.colptr, cnt, sizeof(int64_t) * ((size_t)m + 1));
  p->C.rowidx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  memcpy(p->C.rowidx, p->M.rowidx, sizeof(int32_t) * (size_t)nnz);
  p->C.val = (double *)malloc(sizeof(double) * (size_t)(nnz > 0 ? nnz : 1));
  for (int64_t q = 0; q < nnz; ++q) p->C.val[q] = 1.0;
  return 0;
}

int orc_score_euclidean(orc_problem *p, const double *D1, int32_t d, int64_t n1, const double *D2,
                        int64_t n2, const int32_t *A, int64_t m, double sigma, double epsilon,
                        double mindist, double affinityeps, int nthreads) {
  inv_cfg c = {0, d, sigma, epsilon, mindist, 0.0};
  return score_generic(p, D1, n1, D2, n2, A, m, &c, affinityeps, nthreads);
}

int orc_score_pointnormal(orc_problem *p, const double *D1, int64_t n1, const double *D2, int64_t n2,
                          const int32_t *A, int64_t m, double sigp, double epsp, double sign,
                          double epsn, double affinityeps, int nthreads) {
  inv_cfg c = {1, 6, sigp, epsp, sign, epsn};
  return score_generic(p, D1, n1, D2, n2, A, m, &c, affinityeps, nthreads);
}

/* ---- get / set --------------------------------------------------------------------- */

/* dense column-major m x m -> strict-upper CSC without exact zeros
 * (triangularView<Upper>, diagonal().setZero(), sparseView(): clipper.cpp:149-158) */
static void dense_to_csc_upper(const double *X, int64_t m, orc_csc *s) {
  csc_free(s);
  s->m = m;
  s->colptr = (int64_t *)calloc((size_t)m + 1, sizeof(int64_t));
  for (int64_t j = 0; j < m; ++j) {
    int64_t c = 0;
    for (int64_t i = 0; i < j; ++i) if (X[i + j * m] != 0.0) ++c;
    s->colptr[j + 1] = s->colptr[j] + c;
  }
  const int64_t nnz = s->colptr[m];
  s->rowidx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  s->val = (double *)malloc(sizeof(double) * (size_t)(nnz > 0 ? nnz : 1));
  int64_t q = 0;
  for (int64_t j = 0; j < m; ++j)
    for (int64_t i = 0; i < j; ++i)
      if (X[i + j * m] != 0.0) { s->rowidx[q] = (int32_t)i; s->val[q] = X[i + j * m]; ++q; }
}

int orc_set_dense(orc_problem *p, const double *M, const double *C, int64_t m) {
  p->m = m;
  dense_to_csc_upper(M, m, &p->M);
  dense_to_csc_upper(C, m, &p->C);
  return 0;
}

static void csc_copy_in(orc_csc *s, int64_t m, const int64_t *colptr, const int32_t *rowidx,
                        const double *val) {
  csc_free(s);
  s->m = m;
  const int64_t nnz = colptr[m];
  s->colptr = (int64_t *)malloc(sizeof(int64_t) * ((size_t)m + 1));
  memcpy(s->colptr, colptr, sizeof(int64_t) * ((size_t)m + 1));
  s->rowidx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  s->val = (double *)malloc(sizeof(double) * (size_t)(nnz > 0 ? nnz : 1));
  memcpy(s->rowidx, rowidx, sizeof(int32_t) * (size_t)nnz);
  memcpy(s->val, val, sizeof(double) * (size_t)nnz);
}

/* setSparseMatrixData: stored as given, caller passes strict upper (clipper.cpp:162-166) */
int orc_set_sparse_upper(orc_problem *p, int64_t m, const int64_t *cpM, const int32_t *riM,
                         const double *vM, const int64_t *cpC, const int32_t *riC, const double *vC) {
  p->m = m;
  csc_copy_in(&p->M, m, cpM, riM, vM);
  csc_copy_in(&p->C, m, cpC, riC, vC);
  return 0;
}

int orc_get_csc(const orc_problem *p, int which, int64_t *colptr, int32_t *rowidx, double *val) {
  const orc_csc *s = which ? &p->C : &p->M;
  const int64_t nnz = s->colptr[s->m];
  memcpy(colptr, s->colptr, sizeof(int64_t) * ((size_t)s->m + 1));
  memcpy(rowidx, s->rowidx, sizeof(int32_t) * (size_t)nnz);
  memcpy(val, s->val, sizeof(double) * (size_t)nnz);
  return 0;
}

/* getAffinityMatrix / getConstraintMatrix: sym(upper) + I, dense column-major (clipper.cpp:131-145) */
int orc_get_dense(const orc_problem *p, int which, double *out) {
  const orc_csc *s = which ? &p->C : &p->M;
  const int64_t m = s->m;
  memset(out, 0, sizeof(double) * (size_t)m * (size_t)m);
  for (int64_t j = 0; j < m; ++j) {
    for (int64_t q = s->colptr[j]; q < s->colptr[j + 1]; ++q) {
      const int64_t i = s->rowidx[q];
      out[i + j * m] = s->val[q];
      out[j + i * m] = s->val[q];
    }
    out[j + j * m] += 1.0;
  }
  return 0;
}

int orc_get_associations(const orc_problem *p, int32_t *A) {
  if (!p->A) return 1;
  memcpy(A, p->A, sizeof(int32_t) * 2 * (size_t)p->m);
  return 0;
}

/* ---- linear algebra the reference delegates to Eigen -------------------------------- */

/* y = selfadjointView<Upper>(S) * x, S strict upper CSC, no diagonal.
 * Column sweep (Eigen's sparse self-adjoint x dense kernel visits column j, scatters
 * a_ij*x_j into y_i and gathers a_ij*x_i into a local that is added to y_j). */
static void spmv_sym_upper(const orc_csc *s, const double *x, double *y) {
  const int64_t m = s->m;
  for (int64_t i = 0; i < m; ++i) y[i] = 0.0;
  for (int64_t j = 0; j < m; ++j) {
    const double xj = x[j];
    double rj = 0.0;
    for (int64_t q = s->colptr[j]; q < s->colptr[j + 1]; ++q) {
      const int64_t i = s->rowidx[q];
      const double a = s->val[q];
      rj = rj + a * x[i];
      y[i] = y[i] + a * xj;
    }
    y[j] = y[j] + rj;
  }
}

int orc_matvec(const orc_problem *p, int which, const double *x, double *y) {
  spmv_sym_upper(which ? &p->C : &p->M, x, y);
  return 0;
}

static double vsum(const double *x, int64_t n) { double s = 0.0; for (int64_t i = 0; i < n; ++i) s = s + x[i]; return s; }
static double vdot(const double *x, const double *y, int64_t n) { double s = 0.0; for (int64_t i = 0; i < n; ++i) s = s + x[i] * y[i]; return s; }

static double now_s(void) {
  struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
  return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* ---- the solver: reference src/clipper.cpp:172-323, statement for statement ---------- */

/* ------------------------------------------------------------------------------------------
 * Rounding::DSD -- exact densest edge-weighted subgraph (Goldberg's parametric min-cut).
 * Restates reference src/dsd.cpp:17-272 (graph construction, Dinic max-flow, bisection) and
 * dsd::solve src/dsd.cpp:274-320 (complete weighted graph on S, weights A(min(i,j),max(i,j))).
 * Kept exactly: the edge order (all S x S ordered pairs, then src->v, then v->dest), capacities
 * m/2 (INTEGER division of the edge count, dsd.cpp:25,33,196), paired forward/backward arcs whose
 * reverse arc starts saturated (dsd.cpp:40-51), the current-arc DFS that pushes one path at a time
 * and keeps a lowered bottleneck for the later arcs of the same vertex (dsd.cpp:80-102), the cut =
 * vertices reachable from src in the residual graph (dsd.cpp:106-117), "cut is {src} alone -> U = g,
 * else L = g" and the stopping rule n(n-1)(U-L) < 1 with n = ALL nodes of A, not |S| (dsd.cpp:216).
 * Pinned by tests/test_oracle_golden.py against test/dsd_test.cpp:15,38-43,72-79.
 * ------------------------------------------------------------------------------------------ */
typedef struct {
  int64_t *fin, *nxt, *to, *dist, *Q, *pro, *pro2;
  double *cap, *flow;
} dsd_net;

static void dsd_new_edge(dsd_net *g, int64_t u, int64_t v, double w, int64_t *ne) {
  g->to[*ne] = v; g->cap[*ne] = w; g->flow[*ne] = 0; g->nxt[*ne] = g->fin[u]; g->fin[u] = (*ne)++;
  g->to[*ne] = u; g->cap[*ne] = w; g->flow[*ne] = w; g->nxt[*ne] = g->fin[v]; g->fin[v] = (*ne)++;
}

static int dsd_bfs(dsd_net *g, int64_t nverts, int64_t src, int64_t dest) {
  for (int64_t i = 0; i < nverts; ++i) g->dist[i] = -1;
  int64_t st = 0, en = 0;
  g->dist[src] = 0; g->Q[en++] = src;
  while (st < en) {
    const int64_t u = g->Q[st++];
    for (int64_t e = g->fin[u]; e >= 0; e = g->nxt[e]) {
      const int64_t v = g->to[e];
      if (g->flow[e] < g->cap[e] && g->dist[v] == -1) { g->dist[v] = g->dist[u] + 1; g->Q[en++] = v; }
    }
  }
  return g->dist[dest] != -1;
}

static double dsd_dfs(dsd_net *g, int64_t u, double fl, int64_t src, int64_t dest) {
  if (u == dest) return fl;
  for (int64_t *e = &g->pro[u]; *e >= 0; *e = g->nxt[*e]) {
    const int64_t v = g->to[*e];
    if (g->flow[*e] < g->cap[*e] && g->dist[v] == g->dist[u] + 1) {
      if (u == src || (g->cap[*e] - g->flow[*e]) <= fl) fl = g->cap[*e] - g->flow[*e];
      const double df = dsd_dfs(g, v, fl, src, dest);
      if (df > 0) { g->flow[*e] += df; g->flow[*e ^ 1] -= df; return df; }
    }
  }
  return 0;
}

static void dsd_find_cut(dsd_net *g, int64_t u, int64_t *cut) {
  cut[u] = 1;
  for (int64_t *e = &g->pro2[u]; *e >= 0; *e = g->nxt[*e]) {
    const int64_t v = g->to[*e];
    if (g->flow[*e] < g->cap[*e] && cut[v] == 0) dsd_find_cut(g, v, cut);
  }
}

/* A = strictly-upper CSC of the affinity matrix (n nodes), S = nS node indices (nS == 0: all nodes).
 * out receives the selected nodes in ascending order; returns their number. */
int32_t orc_dsd(const orc_csc *A, const int32_t *S_in, int32_t nS_in, int32_t *out) {
  const int64_t n = A->m;
  int64_t nS = nS_in > 0 ? nS_in : n;
  int32_t *S = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nS > 0 ? nS : 1));
  for (int64_t q = 0; q < nS; ++q) S[q] = nS_in > 0 ? S_in[q] : (int32_t)q;
  const int64_t m = nS * nS - nS;            /* dsd.cpp:285 */
  const int64_t nverts = n + 2, nedges = m + 2 * n;
  double (*ed)[3] = (double (*)[3])malloc(sizeof(double) * 3 * (size_t)(nedges > 0 ? nedges : 1));
  double *degree = (double *)calloc((size_t)(n > 0 ? n : 1), sizeof(double));
  int64_t k = 0;
  for (int64_t a = 0; a < nS; ++a)            /* dsd.cpp:293-305 */
    for (int64_t b = 0; b < nS; ++b) {
      const int64_t i = S[a], j = S[b];
      if (i == j) continue;
      const int64_t r = i < j ? i : j, c = i < j ? j : i;
      double w = 0.0;                          /* A.coeff(r, c): binary search in column c */
      int64_t lo = A->colptr[c], hi = A->colptr[c + 1];
      while (lo < hi) { const int64_t mid = lo + ((hi - lo) >> 1); if (A->rowidx[mid] < r) lo = mid + 1; else hi = mid; }
      if (lo < A->colptr[c + 1] && A->rowidx[lo] == r) w = A->val[lo];
      ed[k][0] = (double)(i + 1); ed[k][1] = (double)(j + 1); ed[k][2] = w;   /* dsd.cpp:186-193 */
      degree[i] += w;
      ++k;
    }
  double L = 0, U = (double)(m / 2);          /* dsd.cpp:195-196, integer division */
  dsd_net g;
  g.Q = (int64_t *)malloc(sizeof(int64_t) * (size_t)nverts);
  g.fin = (int64_t *)malloc(sizeof(int64_t) * (size_t)nverts);
  g.pro = (int64_t *)malloc(sizeof(int64_t) * (size_t)nverts);
  g.pro2 = (int64_t *)malloc(sizeof(int64_t) * (size_t)nverts);
  g.dist = (int64_t *)malloc(sizeof(int64_t) * (size_t)nverts);
  g.flow = (double *)malloc(sizeof(double) * 2 * (size_t)nedges);
  g.cap = (double *)malloc(sizeof(double) * 2 * (size_t)nedges);
  g.nxt = (int64_t *)malloc(sizeof(int64_t) * 2 * (size_t)nedges);
  g.to = (int64_t *)malloc(sizeof(int64_t) * 2 * (size_t)nedges);
  int64_t *cut = (int64_t *)malloc(sizeof(int64_t) * (size_t)nverts);
  int64_t *final_cut = (int64_t *)calloc((size_t)nverts, sizeof(int64_t));
  const int64_t src = 0, dest = nverts - 1;
  while ((double)(n * (n - 1)) * (U - L) >= 1) {   /* dsd.cpp:216 */
    const double gg = (U + L) / 2;
    for (int64_t i = m; i < m + n; ++i) { ed[i][0] = (double)src; ed[i][1] = (double)(i - m + 1); ed[i][2] = (double)(m / 2); }
    for (int64_t i = n + m; i < m + 2 * n; ++i) {
      ed[i][0] = (double)(i - m - n + 1); ed[i][1] = (double)dest;
      ed[i][2] = (double)(m / 2) + 2 * gg - degree[i - m - n];
    }
    for (int64_t i = 0; i < nverts; ++i) { g.fin[i] = -1; cut[i] = 0; }
    int64_t ne = 0;
    for (int64_t i = 0; i < nedges; ++i) dsd_new_edge(&g, (int64_t)ed[i][0], (int64_t)ed[i][1], ed[i][2], &ne);
    for (int64_t i = 0; i < nverts; ++i) g.pro2[i] = g.fin[i];  /* defined even if the first BFS fails */
    while (dsd_bfs(&g, nverts, src, dest)) {
      for (int64_t i = 0; i < nverts; ++i) { g.pro[i] = g.fin[i]; g.pro2[i] = g.fin[i]; }
      for (;;) { const double df = dsd_dfs(&g, src, 0, src, dest); if (!(df != 0)) break; }
    }
    /* NB (dsd.cpp:170): find_cut walks the arc pointers left by the LAST bfs round's copy */
    dsd_find_cut(&g, src, cut);
    int64_t in_cut = 0;
    for (int64_t i = 0; i < nverts; ++i) in_cut += cut[i];
    if (in_cut == 1) U = gg;
    else { L = gg; memcpy(final_cut, cut, sizeof(int64_t) * (size_t)nverts); }
  }
  final_cut[0] = 0; final_cut[nverts - 1] = 0;
  int32_t num = 0;
  for (int64_t i = 1; i < nverts - 1; ++i)
    if (final_cut[i] != 0) out[num++] = (int32_t)(i - 1);
  free(S); free(ed); free(degree); free(g.Q); free(g.fin); free(g.pro); free(g.pro2); free(g.dist);
  free(g.flow); free(g.cap); free(g.nxt); free(g.to); free(cut); free(final_cut);
  return num;
}

/* trace (optional, may be NULL): per OUTER iteration i, trace[3*i+0]=F after the inner loop,
 * trace[3*i+1]=d used in that iteration, trace[3*i+2]=number of inner steps; at most trace_cap rows. */
int orc_solve(const orc_problem *p, const double *u0, const orc_params *P, orc_solution *S,
              double *u_out, int32_t *nodes_out, double *trace, int64_t trace_cap) {
  const double t1 = now_s();
  const int64_t n = p->M.m;
  const orc_csc *M = &p->M, *C = &p->C;
  int64_t n_spmv = 0, n_evals = 0, n_inner = 0;

  double *gradF = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *gradFnew = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *u = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *unew = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *Mu = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *Cu = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *Cbu = (double *)malloc(sizeof(double) * (size_t)(n + 1));

  /* clipper.cpp:193-198 */
  if (P->rescale_u0) {
    spmv_sym_upper(M, u0, Mu); ++n_spmv;
    for (int64_t i = 0; i < n; ++i) u[i] = Mu[i] + u0[i];
  } else {
    for (int64_t i = 0; i < n; ++i) u[i] = u0[i];
  }
  {
    const double nrm = sqrt(vdot(u, u, n));
    for (int64_t i = 0; i < n; ++i) u[i] = u[i] / nrm; /* no zero guard (clipper.cpp:198) */
  }

  /* clipper.cpp:201-209 */
  double d = 0;
  {
    const double su = vsum(u, n);
    spmv_sym_upper(C, u, Cu); ++n_spmv;
    int64_t cnt = 0;
    for (int64_t i = 0; i < n; ++i) {
      Cbu[i] = (1.0 * su - Cu[i]) - u[i];
      if (Cbu[i] > P->eps && u[i] > P->eps) ++cnt;
    }
    if (cnt > 0) {
      spmv_sym_upper(M, u, Mu); ++n_spmv;
      double acc = 0.0;
      for (int64_t i = 0; i < n; ++i)
        if (Cbu[i] > P->eps && u[i] > P->eps) acc = acc + (Mu[i] + u[i]) / Cbu[i];
      d = acc / (double)cnt; /* mean, no abs (clipper.cpp:208) */
    }
  }

  double F = 0;
  int64_t i, j, k;
  for (i = 0; i < (int64_t)P->maxoliters; ++i) {
    /* clipper.cpp:219-220 */
    {
      const double su = vsum(u, n);
      spmv_sym_upper(M, u, Mu); spmv_sym_upper(C, u, Cu); n_spmv += 2;
      for (int64_t q = 0; q < n; ++q)
        gradF[q] = (((1 + d) * u[q] - (d * 1.0) * su) + Mu[q]) + Cu[q] * d;
      F = vdot(u, gradF, n);
    }
    const double d_used = d;

    for (j = 0; j < (int64_t)P->maxiniters; ++j) {
      double alpha = 1;
      double Fnew = 0, deltaF = 0;
      for (k = 0; k < (int64_t)P->maxlsiters; ++k) {
        /* clipper.cpp:235-237 */
        for (int64_t q = 0; q < n; ++q) {
          const double t = u[q] + alpha * gradF[q];
          unew[q] = (t < 0) ? 0 : t; /* cwiseMax(0) */
        }
        {
          const double z = vdot(unew, unew, n);
          if (z > 0) { const double s = sqrt(z); for (int64_t q = 0; q < n; ++q) unew[q] = unew[q] / s; }
        }
        /* clipper.cpp:238-242 */
        {
          const double su = vsum(unew, n);
          spmv_sym_upper(M, unew, Mu); spmv_sym_upper(C, unew, Cu); n_spmv += 2; ++n_evals;
          for (int64_t q = 0; q < n; ++q)
            gradFnew[q] = (((1 + d) * unew[q] - (d * 1.0) * su) + Mu[q]) + Cu[q] * d;
          Fnew = vdot(unew, gradFnew, n);
        }
        deltaF = Fnew - F;
        if (deltaF < -P->eps) alpha = alpha * P->beta; /* clipper.cpp:246-248 */
        else break;
      }
      double du2 = 0.0;
      for (int64_t q = 0; q < n; ++q) { const double t = unew[q] - u[q]; du2 = du2 + t * t; }
      const double deltau = sqrt(du2);
      /* clipper.cpp:256-258: accepted even when the line search ran out */
      F = Fnew;
      { double *t = u; u = unew; unew = t; }
      { double *t = gradF; gradF = gradFnew; gradFnew = t; }
      ++n_inner;
      if (deltau < P->tol_u || fabs(deltaF) < P->tol_F) { ++j; break; }
    }
    if (trace && i < trace_cap) { trace[3 * i] = F; trace[3 * i + 1] = d_used; trace[3 * i + 2] = (double)j; }

    /* clipper.cpp:268-280 */
    {
      const double su = vsum(u, n);
      spmv_sym_upper(C, u, Cu); ++n_spmv;
      int64_t cnt = 0;
      for (int64_t q = 0; q < n; ++q) {
        Cbu[q] = (1.0 * su - Cu[q]) - u[q];
        if (Cbu[q] > P->eps && u[q] > P->eps) ++cnt;
      }
      if (cnt > 0) {
        spmv_sym_upper(M, u, Mu); ++n_spmv;
        double acc = 0.0;
        for (int64_t q = 0; q < n; ++q)
          if (Cbu[q] > P->eps && u[q] > P->eps) acc = acc + fabs((Mu[q] + u[q]) / Cbu[q]);
        d += acc / (double)cnt; /* abs().mean() (clipper.cpp:274) */
      } else {
        break;
      }
    }
  }

  /* clipper.cpp:287-310 */
  int32_t n_nodes = 0;
  if (P->rounding == 0) {
    n_nodes = orc_find_above(u, n, 0.0, nodes_out);
  } else if (P->rounding == 2) {
    /* the reference's (int)std::round(F) is undefined for NaN and F >= 2^31: round(F) is clamped to [0, n] first
     * and NaN keeps no node (a defined divergence, DESIGN section 5) */
    const double r = round(F);
    const int32_t omega = !(r >= 1.0) ? 0 : (r >= (double)n ? (int32_t)n : (int32_t)r);
    n_nodes = orc_find_k_largest(u, n, omega, nodes_out);
  } else {
    /* Rounding::DSD (clipper.cpp:294-300): densest subgraph of M_ restricted to support(u) */
    int32_t *supp = (int32_t *)malloc(sizeof(int32_t) * (size_t)(n > 0 ? n : 1));
    const int32_t nsupp = orc_find_above(u, n, 0.0, supp);
    n_nodes = nsupp > 0 ? orc_dsd(M, supp, nsupp, nodes_out) : 0;
    free(supp);
  }

  S->t = now_s() - t1;
  S->ifinal = (int32_t)i;
  S->n_nodes = n_nodes;
  S->score = F;
  S->d_final = d;
  S->n_evals = n_evals; S->n_spmv = n_spmv; S->n_inner = n_inner;
  memcpy(u_out, u, sizeof(double) * (size_t)n);

  free(gradF); free(gradFnew); free(u); free(unew); free(Mu); free(Cu); free(Cbu);
  return 0;
}

/* helper for the tests: y = gradF(v; d) exactly as clipper.cpp:219 builds it */
int orc_gradf(const orc_problem *p, const double *v, double d, double *y, double *F) {
  const int64_t n = p->M.m;
  double *Mu = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  double *Cu = (double *)malloc(sizeof(double) * (size_t)(n + 1));
  const double su = vsum(v, n);
  spmv_sym_upper(&p->M, v, Mu); spmv_sym_upper(&p->C, v, Cu);
  for (int64_t q = 0; q < n; ++q) y[q] = (((1 + d) * v[q] - (d * 1.0) * su) + Mu[q]) + Cu[q] * d;
  if (F) *F = vdot(v, y, n);
  free(Mu); free(Cu);
  return 0;
}

/* dsd::solve(const Eigen::MatrixXd& A, S) (dsd.cpp:322-325): sparseView of the dense matrix, then the above.
 * Only the strict upper triangle is ever read (dsd.cpp:300-302), so that is what is converted. */
int32_t orc_dsd_dense(const double *A, int64_t n, const int32_t *S, int32_t nS, int32_t *out) {
  orc_csc U;
  U.m = n;
  U.colptr = (int64_t *)calloc((size_t)n + 1, sizeof(int64_t));
  int64_t nnz = 0;
  for (int64_t j = 0; j < n; ++j)
    for (int64_t i = 0; i < j; ++i)
      if (A[(size_t)j * (size_t)n + (size_t)i] != 0.0) ++nnz;
  U.rowidx = (int32_t *)malloc(sizeof(int32_t) * (size_t)(nnz > 0 ? nnz : 1));
  U.val = (double *)malloc(sizeof(double) * (size_t)(nnz > 0 ? nnz : 1));
  int64_t k = 0;
  for (int64_t j = 0; j < n; ++j) {
    U.colptr[j] = k;
    for (int64_t i = 0; i < j; ++i) {
      const double v = A[(size_t)j * (size_t)n + (size_t)i];
      if (v != 0.0) { U.rowidx[k] = (int32_t)i; U.val[k] = v; ++k; }
    }
  }
  U.colptr[n] = k;
  const int32_t r = orc_dsd(&U, S, nS, out);
  free(U.colptr); free(U.rowidx); free(U.val);
  return r;
}
