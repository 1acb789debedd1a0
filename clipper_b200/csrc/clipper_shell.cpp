// clipper_shell.cpp -- bodies of the reference's C++ API (include/clipper/*.h) over the C-ABI.
//
// This is the "reference-side binding": every method of clipper::CLIPPER marshals its Eigen-typed
// arguments into plain pointers and calls include/clipper_b200.h (which launches the sm_90a
// kernels).  Nothing numerical of the hot path happens in this file; what does happen here is
//   * the custom-invariant host path (SURVEY D9): a user-defined PairwiseInvariant other than a
//     CudaInvariant (which is compiled into the scoring kernel, clp_score_custom) is evaluated pair by
//     pair on the host (like reference clipper.cpp:31-56) and the resulting dense matrices are
//     uploaded with clp_set_dense;
//   * single-pair operator() of the two built-in invariants (API completeness; the reference
//     exposes them, e.g. py_clipper.cpp:43), never used for scoring association sets.
#include "clipper/clipper.h"
#include "clipper/utils.h"
#include "clipper_b200.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <iostream>
#include <memory>
#include <random>
#include <stdexcept>
#include <string>

namespace clipper {

namespace {

void check(void* h, int rc, const char* what) {
  if (rc != CLP_OK)
    throw std::runtime_error(std::string("clipper_b200: ") + what + ": " + clp_last_error(static_cast<clp_handle>(h)));
}

double dist3(const invariants::Datum& a, const invariants::Datum& b, int off, int d) {
  double s = 0;
  for (int q = 0; q < d; ++q) { const double t = a(off + q) - b(off + q); s = s + t * t; }
  return std::sqrt(s);
}

}  // namespace

// ---- invariants: single-pair functors ---------------------------------------------------------
namespace invariants {

// reference src/invariants/euclidean_distance.cpp:13-31
double EuclideanDistance::operator()(const Datum& ai, const Datum& aj, const Datum& bi, const Datum& bj)
{
  const int d = (int)ai.size();
  const double l1 = dist3(ai, aj, 0, d);
  const double l2 = dist3(bi, bj, 0, d);
  if (params_.mindist > 0 && (l1 < params_.mindist || l2 < params_.mindist)) return 0.0;
  const double c = std::abs(l1 - l2);
  return (c < params_.epsilon) ? std::exp(-0.5 * c * c / (params_.sigma * params_.sigma)) : 0;
}

// reference src/invariants/pointnormal_distance.cpp:13-35 (acos deliberately not clamped)
double PointNormalDistance::operator()(const Datum& ai, const Datum& aj, const Datum& bi, const Datum& bj)
{
  const double l1 = dist3(ai, aj, 0, 3);
  const double l2 = dist3(bi, bj, 0, 3);
  const double alpha1 = std::acos(ai(3) * aj(3) + ai(4) * aj(4) + ai(5) * aj(5));
  const double alpha2 = std::acos(bi(3) * bj(3) + bi(4) * bj(4) + bi(5) * bj(5));
  const double dp = std::abs(l1 - l2);
  const double dn = std::abs(alpha1 - alpha2);
  if (dp < params_.epsp && dn < params_.epsn) {
    const double sp = std::exp(-0.5 * dp * dp / (params_.sigp * params_.sigp));
    const double sn = std::exp(-0.5 * dn * dn / (params_.sign * params_.sign));
    return sp * sn;
  }
  return 0.0;
}

}  // namespace invariants

// ---- CLIPPER -----------------------------------------------------------------------------------
CLIPPER::CLIPPER(const invariants::PairwiseInvariantPtr& invariant, const Params& params)
: params_(params), invariant_(invariant)
{}

void CLIPPER::setDevice(int device, int storage)
{
  device_ = device; storage_ = storage;
  handle_.reset();
}

void* CLIPPER::handle()
{
  if (!handle_) {
    clp_handle h = nullptr;
    const int rc = clp_create(device_, storage_, &h);
    if (rc != CLP_OK) throw std::runtime_error(std::string("clipper_b200: clp_create: ") + clp_last_error(nullptr));
    handle_ = std::shared_ptr<void>(h, [](void* p) { clp_destroy(static_cast<clp_handle>(p)); });
  }
  clp_params p;
  p.tol_u = params_.tol_u; p.tol_F = params_.tol_F; p.tol_Fop = params_.tol_Fop;
  p.maxiniters = params_.maxiniters; p.maxoliters = params_.maxoliters;
  p.beta = params_.beta; p.maxlsiters = params_.maxlsiters;
  p.eps = params_.eps; p.affinityeps = params_.affinityeps;
  p.rescale_u0 = params_.rescale_u0 ? 1 : 0; p.rounding = (int)params_.rounding;
  check(handle_.get(), clp_set_params(static_cast<clp_handle>(handle_.get()), &p), "clp_set_params");
  return handle_.get();
}

void CLIPPER::scorePairwiseConsistency(const invariants::Data& D1, const invariants::Data& D2, const Association& A)
{
  clp_handle h = static_cast<clp_handle>(handle());
  const int32_t* Ap = (A.size() == 0) ? nullptr : reinterpret_cast<const int32_t*>(A.data());
  const int64_t m = (A.size() == 0) ? 0 : (int64_t)A.rows();
  have_A_ = false;

  if (auto* e = dynamic_cast<invariants::EuclideanDistance*>(invariant_.get())) {
    const auto& ip = e->params();
    check(h, clp_score_euclidean(h, D1.data(), (int32_t)D1.rows(), (int64_t)D1.cols(), D2.data(), (int64_t)D2.cols(),
                                 Ap, m, ip.sigma, ip.epsilon, ip.mindist), "clp_score_euclidean");
    return;
  }
  if (auto* pn = dynamic_cast<invariants::PointNormalDistance*>(invariant_.get())) {
    if (D1.rows() != 6 || D2.rows() != 6) throw std::runtime_error("PointNormalDistance expects 6 x n data");
    const auto& ip = pn->params();
    check(h, clp_score_pointnormal(h, D1.data(), (int64_t)D1.cols(), D2.data(), (int64_t)D2.cols(), Ap, m,
                                   ip.sigp, ip.epsp, ip.sign, ip.epsn), "clp_score_pointnormal");
    return;
  }
  if (auto* cu = dynamic_cast<invariants::CudaInvariant*>(invariant_.get())) {
    if (D1.rows() != D2.rows()) throw std::runtime_error("CudaInvariant expects D1 and D2 of equal dimension");
    const auto& prm = cu->params();
    check(h, clp_score_custom(h, cu->source().c_str(), prm.empty() ? nullptr : prm.data(), (int32_t)prm.size(),
                              D1.data(), (int32_t)D1.rows(), (int64_t)D1.cols(), D2.data(), (int64_t)D2.cols(), Ap, m),
          "clp_score_custom");
    return;
  }

  // custom invariant: host loop over the pairs (reference clipper.cpp:31-56), then upload
  if (A.size() == 0) A_ = utils::createAllToAll(D1.cols(), D2.cols());
  else A_ = A;
  have_A_ = true;
  const size_t mm = A_.rows();
  Eigen::MatrixXd M = Eigen::MatrixXd::Zero(mm, mm);
  Eigen::MatrixXd C = Eigen::MatrixXd::Zero(mm, mm);
  for (size_t j = 0; j < mm; ++j) {
    const invariants::Datum d1j = D1.col(A_(j, 0)), d2j = D2.col(A_(j, 1));
    for (size_t i = 0; i < j; ++i) {
      if (A_(i, 0) == A_(j, 0) || A_(i, 1) == A_(j, 1)) continue;
      const invariants::Datum d1i = D1.col(A_(i, 0)), d2i = D2.col(A_(i, 1));
      const double scr = (*invariant_)(d1i, d1j, d2i, d2j);
      // C_ = pattern of M_ = M.sparseView(), which drops exact zeros (clipper.cpp:53-64)
      if (scr > params_.affinityeps && scr != 0.0) { M(i, j) = scr; C(i, j) = 1; }
    }
  }
  check(h, clp_set_dense(h, M.data(), C.data(), (int64_t)mm), "clp_set_dense");
}

void CLIPPER::solve(const Eigen::VectorXd& u0)
{
  clp_handle h = static_cast<clp_handle>(handle());
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  if (u0.size() != 0 && (int64_t)u0.size() != m) throw std::runtime_error("clipper_b200: u0 has the wrong length");
  clp_solution s;
  Eigen::VectorXd u(m), u0used(m);
  std::vector<int32_t> nodes((size_t)std::max<int64_t>(m, 1));
  check(h, clp_solve(h, u0.size() == 0 ? nullptr : u0.data(), &s, u.data(), nodes.data(), u0used.data()), "clp_solve");
  soln_.t = s.t;
  soln_.ifinal = s.ifinal;
  soln_.nodes.assign(nodes.begin(), nodes.begin() + s.n_nodes);
  soln_.u0 = u0used;
  soln_.u = u;
  soln_.score = s.score;
  kernel_ms_ = s.kernel_ms;
  n_evals_ = s.n_evals;
}

namespace {

// clp_max_clique on a handle that holds the graph; one stats line when verbose
std::vector<int> max_clique_on(clp_handle h, const maxclique::Params& params)
{
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  std::vector<int32_t> nodes((size_t)std::max<int64_t>(m, 1));
  clp_mc_info info;
  check(h, clp_max_clique(h, (int)params.method, (double)params.time_limit, nodes.data(), &info), "clp_max_clique");
  if (params.verbose)
    std::cout << "maxclique: n " << m << " edges " << info.n_edges << " max core " << info.max_core << " lb "
              << info.lower_bound << " ub " << info.upper_bound << " omega " << info.n_nodes << " proven " << info.proven
              << (info.timed_out ? " (time limit)" : "") << " | adjacency " << info.adjacency_ms << " ms, peel "
              << info.peel_ms << " ms, heuristic " << info.heuristic_ms << " ms, search " << info.search_ms << " ms ("
              << info.n_branches << " branches)" << std::endl;
  return std::vector<int>(nodes.begin(), nodes.begin() + info.n_nodes);
}

// the semidefinite relaxation of the matrix a handle holds (clp_sdp_solve) as an sdp::Solution; t_parse starts at
// parse_s (host set-up the caller did), and the SCS timers map to the device call: t_scs its wall time, t_scs_solve the
// kernel, t_scs_cone the eigendecompositions and projections
sdp::Solution sdp_on(clp_handle h, const sdp::Params& params, double parse_s)
{
  utils::Timer tim;
  tim.start();
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  sdp::Solution s;
  clp_sdp_params p;
  clp_sdp_default_params(&p);
  p.max_iters = params.max_iters; p.eps_abs = params.eps_abs; p.eps_rel = params.eps_rel;
  p.time_limit_s = params.time_limit_secs;
  std::vector<int32_t> nodes((size_t)std::max<int64_t>(m, 1));
  s.X = Eigen::MatrixXd::Zero(m, m);
  s.lambdas = Eigen::VectorXd::Zero(m);
  s.evec1 = Eigen::VectorXd::Zero(m);
  clp_sdp_info info;
  tim.stop();
  s.t_parse = parse_s + tim.getElapsedSeconds();
  check(h, clp_sdp_solve(h, &p, &info, nodes.data(), s.X.data(), s.lambdas.data(), s.evec1.data()), "clp_sdp_solve");
  tim.reset();
  tim.start();
  s.nodes.assign(nodes.begin(), nodes.begin() + info.n_nodes);
  s.thr = info.thr;
  s.iters = info.iters;
  s.pobj = (float)-info.value;  // SCS minimises -<M, X>
  s.dobj = (float)-info.bound;
  s.t_scs = info.t;
  s.t_scs_solve = 1e-3 * info.kernel_ms;
  s.t_scs_cone = 1e-3 * info.proj_ms;
  s.t_scs_setup = s.t_scs_linsys = s.t_scs_accel = 0;
  tim.stop();
  s.t_extract = tim.getElapsedSeconds();
  s.t = s.t_parse + s.t_scs + s.t_extract;
  if (params.verbose)
    std::cout << "sdp: n " << m << " iters " << info.iters << (info.converged ? " converged" : "")
              << (info.timed_out ? " (time limit)" : "") << " value " << info.value << " bound " << info.bound << " rho "
              << info.rho << " sweeps " << info.n_sweeps << " nodes " << info.n_nodes << " | kernel " << info.kernel_ms
              << " ms, eig+proj " << info.proj_ms << " ms" << std::endl;
  return s;
}

}  // namespace

// reference clipper.cpp:82-97, on the graph already in HBM (no dense round trip); params.threads is not used
void CLIPPER::solveAsMaximumClique(const maxclique::Params& params)
{
  clp_handle h = static_cast<clp_handle>(handle());
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  utils::Timer tim;
  tim.start();
  std::vector<int> nodes = max_clique_on(h, params);
  tim.stop();
  soln_.t = tim.getElapsedSeconds();
  soln_.ifinal = 0;
  std::swap(soln_.nodes, nodes);
  soln_.u = Eigen::VectorXd::Zero(m);
  soln_.score = -1;
}

// reference clipper.cpp:101-113 without params: a build without SCS (sdp::solve(M, C) selects nothing)
void CLIPPER::solveAsMSRCSDR()
{
  Eigen::MatrixXd M = getAffinityMatrix();
  Eigen::MatrixXd C = getConstraintMatrix();
  sdp::Solution soln = sdp::solve(M, C);
  soln_.t = soln.t;
  soln_.ifinal = 0;
  std::swap(soln_.nodes, soln.nodes);
  soln_.u = Eigen::VectorXd::Zero(M.cols());
  soln_.score = -1;
}

// reference clipper.cpp:101-113 with params: the relaxation on the GPU, of the matrix already in HBM
void CLIPPER::solveAsMSRCSDR(const sdp::Params& params)
{
  clp_handle h = static_cast<clp_handle>(handle());
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  sdp::Solution soln = sdp_on(h, params, 0.0);
  soln_.t = soln.t;
  soln_.ifinal = 0;
  std::swap(soln_.nodes, soln.nodes);
  soln_.u = Eigen::VectorXd::Zero(m);
  soln_.score = -1;
}

Affinity CLIPPER::getAffinityMatrix()
{
  clp_handle h = static_cast<clp_handle>(handle());
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  Affinity M(m, m);
  if (m > 0) check(h, clp_get_dense(h, 0, M.data()), "clp_get_dense");
  return M;
}

Constraint CLIPPER::getConstraintMatrix()
{
  clp_handle h = static_cast<clp_handle>(handle());
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  Constraint C(m, m);
  if (m > 0) check(h, clp_get_dense(h, 1, C.data()), "clp_get_dense");
  return C;
}

void CLIPPER::setMatrixData(const Affinity& M, const Constraint& C)
{
  clp_handle h = static_cast<clp_handle>(handle());
  if (M.rows() != M.cols() || C.rows() != M.rows() || C.cols() != M.cols())
    throw std::runtime_error("clipper_b200: setMatrixData expects square M and C of equal size");
  have_A_ = false;
  check(h, clp_set_dense(h, M.data(), C.data(), (int64_t)M.rows()), "clp_set_dense");
}

void CLIPPER::setSparseMatrixData(const SpAffinity& Min, const SpConstraint& Cin)
{
  clp_handle h = static_cast<clp_handle>(handle());
  SpAffinity M = Min; SpConstraint C = Cin;
  M.makeCompressed(); C.makeCompressed();
  const int64_t m = (int64_t)M.cols();
  auto widen = [m](const int* p) { return std::vector<int64_t>(p, p + m + 1); };
  const std::vector<int64_t> cpM = widen(M.outerIndexPtr()), cpC = widen(C.outerIndexPtr());
  have_A_ = false;
  check(h, clp_set_sparse_upper(h, m, cpM.data(), M.innerIndexPtr(), M.valuePtr(), cpC.data(), C.innerIndexPtr(),
                                C.valuePtr()), "clp_set_sparse_upper");
}

Association CLIPPER::getInitialAssociations()
{
  if (have_A_) return A_;
  clp_handle h = static_cast<clp_handle>(handle());
  int64_t m = 0;
  check(h, clp_num_associations(h, &m), "clp_num_associations");
  Association A(m, 2);
  if (m > 0) check(h, clp_get_associations(h, reinterpret_cast<int32_t*>(A.data())), "clp_get_associations");
  return A;
}

Association CLIPPER::getSelectedAssociations()
{
  return utils::selectInlierAssociations(soln_, getInitialAssociations());
}

// ---- utils -------------------------------------------------------------------------------------
namespace utils {

Eigen::VectorXd randvec(size_t n)
{
  std::random_device rd;
  std::mt19937 gen(rd());
  std::uniform_real_distribution<double> dis(0, 1);
  Eigen::VectorXd v(n);
  for (size_t i = 0; i < n; ++i) v(i) = dis(gen);
  return v;
}

std::vector<int> findIndicesOfkLargest(const Eigen::VectorXd& x, int k)
{
  if (k < 1 || x.size() == 0) return {};
  std::vector<int32_t> out((size_t)std::min<long>(k, (long)x.size()));
  const int n = clp_find_k_largest(x.data(), (int64_t)x.size(), k, out.data());
  return std::vector<int>(out.begin(), out.begin() + n);
}

std::vector<int> findIndicesWhereAboveThreshold(const Eigen::VectorXd& x, double thr)
{
  std::vector<int32_t> out((size_t)std::max<long>(1, (long)x.size()));
  const int n = clp_find_above(x.data(), (int64_t)x.size(), thr, out.data());
  return std::vector<int>(out.begin(), out.begin() + n);
}

Association createAllToAll(size_t n1, size_t n2)
{
  Association A(n1 * n2, 2);
  if (n1 * n2 > 0) clp_create_all_to_all((int64_t)n1, (int64_t)n2, reinterpret_cast<int32_t*>(A.data()));
  return A;
}

// bm_utils.cpp:147-232 on the GPU (clp_correspondences) with a temporary handle on device 0
Association distanceBasedCorrespondences(const invariants::Data& D1, const invariants::Data& D2, size_t knn, double radius,
                                         bool enforce1to1)
{
  if (D1.rows() != D2.rows())
    throw std::runtime_error("clipper_b200: distanceBasedCorrespondences expects D1 and D2 with the same number of rows");
  const int32_t k = (int32_t)std::min<size_t>(knn, (size_t)INT32_MAX);  // the C-ABI checks the range
  const int64_t n1 = (int64_t)D1.cols(), n2 = (int64_t)D2.cols();
  // sized for the cap, not for knn: a knn above it is rejected by the C-ABI (CLP_ERR_UNSUPPORTED) before anything is written
  const int64_t cap = n1 * std::min<int64_t>({(int64_t)std::max<int32_t>(k, 0), (int64_t)CLP_KNN_MAX_K, n2});
  clp_handle h = nullptr;
  if (clp_create(0, CLP_STORE_F32, &h) != CLP_OK)
    throw std::runtime_error(std::string("clipper_b200: clp_create: ") + clp_last_error(nullptr));
  std::shared_ptr<void> guard(h, [](void* p) { clp_destroy(static_cast<clp_handle>(p)); });
  std::vector<int32_t> buf((size_t)std::max<int64_t>(2 * cap, 1));
  int64_t m = 0;
  check(h, clp_correspondences(h, D1.data(), (int32_t)D1.rows(), n1, D2.data(), n2, k, radius,
                               enforce1to1 ? 1 : 0, buf.data(), cap, &m), "clp_correspondences");
  Association A(m, 2);
  if (m > 0) std::memcpy(A.data(), buf.data(), sizeof(int32_t) * (size_t)(2 * m));
  return A;
}

Eigen::VectorXd selectFromIndicator(const Eigen::VectorXd& x, const Eigen::VectorXi& ind)
{
  long cnt = 0;
  for (long i = 0; i < (long)ind.size(); ++i) cnt += ind(i) ? 1 : 0;
  Eigen::VectorXd y(cnt);
  long k = 0;
  for (long i = 0; i < (long)x.size(); ++i) if (ind(i)) y(k++) = x(i);
  return y;
}

Association selectInlierAssociations(const Solution& soln, const Association& A)
{
  Association Ain(soln.nodes.size(), 2);
  for (size_t i = 0; i < soln.nodes.size(); ++i) {
    Ain(i, 0) = A(soln.nodes[i], 0);
    Ain(i, 1) = A(soln.nodes[i], 1);
  }
  return Ain;
}

std::tuple<size_t,size_t> k2ij(size_t k, size_t n)
{
  uint64_t i = 0, j = 0;
  clp_k2ij(k, n, &i, &j);
  return {(size_t)i, (size_t)j};
}

}  // namespace utils

// ---- dsd / sdp / maxclique front-ends -------------------------------------------------------------
namespace dsd {

std::vector<int> solve(const Eigen::MatrixXd& A, const std::vector<int>& S)
{
  const int64_t n = (int64_t)A.rows();
  std::vector<int32_t> out((size_t)std::max<int64_t>(n, 1));
  std::vector<int32_t> Sin(S.begin(), S.end());
  const int k = clp_dsd_dense(A.data(), n, Sin.empty() ? nullptr : Sin.data(), (int32_t)Sin.size(), out.data());
  if (k < 0) throw std::runtime_error("clipper_b200: dsd::solve failed");
  return std::vector<int>(out.begin(), out.begin() + k);
}

std::vector<int> solve(const SpAffinity& Ain, const std::vector<int>& S)
{
  // the sparse overload reads the upper triangle only (reference dsd.cpp:300-302): densify it
  SpAffinity A = Ain;
  A.makeCompressed();
  const long n = (long)A.rows();
  Eigen::MatrixXd D = Eigen::MatrixXd::Zero(n, n);
  for (long j = 0; j < (long)A.cols(); ++j)
    for (int q = A.outerIndexPtr()[j]; q < A.outerIndexPtr()[j + 1]; ++q) {
      const long i = A.innerIndexPtr()[q];
      if (i < j) { D(i, j) = A.valuePtr()[q]; D(j, i) = A.valuePtr()[q]; }
    }
  return solve(D, S);
}

}  // namespace dsd

namespace sdp {
Solution solve(const Eigen::MatrixXd&, const Eigen::MatrixXd&)
{
  std::cout << "Warning: clipper was not built with SCS; SDR solver unavailable." << std::endl;
  return {};
}

// reference sdp.cpp:88-296 on a temporary fp64 handle on device 0: the strict upper triangles of M and C are used
Solution solve(const Eigen::MatrixXd& M, const Eigen::MatrixXd& C, const Params& params)
{
  utils::Timer tim;
  tim.start();
  const int64_t n = (int64_t)M.rows();
  if (M.cols() != M.rows() || C.rows() != M.rows() || C.cols() != M.cols())
    throw std::runtime_error("clipper_b200: sdp::solve expects square M and C of the same size");
  clp_handle h = nullptr;
  if (clp_create(0, CLP_STORE_F64, &h) != CLP_OK)
    throw std::runtime_error(std::string("clipper_b200: clp_create: ") + clp_last_error(nullptr));
  std::shared_ptr<void> guard(h, [](void* p) { clp_destroy(static_cast<clp_handle>(p)); });
  check(h, clp_set_dense(h, M.data(), C.data(), n), "clp_set_dense");
  tim.stop();
  return sdp_on(h, params, tim.getElapsedSeconds());
}
}  // namespace sdp

namespace maxclique {
// reference maxclique.cpp:46-147 on device 0: any nonzero of the strict upper triangle of A is an edge
std::vector<int> solve(const Eigen::MatrixXd& A, const Params& params)
{
  const int64_t n = (int64_t)A.rows();
  if (A.cols() != A.rows()) throw std::runtime_error("clipper_b200: maxclique::solve expects a square matrix");
  if (n == 0) return {};
  clp_handle h = nullptr;
  if (clp_create(0, CLP_STORE_F32, &h) != CLP_OK)
    throw std::runtime_error(std::string("clipper_b200: clp_create: ") + clp_last_error(nullptr));
  std::shared_ptr<void> guard(h, [](void* p) { clp_destroy(static_cast<clp_handle>(p)); });
  Eigen::MatrixXd M = Eigen::MatrixXd::Zero(n, n), C = Eigen::MatrixXd::Zero(n, n);
  for (int64_t j = 0; j < n; ++j)
    for (int64_t i = 0; i < j; ++i) C(i, j) = A(i, j) != 0 ? 1.0 : 0.0;
  check(h, clp_set_dense(h, M.data(), C.data(), n), "clp_set_dense");
  return max_clique_on(h, params);
}
}  // namespace maxclique

}  // namespace clipper
