/**
 * @file clipper.h
 * @brief CLIPPER data association framework -- public API, H100 build.
 *
 * Mirror of reference include/clipper/clipper.h:27-148: same Params / Solution / CLIPPER, same
 * method names, argument meaning and defaults, so test/*.cpp, benchmarks/*.cpp and the pybind11
 * module written against the reference compile against this header.  The method bodies
 * (clipper_b200/csrc/clipper_shell.cpp) marshal into the C-ABI of include/clipper_b200.h, whose
 * entry points launch the sm_90a kernels: the affinity matrix lives in HBM as one dense array,
 * not in Eigen sparse matrices.  Errors reported by the C-ABI surface as std::runtime_error
 * (additive: the reference never throws and none of its callers catch).
 */
#pragma once

#include <memory>
#include <tuple>
#include <vector>

#include "clipper/invariants/abstract.h"
#include "clipper/invariants/builtins.h"
#include "clipper/types.h"

#include "clipper/dsd.h"
#include "clipper/sdp.h"
#include "clipper/maxclique.h"

namespace clipper {

  /// CLIPPER parameters (reference clipper.h:27-60, same fields and defaults)
  struct Params {
    double tol_u = 1e-8;   ///< stop when change in u < tol
    double tol_F = 1e-9;   ///< stop when change in F < tol
    double tol_Fop = 1e-10;///< declared by the reference, never read by its solver
    int maxiniters = 200;  ///< max gradient ascent steps for each d
    int maxoliters = 1000; ///< max outer loop iterations to find d

    double beta = 0.25;    ///< backtracking step size reduction, in (0, 1)
    int maxlsiters = 99;   ///< maximum line search iterations per gradient step

    double eps = 1e-9;     ///< numerical threshold around 0
    double affinityeps = 1e-4; ///< sparsity-promoting threshold for affinities

    bool rescale_u0 = true;///< rescale u0 using one power iteration

    enum Rounding { NONZERO, DSD, DSD_HEU };
    Rounding rounding = Rounding::DSD_HEU;
  };

  /// dense clique solution (reference clipper.h:65-73)
  struct Solution
  {
    double t = 0;           ///< duration spent solving [s]
    int ifinal = 0;         ///< number of outer iterations before convergence
    std::vector<int> nodes; ///< indices of graph vertices in dense clique
    Eigen::VectorXd u0;     ///< initial vector used for local solver
    Eigen::VectorXd u;      ///< characteristic vector associated with graph
    double score = 0;       ///< value of objective function / largest eigenvalue
  };

  /// Convenience class to use CLIPPER for data association (reference clipper.h:78-184)
  class CLIPPER
  {
  public:
    CLIPPER(const invariants::PairwiseInvariantPtr& invariant, const Params& params);
    ~CLIPPER() = default;

    /// consistency scores for the m associations of A (reference clipper.cpp:21-65);
    /// empty A = all-to-all hypothesis
    void scorePairwiseConsistency(const invariants::Data& D1,
                                  const invariants::Data& D2,
                                  const Association& A = Association());

    /// graduated projected gradient ascent (reference clipper.cpp:69-78,172-323);
    /// empty u0 = random start
    void solve(const Eigen::VectorXd& u0 = Eigen::VectorXd());

    void solveAsMaximumClique(const maxclique::Params& params = {});
    /// without params: a build without SCS (nothing selected); with params: the relaxation on the GPU (m <= 128)
    void solveAsMSRCSDR();
    void solveAsMSRCSDR(const sdp::Params& params);

    const Solution& getSolution() const { return soln_; }
    Affinity getAffinityMatrix();
    Constraint getConstraintMatrix();

    /// dense M, C: strict upper triangle is used (reference clipper.cpp:149-158)
    void setMatrixData(const Affinity& M, const Constraint& C);
    /// sparse strictly-upper-triangular M, C (reference clipper.cpp:162-166)
    void setSparseMatrixData(const SpAffinity& M, const SpConstraint& C);

    Association getInitialAssociations();
    Association getSelectedAssociations();

    void setParallelize(bool parallelize) { parallelize_ = parallelize; }

    // -- additive, H100 build only ------------------------------------------------------------
    /// choose the CUDA device and the HBM storage type of M (CLP_STORE_F32 / CLP_STORE_F64)
    /// before the first scoring call; defaults: device 0, fp32 storage
    void setDevice(int device, int storage = 0);
    /// device time of the last solver kernel [ms] and its number of objective evaluations
    double lastKernelMilliseconds() const { return kernel_ms_; }
    long long lastEvaluations() const { return n_evals_; }

  private:
    Params params_;
    invariants::PairwiseInvariantPtr invariant_;
    bool parallelize_ = true; ///< kept for source compatibility; the GPU path is always parallel

    Association A_;  ///< associations of the custom-invariant host path / cache of the scored set
    bool have_A_ = false;
    Solution soln_;
    std::shared_ptr<void> handle_; ///< clp_handle (include/clipper_b200.h), created lazily
    int device_ = 0, storage_ = 0;
    double kernel_ms_ = 0;
    long long n_evals_ = 0;

    void* handle();
  };

} // ns clipper
