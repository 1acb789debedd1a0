/**
 * @file utils.h
 * @brief Utilities of the CLIPPER API (mirror of reference include/clipper/utils.h:20-165)
 */
#pragma once

#include <chrono>
#include <ostream>
#include <string>
#include <tuple>
#include <vector>

#include "clipper/invariants/abstract.h"
#include "clipper/types.h"

namespace clipper {
  struct Solution;
namespace utils {

  /// n x 1 vector with entries drawn from U[0,1), seeded from std::random_device (utils.cpp:22-29)
  Eigen::VectorXd randvec(size_t n);

  /// indices of the k largest elements, descending (utils.cpp:33-55)
  std::vector<int> findIndicesOfkLargest(const Eigen::VectorXd& x, int k);

  /// indices i with x[i] > thr, ascending (utils.cpp:59-68)
  std::vector<int> findIndicesWhereAboveThreshold(const Eigen::VectorXd& x, double thr);

  /// all-to-all association hypothesis, (n1*n2) x 2 (utils.h:61-71)
  Association createAllToAll(size_t n1, size_t n2);

  /// elements of x selected by a 0/1 indicator (utils.cpp:72-83)
  Eigen::VectorXd selectFromIndicator(const Eigen::VectorXd& x, const Eigen::VectorXi& ind);

  /// rows of A picked by the solution's nodes (utils.cpp:101-108)
  Association selectInlierAssociations(const Solution& soln, const Association& A);

  /// flat index k of the strict upper triangle -> (row, col) (utils.cpp:87-97)
  std::tuple<size_t,size_t> k2ij(size_t k, size_t n);

  /**
   * @brief Putative associations by exact k-nearest-neighbour matching on the GPU (device 0, a temporary handle);
   * the reference's benchmarks/bm_utils.cpp:147-232 for any d <= CLP_KNN_MAX_D.  Column i of D1 is matched to its
   * min(knn, n2) nearest columns of D2 (squared distance, ties to the lower index); a pair is kept when its squared
   * distance is <= radius * radius.  Rows (c0, c1) by c0 then rank; with enforce1to1 every c1 keeps its nearest c0
   * (ties to the smallest), rows by c1.  Semantics in full: include/clipper_b200.h, clp_correspondences.
   */
  Association distanceBasedCorrespondences(const invariants::Data& D1, const invariants::Data& D2, size_t knn,
                                           double radius, bool enforce1to1);

  /**
   * @brief distanceBasedCorrespondences of many cloud pairs in one batched call on the GPU (device 0, a temporary
   * clp_batch; clp_batch_correspondences).  Entry p of the result is exactly distanceBasedCorrespondences(D1s[p],
   * D2s[p], knn, radius, enforce1to1).  D1s and D2s have the same length and every cloud the same number of rows; an
   * empty list gives an empty result.
   */
  std::vector<Association> distanceBasedCorrespondencesBatch(const std::vector<invariants::Data>& D1s,
                                                             const std::vector<invariants::Data>& D2s, size_t knn,
                                                             double radius, bool enforce1to1);

  /// the rigid transform that aligns associated points, and how well it is determined (clp_tf_info)
  struct RigidTransformEstimate {
    Eigen::MatrixXd T;   ///< (d+1) x (d+1), last row [0 .. 0 1]: b ~ R a + t maps the frame of D1 into that of D2
    int status = 0;      ///< CLP_TF_OK, CLP_TF_EMPTY, CLP_TF_DEGENERATE or CLP_TF_NONFINITE
    int k = 0;           ///< pairs used
    double rmse = 0.0;   ///< sqrt(sum |R a_i + t - b_i|^2 / k)
    double gap = 0.0;    ///< sv[d-2] + sign(det H) sv[d-1]: R is unique exactly when gap > 0
    Eigen::VectorXd sv;  ///< the 3 singular values of H = sum (b_i - mu_b)(a_i - mu_a)', descending
  };

  /**
   * @brief The proper rigid transform that aligns the pairs (D1.col(A(i,0)), D2.col(A(i,1))) of every row of A, e.g.
   * getSelectedAssociations(), on the GPU (device 0, a temporary handle; clp_estimate_transform).  d is 2 or 3.  An empty
   * A gives CLP_TF_EMPTY (no pairs; not the all-to-all hypothesis).  Semantics in full: include/clipper_b200.h.
   */
  RigidTransformEstimate estimateRigidTransform(const invariants::Data& D1, const invariants::Data& D2,
                                                const Association& A);

  /**
   * @brief estimateRigidTransform of many problems in one batched call on the GPU (device 0, a temporary clp_batch;
   * clp_batch_estimate_transform).  Entry p is bit for bit estimateRigidTransform(D1s[p], D2s[p], As[p]).  The three
   * lists have the same length and every cloud the same number of rows; an empty list gives an empty result.
   */
  std::vector<RigidTransformEstimate> estimateRigidTransformBatch(const std::vector<invariants::Data>& D1s,
                                                                  const std::vector<invariants::Data>& D2s,
                                                                  const std::vector<Association>& As);

  /// simple named profiling timer (utils.h:107-163)
  class Timer
  {
  public:
    Timer() = default;
    Timer(const std::string& name) : name_(name) {}
    void start() { t1_ = clock::now(); running_ = true; }
    void stop()
    {
      t2_ = clock::now();
      if (running_) {
        total_ += std::chrono::duration<double>(t2_ - t1_).count();
        running_ = false;
        count_++;
      }
    }
    void reset() { total_ = 0; }
    double getElapsedSeconds() const { return total_; }

    friend std::ostream& operator<<(std::ostream& os, const Timer& t)
    {
      if (!t.name_.empty()) os << t.name_ << ": ";
      os << t.total_ << " s (" << t.count_ << "x)";
      return os;
    }
    friend Timer operator+(const Timer& lhs, const Timer& rhs) { Timer t; t.total_ = lhs.total_ + rhs.total_; return t; }

  private:
    using clock = std::chrono::high_resolution_clock;
    double total_ = 0;
    std::string name_;
    int count_ = 0;
    bool running_ = false;
    std::chrono::time_point<clock> t1_, t2_;
  };

} // ns utils
} // ns clipper
