/**
 * @file abstract.h
 * @brief Base classes of geometric invariants (mirror of reference invariants/abstract.h:19-74)
 */
#pragma once

#include <memory>

#include "clipper/types.h"

namespace clipper {
namespace invariants {

  using Data = Eigen::MatrixXd;   ///< d x n, one datum per (contiguous) column
  using Datum = Eigen::VectorXd;

  /// An invariant is a quantity that does not change under the transformation between two
  /// sets of objects (reference abstract.h:37-40).
  class Invariant {
  public:
    virtual ~Invariant() = default;
  };
  using InvariantPtr = std::shared_ptr<Invariant>;

  /// Real-valued pairwise scoring function f : A x A x A x A -> R (reference abstract.h:56-72).
  /// EuclideanDistance and PointNormalDistance are evaluated inside the CUDA scoring kernel, and so is
  /// CudaInvariant (cuda_invariant.h), a custom invariant written in CUDA C++ and compiled at run time;
  /// any other subclass is evaluated on the host, pair by pair, like the reference does.
  class PairwiseInvariant : public Invariant
  {
  public:
    virtual ~PairwiseInvariant() = default;
    virtual double operator()(const Datum& ai, const Datum& aj, const Datum& bi, const Datum& bj) = 0;
  };
  using PairwiseInvariantPtr = std::shared_ptr<PairwiseInvariant>;

} // ns invariants
} // ns clipper
