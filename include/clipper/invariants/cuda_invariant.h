/**
 * @file cuda_invariant.h
 * @brief A custom pairwise invariant written in CUDA C++ and scored on the GPU (clp_score_custom, clipper_b200.h)
 */
#pragma once

#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "clipper/invariants/abstract.h"

namespace clipper {
namespace invariants {

  /// `source` defines
  ///   __device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj,
  ///                                   int d, const double* prm);
  /// evaluated for every distinct association pair i < j inside the scoring kernel, with prm = params (at most
  /// CLP_INV_MAX_PARAMS = 16 values).  The source is compiled at run time (NVRTC) the first time it is scored.
  class CudaInvariant : public PairwiseInvariant
  {
  public:
    CudaInvariant(std::string source, std::vector<double> params = {})
    : source_(std::move(source)), params_(std::move(params)) {}
    ~CudaInvariant() = default;

    /// there is no host evaluation: the function exists as CUDA source only
    double operator()(const Datum&, const Datum&, const Datum&, const Datum&) override
    {
      throw std::logic_error("CudaInvariant is evaluated on the GPU only");
    }

    const std::string& source() const { return source_; }
    const std::vector<double>& params() const { return params_; }

  private:
    std::string source_;
    std::vector<double> params_;
  };
  using CudaInvariantPtr = std::shared_ptr<CudaInvariant>;

} // ns invariants
} // ns clipper
