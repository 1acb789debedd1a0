/**
 * @file sdp.h
 * @brief Semidefinite relaxation front-end (mirror of reference sdp.h:20-57).
 *        The reference solves the relaxation with the third-party SCS library (CMakeLists.txt:83-86).
 *        Here solve(M, C, params) solves it on the GPU (clp_sdp_solve: ADMM with a Jacobi eigensolver
 *        in shared memory, m <= 128, on a temporary fp64 handle on device 0) and fills every field:
 *        pobj = -<M, X> and dobj = -bound (SCS's sign), t_scs the device call, t_scs_solve its kernel,
 *        t_scs_cone its eigendecompositions and projections; t_scs_setup, t_scs_linsys and
 *        t_scs_accel are 0.  acceleration_interval, acceleration_lookback and eps_infeas are SCS
 *        settings without effect: the relaxation is always feasible and bounded.  solve(M, C)
 *        without params behaves like a reference build without CLIPPER_HAS_SCS (sdp.cpp:298-302).
 */
#pragma once
#include <vector>
#include "clipper/types.h"

namespace clipper {
namespace sdp {

  struct Solution
  {
    Eigen::MatrixXd X;
    Eigen::VectorXd lambdas;
    Eigen::VectorXd evec1;
    double thr = 0;
    std::vector<int> nodes;
    int iters = 0;
    float pobj = 0, dobj = 0;
    double t = 0, t_parse = 0, t_scs = 0, t_scs_setup = 0, t_scs_solve = 0, t_scs_linsys = 0,
           t_scs_cone = 0, t_scs_accel = 0, t_extract = 0;
  };

  struct Params
  {
    bool verbose = false;
    int max_iters = 2000;
    int acceleration_interval = 10;
    int acceleration_lookback = 10;
    float eps_abs = 1e-3;
    float eps_rel = 1e-3;
    float eps_infeas = 1e-7;
    float time_limit_secs = 0;
  };

  Solution solve(const Eigen::MatrixXd& M, const Eigen::MatrixXd& C);
  Solution solve(const Eigen::MatrixXd& M, const Eigen::MatrixXd& C, const Params& params);

} // ns sdp
} // ns clipper
