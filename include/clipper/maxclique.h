/**
 * @file maxclique.h
 * @brief Maximum-clique front-end (mirror of reference maxclique.h:14-28).  The reference delegates to the
 *        third-party PMC library; here the three methods run on the GPU (clp_max_clique of clipper_b200.h):
 *          KCORE  every vertex whose core number is the max core;
 *          HEU    greedy clique from every seed (highest core number first, ties to the lowest index), the largest
 *                 one, ties to the smallest seed -- our deterministic statement of PMC's "kcore" heuristic;
 *          EXACT  a maximum clique by branch-and-bound (bitset colouring bound), started from the HEU clique;
 *                 when time_limit [s] expires the best clique found is returned (0: the HEU clique).
 *        solve() uses device 0: any nonzero of the strict upper triangle of A is an edge.  `threads` is not used
 *        (the GPU decides its own parallelism); `verbose` prints one statistics line.  Nodes come back ascending.
 */
#pragma once
#include <cstddef>
#include <vector>
#include "clipper/types.h"

namespace clipper {
namespace maxclique {

enum class Method { EXACT, HEU, KCORE };

struct Params
{
  Method method = Method::EXACT;
  size_t threads = 24;   ///< kept for source compatibility; not used
  int time_limit = 3600; ///< [s] EXACT only
  bool verbose = false;
};

std::vector<int> solve(const Eigen::MatrixXd& A, const Params& params = {});

} // ns maxclique
} // ns clipper
