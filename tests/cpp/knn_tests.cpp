// knn_tests.cpp -- utils::distanceBasedCorrespondences of the C++ shell (clp_correspondences on device 0) against a
// plain loop over the same semantics and on hand-built cases.  Every test needs the GPU.  Same assertion harness as
// shell_tests.cpp.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <limits>
#include <map>
#include <random>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include <clipper/clipper.h>
#include <clipper/utils.h>

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("  FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) EXPECT_TRUE((a) == (b))

// the semantics of include/clipper_b200.h (clp_correspondences) as a loop: squared distance accumulated in order,
// neighbours by (sd, j), NaN never one, sd <= radius^2 kept, 1-to-1 by least sd then least c0, rows by c1
static std::vector<std::pair<int, int>> brute(const Eigen::MatrixXd& D1, const Eigen::MatrixXd& D2, size_t knn, double radius,
                                              bool one) {
  std::vector<std::pair<int, int>> rows;
  std::map<int, std::pair<double, int>> best;
  const double r2 = radius * radius;
  for (long i = 0; i < (long)D1.cols(); ++i) {
    std::vector<std::pair<double, int>> c;
    for (long j = 0; j < (long)D2.cols(); ++j) {
      volatile double s = 0;  // volatile: one rounding per operation, as on the device
      for (long k = 0; k < (long)D1.rows(); ++k) {
        volatile double t = D1(k, i) - D2(k, j);
        volatile double p = t * t;
        s = k == 0 ? (double)p : s + p;
      }
      if (s == s) c.push_back({s, (int)j});
    }
    std::sort(c.begin(), c.end());
    for (size_t r = 0; r < std::min(knn, c.size()); ++r)
      if (c[r].first <= r2) {
        rows.push_back({(int)i, c[r].second});
        auto it = best.find(c[r].second);
        if (it == best.end() || c[r].first < it->second.first) best[c[r].second] = {c[r].first, (int)i};
      }
  }
  if (one) {
    rows.clear();
    for (const auto& b : best) rows.push_back({b.second.second, b.first});
  }
  return rows;
}

static bool same(const clipper::Association& A, const std::vector<std::pair<int, int>>& want) {
  if ((size_t)A.rows() != want.size()) return false;
  for (size_t r = 0; r < want.size(); ++r)
    if (A(r, 0) != want[r].first || A(r, 1) != want[r].second) return false;
  return true;
}

static Eigen::MatrixXd random_cloud(int d, int n, unsigned seed) {
  std::mt19937 gen(seed);
  std::normal_distribution<double> g(0.0, 1.0);
  Eigen::MatrixXd D(d, n);
  for (int j = 0; j < n; ++j) for (int k = 0; k < d; ++k) D(k, j) = g(gen);
  return D;
}

// random clouds, d = 3 and 33, with and without a radius and 1-to-1, against the loop
static void Utils_RandomAgainstLoop() {
  for (int d : {3, 33}) {
    const Eigen::MatrixXd D1 = random_cloud(d, 300, 1 + d), D2 = random_cloud(d, 457, 2 + d);
    for (size_t knn : {1, 4, 32})
      for (double radius : {std::numeric_limits<double>::infinity(), d == 3 ? 0.4 : 7.0})
        for (bool one : {false, true}) {
          const clipper::Association A = clipper::utils::distanceBasedCorrespondences(D1, D2, knn, radius, one);
          EXPECT_TRUE(same(A, brute(D1, D2, knn, radius, one)));
        }
  }
}

// duplicate candidates: the lower index wins; knn > n2 is clamped; 1-to-1 keeps the smallest c0 on equal sd
static void Utils_TiesAndClamp() {
  Eigen::MatrixXd D2(1, 4), D1(1, 2);
  D2 << 1, 0, 1, 0;
  D1 << 0, 1;
  const double inf = std::numeric_limits<double>::infinity();
  EXPECT_TRUE(same(clipper::utils::distanceBasedCorrespondences(D1, D2, 2, inf, false), {{0, 1}, {0, 3}, {1, 0}, {1, 2}}));
  EXPECT_EQ((long)clipper::utils::distanceBasedCorrespondences(D1, D2, 10, inf, false).rows(), 8L);
  Eigen::MatrixXd E2(1, 2), E1(1, 5);
  E2 << 0, 10;
  E1 << 1, -1, 1, 9, 11;
  EXPECT_TRUE(same(clipper::utils::distanceBasedCorrespondences(E1, E2, 1, inf, true), {{0, 0}, {3, 1}}));
  EXPECT_EQ((long)clipper::utils::distanceBasedCorrespondences(E1, E2, 1, std::nan(""), false).rows(), 0L);
  EXPECT_EQ((long)clipper::utils::distanceBasedCorrespondences(E1, Eigen::MatrixXd(1, 0), 1, inf, false).rows(), 0L);
}

// the chain of the reference's benchmark: associations from the clouds, then scoring and the solve
static void Utils_FeedsScoring() {
  Eigen::MatrixXd D1 = random_cloud(3, 200, 7);
  Eigen::MatrixXd D2 = D1;
  for (int j = 0; j < 200; ++j) D2(0, j) += 1e-5 * ((j * 37) % 11 - 5);
  const clipper::Association A = clipper::utils::distanceBasedCorrespondences(D1, D2, 1, 1e-3, true);
  EXPECT_EQ((long)A.rows(), 200L);
  for (long r = 0; r < (long)A.rows(); ++r) EXPECT_EQ(A(r, 0), A(r, 1));
  clipper::invariants::EuclideanDistance::Params ip;
  clipper::CLIPPER clipper(std::make_shared<clipper::invariants::EuclideanDistance>(ip), clipper::Params{});
  clipper.scorePairwiseConsistency(D1, D2, A);
  EXPECT_TRUE(clipper.getInitialAssociations() == A);
}

static void Utils_Errors() {
  const Eigen::MatrixXd D = random_cloud(3, 10, 3);
  bool threw = false;
  try { clipper::utils::distanceBasedCorrespondences(D, D, 0, 1.0, false); } catch (const std::runtime_error&) { threw = true; }
  EXPECT_TRUE(threw);
  threw = false;
  try { clipper::utils::distanceBasedCorrespondences(D, D, 33, 1.0, false); } catch (const std::runtime_error&) { threw = true; }
  EXPECT_TRUE(threw);
  threw = false;
  try { clipper::utils::distanceBasedCorrespondences(D, random_cloud(2, 10, 4), 1, 1.0, false); } catch (const std::runtime_error&) { threw = true; }
  EXPECT_TRUE(threw);
  // a knn far above the cap is rejected as unsupported, not by an allocation sized for it
  const Eigen::MatrixXd big = random_cloud(3, 200000, 5);
  std::string msg;
  try { clipper::utils::distanceBasedCorrespondences(big, big, 1u << 20, 1.0, false); }
  catch (const std::runtime_error& e) { msg = e.what(); }
  EXPECT_TRUE(msg.find("CLP_KNN_MAX_K") != std::string::npos);
}

int main() {
  struct T { const char* name; void (*fn)(); };
  const T tests[] = {{"Utils.RandomAgainstLoop", Utils_RandomAgainstLoop}, {"Utils.TiesAndClamp", Utils_TiesAndClamp},
                     {"Utils.FeedsScoring", Utils_FeedsScoring}, {"Utils.Errors", Utils_Errors}};
  int ran = 0;
  for (const T& t : tests) {
    const int before = g_fail;
    std::printf("[ RUN  ] %s\n", t.name);
    try { t.fn(); } catch (const std::exception& e) { ++g_fail; std::printf("  FAIL exception: %s\n", e.what()); }
    std::printf("[ %s ] %s\n", g_fail == before ? " OK " : "FAIL", t.name);
    ++ran;
  }
  std::printf("%d tests, %d checks, %d failures\n", ran, g_checks, g_fail);
  return g_fail ? 1 : 0;
}
