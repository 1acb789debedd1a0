// knn_batch_tests.cpp -- utils::distanceBasedCorrespondencesBatch of the C++ shell (clp_batch_correspondences on
// device 0) against utils::distanceBasedCorrespondences pair by pair.  Every test needs the GPU.  Same assertion harness
// as shell_tests.cpp.
#include <cmath>
#include <cstdio>
#include <limits>
#include <random>
#include <stdexcept>
#include <string>
#include <vector>

#include <clipper/clipper.h>
#include <clipper/utils.h>

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("  FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) EXPECT_TRUE((a) == (b))

static Eigen::MatrixXd random_cloud(int d, int n, unsigned seed, bool ties = false) {
  std::mt19937 gen(seed);
  std::normal_distribution<double> g(0.0, 1.0);
  std::uniform_int_distribution<int> u(0, 2);
  Eigen::MatrixXd D(d, n);
  for (int j = 0; j < n; ++j) for (int k = 0; k < d; ++k) D(k, j) = ties ? (double)u(gen) : g(gen);
  return D;
}

// pairs of mixed sizes, empty clouds among them, d = 3 and 33, against the single call pair by pair
static void Utils_BatchAgainstSingle() {
  const int n1s[] = {300, 0, 1, 129, 2000, 7, 50};
  const int n2s[] = {457, 9, 0, 4097, 33, 1, 50};
  for (int d : {3, 33})
    for (bool ties : {false, true}) {
      std::vector<clipper::invariants::Data> D1s, D2s;
      for (int p = 0; p < 7; ++p) {
        D1s.push_back(random_cloud(d, n1s[p], 10 * p + d, ties));
        D2s.push_back(random_cloud(d, n2s[p], 10 * p + d + 1, ties));
      }
      for (size_t knn : {1, 4, 32})
        for (double radius : {std::numeric_limits<double>::infinity(), d == 3 ? 0.6 : 7.0})
          for (bool one : {false, true}) {
            const std::vector<clipper::Association> As =
                clipper::utils::distanceBasedCorrespondencesBatch(D1s, D2s, knn, radius, one);
            EXPECT_EQ(As.size(), (size_t)7);
            for (size_t p = 0; p < As.size(); ++p)
              EXPECT_TRUE(As[p] == clipper::utils::distanceBasedCorrespondences(D1s[p], D2s[p], knn, radius, one));
            EXPECT_EQ((long)As[1].rows(), 0L);
            EXPECT_EQ((long)As[2].rows(), 0L);
          }
    }
}

// one model against many noisy scans, the benchmark's call: every pair keeps its inliers; the result feeds scoring
static void Utils_BatchFeedsScoring() {
  const Eigen::MatrixXd model = random_cloud(3, 200, 7);
  std::vector<clipper::invariants::Data> D1s, D2s;
  for (int s = 0; s < 5; ++s) {
    Eigen::MatrixXd scan = model;
    for (int j = 0; j < 200; ++j) scan(0, j) += 1e-5 * (((j + s) * 37) % 11 - 5);
    D1s.push_back(model);
    D2s.push_back(scan);
  }
  const std::vector<clipper::Association> As = clipper::utils::distanceBasedCorrespondencesBatch(D1s, D2s, 1, 1e-3, true);
  for (const clipper::Association& A : As) {
    EXPECT_EQ((long)A.rows(), 200L);
    for (long r = 0; r < (long)A.rows(); ++r) EXPECT_EQ(A(r, 0), A(r, 1));
  }
  clipper::invariants::EuclideanDistance::Params ip;
  clipper::CLIPPER clipper(std::make_shared<clipper::invariants::EuclideanDistance>(ip), clipper::Params{});
  clipper.scorePairwiseConsistency(D1s[2], D2s[2], As[2]);
  EXPECT_TRUE(clipper.getInitialAssociations() == As[2]);
  EXPECT_TRUE(clipper::utils::distanceBasedCorrespondencesBatch({}, {}, 1, 1.0, false).empty());
}

static void Utils_BatchErrors() {
  const Eigen::MatrixXd D = random_cloud(3, 10, 3);
  auto throws = [](auto&& f, const char* needle) {
    std::string msg;
    try { f(); } catch (const std::runtime_error& e) { msg = e.what(); }
    return !msg.empty() && msg.find(needle) != std::string::npos;
  };
  using V = std::vector<clipper::invariants::Data>;
  EXPECT_TRUE(throws([&] { clipper::utils::distanceBasedCorrespondencesBatch(V{D, D}, V{D}, 1, 1.0, false); }, "as many"));
  EXPECT_TRUE(throws([&] { clipper::utils::distanceBasedCorrespondencesBatch(V{D}, V{random_cloud(2, 10, 4)}, 1, 1.0, false); },
                     "rows"));
  EXPECT_TRUE(throws([&] { clipper::utils::distanceBasedCorrespondencesBatch(V{D}, V{D}, 0, 1.0, false); }, "knn"));
  EXPECT_TRUE(throws([&] { clipper::utils::distanceBasedCorrespondencesBatch(V{D, D}, V{D, D}, 33, 1.0, false); },
                     "CLP_KNN_MAX_K"));
  // the batch of the call is gone: a call after the errors works
  EXPECT_EQ(clipper::utils::distanceBasedCorrespondencesBatch(V{D}, V{D}, 1, 1.0, false)[0].rows(), 10L);
}

int main() {
  struct T { const char* name; void (*fn)(); };
  const T tests[] = {{"Utils.BatchAgainstSingle", Utils_BatchAgainstSingle}, {"Utils.BatchFeedsScoring", Utils_BatchFeedsScoring},
                     {"Utils.BatchErrors", Utils_BatchErrors}};
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
