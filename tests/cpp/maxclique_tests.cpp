// maxclique_tests.cpp -- maxclique::solve and CLIPPER::solveAsMaximumClique of the C++ shell on known graphs.
// Every test needs the GPU.  Same 20-line assertion harness as shell_tests.cpp.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include <clipper/clipper.h>
#include <clipper/utils.h>

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("  FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) EXPECT_TRUE((a) == (b))

using clipper::maxclique::Method;

static clipper::maxclique::Params mc(Method method, int time_limit = 60) {
  clipper::maxclique::Params p;
  p.method = method;
  p.time_limit = time_limit;
  return p;
}

// two disjoint cliques {0..4} and {10..15} plus a path 5-6-7-8-9 and a pendant 16-0; A full (both triangles)
static Eigen::MatrixXd two_cliques() {
  Eigen::MatrixXd A = Eigen::MatrixXd::Zero(17, 17);
  auto edge = [&](int i, int j) { A(i, j) = 1; A(j, i) = 1; };
  for (int i = 0; i < 5; ++i) for (int j = i + 1; j < 5; ++j) edge(i, j);
  for (int i = 10; i < 16; ++i) for (int j = i + 1; j < 16; ++j) edge(i, j);
  for (int i = 5; i < 9; ++i) edge(i, i + 1);
  edge(16, 0);
  return A;
}

static void MaxClique_Solve() {
  const Eigen::MatrixXd A = two_cliques();
  const std::vector<int> want = {10, 11, 12, 13, 14, 15};
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::EXACT)) == want);
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::HEU)) == want);
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::KCORE)) == want);  // the 5-core is the 6-clique
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::EXACT, 0)) == want);
}

static void MaxClique_Edgeless() {
  const Eigen::MatrixXd A = Eigen::MatrixXd::Zero(5, 5);
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::KCORE)) == std::vector<int>({0, 1, 2, 3, 4}));
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::HEU)) == std::vector<int>({0}));
  EXPECT_TRUE(clipper::maxclique::solve(A, mc(Method::EXACT)) == std::vector<int>({0}));
  const Eigen::MatrixXd one = Eigen::MatrixXd::Zero(1, 1);
  EXPECT_TRUE(clipper::maxclique::solve(one, mc(Method::EXACT)) == std::vector<int>({0}));
}

// the reference's toy problem (test/clipper_test.cpp): the inliers 0, 4, 8 are the maximum clique of C
static void CLIPPER_SolveAsMaximumClique() {
  Eigen::MatrixXd model(3, 4);
  const double pts[4][3] = {{0, 0, 0}, {2, 0, 0}, {0, 3, 0}, {2, 2, 0}};
  for (int j = 0; j < 4; ++j) for (int i = 0; i < 3; ++i) model(i, j) = pts[j][i];
  const double th = M_PI / 8, c = std::cos(th), s = std::sin(th), t[3] = {5, 3, 0};
  Eigen::MatrixXd data(3, 3);
  for (int j = 0; j < 3; ++j) {
    const double x = model(0, j) - t[0], y = model(1, j) - t[1], z = model(2, j) - t[2];
    data(0, j) = c * x + s * y;
    data(1, j) = -s * x + c * y;
    data(2, j) = z;
  }
  clipper::invariants::EuclideanDistance::Params iparams;
  clipper::CLIPPER clipper(std::make_shared<clipper::invariants::EuclideanDistance>(iparams), clipper::Params());
  clipper.scorePairwiseConsistency(model, data);
  clipper.solveAsMaximumClique();
  const clipper::Solution& soln = clipper.getSolution();
  EXPECT_TRUE(soln.nodes == std::vector<int>({0, 4, 8}));
  EXPECT_EQ(soln.score, -1);
  EXPECT_EQ(soln.ifinal, 0);
  EXPECT_EQ((long)soln.u.size(), 12L);
  double unorm = 0;
  for (long i = 0; i < (long)soln.u.size(); ++i) unorm += std::abs(soln.u(i));
  EXPECT_EQ(unorm, 0.0);
  const clipper::Association Ain = clipper.getSelectedAssociations();
  EXPECT_EQ((long)Ain.rows(), 3L);
  for (long i = 0; i < (long)Ain.rows(); ++i) EXPECT_EQ(Ain(i, 0), Ain(i, 1));
}

int main() {
  struct T { const char* name; void (*fn)(); };
  const T tests[] = {{"MaxClique.Solve", MaxClique_Solve}, {"MaxClique.Edgeless", MaxClique_Edgeless},
                     {"CLIPPER.SolveAsMaximumClique", CLIPPER_SolveAsMaximumClique}};
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
