// sdp_tests.cpp -- sdp::solve and CLIPPER::solveAsMSRCSDR of the C++ shell: the GPU relaxation with params, the
// build-without-SCS behaviour without them.  Every test needs the GPU.  Same assertion harness as shell_tests.cpp.
#include <algorithm>
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

// the 20 x 20 weighted matrix of the reference's test/sdp_test.cpp (values only)
static Eigen::MatrixXd m20() {
  Eigen::MatrixXd M = Eigen::MatrixXd::Identity(20, 20);
  const struct { int i, j; double v; } e[] = {
    {0,18,0.2964},{1,13,0.0138},{2,11,0.0016},{2,18,0.0747},{3,5,0.0555},{3,6,0.2547},{3,13,0.0102},{3,15,0.7715},
    {4,5,0.0063},{4,7,0.3846},{4,9,0.0003},{4,10,0.0014},{4,15,0.0063},{5,12,0.9927},{5,15,0.9722},{6,8,0.0023},
    {6,11,0.8775},{7,8,0.0001},{8,9,0.7914},{8,13,0.0617},{8,16,0.9938},{8,19,0.0007},{9,12,0.0001},{9,13,0.0091},
    {9,15,0.2503},{9,16,0.0222},{9,17,0.0549},{10,19,0.0008},{11,18,0.7007},{12,14,0.9978},{13,17,0.0003},
    {14,15,0.0012},{14,19,0.0074},{15,16,0.0026},{15,17,0.0217},{17,18,0.0007}};
  for (const auto& x : e) { M(x.i, x.j) = x.v; M(x.j, x.i) = x.v; }
  return M;
}

static Eigen::MatrixXd pattern(const Eigen::MatrixXd& M) {
  Eigen::MatrixXd C(M.rows(), M.cols());
  for (long j = 0; j < (long)M.cols(); ++j) for (long i = 0; i < (long)M.rows(); ++i) C(i, j) = M(i, j) > 0 ? 1.0 : 0.0;
  return C;
}

// sdp::solve with params on the reference's matrix: nodes {8, 9, 16}, and X, lambdas, evec1, thr consistent
static void SDP_SolveReferenceMatrix() {
  const Eigen::MatrixXd M = m20(), C = pattern(M);
  const clipper::sdp::Solution s = clipper::sdp::solve(M, C, clipper::sdp::Params{});
  EXPECT_TRUE(s.nodes == std::vector<int>({8, 9, 16}));
  EXPECT_EQ((long)s.X.rows(), 20L);
  EXPECT_EQ((long)s.lambdas.size(), 20L);
  EXPECT_EQ((long)s.evec1.size(), 20L);
  double tr = 0, lsum = 0, vmax = 0, value = 0;
  for (int i = 0; i < 20; ++i) { tr += s.X(i, i); lsum += s.lambdas(i); vmax = std::max(vmax, std::abs(s.evec1(i))); }
  for (int j = 0; j < 20; ++j) for (int i = 0; i < 20; ++i) value += M(i, j) * s.X(i, j);
  EXPECT_TRUE(std::abs(tr - 1) < 1e-9);
  EXPECT_TRUE(std::abs(lsum - 1) < 1e-9);
  for (int i = 1; i < 20; ++i) EXPECT_TRUE(s.lambdas(i - 1) <= s.lambdas(i));
  EXPECT_TRUE(std::abs(s.thr - vmax / 2) < 1e-15);
  for (int i = 0; i < 20; ++i)
    EXPECT_EQ(std::abs(s.evec1(i)) > s.thr, std::find(s.nodes.begin(), s.nodes.end(), i) != s.nodes.end());
  EXPECT_TRUE(std::abs(s.pobj + value) < 1e-4 * std::abs(value));  // SCS's sign, stored as float
  EXPECT_TRUE(s.dobj <= s.pobj + 1e-3f);
  EXPECT_TRUE(s.iters >= 1 && s.iters <= 2000);
  EXPECT_TRUE(s.t > 0 && s.t_scs > 0 && s.t_scs_solve > 0 && s.t_scs_cone > 0);
  EXPECT_EQ(s.t_scs_setup, 0.0);
  EXPECT_EQ(s.t_scs_linsys, 0.0);
  EXPECT_EQ(s.t_scs_accel, 0.0);
}

// without params: a build without SCS, nothing selected
static void SDP_NoParamsIsTheStub() {
  const Eigen::MatrixXd M = m20(), C = pattern(M);
  EXPECT_TRUE(clipper::sdp::solve(M, C).nodes.empty());
  clipper::invariants::EuclideanDistance::Params iparams;
  clipper::CLIPPER clipper(std::make_shared<clipper::invariants::EuclideanDistance>(iparams), clipper::Params());
  clipper.setMatrixData(M, C);
  clipper.solveAsMSRCSDR();
  EXPECT_TRUE(clipper.getSolution().nodes.empty());
  EXPECT_EQ(clipper.getSolution().score, -1);
}

// the reference's toy problem (test/clipper_test.cpp): solveAsMSRCSDR with params selects the three inliers
static void CLIPPER_SolveAsMSRCSDR() {
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
  clipper::sdp::Params sp;
  sp.verbose = true;
  clipper.solveAsMSRCSDR(sp);
  const clipper::Solution& soln = clipper.getSolution();
  EXPECT_TRUE(soln.nodes == std::vector<int>({0, 4, 8}));
  EXPECT_EQ(soln.score, -1);
  EXPECT_EQ(soln.ifinal, 0);
  EXPECT_EQ((long)soln.u.size(), 12L);
  const clipper::Association Ain = clipper.getSelectedAssociations();
  EXPECT_EQ((long)Ain.rows(), 3L);
  for (long i = 0; i < (long)Ain.rows(); ++i) EXPECT_EQ(Ain(i, 0), Ain(i, 1));
}

int main() {
  struct T { const char* name; void (*fn)(); };
  const T tests[] = {{"SDP.SolveReferenceMatrix", SDP_SolveReferenceMatrix}, {"SDP.NoParamsIsTheStub", SDP_NoParamsIsTheStub},
                     {"CLIPPER.SolveAsMSRCSDR", CLIPPER_SolveAsMSRCSDR}};
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
