// custom_invariant_tests.cpp -- clipper::invariants::CudaInvariant through the C++ shell (libclipper.so):
// the reference's m = 12 toy problem (test/affinity_test.cpp:14-108, test/clipper_test.cpp:15-68) scored by a CUDA
// restatement of EuclideanDistance compiled at run time, and the functor's host call.  Needs a GPU.
#include <cmath>
#include <cstdio>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include <clipper/clipper.h>
#include <clipper/utils.h>

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("  FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) EXPECT_TRUE((a) == (b))
#define ASSERT_EQ(a, b) do { ++g_checks; if (!((a) == (b))) { ++g_fail; std::printf("  FAIL %s:%d  %s == %s\n", __FILE__, __LINE__, #a, #b); return; } } while (0)

// EuclideanDistance (reference euclidean_distance.cpp:13-31) with the scoring kernel's operation order;
// prm = (sigma, epsilon, mindist)
static const char* kEuclid = R"(
__device__ double clp_invariant(const double* ai, const double* aj, const double* bi, const double* bj, int d,
                                const double* prm) {
  double s1 = 0.0, s2 = 0.0;
  for (int q = 0; q < d; ++q) { const double t = __dsub_rn(ai[q], aj[q]); s1 = __dadd_rn(s1, __dmul_rn(t, t)); }
  for (int q = 0; q < d; ++q) { const double t = __dsub_rn(bi[q], bj[q]); s2 = __dadd_rn(s2, __dmul_rn(t, t)); }
  const double l1 = __dsqrt_rn(s1), l2 = __dsqrt_rn(s2);
  if (prm[2] > 0 && (l1 < prm[2] || l2 < prm[2])) return 0.0;
  const double c = fabs(__dsub_rn(l1, l2));
  if (!(c < prm[1])) return 0.0;
  return exp(__ddiv_rn(__dmul_rn(__dmul_rn(-0.5, c), c), __dmul_rn(prm[0], prm[0])));
}
)";

// model: 4 points; data = T_MD^-1 * model with T_MD = (Rz(pi/8), t = (5,3,0)), first 3 points
static void toy(Eigen::MatrixXd& model, Eigen::MatrixXd& data) {
  model = Eigen::MatrixXd(3, 4);
  const double pts[4][3] = {{0, 0, 0}, {2, 0, 0}, {0, 3, 0}, {2, 2, 0}};
  for (int j = 0; j < 4; ++j) for (int i = 0; i < 3; ++i) model(i, j) = pts[j][i];
  const double th = M_PI / 8, c = std::cos(th), s = std::sin(th), t[3] = {5, 3, 0};
  data = Eigen::MatrixXd(3, 3);
  for (int j = 0; j < 3; ++j) {
    const double x = model(0, j) - t[0], y = model(1, j) - t[1], z = model(2, j) - t[2];
    data(0, j) = c * x + s * y;   // R^T (p - t)
    data(1, j) = -s * x + c * y;
    data(2, j) = z;
  }
}

static std::shared_ptr<clipper::invariants::CudaInvariant> make_invariant() {
  const clipper::invariants::EuclideanDistance::Params p;  // the reference's defaults
  return std::make_shared<clipper::invariants::CudaInvariant>(kEuclid, std::vector<double>{p.sigma, p.epsilon, p.mindist});
}

static void CudaInvariant_Toy() {
  clipper::Params params;
  clipper::CLIPPER clipper(make_invariant(), params);
  Eigen::MatrixXd model, data;
  toy(model, data);
  clipper.scorePairwiseConsistency(model, data);
  clipper::Affinity M = clipper.getAffinityMatrix();
  clipper::Constraint C = clipper.getConstraintMatrix();
  ASSERT_EQ(M.rows(), 12);
  Eigen::MatrixXd Mtrue(M.rows(), M.cols());
  Mtrue << 1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0,
           0, 1, 0, 1, 0, 0, 0, 0, 0, 0, 0, 0,
           0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0,
           0, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0,
           1, 0, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0,
           0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0,
           0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 0, 0,
           0, 0, 0, 0, 0, 1, 0, 1, 0, 0, 0, 0,
           1, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0,
           0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0,
           0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0,
           0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1;
  EXPECT_EQ(M, Mtrue);
  EXPECT_EQ(C, Mtrue);
  clipper.solve(Eigen::VectorXd::Ones(12));
  clipper::Association Ainliers = clipper.getSelectedAssociations();
  ASSERT_EQ(Ainliers.rows(), 3);
  int seen = 0;  // the inliers {(0,0), (1,1), (2,2)}, in the solver's order
  for (int i = 0; i < 3; ++i) {
    EXPECT_EQ(Ainliers(i, 0), Ainliers(i, 1));
    if (Ainliers(i, 0) >= 0 && Ainliers(i, 0) < 3) seen |= 1 << Ainliers(i, 0);
  }
  EXPECT_EQ(seen, 7);
}

static void CudaInvariant_HostCallThrows() {
  auto inv = make_invariant();
  EXPECT_EQ(inv->source(), std::string(kEuclid));
  EXPECT_EQ(inv->params().size(), (size_t)3);
  const clipper::invariants::Datum a = Eigen::VectorXd::Zero(3);
  bool threw = false;
  try { (*inv)(a, a, a, a); } catch (const std::logic_error&) { threw = true; }
  EXPECT_TRUE(threw);
}

int main() {
  struct T { const char* name; void (*fn)(); };
  const T tests[] = {{"CudaInvariant.Toy", CudaInvariant_Toy}, {"CudaInvariant.HostCallThrows", CudaInvariant_HostCallThrows}};
  int ran = 0;
  for (const T& t : tests) {
    const int before = g_fail;
    std::printf("[ RUN  ] %s\n", t.name);
    try { t.fn(); } catch (const std::exception& e) { ++g_fail; std::printf("  EXCEPTION %s\n", e.what()); }
    std::printf("[ %s ] %s\n", g_fail == before ? " OK " : "FAIL", t.name);
    ++ran;
  }
  std::printf("%d tests, %d checks, %d failures\n", ran, g_checks, g_fail);
  return g_fail ? 1 : 0;
}
