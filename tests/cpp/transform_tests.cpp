// transform_tests.cpp -- utils::estimateRigidTransform(Batch) of the C++ shell (clp_estimate_transform and
// clp_batch_estimate_transform on device 0): the reference's toy problem as a known answer, a batch against single
// calls, and an empty A.  Every test needs the GPU.  Same assertion harness as shell_tests.cpp.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <random>
#include <stdexcept>
#include <vector>

#include <clipper/clipper.h>
#include <clipper/utils.h>
#include <clipper_b200.h>

static int g_fail = 0, g_checks = 0;
#define EXPECT_TRUE(c) do { ++g_checks; if (!(c)) { ++g_fail; std::printf("  FAIL %s:%d  %s\n", __FILE__, __LINE__, #c); } } while (0)
#define EXPECT_EQ(a, b) EXPECT_TRUE((a) == (b))

// the reference's toy problem (test/clipper_test.cpp:34-49): data = Rz(pi/8)' (model - (5, 3, 0)), first 3 points
static void toy(Eigen::MatrixXd& model, Eigen::MatrixXd& data) {
  const double pts[4][3] = {{0, 0, 0}, {2, 0, 0}, {0, 3, 0}, {2, 2, 0}};
  const double th = M_PI / 8, c = std::cos(th), s = std::sin(th);
  model.resize(3, 4);
  data.resize(3, 3);
  for (int j = 0; j < 4; ++j)
    for (int k = 0; k < 3; ++k) model(k, j) = pts[j][k];
  for (int j = 0; j < 3; ++j) {
    const double x = pts[j][0] - 5, y = pts[j][1] - 3, z = pts[j][2];
    data(0, j) = c * x + s * y; data(1, j) = -s * x + c * y; data(2, j) = z;
  }
}

static clipper::Association diag(int n) {
  clipper::Association A(n, 2);
  for (int i = 0; i < n; ++i) { A(i, 0) = i; A(i, 1) = i; }
  return A;
}

// R = Rz(pi/8)' and t = -Rz(pi/8)' (5, 3, 0): the transform from the model's frame into the data's
static void Transform_ToyKnownAnswer() {
  Eigen::MatrixXd model, data;
  toy(model, data);
  const auto r = clipper::utils::estimateRigidTransform(model, data, diag(3));
  const double th = M_PI / 8, c = std::cos(th), s = std::sin(th);
  const double want[4][4] = {{c, s, 0, -(c * 5 + s * 3)}, {-s, c, 0, -(-s * 5 + c * 3)}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  EXPECT_EQ(r.status, CLP_TF_OK);
  EXPECT_EQ(r.k, 3);
  EXPECT_EQ(r.T.rows(), 4);
  double err = 0;
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) err = std::fmax(err, std::fabs(r.T(i, j) - want[i][j]));
  EXPECT_TRUE(err <= 1e-14);
  EXPECT_TRUE(r.rmse <= 1e-14);
  EXPECT_TRUE(r.gap > 0 && r.sv(0) >= r.sv(1) && r.sv(1) >= r.sv(2));
}

// a batch of random problems (d = 2 and 3, sizes 0 to 300) is bit for bit the single calls
static void Transform_BatchEqualsSingle() {
  std::mt19937 gen(7);
  std::normal_distribution<double> g(0.0, 1.0);
  for (int d : {2, 3}) {
    std::vector<Eigen::MatrixXd> D1s, D2s;
    std::vector<clipper::Association> As;
    for (int p = 0; p < 9; ++p) {
      const int n = p == 0 ? 0 : 1 + 37 * p;
      Eigen::MatrixXd a(d, n), b(d, n);
      for (int j = 0; j < n; ++j)
        for (int k = 0; k < d; ++k) { a(k, j) = g(gen) + 10 * p; b(k, j) = g(gen); }
      D1s.push_back(a); D2s.push_back(b); As.push_back(diag(n));
    }
    const auto batch = clipper::utils::estimateRigidTransformBatch(D1s, D2s, As);
    EXPECT_EQ(batch.size(), D1s.size());
    for (size_t p = 0; p < D1s.size(); ++p) {
      const auto one = clipper::utils::estimateRigidTransform(D1s[p], D2s[p], As[p]);
      EXPECT_EQ(batch[p].status, one.status);
      EXPECT_EQ(batch[p].k, one.k);
      EXPECT_TRUE(std::memcmp(batch[p].T.data(), one.T.data(), sizeof(double) * (d + 1) * (d + 1)) == 0);
      EXPECT_TRUE(std::memcmp(&batch[p].rmse, &one.rmse, sizeof(double)) == 0);
      EXPECT_TRUE(std::memcmp(batch[p].sv.data(), one.sv.data(), 3 * sizeof(double)) == 0);
    }
  }
  EXPECT_TRUE(clipper::utils::estimateRigidTransformBatch({}, {}, {}).empty());
}

// an empty A is no pairs (CLP_TF_EMPTY, T = I), not the all-to-all hypothesis
static void Transform_EmptyA() {
  Eigen::MatrixXd model, data;
  toy(model, data);
  const auto r = clipper::utils::estimateRigidTransform(model, data, clipper::Association());
  EXPECT_EQ(r.status, CLP_TF_EMPTY);
  EXPECT_EQ(r.k, 0);
  EXPECT_EQ(r.rmse, 0.0);
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) EXPECT_EQ(r.T(i, j), i == j ? 1.0 : 0.0);
  const auto b = clipper::utils::estimateRigidTransformBatch({model}, {data}, {clipper::Association()});
  EXPECT_EQ(b[0].status, CLP_TF_EMPTY);
  bool threw = false;
  try { clipper::utils::estimateRigidTransform(Eigen::MatrixXd(4, 3), Eigen::MatrixXd(4, 3), diag(3)); }
  catch (const std::runtime_error&) { threw = true; }
  EXPECT_TRUE(threw);  // d = 4: CLP_ERR_UNSUPPORTED
}

int main() {
  struct T { const char* name; void (*fn)(); };
  const T tests[] = {{"Transform.ToyKnownAnswer", Transform_ToyKnownAnswer},
                     {"Transform.BatchEqualsSingle", Transform_BatchEqualsSingle}, {"Transform.EmptyA", Transform_EmptyA}};
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
