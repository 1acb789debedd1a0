// py_clipperpy.cpp -- the reference's pybind11 module `clipperpy`, built over the H100 C++ shell.
//
// Same module layout, class / method / attribute names and keyword arguments as
// reference bindings/python/py_clipper.cpp:116-232 and trampolines.h:20-29.  With Eigen installed
// the reference's own py_clipper.cpp compiles unchanged against include/clipper/*.h; this file is
// the variant that needs no Eigen (numpy <-> column-major buffers are converted by hand, because
// pybind11/eigen.h requires the real Eigen).  D1, D2, A, u0, M, C are "noconvert" like upstream:
// float64 / int32 numpy arrays are required.
#include <cstring>
#include <optional>
#include <sstream>

#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "clipper/clipper.h"
#include "clipper/utils.h"

#ifndef CLIPPER_VERSION
#define CLIPPER_VERSION "0.2.4"
#endif

namespace py = pybind11;
using namespace pybind11::literals;

namespace {

using arr_d = py::array_t<double>;
using arr_i = py::array_t<int>;

void require_dtype(const py::array& a, const char* name, bool want_double) {
  const bool ok = want_double ? py::isinstance<arr_d>(a) : py::isinstance<arr_i>(a);
  if (!ok) throw py::type_error(std::string(name) + ": incompatible dtype (noconvert: float64 / int32 required)");
}

Eigen::MatrixXd to_matrix(const py::array& a, const char* name) {
  require_dtype(a, name, true);
  auto f = py::array_t<double, py::array::f_style | py::array::forcecast>::ensure(a);
  if (!f || f.ndim() != 2) throw py::type_error(std::string(name) + ": expected a 2-D array");
  Eigen::MatrixXd M(f.shape(0), f.shape(1));
  std::memcpy(M.data(), f.data(), sizeof(double) * (size_t)M.size());
  return M;
}

Eigen::VectorXd to_vector(const py::array& a, const char* name) {
  if (a.size() == 0) return Eigen::VectorXd();
  require_dtype(a, name, true);
  auto f = py::array_t<double, py::array::c_style | py::array::forcecast>::ensure(a);
  Eigen::VectorXd v(f.size());
  std::memcpy(v.data(), f.data(), sizeof(double) * (size_t)v.size());
  return v;
}

clipper::Association to_assoc(const py::array& a, const char* name) {
  if (a.size() == 0) return clipper::Association();
  require_dtype(a, name, false);
  auto f = py::array_t<int, py::array::f_style | py::array::forcecast>::ensure(a);
  if (!f || f.ndim() != 2 || f.shape(1) != 2) throw py::type_error(std::string(name) + ": expected an (m, 2) int32 array");
  clipper::Association A(f.shape(0), 2);
  std::memcpy(A.data(), f.data(), sizeof(int) * (size_t)A.size());
  return A;
}

arr_d from_matrix(const Eigen::MatrixXd& M) {
  arr_d out({(py::ssize_t)M.rows(), (py::ssize_t)M.cols()},
            {(py::ssize_t)sizeof(double), (py::ssize_t)(sizeof(double) * M.rows())});
  std::memcpy(out.mutable_data(), M.data(), sizeof(double) * (size_t)M.size());
  return out;
}

arr_d from_vector(const Eigen::VectorXd& v) {
  arr_d out((py::ssize_t)v.size());
  if (v.size()) std::memcpy(out.mutable_data(), v.data(), sizeof(double) * (size_t)v.size());
  return out;
}

arr_i from_assoc(const clipper::Association& A) {
  arr_i out({(py::ssize_t)A.rows(), (py::ssize_t)2}, {(py::ssize_t)sizeof(int), (py::ssize_t)(sizeof(int) * A.rows())});
  if (A.size()) std::memcpy(out.mutable_data(), A.data(), sizeof(int) * (size_t)A.size());
  return out;
}

// trampoline so that Python can subclass PairwiseInvariant (reference trampolines.h:20-29)
class PyPairwiseInvariant : public clipper::invariants::PairwiseInvariant {
 public:
  using clipper::invariants::PairwiseInvariant::PairwiseInvariant;
  double operator()(const clipper::invariants::Datum& ai, const clipper::invariants::Datum& aj,
                    const clipper::invariants::Datum& bi, const clipper::invariants::Datum& bj) override {
    py::gil_scoped_acquire acquire;
    py::function f = py::get_override(static_cast<const clipper::invariants::PairwiseInvariant*>(this), "__call__");
    if (!f) throw std::runtime_error("PairwiseInvariant.__call__ is pure virtual");
    return f(from_vector(ai), from_vector(aj), from_vector(bi), from_vector(bj)).cast<double>();
  }
};

double call_builtin(clipper::invariants::PairwiseInvariant& inv, const py::array& ai, const py::array& aj,
                    const py::array& bi, const py::array& bj) {
  return inv(to_vector(ai, "ai"), to_vector(aj, "aj"), to_vector(bi, "bi"), to_vector(bj, "bj"));
}

}  // namespace

void pybind_invariants(py::module& m)
{
  m.doc() = "Invariants are quantities that do not change under the transformation between two sets "
            "of objects. They are used to build a consistency graph. Some built-in invariants are provided.";
  using namespace clipper::invariants;

  py::class_<Invariant, std::shared_ptr<Invariant>>(m, "Invariant");
  py::class_<PairwiseInvariant, Invariant, PyPairwiseInvariant, std::shared_ptr<PairwiseInvariant>>(m, "PairwiseInvariant")
    .def(py::init<>())
    .def("__call__", &call_builtin);

  py::class_<EuclideanDistance::Params>(m, "EuclideanDistanceParams")
    .def(py::init<>())
    .def("__repr__", [](const EuclideanDistance::Params& p) {
      std::ostringstream r;
      r << "<EuclideanDistanceParams : sigma=" << p.sigma << " epsilon=" << p.epsilon << " mindist=" << p.mindist << ">";
      return r.str();
    })
    .def_readwrite("sigma", &EuclideanDistance::Params::sigma)
    .def_readwrite("epsilon", &EuclideanDistance::Params::epsilon)
    .def_readwrite("mindist", &EuclideanDistance::Params::mindist);
  py::class_<EuclideanDistance, PairwiseInvariant, std::shared_ptr<EuclideanDistance>>(m, "EuclideanDistance")
    .def(py::init<const EuclideanDistance::Params&>());

  py::class_<PointNormalDistance::Params>(m, "PointNormalDistanceParams")
    .def(py::init<>())
    .def("__repr__", [](const PointNormalDistance::Params& p) {
      std::ostringstream r;
      r << "<PointNormalDistanceParams : sigp=" << p.sigp << " epsp=" << p.epsp << " sign=" << p.sign << " epsn=" << p.epsn << ">";
      return r.str();
    })
    .def_readwrite("sigp", &PointNormalDistance::Params::sigp)
    .def_readwrite("epsp", &PointNormalDistance::Params::epsp)
    .def_readwrite("sign", &PointNormalDistance::Params::sign)
    .def_readwrite("epsn", &PointNormalDistance::Params::epsn);
  py::class_<PointNormalDistance, PairwiseInvariant, std::shared_ptr<PointNormalDistance>>(m, "PointNormalDistance")
    .def(py::init<const PointNormalDistance::Params&>());

  // additive: a custom invariant written in CUDA C++, scored on the GPU (not a Python subclass: parallelize stays on)
  py::class_<CudaInvariant, PairwiseInvariant, std::shared_ptr<CudaInvariant>>(m, "CudaInvariant")
    .def(py::init<std::string, std::vector<double>>(), "source"_a, "params"_a = std::vector<double>{})
    .def("source", &CudaInvariant::source)
    .def("params", &CudaInvariant::params);
}

void pybind_utils(py::module& m)
{
  m.doc() = "Various convenience utilities for working with CLIPPER";
  m.def("create_all_to_all", [](size_t n1, size_t n2) { return from_assoc(clipper::utils::createAllToAll(n1, n2)); },
        "n1"_a, "n2"_a,
        "Create an all-to-all hypothesis for association. Useful for the case of no prior information or putative associations.");
  m.def("k2ij", clipper::utils::k2ij, "k"_a, "n"_a,
        "Maps a flat index k to coordinate of a square nxn symmetric matrix");
}

// additive: putative associations by exact kNN on the GPU (registered on utils only, not on the dsd alias)
void pybind_correspondences(py::module& m)
{
  m.def("distance_based_correspondences",
        [](const py::array& D1, const py::array& D2, size_t knn, double radius, bool enforce_1to1) {
          return from_assoc(clipper::utils::distanceBasedCorrespondences(to_matrix(D1, "D1"), to_matrix(D2, "D2"), knn,
                                                                         radius, enforce_1to1));
        },
        "D1"_a, "D2"_a, "knn"_a, "radius"_a, "enforce_1to1"_a,
        "Associations (m, 2) int32: every column of D1 (d x n1) to its knn nearest columns of D2 within radius, on the GPU.");
}

void pybind_dsd(py::module& m)
{
  // the reference registers pybind_utils on this submodule by mistake (py_clipper.cpp:127-128, SURVEY D8b);
  // the intended `solve` is exported here next to those names
  m.def("solve", [](const py::array& A, const std::vector<int>& S) { return clipper::dsd::solve(to_matrix(A, "A"), S); },
        "A"_a, "S"_a = std::vector<int>{}, "Find densest edge-weighted subgraph of weighted adj mat A.");
}

PYBIND11_MODULE(clipperpy, m)
{
  m.doc() = "A graph-theoretic framework for robust data association (H100 build)";
  m.attr("__version__") = CLIPPER_VERSION;

  py::module m_invariants = m.def_submodule("invariants");
  pybind_invariants(m_invariants);
  py::module m_utils = m.def_submodule("utils");
  pybind_utils(m_utils);
  pybind_correspondences(m_utils);
  py::module m_dsd = m.def_submodule("dsd");
  pybind_utils(m_dsd);
  pybind_dsd(m_dsd);

  py::enum_<clipper::maxclique::Method>(m, "MCMethod")
    .value("EXACT", clipper::maxclique::Method::EXACT)
    .value("HEU", clipper::maxclique::Method::HEU)
    .value("KCORE", clipper::maxclique::Method::KCORE);
  py::class_<clipper::maxclique::Params>(m, "MCParams")
    .def(py::init<>())
    .def("__repr__", [](const clipper::maxclique::Params&) { return std::string("<CLIPPER Maximum Clique Parameters>"); })
    .def_readwrite("method", &clipper::maxclique::Params::method)
    .def_readwrite("threads", &clipper::maxclique::Params::threads)
    .def_readwrite("time_limit", &clipper::maxclique::Params::time_limit)
    .def_readwrite("verbose", &clipper::maxclique::Params::verbose);

  py::class_<clipper::sdp::Params>(m, "SDPParams")
    .def(py::init<>())
    .def("__repr__", [](const clipper::sdp::Params&) { return std::string("<CLIPPER SDP Parameters>"); })
    .def_readwrite("verbose", &clipper::sdp::Params::verbose)
    .def_readwrite("max_iters", &clipper::sdp::Params::max_iters)
    .def_readwrite("acceleration_interval", &clipper::sdp::Params::acceleration_interval)
    .def_readwrite("acceleration_lookback", &clipper::sdp::Params::acceleration_lookback)
    .def_readwrite("eps_abs", &clipper::sdp::Params::eps_abs)
    .def_readwrite("eps_rel", &clipper::sdp::Params::eps_rel)
    .def_readwrite("eps_infeas", &clipper::sdp::Params::eps_infeas)
    .def_readwrite("time_limit_secs", &clipper::sdp::Params::time_limit_secs);

  py::enum_<clipper::Params::Rounding>(m, "Rounding")
    .value("NONZERO", clipper::Params::Rounding::NONZERO)
    .value("DSD", clipper::Params::Rounding::DSD)
    .value("DSD_HEU", clipper::Params::Rounding::DSD_HEU)
    .export_values();

  py::class_<clipper::Params>(m, "Params")
    .def(py::init<>())
    .def("__repr__", [](const clipper::Params&) { return std::string("<CLIPPER Parameters>"); })
    .def_readwrite("tol_u", &clipper::Params::tol_u)
    .def_readwrite("tol_F", &clipper::Params::tol_F)
    .def_readwrite("tol_Fop", &clipper::Params::tol_Fop)
    .def_readwrite("maxiniters", &clipper::Params::maxiniters)
    .def_readwrite("maxoliters", &clipper::Params::maxoliters)
    .def_readwrite("beta", &clipper::Params::beta)
    .def_readwrite("maxlsiters", &clipper::Params::maxlsiters)
    .def_readwrite("eps", &clipper::Params::eps)
    .def_readwrite("affinityeps", &clipper::Params::affinityeps)
    .def_readwrite("rescale_u0", &clipper::Params::rescale_u0)
    .def_readwrite("rounding", &clipper::Params::rounding);

  py::class_<clipper::Solution>(m, "Solution")
    .def(py::init<>())
    .def("__repr__", [](const clipper::Solution&) { return std::string("<CLIPPER Solution>"); })
    .def_readwrite("t", &clipper::Solution::t)
    .def_readwrite("ifinal", &clipper::Solution::ifinal)
    .def_readwrite("nodes", &clipper::Solution::nodes)
    .def_property("u0", [](const clipper::Solution& s) { return from_vector(s.u0); },
                  [](clipper::Solution& s, const py::array& a) { s.u0 = to_vector(a, "u0"); })
    .def_property("u", [](const clipper::Solution& s) { return from_vector(s.u); },
                  [](clipper::Solution& s, const py::array& a) { s.u = to_vector(a, "u"); })
    .def_readwrite("score", &clipper::Solution::score);

  py::class_<clipper::CLIPPER>(m, "CLIPPER")
    .def(py::init([](const clipper::invariants::PairwiseInvariantPtr& invariant, const clipper::Params& params) {
      clipper::CLIPPER* c = new clipper::CLIPPER(invariant, params);
      // Python-extended invariants cannot be evaluated in parallel (GIL), py_clipper.cpp:203-208
      const bool parallelize = (std::dynamic_pointer_cast<PyPairwiseInvariant>(invariant)) ? false : true;
      c->setParallelize(parallelize);
      return c;
    }), py::keep_alive<1, 2>())  // a Python-subclassed invariant must outlive the temporary it was passed as
    .def("__repr__", [](const clipper::CLIPPER&) { return std::string("<CLIPPER>"); })
    .def("score_pairwise_consistency",
         [](clipper::CLIPPER& c, const py::array& D1, const py::array& D2, const py::array& A) {
           c.scorePairwiseConsistency(to_matrix(D1, "D1"), to_matrix(D2, "D2"), to_assoc(A, "A"));
         }, "D1"_a.noconvert(), "D2"_a.noconvert(), "A"_a.noconvert())
    .def("solve", [](clipper::CLIPPER& c, const py::array& u0) { c.solve(to_vector(u0, "u0")); },
         "u0"_a.noconvert() = arr_d(0))
    .def("solve_as_maximum_clique", &clipper::CLIPPER::solveAsMaximumClique, "params"_a = clipper::maxclique::Params{})
    // without params: a build without SCS (nothing selected); with params: the GPU relaxation
    .def("solve_as_msrc_sdr",
         [](clipper::CLIPPER& c, std::optional<clipper::sdp::Params> params) {
           if (params) c.solveAsMSRCSDR(*params);
           else c.solveAsMSRCSDR();
         },
         "params"_a = py::none())
    .def("get_initial_associations", [](clipper::CLIPPER& c) { return from_assoc(c.getInitialAssociations()); })
    .def("get_selected_associations", [](clipper::CLIPPER& c) { return from_assoc(c.getSelectedAssociations()); })
    .def("get_solution", &clipper::CLIPPER::getSolution)
    .def("get_affinity_matrix", [](clipper::CLIPPER& c) { return from_matrix(c.getAffinityMatrix()); })
    .def("get_constraint_matrix", [](clipper::CLIPPER& c) { return from_matrix(c.getConstraintMatrix()); })
    .def("set_matrix_data", [](clipper::CLIPPER& c, const py::array& M, const py::array& C) {
           c.setMatrixData(to_matrix(M, "M"), to_matrix(C, "C"));
         }, "M"_a.noconvert(), "C"_a.noconvert())
    .def("set_parallelize", &clipper::CLIPPER::setParallelize)
    // additive
    .def("set_device", &clipper::CLIPPER::setDevice, "device"_a, "storage"_a = 0)
    .def("last_kernel_milliseconds", &clipper::CLIPPER::lastKernelMilliseconds)
    .def("last_evaluations", &clipper::CLIPPER::lastEvaluations);
}
