// pybind11 bindings of the CUDA-free C++ core: allocator (even / dynamic / exact), cost model,
// stimulator.  Importable on CPU-only machines.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <limits>

#include "alloc/allocator.h"
#include "alloc/stimulator.h"

namespace py = pybind11;
using namespace sky;

namespace {
AllocProblem make_problem(const std::vector<double>& layer_flops,
                          const std::vector<double>& layer_mem,
                          const std::vector<double>& dev_time, const std::vector<double>& dev_mem,
                          const std::vector<double>& cut_penalty) {
  AllocProblem p;
  p.layer_flops = layer_flops;
  p.layer_mem = layer_mem;
  p.dev_time = dev_time;
  p.dev_mem = dev_mem;
  p.cut_penalty = cut_penalty;
  return p;
}
py::dict to_dict(const AllocResult& r) {
  py::dict d;
  d["order"] = r.order;
  d["boundaries"] = r.boundaries;
  d["bottleneck"] = r.bottleneck;
  d["exact"] = r.exact;
  d["method"] = r.method;
  return d;
}
}  // namespace

PYBIND11_MODULE(_core, m) {
  m.doc() = "skycomputing_b200 C++ core (allocator, cost model, stimulator)";
  m.def("even_partition", &even_partition, py::arg("num_layers"), py::arg("num_devices"));
  m.def(
      "dynamic_partition",
      [](const std::vector<double>& lf, const std::vector<double>& lm,
         const std::vector<double>& dt, const std::vector<double>& dm, int break_iter, bool compat,
         const std::vector<double>& cut_penalty) {
        return to_dict(dynamic_partition(make_problem(lf, lm, dt, dm, cut_penalty), break_iter,
                                         compat));
      },
      py::arg("layer_flops"), py::arg("layer_mem"), py::arg("dev_time"), py::arg("dev_mem"),
      py::arg("break_iter") = 1000, py::arg("compat") = false,
      py::arg("cut_penalty") = std::vector<double>());
  m.def(
      "optimal_partition",
      [](const std::vector<double>& lf, const std::vector<double>& lm,
         const std::vector<double>& dt, const std::vector<double>& dm, bool permute,
         int min_layers, const std::vector<double>& cut_penalty) {
        return to_dict(
            optimal_partition(make_problem(lf, lm, dt, dm, cut_penalty), permute, min_layers));
      },
      py::arg("layer_flops"), py::arg("layer_mem"), py::arg("dev_time"), py::arg("dev_mem"),
      py::arg("permute") = true, py::arg("min_layers") = 1,
      py::arg("cut_penalty") = std::vector<double>());
  m.def(
      "partition_bottleneck",
      [](const std::vector<double>& lf, const std::vector<double>& lm,
         const std::vector<double>& dt, const std::vector<double>& dm,
         const std::vector<int>& order, const std::vector<int>& boundaries,
         const std::vector<double>& cut_penalty) {
        return partition_bottleneck(make_problem(lf, lm, dt, dm, cut_penalty), order, boundaries);
      },
      py::arg("layer_flops"), py::arg("layer_mem"), py::arg("dev_time"), py::arg("dev_mem"),
      py::arg("order"), py::arg("boundaries"), py::arg("cut_penalty") = std::vector<double>());
  m.def(
      "refine_looped_partition",
      [](const std::vector<double>& lf, const std::vector<double>& lm,
         const std::vector<double>& dt, const std::vector<double>& dm,
         const std::vector<int>& boundaries, double max_chunk) {
        return refine_looped_partition(make_problem(lf, lm, dt, dm, {}), boundaries, max_chunk);
      },
      py::arg("layer_flops"), py::arg("layer_mem"), py::arg("dev_time"), py::arg("dev_mem"),
      py::arg("boundaries"), py::arg("max_chunk") = std::numeric_limits<double>::infinity(),
      "looped pipelines: refine a v * D chunk partition towards balanced per-device loads");
  m.def("numpy_default_rng_random", &numpy_default_rng_random, py::arg("seed"), py::arg("n"));
  py::class_<Stimulator>(m, "Stimulator")
      .def(py::init<int, uint64_t, uint64_t, uint64_t>(), py::arg("worker_num"),
           py::arg("mem_seed") = 22, py::arg("net_seed") = 32, py::arg("comp_seed") = 32)
      .def_property_readonly("worker_num", &Stimulator::worker_num)
      .def_readonly("m_slowdown", &Stimulator::m_slowdown)
      .def_readonly("n_slowdown", &Stimulator::n_slowdown)
      .def_readonly("c_slowdown", &Stimulator::c_slowdown)
      .def("memory_slowdown", &Stimulator::memory_slowdown)
      .def("compute_slowdown", &Stimulator::compute_slowdown)
      .def("network_stimulate", &Stimulator::network_stimulate);
}
