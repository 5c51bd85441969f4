// pymadtree -- reference: mad_icp/src/pybind/tools/pymadtree.cpp:36-48 (MADtree: build / search /
// searchCloud / searchCloudDist), same names, defaults and return shapes; the search runs on the GPU.
#include "py_common.hpp"
PYBIND11_MODULE(pymadtree, m) {
  bind_vector_eigen3d(m);
  py::class_<mb::MADtreeWrapper>(m, "MADtree")
      .def(py::init<>())
      .def("build",
           [](mb::MADtreeWrapper& t, const py::object& vec, double b_max, double b_min, int max_parallel_level) {
             t.build(cloud_arg(vec), b_max, b_min, max_parallel_level);
           },
           py::arg("vec"), py::arg("b_max") = 1e-5, py::arg("b_min") = 0.1, py::arg("max_parallel_level") = 2)
      .def("search",
           [](mb::MADtreeWrapper& t, const NpArr& q) {
             if (q.size() != 3) throw py::cast_error();
             mb::ContainerType one{{q.data()[0], q.data()[1], q.data()[2]}};
             auto r = t.searchCloud(one, false);
             return py::make_tuple(numpy3(r.points[0]), numpy3(r.normals[0]));
           },
           py::arg("query"))
      .def("searchCloud",
           [](mb::MADtreeWrapper& t, const py::object& cloud) {
             auto r = t.searchCloud(cloud_arg(cloud), false);
             py::list out;
             for (size_t i = 0; i < r.points.size(); ++i)
               out.append(py::make_tuple(numpy3(r.points[i]), numpy3(r.normals[i])));
             return out;
           },
           py::arg("query_cloud"))
      .def("searchCloudDist",
           [](mb::MADtreeWrapper& t, const py::object& cloud) {
             auto r = t.searchCloud(cloud_arg(cloud), true);
             py::list out;
             for (size_t i = 0; i < r.points.size(); ++i)
               out.append(py::make_tuple(numpy3(r.points[i]), numpy3(r.normals[i]), r.dists[i]));
             return out;
           },
           py::arg("query_cloud"))
      // array form of the same operator (SURVEY 8f next-4): (points N x 3, normals N x 3, dists N); device queries (a CUDA
      // tensor, a CuPy array) are read in place and answered with float64 torch tensors on their device, ready on the
      // caller's current stream (records.search_cloud_arrays_dev)
      .def("searchCloudArrays", [](py::object self, const py::object& cloud) -> py::object {
        if (py::hasattr(cloud, "__cuda_array_interface__"))
          return py::module_::import("mad_icp_b200.records").attr("search_cloud_arrays_dev")(self.attr("_searchCloudDev"), cloud);
        mb::MADtreeWrapper& t = self.cast<mb::MADtreeWrapper&>();
        auto r = t.searchCloud(cloud_arg(cloud), true);
        const size_t n = r.points.size();
        py::array_t<double> P({n, size_t(3)}), N({n, size_t(3)}), D(n);
        if (n) {
          std::memcpy(P.mutable_data(), r.points[0].data(), 24 * n);
          std::memcpy(N.mutable_data(), r.normals[0].data(), 24 * n);
          std::memcpy(D.mutable_data(), r.dists.data(), 8 * n);
        }
        return py::make_tuple(P, N, D);
      })
      .def("_searchCloudDev", [](mb::MADtreeWrapper& t, uintptr_t q, int64_t n, int64_t stride, bool is_f32, uintptr_t P,
                                 uintptr_t N, uintptr_t D, uintptr_t stream) {
        t.searchCloudDev(reinterpret_cast<const void*>(q), n, stride, is_f32, reinterpret_cast<double*>(P),
                         reinterpret_cast<double*>(N), reinterpret_cast<double*>(D), reinterpret_cast<void*>(stream));
      });
}
