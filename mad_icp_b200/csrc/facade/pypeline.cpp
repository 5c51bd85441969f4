// pypeline -- reference: mad_icp/src/pybind/pypeline.cpp:52-75 (Pipeline + VectorEigen3d), same ctor
// arguments and method names; registration runs on the GPU.
#include <limits>

#include "pipeline.hpp"
#include "py_common.hpp"

// an object exporting __cuda_array_interface__ (a CUDA tensor, a CuPy array): its records are device memory
static bool on_device(const py::object& o) { return py::hasattr(o, "__cuda_array_interface__"); }
// a device array copied to the host once (records.to_host), for host-built trees (MADICP_GPU_BUILD=0)
static py::object to_host(const py::object& o) { return py::module_::import("mad_icp_b200.records").attr("to_host")(o); }

// records (2-D float array with >= 3 columns, or 1-D structured with x/y/z; host or device memory) -> madicp_points_t, by
// records.layout; dev receives the producer stream of device records (and is left alone for host records)
static madicp_points_t records_arg(const py::object& records, double min_range, double max_range, bool inclusive,
                                   bool drop_nan, mb::DevScan* dev = nullptr, bool* is_dev = nullptr) {
  const py::tuple t = py::module_::import("mad_icp_b200.records")
                          .attr("layout")(records, min_range, max_range, inclusive, drop_nan)
                          .cast<py::tuple>();
  if (is_dev) *is_dev = t[11].cast<bool>();
  if (dev && t[11].cast<bool>()) dev->stream = reinterpret_cast<void*>(t[12].cast<uintptr_t>());
  madicp_points_t d{};
  d.data = reinterpret_cast<const void*>(t[0].cast<uintptr_t>());
  d.n = t[1].cast<int64_t>();
  d.stride = t[2].cast<int64_t>();
  for (int c = 0; c < 3; ++c) d.offset[c] = t[size_t(3 + c)].cast<int32_t>();
  d.is_f32 = t[6].cast<int32_t>();
  d.min_range = t[7].cast<double>();
  d.max_range = t[8].cast<double>();
  d.range_mode = t[9].cast<int32_t>();
  d.drop_nan = t[10].cast<int32_t>();
  return d;
}

// time_field / time_scale / time_end -> madicp_times_t (records.time_layout; type MADICP_TIME_NONE without a field)
static madicp_times_t times_arg(const py::object& records, const py::object& field, double scale, const py::object& t_end) {
  madicp_times_t t{};
  if (field.is_none()) return t;
  const py::tuple l = py::module_::import("mad_icp_b200.records").attr("time_layout")(records, field, scale, t_end).cast<py::tuple>();
  t.offset = l[0].cast<int32_t>();
  t.type = l[1].cast<int32_t>();
  t.scale = l[2].cast<double>();
  t.t_end = l[3].cast<double>();
  t.has_t_end = l[4].cast<int32_t>();
  return t;
}

// apply_correction / vertical_angle_offset (KittiReader's names) -> madicp_vcorr_t
static madicp_vcorr_t vcorr_arg(bool apply_correction, double vertical_angle_offset) {
  madicp_vcorr_t v{};
  v.angle = vertical_angle_offset;
  v.enabled = apply_correction ? 1 : 0;
  return v;
}

// currentLeaves (model == false) / modelLeaves as an (N, 3) float64 numpy array, or with `device` as a float64 CUDA tensor
// on the pipeline's device, written in place and ready on torch's current stream (records.leaves_array_dev)
static py::object leaves_array(const py::object& self, bool model, bool device) {
  if (device) return py::module_::import("mad_icp_b200.records").attr("leaves_array_dev")(self, model);
  const mb::Pipeline& p = self.cast<const mb::Pipeline&>();
  py::array_t<double> out({p.numLeaves(model), size_t(3)});
  if (out.shape(0)) p.leafMeans(model, out.mutable_data());
  return std::move(out);
}

// currentCloudArray's frame: "map" or "sensor"
static bool map_frame(const std::string& frame) {
  if (frame != "map" && frame != "sensor") throw py::value_error("currentCloudArray: frame must be \"map\" or \"sensor\"");
  return frame == "map";
}

// currentCloudArray / currentCloudIndices as numpy arrays, or with `device` as CUDA tensors on the pipeline's device,
// ready on torch's current stream (records.cloud_array_dev)
static py::object cloud_array(const py::object& self, bool device, bool map) {
  const mb::Pipeline& p = self.cast<const mb::Pipeline&>();
  const size_t n = p.numCloudPoints();
  if (device) return py::module_::import("mad_icp_b200.records").attr("cloud_array_dev")(self, false, map);
  py::array_t<double> out({n, size_t(3)});
  if (n) p.cloud(map, out.mutable_data(), nullptr);
  return std::move(out);
}
static py::object cloud_indices(const py::object& self, bool device) {
  const mb::Pipeline& p = self.cast<const mb::Pipeline&>();
  const size_t n = p.numCloudPoints();
  if (device) return py::module_::import("mad_icp_b200.records").attr("cloud_array_dev")(self, true, false);
  py::array_t<int64_t> out(n);
  if (n) p.cloud(false, nullptr, out.mutable_data());
  return std::move(out);
}

PYBIND11_MODULE(pypeline, m) {
  bind_vector_eigen3d(m);
  // KittiReader.vertical_angle_offset, np.radians(0.205), as records.py computes it: the default bit for bit
  const double kVerticalAngle = py::module_::import("mad_icp_b200.records").attr("VERTICAL_ANGLE_OFFSET").cast<double>();
  py::class_<mb::Pipeline>(m, "Pipeline")
      // keep_cloud (not in the reference): the current scan's deskewed cloud and its record indices stay available
      // (currentCloudArray / currentCloudIndices)
      .def(py::init([](double sensor_hz, bool deskew, double b_max, double rho_ker, double p_th, double b_min, double b_ratio,
                       int num_keyframes, int num_threads, bool realtime, bool keep_cloud) {
             return new mb::Pipeline(sensor_hz, deskew, b_max, rho_ker, p_th, b_min, b_ratio, num_keyframes, num_threads,
                                     realtime, -1, keep_cloud);
           }),
           py::arg("sensor_hz"), py::arg("deskew"), py::arg("b_max"), py::arg("rho_ker"), py::arg("p_th"), py::arg("b_min"),
           py::arg("b_ratio"), py::arg("num_keyframes"), py::arg("num_threads"), py::arg("realtime"),
           py::arg("keep_cloud") = false)
      .def("currentPose", [](const mb::Pipeline& p) { return pose_to_numpy(p.currentPose()); })
      .def("trajectory",
           [](const mb::Pipeline& p) {
             py::list out;
             for (const auto& T : p.trajectory()) out.append(pose_to_numpy(T));
             return out;
           })
      .def("keyframePose", [](const mb::Pipeline& p) { return pose_to_numpy(p.keyframePose()); })
      .def("isInitialized", &mb::Pipeline::isInitialized)
      .def("isMapUpdated", &mb::Pipeline::isMapUpdated)
      .def("currentID", &mb::Pipeline::currentID)
      .def("keyframeID", &mb::Pipeline::keyframeID)
      .def("modelLeaves", &mb::Pipeline::modelLeaves)
      .def("currentLeaves", &mb::Pipeline::currentLeaves)
      // additions (not in the reference): the same points as arrays, gathered on the device, or as CUDA tensors
      .def("currentLeavesArray", [](const py::object& self, bool device) { return leaves_array(self, false, device); },
           py::arg("device") = false)
      .def("modelLeavesArray", [](const py::object& self, bool device) { return leaves_array(self, true, device); },
           py::arg("device") = false)
      // the current scan's deskewed cloud (keep_cloud): points in the map frame (currentPose) or the sensor frame, and
      // the index of every point's record in the array the scan was handed over as
      .def("currentCloudArray", [](const py::object& self, bool device, const std::string& frame) {
             return cloud_array(self, device, map_frame(frame));
           }, py::arg("device") = false, py::arg("frame") = "map")
      .def("currentCloudIndices", [](const py::object& self, bool device) { return cloud_indices(self, device); },
           py::arg("device") = false)
      .def("_numCloudPoints", &mb::Pipeline::numCloudPoints)
      .def("_kernelLaunches", &mb::Pipeline::kernelLaunches)
      .def("_cloudDev", [](const mb::Pipeline& p, bool map, uintptr_t xyz, uintptr_t idx, uintptr_t stream) {
        p.cloudDev(map, reinterpret_cast<double*>(xyz), reinterpret_cast<int64_t*>(idx), reinterpret_cast<void*>(stream));
      })
      .def("_numLeaves", &mb::Pipeline::numLeaves)
      .def("_device", &mb::Pipeline::device)
      .def("_leafMeansDev", [](const mb::Pipeline& p, bool model, uintptr_t out, uintptr_t stream) {
        p.leafMeansDev(model, reinterpret_cast<double*>(out), reinterpret_cast<void*>(stream));
      })
      .def("compute", [](mb::Pipeline& p, double stamp, py::object cloud) {
        // read the points where they are: a bound VectorEigen3d by reference, a numpy array through its buffer, a device
        // array in place (as records without a gate)
        if (on_device(cloud)) {
          if (p.gpuBuild()) {
            mb::DevScan dev;
            madicp_points_t d = records_arg(cloud, 0.0, std::numeric_limits<double>::infinity(), true, false, &dev);
            d.range_mode = MADICP_RANGE_NONE;
            p.computeRecords(stamp, d, nullptr, &dev);
            return;
          }
          cloud = to_host(cloud);
        }
        if (py::isinstance<mb::ContainerType>(cloud)) {
          const mb::ContainerType& v = cloud.cast<const mb::ContainerType&>();
          p.compute(stamp, v.empty() ? nullptr : v[0].data(), v.size());
        } else if (py::isinstance<py::array>(cloud) && py::array::ensure(cloud).dtype().is(py::dtype::of<float>())) {
          // float32 as the dataset readers deliver it: converted on the device (no host copy in float64)
          const auto a = cloud.cast<py::array_t<float, py::array::c_style | py::array::forcecast>>();
          if (a.ndim() != 2 || a.shape(1) != 3) throw py::cast_error();
          p.computeF32(stamp, a.shape(0) ? a.data() : nullptr, size_t(a.shape(0)));
        } else {
          const NpArr a = cloud.cast<NpArr>();  // a view when the array already is C-contiguous float64
          if (a.ndim() != 2 || a.shape(1) != 3) throw py::cast_error();
          p.compute(stamp, a.shape(0) ? a.data() : nullptr, size_t(a.shape(0)));
        }
      })
      // additions (not in the reference): diagnostics
      .def_static("_deskewOnly", [](const py::object& cloud, const NpArr& a, const NpArr& b, double sensor_hz, int num_threads) {
        return mb::Pipeline::deskewOnly(cloud_arg(cloud), pose_from_numpy(a), pose_from_numpy(b), sensor_hz, num_threads);
      }, py::arg("cloud"), py::arg("T_prev"), py::arg("T_now"), py::arg("sensor_hz"), py::arg("num_threads") = 1)
      .def("prefetch", [](mb::Pipeline& p, const py::object& cloud, bool deskew_ahead) {
        // the array is read in place when the batch is built (inside a later compute()): a reference keeps it alive
        // until then (it is dropped there, on the calling thread, with the GIL held)
        auto hold = [](const py::object& o) {
          py::object* ref = new py::object(o);
          return std::shared_ptr<void>(ref, [](void* q) { delete static_cast<py::object*>(q); });
        };
        if (on_device(cloud)) {  // (host-built trees: no look-ahead, as for host arrays)
          if (!p.gpuBuild()) return false;
          mb::DevScan dev;
          madicp_points_t d = records_arg(cloud, 0.0, std::numeric_limits<double>::infinity(), true, false, &dev);
          d.range_mode = MADICP_RANGE_NONE;
          return p.prefetchRecords(d, hold(cloud), nullptr, deskew_ahead, &dev);
        }
        if (py::isinstance<mb::ContainerType>(cloud)) {
          const mb::ContainerType& v = cloud.cast<const mb::ContainerType&>();
          return p.prefetch(v.empty() ? nullptr : v[0].data(), v.size(), false, hold(cloud), nullptr, nullptr, deskew_ahead);
        }
        if (py::isinstance<py::array>(cloud) && py::array::ensure(cloud).dtype().is(py::dtype::of<float>())) {
          const auto a = cloud.cast<py::array_t<float, py::array::c_style | py::array::forcecast>>();
          if (a.ndim() != 2 || a.shape(1) != 3) throw py::cast_error();
          return p.prefetch(a.data(), size_t(a.shape(0)), true, hold(a), nullptr, nullptr, deskew_ahead);
        }
        const NpArr a = cloud.cast<NpArr>();
        if (a.ndim() != 2 || a.shape(1) != 3) throw py::cast_error();
        return p.prefetch(a.data(), size_t(a.shape(0)), false, hold(a), nullptr, nullptr, deskew_ahead);
      }, py::arg("cloud"), py::arg("deskew_ahead") = false)
      // additions (not in the reference): raw sensor records, filtered on the way in like the dataset readers do
      // (mad_icp_b200/records.py describes the array; it is read in place); apply_correction: KITTI's vertical-angle
      // correction of the kept points, as KittiReader applies it
      // time_field (a structured field name, or a column index of a 2-D array): the records' per-point time stamps, in
      // units of time_scale seconds; a deskewing pipeline takes each point's chunk from its own stamp (time_end: the
      // sweep's end in field units, default the largest kept stamp) -- no azimuth sort
      .def("computeRecords", [](mb::Pipeline& p, double stamp, const py::object& records, double min_range, double max_range,
                                bool inclusive, bool drop_nan, bool apply_correction, double vertical_angle_offset,
                                const py::object& time_field, double time_scale, const py::object& time_end) {
        const madicp_vcorr_t v = vcorr_arg(apply_correction, vertical_angle_offset);
        const py::object recs = (on_device(records) && !p.gpuBuild()) ? to_host(records) : records;
        mb::DevScan dev;
        bool is_dev = false;
        const madicp_points_t d = records_arg(recs, min_range, max_range, inclusive, drop_nan, &dev, &is_dev);
        const madicp_times_t t = times_arg(recs, time_field, time_scale, time_end);
        p.computeRecords(stamp, d, &v, is_dev ? &dev : nullptr, t.type ? &t : nullptr);
      }, py::arg("stamp"), py::arg("records"), py::arg("min_range") = 0.0,
         py::arg("max_range") = std::numeric_limits<double>::infinity(), py::arg("inclusive") = true, py::arg("drop_nan") = false,
         py::arg("apply_correction") = false, py::arg("vertical_angle_offset") = kVerticalAngle, py::arg("time_field") = py::none(),
         py::arg("time_scale") = 1.0, py::arg("time_end") = py::none())
      // deskew_ahead (prefetch, prefetchRecords): on a deskewing pipeline the scan is planned ahead -- uploaded, gated,
      // corrected and sorted by azimuth while earlier scans register -- and compute applies its chunk poses
      .def("prefetchRecords", [](mb::Pipeline& p, const py::object& records, double min_range, double max_range,
                                 bool inclusive, bool drop_nan, bool apply_correction, double vertical_angle_offset,
                                 bool deskew_ahead, const py::object& time_field, double time_scale, const py::object& time_end) {
        if (on_device(records) && !p.gpuBuild()) return false;  // (host-built trees: no look-ahead)
        mb::DevScan dev;
        bool is_dev = false;
        const madicp_points_t d = records_arg(records, min_range, max_range, inclusive, drop_nan, &dev, &is_dev);
        const madicp_vcorr_t v = vcorr_arg(apply_correction, vertical_angle_offset);
        const madicp_times_t t = times_arg(records, time_field, time_scale, time_end);
        py::object* ref = new py::object(records);  // dropped once the scan's tree is built (see prefetch)
        return p.prefetchRecords(d, std::shared_ptr<void>(ref, [](void* q) { delete static_cast<py::object*>(q); }), &v,
                                 deskew_ahead, is_dev ? &dev : nullptr, t.type ? &t : nullptr);
      }, py::arg("records"), py::arg("min_range") = 0.0,
         py::arg("max_range") = std::numeric_limits<double>::infinity(), py::arg("inclusive") = true, py::arg("drop_nan") = false,
         py::arg("apply_correction") = false, py::arg("vertical_angle_offset") = kVerticalAngle, py::arg("deskew_ahead") = false,
         py::arg("time_field") = py::none(), py::arg("time_scale") = 1.0, py::arg("time_end") = py::none())
      .def("prefetched", &mb::Pipeline::prefetched)
      .def("lastIcpIterations", &mb::Pipeline::lastIcpIterations)
      .def("gpuBuild", &mb::Pipeline::gpuBuild)
      .def("inliersRatio", &mb::Pipeline::inliersRatio)
      .def("numKeyframes", &mb::Pipeline::numKeyframes);
  py::register_exception<mb::Error>(m, "MadIcpError", PyExc_RuntimeError);
}
