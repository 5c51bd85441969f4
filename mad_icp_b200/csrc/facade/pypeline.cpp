// pypeline -- reference: mad_icp/src/pybind/pypeline.cpp:52-75 (Pipeline + VectorEigen3d), same ctor
// arguments and method names; registration runs on the GPU.
#include <limits>

#include "pipeline.hpp"
#include "py_common.hpp"

// an object exporting __cuda_array_interface__ (a CUDA tensor, a CuPy array): its records are device memory
static bool on_device(const py::object& o) { return py::hasattr(o, "__cuda_array_interface__"); }
// a device array copied to the host once (records.to_host), for host-built trees (MADICP_GPU_BUILD=0)
static py::object to_host(const py::object& o) { return py::module_::import("mad_icp_b200.records").attr("to_host")(o); }

// keeps a Python object alive until a queued scan is done with it (dropped on the thread that calls compute, with the
// GIL held)
static std::shared_ptr<void> keepalive(const py::object& o) {
  return std::shared_ptr<void>(new py::object(o), [](void* q) { delete static_cast<py::object*>(q); });
}

// A scan as a Pipeline call takes it, and the Python object that keeps its memory alive
struct ScanArg {
  madicp_points_t d{};
  madicp_vcorr_t v{};
  madicp_times_t t{};  // type MADICP_TIME_NONE without a time field
  bool on_dev = false;
  mb::DevScan dev;     // device records: the stream they are ready on
  py::object hold;
  const mb::DevScan* devScan() const { return on_dev ? &dev : nullptr; }
  const madicp_times_t* times() const { return t.type ? &t : nullptr; }
};

// records (2-D float array with >= 3 columns, or 1-D structured with x/y/z; host or device memory) -> madicp_points_t, by
// records.layout; apply_correction / vertical_angle_offset (KittiReader's names) -> madicp_vcorr_t; time_field /
// time_scale / time_end -> madicp_times_t, by records.time_layout
static ScanArg records_arg(const py::object& records, double min_range, double max_range, bool inclusive, bool drop_nan,
                           bool apply_correction = false, double vertical_angle_offset = 0.0,
                           const py::object& time_field = py::none(), double time_scale = 1.0,
                           const py::object& time_end = py::none()) {
  const py::module_ rec = py::module_::import("mad_icp_b200.records");
  const py::tuple l = rec.attr("layout")(records, min_range, max_range, inclusive, drop_nan).cast<py::tuple>();
  ScanArg r;
  r.d.data = reinterpret_cast<const void*>(l[0].cast<uintptr_t>());
  r.d.n = l[1].cast<int64_t>();
  r.d.stride = l[2].cast<int64_t>();
  for (int c = 0; c < 3; ++c) r.d.offset[c] = l[size_t(3 + c)].cast<int32_t>();
  r.d.is_f32 = l[6].cast<int32_t>();
  r.d.min_range = l[7].cast<double>();
  r.d.max_range = l[8].cast<double>();
  r.d.range_mode = l[9].cast<int32_t>();
  r.d.drop_nan = l[10].cast<int32_t>();
  r.on_dev = l[11].cast<bool>();
  if (r.on_dev) r.dev.stream = reinterpret_cast<void*>(l[12].cast<uintptr_t>());
  r.v.angle = vertical_angle_offset;
  r.v.enabled = apply_correction ? 1 : 0;
  if (!time_field.is_none()) {
    const py::tuple t = rec.attr("time_layout")(records, time_field, time_scale, time_end).cast<py::tuple>();
    r.t.offset = t[0].cast<int32_t>();
    r.t.type = t[1].cast<int32_t>();
    r.t.scale = t[2].cast<double>();
    r.t.t_end = t[3].cast<double>();
    r.t.has_t_end = t[4].cast<int32_t>();
  }
  r.hold = records;
  return r;
}

// A compute / prefetch cloud, read where it is: a device array as records without a gate (for host-built trees it is
// copied to the host first); in host memory a packed N x 3 cloud -- a bound VectorEigen3d by reference, a float32 array
// as the dataset readers deliver it (the conversion to float64 runs on the device), any other array as C-contiguous
// float64 (a view when it already is one)
static ScanArg scan_arg(py::object cloud, bool gpu_build) {
  if (on_device(cloud)) {
    if (gpu_build) {
      ScanArg r = records_arg(cloud, 0.0, std::numeric_limits<double>::infinity(), true, false);
      r.d.range_mode = MADICP_RANGE_NONE;
      return r;
    }
    cloud = to_host(cloud);
  }
  ScanArg r;
  if (py::isinstance<mb::ContainerType>(cloud)) {
    const mb::ContainerType& v = cloud.cast<const mb::ContainerType&>();
    r.d = madicp::packed_points(v.empty() ? nullptr : v[0].data(), int64_t(v.size()), 0);
    r.hold = cloud;
    return r;
  }
  const bool f32 = py::isinstance<py::array>(cloud) && py::array::ensure(cloud).dtype().is(py::dtype::of<float>());
  const py::array a = f32 ? py::array(cloud.cast<py::array_t<float, py::array::c_style | py::array::forcecast>>())
                          : py::array(cloud.cast<NpArr>());
  if (a.ndim() != 2 || a.shape(1) != 3) throw py::cast_error();
  r.d = madicp::packed_points(a.shape(0) ? a.data() : nullptr, a.shape(0), f32 ? 1 : 0);
  r.hold = a;
  return r;
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

// mapArray / mapIndices as numpy arrays, or with `device` as CUDA tensors on the pipeline's device, ready on torch's current
// stream (records.map_array_dev)
static py::object map_array(const py::object& self, bool device, bool indices) {
  if (device) return py::module_::import("mad_icp_b200.records").attr("map_array_dev")(self, indices);
  mb::Pipeline& p = self.cast<mb::Pipeline&>();
  const size_t n = p.mapSize();
  py::array_t<double> xyz({indices ? size_t(0) : n, size_t(3)});
  py::array_t<int64_t> sr({indices ? n : size_t(0), size_t(2)});
  if (n) p.mapPoints(indices ? nullptr : xyz.mutable_data(), indices ? sr.mutable_data() : nullptr);
  if (indices) return std::move(sr);
  return std::move(xyz);
}

PYBIND11_MODULE(pypeline, m) {
  bind_vector_eigen3d(m);
  // KittiReader.vertical_angle_offset, np.radians(0.205), as records.py computes it: the default bit for bit
  const double kVerticalAngle = py::module_::import("mad_icp_b200.records").attr("VERTICAL_ANGLE_OFFSET").cast<double>();
  py::class_<mb::Pipeline>(m, "Pipeline")
      // keep_cloud (not in the reference): the current scan's deskewed cloud and its record indices stay available
      // (currentCloudArray / currentCloudIndices)
      // map_voxel_size > 0 (not in the reference): a voxel map of every scan builds itself on the device, keeping the
      // first map_points_per_voxel points of each voxel (mapArray / mapIndices); map_max_distance > 0 bounds it to the
      // voxels whose centre lies within that distance of the sensor after each scan; map_carve = r in (0, 1] carves it
      // along each scan's rays after its insert: the voxels the first r of a ray's steps pass through go unless they
      // hold a point of the scan (madicp_map_carve)
      .def(py::init([](double sensor_hz, bool deskew, double b_max, double rho_ker, double p_th, double b_min, double b_ratio,
                       int num_keyframes, int num_threads, bool realtime, bool keep_cloud, double map_voxel_size,
                       int map_points_per_voxel, double map_max_distance, double map_carve) {
             return new mb::Pipeline(sensor_hz, deskew, b_max, rho_ker, p_th, b_min, b_ratio, num_keyframes, num_threads,
                                     realtime, -1, keep_cloud, map_voxel_size, map_points_per_voxel,
                                     map_max_distance, map_carve);
           }),
           py::arg("sensor_hz"), py::arg("deskew"), py::arg("b_max"), py::arg("rho_ker"), py::arg("p_th"), py::arg("b_min"),
           py::arg("b_ratio"), py::arg("num_keyframes"), py::arg("num_threads"), py::arg("realtime"),
           py::arg("keep_cloud") = false, py::arg("map_voxel_size") = 0.0, py::arg("map_points_per_voxel") = 1,
           py::arg("map_max_distance") = 0.0, py::arg("map_carve") = 0.0)
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
      // the voxel map (map_voxel_size > 0): its points in the map frame (M, 3) float64, and (scan, record) per point
      // (M, 2) int64 -- scan: currentID() before that scan was computed, record: its currentCloudIndices() value
      .def("mapSize", &mb::Pipeline::mapSize)
      .def("mapArray", [](const py::object& self, bool device) { return map_array(self, device, false); },
           py::arg("device") = false)
      .def("mapIndices", [](const py::object& self, bool device) { return map_array(self, device, true); },
           py::arg("device") = false)
      .def("mapDropped", &mb::Pipeline::mapDropped)
      .def("clearMap", &mb::Pipeline::clearMap)
      // the nearest map row within max_distance (<= 4 map voxel sizes) of each point (N x 3), among the rows whose scan
      // is < scan_below (None: every row): (row (N,) int64, -1 for none; d2 (N,) float64, +inf for none), as numpy
      // arrays, or for device points (a CUDA tensor, a CuPy array, read in place) as torch tensors on the pipeline's
      // device, ready on torch's current stream (records.map_nearest_dev)
      .def("mapNearest", [](py::object self, const py::object& points, double max_distance, const py::object& scan_below)
               -> py::object {
             const int64_t below = scan_below.is_none() ? std::numeric_limits<int64_t>::max() : scan_below.cast<int64_t>();
             if (on_device(points))
               return py::module_::import("mad_icp_b200.records").attr("map_nearest_dev")(
                   self.attr("_mapNearestDev"), self.attr("_device")(), points, max_distance, below);
             mb::Pipeline& p = self.cast<mb::Pipeline&>();
             const mb::ContainerType q = cloud_arg(points);
             py::array_t<int64_t> row(q.size());
             py::array_t<double> d2(q.size());
             p.mapNearest(q.empty() ? nullptr : q[0].data(), int64_t(q.size()), max_distance, below, row.mutable_data(),
                          d2.mutable_data());
             return py::make_tuple(row, d2);
           }, py::arg("points"), py::arg("max_distance"), py::arg("scan_below") = py::none())
      .def("_mapNearestDev", [](mb::Pipeline& p, uintptr_t q, int64_t n, int64_t stride, bool is_f32, double max_distance,
                                int64_t scan_below, uintptr_t row, uintptr_t d2, uintptr_t stream) {
        p.mapNearestDev(reinterpret_cast<const void*>(q), n, stride, is_f32, max_distance, scan_below,
                        reinterpret_cast<int64_t*>(row), reinterpret_cast<double*>(d2), reinterpret_cast<void*>(stream));
      })
      .def("_mapDev", [](mb::Pipeline& p, uintptr_t xyz, uintptr_t sr, uintptr_t stream) {
        p.mapPointsDev(reinterpret_cast<double*>(xyz), reinterpret_cast<int64_t*>(sr), reinterpret_cast<void*>(stream));
      })
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
      .def("compute", [](mb::Pipeline& p, double stamp, const py::object& cloud) {
        const ScanArg c = scan_arg(cloud, p.gpuBuild());
        if (c.on_dev) p.computeRecords(stamp, c.d, nullptr, &c.dev);
        else if (c.d.is_f32) p.computeF32(stamp, static_cast<const float*>(c.d.data), size_t(c.d.n));
        else p.compute(stamp, static_cast<const double*>(c.d.data), size_t(c.d.n));
      })
      // additions (not in the reference): diagnostics
      .def_static("_deskewOnly", [](const py::object& cloud, const NpArr& a, const NpArr& b, double sensor_hz, int num_threads) {
        return mb::Pipeline::deskewOnly(cloud_arg(cloud), pose_from_numpy(a), pose_from_numpy(b), sensor_hz, num_threads);
      }, py::arg("cloud"), py::arg("T_prev"), py::arg("T_now"), py::arg("sensor_hz"), py::arg("num_threads") = 1)
      .def("prefetch", [](mb::Pipeline& p, const py::object& cloud, bool deskew_ahead) {
        // the array is read in place when the batch is built (inside a later compute()): a reference keeps it alive
        if (on_device(cloud) && !p.gpuBuild()) return false;  // (host-built trees: no look-ahead, as for host arrays)
        const ScanArg c = scan_arg(cloud, true);
        if (c.on_dev) return p.prefetchRecords(c.d, keepalive(c.hold), nullptr, deskew_ahead, &c.dev);
        return p.prefetch(c.d.data, size_t(c.d.n), c.d.is_f32 != 0, keepalive(c.hold), nullptr, nullptr, deskew_ahead);
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
        const py::object recs = (on_device(records) && !p.gpuBuild()) ? to_host(records) : records;
        const ScanArg r = records_arg(recs, min_range, max_range, inclusive, drop_nan, apply_correction,
                                      vertical_angle_offset, time_field, time_scale, time_end);
        p.computeRecords(stamp, r.d, &r.v, r.devScan(), r.times());
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
        const ScanArg r = records_arg(records, min_range, max_range, inclusive, drop_nan, apply_correction,
                                      vertical_angle_offset, time_field, time_scale, time_end);
        return p.prefetchRecords(r.d, keepalive(r.hold), &r.v, deskew_ahead, r.devScan(), r.times());
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
