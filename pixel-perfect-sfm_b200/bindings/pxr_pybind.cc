// pxr_pybind.cc — the pybind11 form of the binding INTEGRATION.md describes: what a maintainer of the reference puts
// in place of `pixsfm/_pixsfm/bindings.cc:34-63` to reach libpxr.so from C++.  It binds the C-ABI of include/pxr.h
// one to one (flat numpy arrays in, numpy arrays / dicts out), the problem construction of BundleOptimizer::SetUp /
// Parameterize included (`build_problem` -> pxr_problem_build, csrc/pxr_problem.cu).  Error codes become the exception types the reference throws:
// PXR_ERR_INVALID_ARGUMENT / PXR_ERR_UNSUPPORTED -> ValueError (THROW_CHECK*, util/src/log_exceptions.h:52-84),
// everything else -> RuntimeError.  The module is thin by design: no algorithm lives here.
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/pxr.h"

namespace py = pybind11;
using namespace pybind11::literals;

namespace {

template <typename T>
using carray = py::array_t<T, py::array::c_style | py::array::forcecast>;

void check(int status) {
  if (status == PXR_OK) return;
  const std::string msg = pxr_last_error();
  if (status == PXR_ERR_INVALID_ARGUMENT || status == PXR_ERR_UNSUPPORTED) throw py::value_error(msg);
  throw std::runtime_error("pxr status " + std::to_string(status) + ": " + msg);
}

// dict lookups with the conversions a desc needs; arrays are kept alive in `keep` for the duration of the call
struct Fields {
  py::dict d;
  std::vector<py::object> keep;
  template <typename T>
  T* arr(const char* key, bool required = true) {
    if (!d.contains(key) || d[key].is_none()) {
      if (required) throw py::value_error(std::string("missing field '") + key + "'");
      return nullptr;
    }
    carray<T> a = carray<T>::ensure(d[key]);
    if (!a) throw py::value_error(std::string("field '") + key + "' has the wrong type");
    keep.push_back(a);
    return a.size() ? a.mutable_data() : nullptr;
  }
  template <typename T>
  T* inout(const char* key) {      // must already be a C-contiguous array of T: the library writes into it
    if (!d.contains(key)) throw py::value_error(std::string("missing field '") + key + "'");
    py::array a = py::array::ensure(d[key]);
    if (!a || !(a.flags() & py::array::c_style) || !py::dtype::of<T>().is(a.dtype()) || !a.writeable())
      throw py::value_error(std::string("field '") + key + "' must be a writeable C-contiguous array of the right dtype");
    keep.push_back(a);
    return static_cast<T*>(a.mutable_data());
  }
  int64_t len(const char* key) { return d.contains(key) && !d[key].is_none() ? (int64_t)py::len(d[key]) : 0; }
  template <typename T>
  T scalar(const char* key, T dflt) { return d.contains(key) ? d[key].cast<T>() : dflt; }
};

int dtype_id(const py::array& a) {
  if (a.dtype().is(py::dtype("float16"))) return PXR_F16;
  if (a.dtype().is(py::dtype::of<float>())) return PXR_F32;
  if (a.dtype().is(py::dtype::of<double>())) return PXR_F64;
  throw py::value_error("patches must be float16, float32 or float64");
}

// the geometry and observation lists of a problem dict (every pxr_ba_desc field but the patch ones)
pxr_ba_desc ba_geometry(Fields& f) {
  pxr_ba_desc d;
  std::memset(&d, 0, sizeof(d));
  d.n_cameras = (int32_t)f.len("cam_model");
  d.cam_model = f.arr<int32_t>("cam_model");
  d.cam_params = f.inout<double>("cam_params");
  d.cam_const_mask = f.arr<uint32_t>("cam_const_mask");
  d.n_images = (int32_t)f.len("img_cam");
  d.qvec = f.inout<double>("qvec");
  d.tvec = f.inout<double>("tvec");
  d.img_cam = f.arr<int32_t>("img_cam");
  d.pose_const = f.arr<uint8_t>("pose_const");
  d.tvec_const_mask = f.arr<uint8_t>("tvec_const_mask");
  d.n_points = f.len("point_const");
  d.xyz = f.inout<double>("xyz");
  d.point_const = f.arr<uint8_t>("point_const");
  d.n_obs = f.len("obs_img");
  d.obs_img = f.arr<int32_t>("obs_img");
  d.obs_pt = f.arr<int64_t>("obs_pt");
  return d;
}

pxr_ba_desc ba_desc(Fields& f) {
  pxr_ba_desc d = ba_geometry(f);
  d.obs_patch = f.arr<int64_t>("obs_patch", false);
  py::array patches = py::array::ensure(f.d["patches"]);
  if (!patches || patches.ndim() != 4 || !(patches.flags() & py::array::c_style))
    throw py::value_error("patches must be a C-contiguous [N,H,W,C] array");
  f.keep.push_back(patches);
  d.n_patches = patches.shape(0);
  d.patches = patches.data();
  d.patch_dtype = dtype_id(patches);
  d.ph = (int32_t)patches.shape(1); d.pw = (int32_t)patches.shape(2); d.channels = (int32_t)patches.shape(3);
  d.corner = f.arr<int32_t>("corner");
  d.scale = f.arr<double>("scale");
  d.upsampling_factor = f.scalar<double>("upsampling_factor", 1.0);
  d.refs = f.arr<double>("refs", false);
  return d;
}

pxr_interp_config interp_config(const py::dict& c) {
  pxr_interp_config ic;
  pxr_default_interp_config(&ic);
  if (c.contains("l2_normalize")) ic.l2_normalize = c["l2_normalize"].cast<bool>();
  if (c.contains("use_float_simd")) ic.use_float_simd = c["use_float_simd"].cast<bool>();
  if (c.contains("check_bounds")) ic.check_bounds = c["check_bounds"].cast<bool>();
  return ic;
}

void apply_options(pxr_solver_options& o, const py::dict& c) {
  auto geti = [&](const char* k, int32_t& v) { if (c.contains(k)) v = c[k].cast<int32_t>(); };
  auto getd = [&](const char* k, double& v) { if (c.contains(k)) v = c[k].cast<double>(); };
  geti("loss_type", o.loss_type); getd("loss_scale", o.loss_scale); geti("linear_solver", o.linear_solver);
  geti("max_num_iterations", o.max_num_iterations); geti("max_linear_solver_iterations", o.max_linear_solver_iterations);
  geti("max_num_consecutive_invalid_steps", o.max_num_consecutive_invalid_steps);
  getd("function_tolerance", o.function_tolerance); getd("gradient_tolerance", o.gradient_tolerance);
  getd("parameter_tolerance", o.parameter_tolerance); geti("use_inner_iterations", o.use_inner_iterations);
  getd("initial_trust_region_radius", o.initial_trust_region_radius);
  getd("inner_iteration_tolerance", o.inner_iteration_tolerance); getd("max_trust_region_radius", o.max_trust_region_radius);
  getd("min_trust_region_radius", o.min_trust_region_radius); getd("min_relative_decrease", o.min_relative_decrease);
  getd("min_lm_diagonal", o.min_lm_diagonal); getd("max_lm_diagonal", o.max_lm_diagonal);
  geti("jacobi_scaling", o.jacobi_scaling); geti("deterministic", o.deterministic);
  geti("use_nonmonotonic_steps", o.use_nonmonotonic_steps);
  geti("max_consecutive_nonmonotonic_steps", o.max_consecutive_nonmonotonic_steps);
  for (auto item : c) {
    const std::string k = py::str(item.first);
    static const char* known[] = {"loss_type", "loss_scale", "linear_solver", "max_num_iterations", "max_linear_solver_iterations",
                                  "max_num_consecutive_invalid_steps", "function_tolerance", "gradient_tolerance",
                                  "parameter_tolerance", "use_inner_iterations", "initial_trust_region_radius",
                                  "inner_iteration_tolerance", "max_trust_region_radius", "min_trust_region_radius",
                                  "min_relative_decrease", "min_lm_diagonal", "max_lm_diagonal", "jacobi_scaling",
                                  "deterministic", "use_nonmonotonic_steps", "max_consecutive_nonmonotonic_steps"};
    bool ok = false;
    for (const char* n : known) ok = ok || k == n;
    if (!ok) throw py::value_error("unknown solver option '" + k + "'");   // strict keys, like _pixsfm/src/helpers.h:149-232
  }
}

py::dict summary_dict(const pxr_summary& s, const std::vector<pxr_iteration_summary>& its) {
  py::list iterations;
  const int n = std::min<int>(s.num_iterations, (int)its.size());
  for (int i = 0; i < n; ++i)
    iterations.append(py::dict("iteration"_a = its[i].iteration, "cost"_a = its[i].cost, "step_is_valid"_a = its[i].step_is_valid,
                               "step_is_successful"_a = its[i].step_is_successful));
  return py::dict("initial_cost"_a = s.initial_cost, "final_cost"_a = s.final_cost, "num_residual_blocks"_a = s.num_residual_blocks,
                  "num_residuals"_a = s.num_residuals, "num_successful_steps"_a = s.num_successful_steps,
                  "num_unsuccessful_steps"_a = s.num_unsuccessful_steps, "termination_type"_a = s.termination_type,
                  "total_time_s"_a = s.total_time_s, "solve_time_s"_a = s.solve_time_s, "h2d_bytes"_a = s.h2d_bytes,
                  "d2h_bytes"_a = s.d2h_bytes, "kernel_launches"_a = s.kernel_launches, "message"_a = std::string(s.message),
                  "iterations"_a = iterations);
}

struct Blocks {
  std::vector<const void*> ptrs;
  std::vector<int64_t> counts;
  int32_t dtype = PXR_F16, ph = 1, pw = 1, channels = 8;
};

// `patch_blocks`: one host [n_q,H,W,C] array per query, one dtype and patch shape
Blocks patch_blocks(Fields& f, int64_t n_queries) {
  if (!f.d.contains("patch_blocks")) throw py::value_error("missing field 'patch_blocks'");
  py::list blocks = f.d["patch_blocks"];
  if ((int64_t)py::len(blocks) != n_queries) throw py::value_error("one patch block per query is required");
  Blocks b;
  for (auto item : blocks) {
    py::array a = py::array::ensure(item);
    if (!a || a.ndim() != 4 || !(a.flags() & py::array::c_style))
      throw py::value_error("patch blocks must be C-contiguous [N,H,W,C] arrays");
    f.keep.push_back(a);
    if (b.ptrs.empty()) {
      b.dtype = dtype_id(a);
      b.ph = (int32_t)a.shape(1); b.pw = (int32_t)a.shape(2); b.channels = (int32_t)a.shape(3);
    } else if (dtype_id(a) != b.dtype || a.shape(1) != b.ph || a.shape(2) != b.pw || a.shape(3) != b.channels) {
      throw py::value_error("patch blocks must share one dtype and patch shape");
    }
    b.ptrs.push_back(a.data());
    b.counts.push_back((int64_t)a.shape(0));
  }
  return b;
}

struct Context {
  pxr_ctx* h = nullptr;
  explicit Context(int device) { check(pxr_ctx_create(device, &h)); }
  ~Context() { if (h) pxr_ctx_destroy(h); }
  Context(const Context&) = delete;
  Context& operator=(const Context&) = delete;
};

}  // namespace

PYBIND11_MODULE(_pxr_pybind, m) {
  m.doc() = "pybind11 binding of libpxr.so (include/pxr.h)";
  m.def("version", &pxr_version);

  py::class_<Context>(m, "Context")
      .def(py::init<int>(), "device"_a = -1)
      .def("sync", [](Context& c) { check(pxr_ctx_sync(c.h)); });

  // ---- host-side integer algorithms (base/src/graph.cc:126-256, keypoint_adjustment/main.py:13-57)
  m.def("compute_track_labels", [](carray<int32_t> node_image, carray<int64_t> es, carray<int64_t> ed, carray<double> sim) {
    if (es.size() != ed.size() || es.size() != sim.size()) throw py::value_error("edge arrays differ in length");
    carray<int64_t> out(node_image.size());
    check(pxr_graph_track_labels(node_image.size(), node_image.data(), es.size(), es.data(), ed.data(), sim.data(), out.mutable_data()));
    return out;
  }, "node_image"_a, "edge_src"_a, "edge_dst"_a, "edge_sim"_a);
  m.def("compute_score_labels", [](int64_t n_nodes, carray<int64_t> es, carray<int64_t> ed, carray<double> sim, carray<int64_t> tl) {
    if (tl.size() != n_nodes) throw py::value_error("one track label per node is required");
    carray<double> out(n_nodes);
    check(pxr_graph_score_labels(n_nodes, es.size(), es.data(), ed.data(), sim.data(), tl.data(), out.mutable_data()));
    return out;
  }, "n_nodes"_a, "edge_src"_a, "edge_dst"_a, "edge_sim"_a, "track_labels"_a);
  m.def("compute_root_labels", [](carray<int64_t> tl, carray<double> scores) {
    if (tl.size() != scores.size()) throw py::value_error("one score per node is required");
    carray<uint8_t> out(tl.size());
    check(pxr_graph_root_labels(tl.size(), tl.data(), scores.data(), out.mutable_data()));
    return out;
  }, "track_labels"_a, "scores"_a);
  m.def("ka_problem_labels", [](carray<int64_t> tl, int max_per_problem) {
    carray<int32_t> out(tl.size());
    int32_t n = 0;
    check(pxr_ka_problem_labels(tl.size(), tl.data(), max_per_problem, out.mutable_data(), &n));
    return py::make_tuple(out, n);
  }, "track_labels"_a, "max_per_problem"_a = 50);
  m.def("shard_points", [](int64_t n_points, carray<int64_t> obs_pt, int world) {
    if (world < 1) throw py::value_error("world must be >= 1");
    carray<int64_t> pb(world + 1), ob(world + 1);
    check(pxr_shard_points(n_points, obs_pt.size(), obs_pt.data(), world, pb.mutable_data(), ob.mutable_data()));
    return py::make_tuple(pb, ob);
  }, "n_points"_a, "obs_pt"_a, "world"_a);
  m.def("shard_ka_problems", [](carray<int64_t> weight, int world) {
    carray<int32_t> out(weight.size());
    check(pxr_shard_ka_problems((int32_t)weight.size(), weight.data(), world, out.mutable_data()));
    return out;
  }, "weight"_a, "world"_a);

  // ---- problem construction: BundleOptimizer::SetUp + Parameterize (bundle_optimizer.h:139-165,247-442) and
  // ReferenceExtractor::GetVisibleObservations (reference_extractor.h:171-205) over a structure-of-arrays reconstruction.
  // `recon`: image_id, image_camera_id, p2d_begin, p2d_point3D_id, camera_id, camera_model, point3D_id, track_begin,
  // track_image_id, track_point2D_idx.  `setup` (BA mode): image_ids, const_pose_ids, const_tvec_ids, const_tvec_masks,
  // const_camera_ids, var_point_ids, const_point_ids.  `options`: refine_* flags, min_track_length; or mode = 1 with
  // ref_point_ids (+ track_has_patch).  Returns the arrays of pxr_problem_copy by name.
  m.def("build_problem", [](py::dict recon, py::dict setup, py::dict options) {
    Fields r{recon, {}}, su{setup, {}}, op{options, {}};
    pxr_recon_view v; std::memset(&v, 0, sizeof(v));
    v.n_images = r.len("image_id"); v.image_id = r.arr<int64_t>("image_id"); v.image_camera_id = r.arr<int64_t>("image_camera_id");
    v.p2d_begin = r.arr<int64_t>("p2d_begin"); v.p2d_point3D_id = r.arr<int64_t>("p2d_point3D_id", false);
    v.n_cameras = r.len("camera_id"); v.camera_id = r.arr<int64_t>("camera_id"); v.camera_model = r.arr<int32_t>("camera_model");
    v.n_points = r.len("point3D_id"); v.point3D_id = r.arr<int64_t>("point3D_id", false); v.track_begin = r.arr<int64_t>("track_begin");
    v.track_image_id = r.arr<int64_t>("track_image_id", false); v.track_point2D_idx = r.arr<int64_t>("track_point2D_idx", false);
    pxr_ba_build_options bo; std::memset(&bo, 0, sizeof(bo));
    bo.refine_focal_length = op.scalar<int>("refine_focal_length", 1); bo.refine_principal_point = op.scalar<int>("refine_principal_point", 0);
    bo.refine_extra_params = op.scalar<int>("refine_extra_params", 1); bo.refine_extrinsics = op.scalar<int>("refine_extrinsics", 1);
    bo.min_track_length = op.scalar<int>("min_track_length", -1); bo.mode = op.scalar<int>("mode", 0);
    bo.n_ref_points = op.len("ref_point_ids"); bo.ref_point_ids = op.arr<int64_t>("ref_point_ids", false);
    bo.track_has_patch = op.arr<uint8_t>("track_has_patch", false);
    pxr_ba_setup_view sv; std::memset(&sv, 0, sizeof(sv));
    if (bo.mode == 0) {
      sv.n_images = su.len("image_ids"); sv.image_ids = su.arr<int64_t>("image_ids", false);
      sv.n_const_poses = su.len("const_pose_ids"); sv.const_pose_ids = su.arr<int64_t>("const_pose_ids", false);
      sv.n_const_tvecs = su.len("const_tvec_ids"); sv.const_tvec_ids = su.arr<int64_t>("const_tvec_ids", false);
      sv.const_tvec_masks = su.arr<uint8_t>("const_tvec_masks", false);
      sv.n_const_cameras = su.len("const_camera_ids"); sv.const_camera_ids = su.arr<int64_t>("const_camera_ids", false);
      sv.n_var_points = su.len("var_point_ids"); sv.var_point_ids = su.arr<int64_t>("var_point_ids", false);
      sv.n_const_points = su.len("const_point_ids"); sv.const_point_ids = su.arr<int64_t>("const_point_ids", false);
    }
    pxr_problem_ir* ir = nullptr;
    check(pxr_problem_build(&v, bo.mode == 0 ? &sv : nullptr, &bo, &ir));
    int64_t n_obs = 0, n_img = 0, n_cam = 0, n_pts = 0;
    pxr_problem_sizes(ir, &n_obs, &n_img, &n_cam, &n_pts);
    carray<int64_t> o_pid(n_obs), o_img(n_obs), o_p2d(n_obs), obs_pt(n_obs), image_ids(n_img), camera_ids(n_cam), point_ids(n_pts);
    carray<int32_t> obs_img(n_obs), img_cam(n_img);
    carray<uint8_t> pose_const(n_img), tmask(n_img), point_const(n_pts);
    carray<uint32_t> cam_mask(n_cam);
    const int rc = pxr_problem_copy(ir, o_pid.mutable_data(), o_img.mutable_data(), o_p2d.mutable_data(), obs_img.mutable_data(),
                                    obs_pt.mutable_data(), image_ids.mutable_data(), camera_ids.mutable_data(), point_ids.mutable_data(),
                                    img_cam.mutable_data(), pose_const.mutable_data(), tmask.mutable_data(), point_const.mutable_data(),
                                    cam_mask.mutable_data());
    pxr_problem_destroy(ir);
    check(rc);
    return py::dict("obs_point3D_id"_a = o_pid, "obs_image_id"_a = o_img, "obs_point2D_idx"_a = o_p2d, "obs_img"_a = obs_img,
                    "obs_pt"_a = obs_pt, "image_ids"_a = image_ids, "camera_ids"_a = camera_ids, "point_ids"_a = point_ids,
                    "img_cam"_a = img_cam, "pose_const"_a = pose_const, "tvec_const_mask"_a = tmask, "point_const"_a = point_const,
                    "cam_const_mask"_a = cam_mask);
  }, "recon"_a, "setup"_a = py::dict(), "options"_a = py::dict());

  // ---- defaults (base/main.py:1-22, bundle_adjustment/main.py:30-62, keypoint_adjustment/main.py:60-83)
  m.def("default_ba_options", []() {
    pxr_solver_options o; pxr_default_ba_options(&o);
    return py::dict("loss_type"_a = o.loss_type, "loss_scale"_a = o.loss_scale, "max_num_iterations"_a = o.max_num_iterations,
                    "use_inner_iterations"_a = o.use_inner_iterations, "parameter_tolerance"_a = o.parameter_tolerance,
                    "linear_solver"_a = o.linear_solver);
  });
  m.def("default_ka_options", []() {
    pxr_solver_options o; pxr_default_ka_options(&o);
    return py::dict("loss_type"_a = o.loss_type, "loss_scale"_a = o.loss_scale, "max_num_iterations"_a = o.max_num_iterations,
                    "use_inner_iterations"_a = o.use_inner_iterations, "parameter_tolerance"_a = o.parameter_tolerance,
                    "linear_solver"_a = o.linear_solver);
  });

  // ---- device entry points: the problem is a dict of flat arrays named like the fields of pxr_ba_desc;
  // cam_params / qvec / tvec / xyz are refined IN PLACE, as the reference refines the Reconstruction in place
  m.def("describe_ba_problem", [](py::dict problem) {      // what the binding would hand to the library (no device needed)
    Fields f{problem, {}};
    const pxr_ba_desc d = ba_desc(f);
    return py::dict("n_cameras"_a = d.n_cameras, "n_images"_a = d.n_images, "n_points"_a = d.n_points, "n_obs"_a = d.n_obs,
                    "n_patches"_a = d.n_patches, "patch_dtype"_a = d.patch_dtype, "ph"_a = d.ph, "pw"_a = d.pw,
                    "channels"_a = d.channels, "has_refs"_a = d.refs != nullptr, "has_obs_patch"_a = d.obs_patch != nullptr);
  }, "problem"_a);
  m.def("ba_run", [](Context& ctx, py::dict problem, py::dict interpolation, py::dict options) {
    Fields f{problem, {}};
    pxr_ba_desc d = ba_desc(f);
    const pxr_interp_config ic = interp_config(interpolation);
    pxr_solver_options so; pxr_default_ba_options(&so); apply_options(so, options);
    std::vector<pxr_iteration_summary> its(512);
    pxr_summary s; std::memset(&s, 0, sizeof(s));
    s.iterations = its.data(); s.iterations_capacity = (int32_t)its.size();
    int rc;
    { py::gil_scoped_release nogil; rc = pxr_ba_run(ctx.h, &d, &ic, &so, &s); }
    check(rc);
    return summary_dict(s, its);
  }, "ctx"_a, "problem"_a, "interpolation"_a = py::dict(), "options"_a = py::dict());
  // geometric BA (GeometricBundleOptimizer.run): the problem dict holds the geometry and `obs_xy` [n_obs, 2], no patches
  m.def("ba_run_geometric", [](Context& ctx, py::dict problem, py::dict options) {
    Fields f{problem, {}};
    pxr_ba_desc d = ba_geometry(f);
    const double* obs_xy = f.arr<double>("obs_xy");
    if (f.len("obs_xy") != d.n_obs) throw py::value_error("obs_xy must hold one keypoint per observation");
    pxr_solver_options so; pxr_default_ba_options(&so); apply_options(so, options);
    std::vector<pxr_iteration_summary> its(512);
    pxr_summary s; std::memset(&s, 0, sizeof(s));
    s.iterations = its.data(); s.iterations_capacity = (int32_t)its.size();
    int rc;
    { py::gil_scoped_release nogil; rc = pxr_ba_run_geometric(ctx.h, &d, obs_xy, &so, &s); }
    check(rc);
    return summary_dict(s, its);
  }, "ctx"_a, "problem"_a, "options"_a = py::dict());
  // batched query BA (a loop of QueryBundleOptimizer.run): per query cam_model, cam_params [nq,12] / qvec [nq,4] /
  // tvec [nq,3] (refined IN PLACE), cam_const_mask, obs_begin [nq+1]; per residual block xyz, obs_patch, refs;
  // `patch_blocks` one host [n_q,H,W,C] array per query, `corner` / `scale` of their patches back to back
  m.def("qba_run", [](Context& ctx, py::dict problem, py::dict interpolation, py::dict options) {
    Fields f{problem, {}};
    pxr_qba_desc d;
    std::memset(&d, 0, sizeof(d));
    d.n_queries = (int32_t)f.len("cam_model");
    d.cam_model = f.arr<int32_t>("cam_model");
    d.cam_params = f.inout<double>("cam_params");
    d.cam_const_mask = f.arr<uint32_t>("cam_const_mask");
    d.qvec = f.inout<double>("qvec");
    d.tvec = f.inout<double>("tvec");
    d.obs_begin = f.arr<int64_t>("obs_begin");
    if (f.len("obs_begin") != (int64_t)d.n_queries + 1) throw py::value_error("obs_begin must hold n_queries + 1 entries");
    d.xyz = f.arr<double>("xyz", false);
    d.obs_patch = f.arr<int64_t>("obs_patch", false);
    d.refs = f.arr<double>("refs", false);
    Blocks pb = patch_blocks(f, d.n_queries);
    d.patch_dtype = pb.dtype; d.ph = pb.ph; d.pw = pb.pw; d.channels = pb.channels;
    std::vector<const void*>& ptrs = pb.ptrs;
    std::vector<int64_t>& counts = pb.counts;
    d.patch_blocks = ptrs.data();
    d.patch_counts = counts.data();
    d.corner = f.arr<int32_t>("corner", false);
    d.scale = f.arr<double>("scale", false);
    d.upsampling_factor = f.scalar<double>("upsampling_factor", 1.0);
    d.max_wave_bytes = f.scalar<double>("max_wave_bytes", 0.0);
    const pxr_interp_config ic = interp_config(interpolation);
    pxr_solver_options so; pxr_default_ba_options(&so); so.use_inner_iterations = 0; apply_options(so, options);
    std::vector<pxr_qba_result> res((size_t)std::max(d.n_queries, 1));
    int32_t n_waves = 0;
    pxr_summary s; std::memset(&s, 0, sizeof(s));
    int rc;
    { py::gil_scoped_release nogil; rc = pxr_qba_run(ctx.h, &d, &ic, &so, res.data(), nullptr, 0, &n_waves, &s); }
    check(rc);
    py::list out;
    for (int q = 0; q < d.n_queries; ++q) {
      const pxr_qba_result& r = res[q];
      out.append(py::dict("status"_a = r.status, "num_residual_blocks"_a = r.num_residual_blocks,
                          "initial_cost"_a = r.initial_cost, "final_cost"_a = r.final_cost,
                          "num_iterations"_a = r.num_iterations, "num_successful_steps"_a = r.num_successful_steps,
                          "num_unsuccessful_steps"_a = r.num_unsuccessful_steps, "termination_type"_a = r.termination_type,
                          "block_evaluations"_a = r.block_evaluations));
    }
    return py::dict("results"_a = out, "n_waves"_a = n_waves, "h2d_bytes"_a = s.h2d_bytes, "solve_time_s"_a = s.solve_time_s,
                    "total_time_s"_a = s.total_time_s);
  }, "ctx"_a, "problem"_a, "interpolation"_a = py::dict(), "options"_a = py::dict());
  // batched absolute pose estimation: per query corr_begin [nq+1], cam_model, cam_params [nq,12] (in/out), seed [nq]
  // (uint64), qvec [nq,4] / tvec [nq,3] (written for successful queries); per correspondence points2D [n,2],
  // points3D [n,3], inlier_mask [n] (uint8, written); `options` takes pxr_pnp_options' field names
  m.def("pnp_run", [](Context& ctx, py::dict problem, py::dict options) {
    Fields f{problem, {}};
    pxr_pnp_desc d;
    std::memset(&d, 0, sizeof(d));
    d.n_queries = (int32_t)f.len("cam_model");
    d.cam_model = f.arr<int32_t>("cam_model");
    d.cam_params = f.inout<double>("cam_params");
    d.seed = f.arr<uint64_t>("seed");
    d.qvec = f.inout<double>("qvec");
    d.tvec = f.inout<double>("tvec");
    d.corr_begin = f.arr<int64_t>("corr_begin");
    if (f.len("corr_begin") != (int64_t)d.n_queries + 1) throw py::value_error("corr_begin must hold n_queries + 1 entries");
    d.points2D = f.arr<double>("points2D", false);
    d.points3D = f.arr<double>("points3D", false);
    d.inlier_mask = f.inout<uint8_t>("inlier_mask");
    pxr_pnp_options o; pxr_default_pnp_options(&o);
    for (auto item : options) {
      const std::string k = py::str(item.first);
      py::handle v = item.second;
      if (k == "max_error") o.max_error = v.cast<double>();
      else if (k == "min_inlier_ratio") o.min_inlier_ratio = v.cast<double>();
      else if (k == "min_num_trials") o.min_num_trials = v.cast<int32_t>();
      else if (k == "max_num_trials") o.max_num_trials = v.cast<int32_t>();
      else if (k == "confidence") o.confidence = v.cast<double>();
      else if (k == "dyn_num_trials_multiplier") o.dyn_num_trials_multiplier = v.cast<double>();
      else if (k == "estimate_focal_length") o.estimate_focal_length = v.cast<bool>();
      else if (k == "refine") o.refine = v.cast<bool>();
      else if (k == "gradient_tolerance") o.gradient_tolerance = v.cast<double>();
      else if (k == "max_num_iterations") o.max_num_iterations = v.cast<int32_t>();
      else if (k == "loss_function_scale") o.loss_function_scale = v.cast<double>();
      else if (k == "refine_focal_length") o.refine_focal_length = v.cast<bool>();
      else if (k == "refine_extra_params") o.refine_extra_params = v.cast<bool>();
      else if (k == "function_tolerance") o.function_tolerance = v.cast<double>();
      else if (k == "parameter_tolerance") o.parameter_tolerance = v.cast<double>();
      else throw py::value_error("unknown pnp option '" + k + "'");
    }
    std::vector<pxr_pnp_result> res((size_t)std::max(d.n_queries, 1));
    pxr_summary s; std::memset(&s, 0, sizeof(s));
    int rc;
    { py::gil_scoped_release nogil; rc = pxr_pnp_run(ctx.h, &d, &o, res.data(), &s); }
    check(rc);
    py::list out;
    for (int q = 0; q < d.n_queries; ++q) {
      const pxr_pnp_result& r = res[q];
      out.append(py::dict("status"_a = r.status, "success"_a = (bool)r.success, "num_inliers"_a = r.num_inliers,
                          "num_trials"_a = r.num_trials, "best_trial"_a = r.best_trial, "best_solution"_a = r.best_solution,
                          "local_optimized"_a = (bool)r.local_optimized, "num_iterations"_a = r.num_iterations,
                          "termination_type"_a = r.termination_type, "initial_cost"_a = r.initial_cost,
                          "final_cost"_a = r.final_cost));
    }
    return py::dict("results"_a = out, "solve_time_s"_a = s.solve_time_s, "total_time_s"_a = s.total_time_s);
  }, "ctx"_a, "problem"_a, "options"_a = py::dict());
  // triangulation from known poses: `problem` holds cam_model [nc], cam_params [nc,12], img_cam [ni], qvec [ni,4],
  // tvec [ni,3] and, for tri_run, track_begin [nt+1], obs_img [n], obs_xy [n,2] and optionally track_key [nt]
  auto tri_desc = [](Fields& f, bool tracks) {
    pxr_tri_desc d;
    std::memset(&d, 0, sizeof(d));
    d.n_cameras = (int32_t)f.len("cam_model");
    d.cam_model = f.arr<int32_t>("cam_model");
    d.cam_params = f.arr<double>("cam_params");
    d.n_images = (int32_t)f.len("img_cam");
    d.img_cam = f.arr<int32_t>("img_cam");
    d.qvec = f.arr<double>("qvec");
    d.tvec = f.arr<double>("tvec");
    if (tracks) {
      d.track_begin = f.arr<int64_t>("track_begin");
      d.n_tracks = f.len("track_begin") - 1;
      if (d.n_tracks < 0) throw py::value_error("track_begin must hold n_tracks + 1 entries");
      d.track_key = f.arr<int64_t>("track_key", false);
      if (d.track_key && f.len("track_key") != d.n_tracks) throw py::value_error("track_key must hold n_tracks entries");
      d.obs_img = f.arr<int32_t>("obs_img", false);
      d.obs_xy = f.arr<double>("obs_xy", false);
      if (f.len("obs_img") != d.track_begin[d.n_tracks] || f.len("obs_xy") != d.track_begin[d.n_tracks])
        throw py::value_error("obs_img / obs_xy must hold track_begin[-1] entries");
    }
    return d;
  };
  m.def("tri_verify", [tri_desc](Context& ctx, py::dict problem, carray<int32_t> match_img, carray<double> match_xy,
                                 carray<double> match_noise, double max_error) {
    Fields f{problem, {}};
    const pxr_tri_desc d = tri_desc(f, false);
    const int64_t n = match_img.size() / 2;
    if (match_img.size() != 2 * n || match_xy.size() != 4 * n || match_noise.size() != 2 * n)
      throw py::value_error("match_img [n,2], match_xy [n,4] and match_noise [n,2] differ in n");
    carray<uint8_t> keep(n);
    carray<double> err({n, (int64_t)2});
    int rc;
    { py::gil_scoped_release nogil;
      rc = pxr_tri_verify(ctx.h, &d, n, match_img.data(), match_xy.data(), match_noise.data(), max_error,
                          keep.mutable_data(), err.mutable_data(), nullptr); }
    check(rc);
    return py::dict("keep"_a = keep, "err"_a = err);
  }, "ctx"_a, "problem"_a, "match_img"_a, "match_xy"_a, "match_noise"_a, "max_error"_a = 4.0);
  m.def("tri_run", [tri_desc](Context& ctx, py::dict problem, py::dict options) {
    Fields f{problem, {}};
    const pxr_tri_desc d = tri_desc(f, true);
    pxr_tri_options o; pxr_default_tri_options(&o);
    for (auto item : options) {
      const std::string k = py::str(item.first);
      py::handle v = item.second;
      if (k == "min_angle") o.min_angle = v.cast<double>();
      else if (k == "create_max_angle_error") o.create_max_angle_error = v.cast<double>();
      else if (k == "tri_max_pairs") o.tri_max_pairs = v.cast<int32_t>();
      else if (k == "seed") o.seed = v.cast<uint64_t>();
      else throw py::value_error("unknown triangulation option '" + k + "'");
    }
    const int64_t nt = d.n_tracks, no = d.track_begin[nt];
    carray<double> xyz({nt, (int64_t)3}), angle(nt), err(no);
    carray<int32_t> status(nt), n_inl(nt);
    carray<uint8_t> inl(no);
    int rc;
    { py::gil_scoped_release nogil;
      rc = pxr_tri_run(ctx.h, &d, &o, xyz.mutable_data(), status.mutable_data(), n_inl.mutable_data(), angle.mutable_data(),
                       inl.mutable_data(), err.mutable_data(), nullptr); }
    check(rc);
    return py::dict("xyz"_a = xyz, "status"_a = status, "n_inliers"_a = n_inl, "tri_angle"_a = angle,
                    "obs_inlier"_a = inl, "obs_error"_a = err);
  }, "ctx"_a, "problem"_a, "options"_a = py::dict());
  // batched query KA (a loop of QueryKeypointOptimizer.run): per query kp_begin [nq+1], patches_are_sparse [nq] and
  // one host patch block (`patch_blocks`, `corner` / `scale` back to back); per keypoint keypoints [n,2] (refined IN
  // PLACE), kp_patch (within its query's block) and desc_begin [n+1] into descs [m, C]
  m.def("qka_run", [](Context& ctx, py::dict problem, py::dict interpolation, py::dict options) {
    Fields f{problem, {}};
    pxr_qka_desc d;
    std::memset(&d, 0, sizeof(d));
    d.kp_begin = f.arr<int64_t>("kp_begin");
    d.n_queries = (int32_t)(f.len("kp_begin") - 1);
    if (d.n_queries < 0) throw py::value_error("kp_begin must hold n_queries + 1 entries");
    Blocks pb = patch_blocks(f, d.n_queries);
    d.patch_dtype = pb.dtype; d.ph = pb.ph; d.pw = pb.pw; d.channels = pb.channels;
    d.patch_blocks = pb.ptrs.data(); d.patch_counts = pb.counts.data();
    d.patches_are_sparse = f.arr<uint8_t>("patches_are_sparse", d.n_queries > 0);
    if (f.len("patches_are_sparse") != d.n_queries) throw py::value_error("one patches_are_sparse flag per query");
    d.keypoints = f.inout<double>("keypoints");
    d.kp_patch = f.arr<int64_t>("kp_patch", false);
    d.desc_begin = f.arr<int64_t>("desc_begin", false);
    const int64_t n_kp = f.len("keypoints");
    if (f.len("kp_patch") != n_kp || f.len("desc_begin") != (n_kp ? n_kp + 1 : f.len("desc_begin")))
      throw py::value_error("kp_patch must hold one entry per keypoint and desc_begin n_keypoints + 1");
    d.descs = f.arr<double>("descs", false);
    d.corner = f.arr<int32_t>("corner", false);
    d.scale = f.arr<double>("scale", false);
    d.upsampling_factor = f.scalar<double>("upsampling_factor", 1.0);
    d.bound = f.scalar<double>("bound", 4.0);
    d.max_wave_bytes = f.scalar<double>("max_wave_bytes", 0.0);
    const pxr_interp_config ic = interp_config(interpolation);
    pxr_solver_options so; pxr_default_ka_options(&so); apply_options(so, options);
    std::vector<pxr_qka_result> res((size_t)std::max(d.n_queries, 1));
    int32_t n_waves = 0;
    pxr_summary s; std::memset(&s, 0, sizeof(s));
    int rc;
    { py::gil_scoped_release nogil; rc = pxr_qka_run(ctx.h, &d, &ic, &so, res.data(), &n_waves, &s); }
    check(rc);
    py::list out;
    for (int q = 0; q < d.n_queries; ++q) {
      const pxr_qka_result& r = res[q];
      out.append(py::dict("status"_a = r.status, "num_residual_blocks"_a = r.num_residual_blocks,
                          "initial_cost"_a = r.initial_cost, "final_cost"_a = r.final_cost,
                          "num_iterations"_a = r.num_iterations, "num_successful_steps"_a = r.num_successful_steps,
                          "num_unsuccessful_steps"_a = r.num_unsuccessful_steps, "termination_type"_a = r.termination_type));
    }
    return py::dict("results"_a = out, "n_waves"_a = n_waves, "h2d_bytes"_a = s.h2d_bytes, "solve_time_s"_a = s.solve_time_s,
                    "total_time_s"_a = s.total_time_s);
  }, "ctx"_a, "problem"_a, "interpolation"_a = py::dict(), "options"_a = py::dict());
  // nearest candidate descriptor (FindNearestReferences for many queries): `patch_blocks` / `corner` / `scale` as in
  // qka_run; per item item_query, item_patch, xy [n,2] and the candidate rows [cand_begin, cand_end) of cand [m, C]
  // (host) -> dict(best, d_min, desc)
  m.def("query_match_run", [](Context& ctx, py::dict problem, py::dict interpolation) {
    Fields f{problem, {}};
    const int64_t n_queries = f.len("patch_blocks");
    Blocks pb = patch_blocks(f, n_queries);
    const int64_t n = f.len("item_query");
    const int32_t* iq = f.arr<int32_t>("item_query", false);
    const int64_t* ip = f.arr<int64_t>("item_patch", false);
    const double* xy = f.arr<double>("xy", false);
    const int64_t* cb = f.arr<int64_t>("cand_begin", false);
    const int64_t* ce = f.arr<int64_t>("cand_end", false);
    if (f.len("item_patch") != n || f.len("xy") != n || f.len("cand_begin") != n || f.len("cand_end") != n)
      throw py::value_error("one item_patch, xy, cand_begin and cand_end per item");
    const double* cand = f.arr<double>("cand", false);
    const int64_t n_cand = f.len("cand");
    if (n_cand && carray<double>::ensure(problem["cand"]).size() != n_cand * pb.channels)
      throw py::value_error("cand must be [n, channels]");
    const int32_t* corner = f.arr<int32_t>("corner", false);
    const double* scale = f.arr<double>("scale", false);
    const pxr_interp_config ic = interp_config(interpolation);
    carray<int64_t> best(n);
    carray<double> dmin(n), desc({(py::ssize_t)n, (py::ssize_t)pb.channels});
    int rc;
    {
      py::gil_scoped_release nogil;
      rc = pxr_query_match_run(ctx.h, (int32_t)n_queries, pb.ptrs.data(), pb.counts.data(), corner, scale, 1.0, pb.ph, pb.pw, pb.channels, pb.dtype, n, iq, ip, xy, cb, ce,
                               cand, n_cand, 0, &ic, best.mutable_data(), dmin.mutable_data(), desc.mutable_data());
    }
    check(rc);
    return py::dict("best"_a = best, "d_min"_a = dmin, "desc"_a = desc);
  }, "ctx"_a, "problem"_a, "interpolation"_a = py::dict());
  m.def("refs_compute", [](Context& ctx, py::dict problem, py::dict interpolation, int loss_type, double loss_scale, int iters) {
    Fields f{problem, {}};
    pxr_ba_desc d = ba_desc(f);
    const pxr_interp_config ic = interp_config(interpolation);
    carray<double> refs({(py::ssize_t)d.n_points, (py::ssize_t)d.channels});
    carray<int64_t> src(d.n_points);
    int rc;
    { py::gil_scoped_release nogil; rc = pxr_refs_compute(ctx.h, &d, &ic, loss_type, loss_scale, iters, refs.mutable_data(), src.mutable_data(), nullptr); }
    check(rc);
    return py::make_tuple(refs, src);
  }, "ctx"_a, "problem"_a, "interpolation"_a = py::dict(), "loss_type"_a = (int)PXR_LOSS_CAUCHY, "loss_scale"_a = 0.25, "iters"_a = 100);
}
