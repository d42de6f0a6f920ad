"""Geometric (reprojection-error) bundle adjustment without a device: the CPU restatement converges to scipy's
optimum on the nine setups of the reference's bundle_optimizer_test.cc, the Python surface runs end to end with the
oracle standing in for the device entry points, and the C-ABI rejects malformed geometric problems on the host."""
import ctypes as C

import numpy as np
import pytest

import geo_scenes as G
import geo_oracle_lib as GO
from conftest import HAS_GPU
from pixsfm._pixsfm import _bundle_adjustment as ba, _capi, _engine


def _solver_options(opts):
    return ba.solver_options_from(opts.loss, opts.solver, _capi.default_ba_options(use_inner_iterations=0))


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_oracle_geometric_ba_matches_scipy(name):
    """Where the gauge-fixed problem has an isolated minimum (every pose constant), the oracle's LM and scipy's land
    on it within 1e-4.  With a variable second pose and a free focal length the two-view cost keeps falling along
    focal length against depth, so there the solve must lower the cost and the GPU is held to the oracle's trajectory
    instead (tests/test_gpu_geometric_ba.py), as the reference holds its optimizer to COLMAP's."""
    rec, setup, opts = G.case(name)
    prob, _ = G.geometric_problem(rec, setup, opts)
    start = prob.copy()
    s = GO.ba_solve_geometric(prob, _solver_options(opts))
    assert s["final_cost"] < s["initial_cost"]
    assert s["num_residuals"] == 2 * prob.n_obs
    if not prob.pose_const.all():
        return
    ref = G.scipy_solve(start)
    G.assert_close_to((prob.cam_params, prob.qvec, prob.tvec, prob.xyz), ref)


def test_oracle_geometric_residual_and_jacobian():
    """r = WorldToImage(X) - keypoint, with the Jacobian of that projection (finite differences)"""
    from pixsfm.util.cameras import world_to_image
    rec, setup, opts = G.case("variable_image")
    prob, _ = G.geometric_problem(rec, setup, opts)
    so = _solver_options(opts)
    ev = GO.ba_evaluate_geometric(prob, so, residuals=True)
    r, J = GO.ba_block_jacobians_geometric(prob)
    for o in (0, 57, prob.n_obs - 1):
        i = int(prob.obs_img[o]); c = int(prob.img_cam[i])
        xy = world_to_image(2, prob.cam_params[c, :4], prob.qvec[i], prob.tvec[i], prob.xyz[prob.obs_pt[o]])[0]
        np.testing.assert_allclose(ev["residuals"][o], xy - prob.obs_xy[o], atol=1e-9)
        np.testing.assert_allclose(r[o], ev["residuals"][o], atol=0)
        X = prob.xyz[prob.obs_pt[o]].copy()
        for a in range(3):
            e = np.zeros(3); e[a] = 1e-6
            num = (world_to_image(2, prob.cam_params[c, :4], prob.qvec[i], prob.tvec[i], X + e)[0]
                   - world_to_image(2, prob.cam_params[c, :4], prob.qvec[i], prob.tvec[i], X - e)[0]) / 2e-6
            np.testing.assert_allclose(J[o, :, 7 + a], num, rtol=1e-5, atol=1e-4)
    np.testing.assert_array_equal(ev["gtr"], ev["residuals"])
    np.testing.assert_array_equal(ev["gtg"], np.tile([1.0, 0.0, 1.0], (prob.n_obs, 1)))
    assert abs(ev["cost"] - 0.5 * (ev["residuals"] ** 2).sum()) <= 1e-9 * ev["cost"]


# ---- the Python surface with the oracle standing in for the device ----------------------------------------------
def _ba_run_oracle(problem, interp=None, options=None, ctx=None, capacity=512):
    assert problem.obs_xy is not None
    out = GO.ba_solve_geometric(problem, options or _capi.default_ba_options())
    out.setdefault("num_residual_blocks", problem.n_obs)
    return out


@pytest.fixture
def oracle_device(monkeypatch):
    monkeypatch.setattr(_engine, "ba_run", _ba_run_oracle)
    yield


def _reprojection_error(rec):
    from pixsfm.util.cameras import world_to_image
    err = []
    for image in rec.images.values():
        cam = rec.cameras[image.camera_id]
        for p2 in image.points2D:
            if p2.has_point3D():
                xy = world_to_image(cam.model_id, cam.params, image.qvec, image.tvec, rec.points3D[p2.point3D_id].xyz)[0]
                err.append(np.linalg.norm(xy - p2.xy))
    return float(np.mean(err))


def test_geometric_adjuster_refines_and_writes_back(oracle_device):
    from pixsfm.bundle_adjustment.main import BundleAdjuster, GeometricBundleAdjuster
    rec = G.make_reconstruction(3, seed=4)
    rng = np.random.default_rng(1)
    for p in rec.points3D.values():
        p.xyz += rng.normal(0, 0.01, 3)
    before = _reprojection_error(rec)
    xyz0 = np.array([p.xyz.copy() for p in rec.points3D.values()])
    adjuster = BundleAdjuster.create({"strategy": "geometric"})
    assert isinstance(adjuster, GeometricBundleAdjuster)
    out = adjuster.refine(rec)
    s = out["summary"]
    assert s["final_cost"] < s["initial_cost"]
    assert _reprojection_error(rec) < before
    assert not np.array_equal(np.array([p.xyz for p in rec.points3D.values()]), xyz0)


def test_geometric_optimizer_surface(oracle_device):
    rec, setup, opts = G.case("two_view")
    opt = ba.GeometricBundleOptimizer(opts, setup)
    assert opt.run(rec)
    assert opt.problem.obs_xy.shape == (opt.problem.n_obs, 2)
    assert opt.summary()["num_residuals"] == 2 * opt.problem.n_obs
    with pytest.raises(ValueError):
        opt.run(rec)                       # one-shot, as BundleOptimizer
    opt.reset()
    assert opt.run(rec)


def test_refine_multilevel_honours_a_positional_setup(oracle_device):
    """refine_multilevel passes the setup positionally; the adjuster uses it (here: every pose constant)"""
    from pixsfm.bundle_adjustment.main import GeometricBundleAdjuster
    import types
    rec = G.make_reconstruction(2, seed=2)
    q0 = {i: im.qvec.copy() for i, im in rec.images.items()}
    t0 = {i: im.tvec.copy() for i, im in rec.images.items()}
    setup = ba.BundleAdjustmentSetup()
    setup.add_images([1, 2]); setup.set_constant_pose(1); setup.set_constant_pose(2)
    fm = types.SimpleNamespace(num_levels=2, fset=lambda level: None)
    out = GeometricBundleAdjuster({}).refine_multilevel(rec, fm, setup)
    assert len(out["summary"]) == 2
    for i, im in rec.images.items():
        np.testing.assert_array_equal(im.tvec, t0[i])
        np.testing.assert_allclose(im.qvec, q0[i] / np.linalg.norm(q0[i]), atol=0)


# ---- C-ABI argument checks (host side, no device needed) ---------------------------------------------------------
def _geo_desc():
    rec, setup, opts = G.case("two_view")
    prob, _ = G.geometric_problem(rec, setup, opts)
    return prob


def _create(lib, d, xy):
    h = C.c_void_p()
    so = _capi.default_ba_options()
    return lib.pxr_ba_create_geometric(None, C.byref(d), xy, C.byref(so), C.byref(h))


def _run(lib, d, xy):
    so = _capi.default_ba_options()
    s = _capi.make_summary(0)
    return lib.pxr_ba_run_geometric(None, C.byref(d), xy, C.byref(so), C.byref(s))


@pytest.mark.parametrize("call", [_create, _run])
def test_geometric_entry_points_reject_bad_arguments(call):
    lib = _capi.load_lib()
    prob = _geo_desc()
    d = prob.desc()
    assert call(lib, d, None) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert b"obs_xy" in lib.pxr_last_error()
    bad = prob.obs_xy.copy(); bad[5, 1] = np.nan
    assert call(lib, d, _capi.ptr(bad)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert b"finite" in lib.pxr_last_error()
    bad[5, 1] = np.inf
    assert call(lib, d, _capi.ptr(bad)) == _capi.PXR_ERR_INVALID_ARGUMENT
    patches = np.zeros((prob.n_obs, 4, 4, 3), np.float32)
    d2 = prob.desc(); d2.patches = patches.ctypes.data_as(C.c_void_p); d2.channels = 3; d2.ph = d2.pw = 4
    assert call(lib, d2, _capi.ptr(prob.obs_xy)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert b"no feature patches" in lib.pxr_last_error()
    d3 = prob.desc(); d3.channels = 128
    assert call(lib, d3, _capi.ptr(prob.obs_xy)) == _capi.PXR_ERR_INVALID_ARGUMENT
    refs = np.zeros((len(prob.xyz), 1))
    d4 = prob.desc(); d4.refs = refs.ctypes.data_as(C.c_void_p)
    assert call(lib, d4, _capi.ptr(prob.obs_xy)) == _capi.PXR_ERR_INVALID_ARGUMENT


@pytest.mark.skipif(HAS_GPU, reason="only meaningful on a box without a GPU")
@pytest.mark.parametrize("call", [_create, _run])
def test_geometric_entry_points_need_a_device(call):
    lib = _capi.load_lib()
    prob = _geo_desc()
    assert call(lib, prob.desc(), _capi.ptr(prob.obs_xy)) == _capi.PXR_ERR_NO_DEVICE
    assert b"no CPU fallback" in lib.pxr_last_error()


def test_memory_estimate_of_a_geometric_problem():
    prob = _geo_desc()
    need = _engine.ba_estimate_device_bytes(prob, _capi.default_ba_options())
    assert need["patches"] == 0
    assert need["state"] > 0 and need["reduced_system"] > 0
