"""Geometric (reprojection-error) bundle adjustment on the GPU against the CPU oracle: residual blocks and Jacobian
factors for every camera model, the normal equations / Schur system / step under every loss (also on every scene of
the dispatch catalogue, so the assembly kernels run on geometric records), full LM trajectories through every linear
solver, block mode and the inner iterations, and the Python surface (GeometricBundleOptimizer, the adjuster)."""
import numpy as np
import pytest

import dispatch_scenes as DS
import geo_scenes as G
import geo_oracle_lib as GO
from pixsfm._pixsfm import _bundle_adjustment as ba, _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu


def geometric(prob, seed=0, noise=0.5):
    """the same geometry and observations as a geometric problem: keypoints = projections + seeded N(0, noise) px"""
    g = _capi.BAProblem(prob.cam_model, prob.cam_params, prob.cam_const_mask, prob.qvec, prob.tvec, prob.img_cam,
                        prob.pose_const, prob.tvec_const_mask, prob.xyz, prob.point_const, prob.obs_img, prob.obs_pt,
                        None, None, None, obs_xy=np.zeros((prob.n_obs, 2)))
    xy = GO.ba_evaluate_geometric(g, _capi.default_ba_options())["xy"]
    g.obs_xy[:] = xy + np.random.default_rng(seed).normal(0, noise, xy.shape)
    return g


def _scene(**kw):
    args = dict(n_cams=6, n_points=60, track_len=4, channels=4, seed=0)
    args.update(kw)
    prob, _ = synthetic.make_ba_scene(**args)
    return geometric(prob, seed=args["seed"])


def _pose_mix(prob):
    """image 0 constant pose, image 1 a partial tvec mask: constant-pose and variable-pose residual blocks"""
    prob.pose_const[:] = 0; prob.pose_const[0] = 1
    prob.tvec_const_mask[:] = 0; prob.tvec_const_mask[1] = 1
    return prob


@pytest.mark.parametrize("model", range(7))
def test_residual_blocks_and_jacobians_match_oracle(model):
    prob = _pose_mix(geometric(DS._one_model(model, "f", 40 + model), seed=model))
    so = _capi.default_ba_options(use_inner_iterations=0, loss_type=0)
    ref = GO.ba_evaluate_geometric(prob, so, residuals=True)
    h = _engine.BAHandle(prob, options=so)
    got = h.evaluate(residuals=True)
    np.testing.assert_allclose(got["xy"], ref["xy"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(got["residuals"], ref["residuals"], rtol=0, atol=1e-9)
    np.testing.assert_array_equal(got["gtr"], got["residuals"])
    np.testing.assert_array_equal(got["gtg"], np.tile([1.0, 0.0, 1.0], (prob.n_obs, 1)))
    np.testing.assert_allclose(got["sq_norm"], ref["sq_norm"], rtol=1e-9, atol=1e-12)
    assert abs(got["cost"] - ref["cost"]) <= 1e-10 * ref["cost"]
    jac = h.evaluate_jacobians()
    np.testing.assert_array_equal(jac["grad"], np.tile(np.eye(2), (prob.n_obs, 1, 1)))
    np.testing.assert_array_equal(jac["residuals"], got["residuals"])
    # J = juv against the Jets of the oracle: point and intrinsics columns directly, the rotation through the tangent
    r_ref, J_ref = GO.ba_block_jacobians_geometric(prob)
    K = _capi.CAMERA_NUM_PARAMS[model]
    P = jac["juv"]
    scale = np.abs(J_ref).max()
    assert np.abs(P[:, :, 6:9] - J_ref[:, :, 7:10]).max() <= 1e-9 * scale
    assert np.abs(P[:, :, 9:9 + K] - J_ref[:, :, 10:10 + K]).max() <= 1e-9 * scale
    assert np.abs(P[:, :, 3:6] - J_ref[:, :, 4:7]).max() <= 1e-9 * scale


def _compare_linearization(got, ref):
    tril = np.tril
    assert abs(got["cost"] - ref["cost"]) <= 1e-11 * ref["cost"]
    if "Hcc" in got:
        assert np.abs(tril(got["Hcc"]) - tril(ref["Hcc"])).max() <= 1e-10 * np.abs(ref["Hcc"]).max()
        assert np.abs(tril(got["S"]) - tril(ref["S"])).max() <= 1e-9 * np.abs(ref["S"]).max()
        assert np.allclose(got["rhs"], ref["rhs"], rtol=1e-7, atol=1e-9 * np.abs(ref["rhs"]).max())
    assert np.allclose(got["gc"], ref["gc"], rtol=1e-8, atol=1e-10 * np.abs(ref["gc"]).max())
    assert np.allclose(got["Hpp"], ref["Hpp"], rtol=1e-9, atol=1e-10 * np.abs(ref["Hpp"]).max())
    assert np.allclose(got["gp"], ref["gp"], rtol=1e-8, atol=1e-10 * np.abs(ref["gp"]).max())
    assert np.allclose(got["delta"], ref["delta"], rtol=1e-5, atol=1e-8 * np.abs(ref["delta"]).max())
    assert abs(got["model_cost_change"] - ref["model_cost_change"]) <= 1e-7 * abs(ref["model_cost_change"])


@pytest.mark.parametrize("loss", ["trivial", "cauchy", "huber", "soft_l1", "arctan"])
def test_normal_equations_schur_and_step_match_oracle(loss):
    prob = _pose_mix(_scene())
    so = _capi.default_ba_options(use_inner_iterations=0, loss_type=_capi.LOSS_IDS[loss], loss_scale=0.5)
    ref = GO.ba_linearize_geometric(prob, so, radius=1e4)
    got = _engine.BAHandle(prob, options=so).debug_linearize(ref["nc"], ref["nl"], radius=1e4)
    _compare_linearization(got, ref)


@pytest.mark.parametrize("name", sorted(DS.SCENES))
def test_dispatch_scenes_as_geometric_problems(name):
    prob = geometric(DS.SCENES[name](), seed=7)
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = GO.ba_linearize_geometric(prob, so, radius=1e4)
    got = _engine.BAHandle(prob, options=so).debug_linearize(ref["nc"], ref["nl"], radius=1e4)
    _compare_linearization(got, ref)


def _check_trajectory(s_gpu, s_ref, p_gpu, p_ref, cost_tol=1e-6, param_tol=1e-4):
    assert s_gpu["num_iterations"] == s_ref["num_iterations"]
    assert s_gpu["num_residuals"] == s_ref["num_residuals"]
    assert abs(s_gpu["initial_cost"] - s_ref["initial_cost"]) <= 1e-10 * s_ref["initial_cost"]
    for ig, ir in zip(s_gpu["iterations"], s_ref["iterations"]):
        assert ig["step_is_successful"] == ir["step_is_successful"]
        assert abs(ig["cost"] - ir["cost"]) <= cost_tol * abs(ir["cost"])
    assert s_gpu["num_inner_iteration_steps"] == s_ref["num_inner_iteration_steps"]
    for a in ("qvec", "tvec", "xyz"):
        assert np.abs(getattr(p_gpu, a) - getattr(p_ref, a)).max() < param_tol
    assert np.abs(p_gpu.cam_params[:, 0] / p_ref.cam_params[:, 0] - 1).max() < param_tol
    assert np.abs(p_gpu.cam_params[:, 1:] - p_ref.cam_params[:, 1:]).max() < param_tol


@pytest.mark.parametrize("inner", [0, 1])
@pytest.mark.parametrize("variant", ["dense", "iterative", "pcg_sparse", "block"])
def test_full_solve_follows_oracle(inner, variant, monkeypatch):
    prob = _pose_mix(_scene(n_points=80))
    so = _capi.default_ba_options(use_inner_iterations=inner, max_num_iterations=15,
                                  linear_solver=3 if variant in ("iterative", "pcg_sparse") else 1)
    if variant == "pcg_sparse":
        monkeypatch.setenv("PXR_PCG_SPARSE", "1")
    if variant == "block":
        monkeypatch.setenv("PXR_BLOCK_ASSEMBLY", "1")
    p_gpu, p_ref = prob.copy(), prob.copy()
    s_gpu = _engine.ba_run(p_gpu, options=so)
    s_ref = GO.ba_solve_geometric(p_ref, so)
    exact = variant in ("dense", "block")
    _check_trajectory(s_gpu, s_ref, p_gpu, p_ref, cost_tol=1e-6 if exact else 1e-4)
    assert s_gpu["kernel_launches"] > 0
    assert s_gpu["final_cost"] < s_gpu["initial_cost"]


def test_inner_iterations_match_oracle_points():
    prob = _scene(n_points=80)
    so = _capi.default_ba_options(use_inner_iterations=1)
    p_ref = prob.copy()
    GO.ba_inner_iterations_geometric(p_ref, so)
    h = _engine.BAHandle(prob.copy(), options=so)
    h.debug_inner_iterations()
    h.read_params()
    assert np.abs(h.problem.xyz - p_ref.xyz).max() < 1e-7
    assert np.abs(p_ref.xyz - prob.xyz).max() > 1e-5


def test_eval_list_matches_full_range_records():
    prob = _scene(n_points=60)
    h = _engine.BAHandle(prob, options=_capi.default_ba_options())
    full = h.debug_eval_list(np.arange(prob.n_obs))
    items = np.arange(0, prob.n_obs, 3)
    for on_dev in (False, True):
        got = h.debug_eval_list(items, count_on_device=on_dev)
        np.testing.assert_array_equal(got[items, :6], full[items, :6])
        assert np.isnan(got[1, 0])


def test_deterministic_runs_are_bit_identical():
    prob = _scene(n_points=80)
    so = _capi.default_ba_options(use_inner_iterations=1, max_num_iterations=10, deterministic=1)
    a, b = prob.copy(), prob.copy()
    sa = _engine.ba_run(a, options=so)
    sb = _engine.ba_run(b, options=so)
    assert [i["cost"] for i in sa["iterations"]] == [i["cost"] for i in sb["iterations"]]
    for k in ("cam_params", "qvec", "tvec", "xyz"):
        np.testing.assert_array_equal(getattr(a, k), getattr(b, k))


def test_handle_reset_and_time_stage():
    prob = _scene(n_points=60)
    so = _capi.default_ba_options(use_inner_iterations=0)
    h = _engine.BAHandle(prob.copy(), options=so)
    s1 = h.iterate(3)
    h.reset(prob.cam_params, prob.qvec, prob.tvec, prob.xyz)
    s2 = h.iterate(3)
    assert [i["cost"] for i in s1["iterations"]] == [i["cost"] for i in s2["iterations"]]
    assert h.time_stage(0, 2) > 0 and h.time_stage(3, 2) > 0
    h.kernel_timing(enable=1)
    h.iterate(2)
    ms, n = h.kernel_timing(which=1)
    assert n > 0 and ms > 0


@pytest.mark.parametrize("name", sorted(G.CASES))
def test_reference_cases_through_the_optimizer_match_oracle(name):
    rec, setup, opts = G.case(name)
    prob, _ = G.geometric_problem(rec, setup, opts)
    so = ba.solver_options_from(opts.loss, opts.solver, _capi.default_ba_options(use_inner_iterations=0))
    s_ref = GO.ba_solve_geometric(prob, so)
    opt = ba.GeometricBundleOptimizer(opts, setup)
    assert opt.run(rec)
    # the reference's BA-vs-BA tolerance (bundle_optimizer_test.cc): 1e-4, relative for the focal lengths.  A few
    # two-view points end far out on their rays, where the cost is flat along the ray: 99% of the points are held to
    # 1e-4, and the final costs to 1e-8
    g = opt.problem
    assert abs(opt.summary()["final_cost"] - s_ref["final_cost"]) <= 1e-8 * s_ref["final_cost"]
    assert np.abs(g.cam_params[:, 0] / prob.cam_params[:, 0] - 1).max() < 1e-4
    assert np.abs(g.cam_params[:, 1:] - prob.cam_params[:, 1:]).max() < 1e-4
    for a in ("qvec", "tvec"):
        assert np.abs(getattr(g, a) - getattr(prob, a)).max() < 1e-4
    assert np.mean(np.abs(g.xyz - prob.xyz).max(axis=1) < 1e-4) >= 0.99
    image = rec.images[2]
    k = list(opt._ir.image_ids).index(2)
    np.testing.assert_array_equal(image.tvec, opt.problem.tvec[k])


def test_refine_multilevel_returns_one_summary_per_level():
    import types
    from pixsfm.bundle_adjustment.main import BundleAdjuster
    rec = G.make_reconstruction(3, seed=5)
    fm = types.SimpleNamespace(num_levels=2, fset=lambda level: None)
    out = BundleAdjuster.create({"strategy": "geometric"}).refine_multilevel(rec, fm)
    assert len(out["summary"]) == 2
    assert out["summary"][1]["final_cost"] <= out["summary"][0]["initial_cost"]
