"""An LM iteration with inner iterations evaluates each point once: the trial cost is reduced from inner-iteration
round 0's records (round 0 evaluates every observation at the trial point), and the pass after the rounds runs in
Jacobian mode into the alternate buffer set, so an accepted step adopts it as the next linearisation.  PXR_NO_SPECULATION
keeps separate cost-only passes and evaluates the accepted point again; it is the reference here.

Round 0 projects with the point-only K0 and the pass after the rounds with the Jacobian K0, where the separate trial
pass used the cost-only K0: all three must give the same uv (and xy) bits on every camera model."""
import numpy as np
import pytest

import dispatch_scenes as DS
import oracle_lib as O
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    """the 70 000-observation scene of test_gpu_inner_rounds.py"""
    prob, _ = synthetic.make_ba_scene(n_cams=40, n_points=7000, track_len=10, channels=128, ps=8, seed=1)
    prob.refs, _ = _engine.refs_compute(prob, _capi.default_interp())
    return prob


def _geometric(prob):
    g = _capi.BAProblem(prob.cam_model, prob.cam_params, prob.cam_const_mask, prob.qvec, prob.tvec, prob.img_cam,
                        prob.pose_const, prob.tvec_const_mask, prob.xyz, prob.point_const, prob.obs_img, prob.obs_pt,
                        None, None, None, obs_xy=np.zeros((prob.n_obs, 2)))
    g.obs_xy[:] = 100.0
    return g


@pytest.mark.parametrize("geometric", [False, True], ids=["featuremetric", "geometric"])
@pytest.mark.parametrize("model", range(7))
def test_cost_only_projection_matches_the_jacobian_projections(model, geometric):
    prob = DS._one_model(model, "f", 60 + model)
    prob.xyz += np.random.default_rng(model).normal(0, 0.01, prob.xyz.shape)
    if geometric:
        prob = _geometric(prob)
    h = _engine.BAHandle(prob, _capi.default_interp(), _capi.default_ba_options())
    cost_only, full = h.debug_project(False), h.debug_project(True)
    point = h.debug_project_point(np.arange(prob.n_obs))
    h.close()
    assert np.isfinite(cost_only["uv"]).all()
    np.testing.assert_array_equal(cost_only["uv"], full["uv"])
    np.testing.assert_array_equal(cost_only["xy"], full["xy"])
    np.testing.assert_array_equal(cost_only["uv"], point["uv"])
    np.testing.assert_array_equal(cost_only["uv"], point["uv_full"])


def _bits(s, p):
    its = [(i["cost"], i["cost_change"], i["step_norm"], i["relative_decrease"], i["trust_region_radius"],
            i["gradient_max_norm"], i["step_is_successful"], i["step_is_valid"]) for i in s["iterations"]]
    return its, s["num_inner_iteration_steps"], p.qvec.tobytes(), p.tvec.tobytes(), p.xyz.tobytes(), p.cam_params.tobytes()


def _solve(prob, so, monkeypatch, no_speculation):
    if no_speculation:
        monkeypatch.setenv("PXR_NO_SPECULATION", "1")
    else:
        monkeypatch.delenv("PXR_NO_SPECULATION", raising=False)
    p = prob.copy()
    s = _engine.ba_run(p, _capi.default_interp(), so)
    monkeypatch.delenv("PXR_NO_SPECULATION", raising=False)
    return s, p


@pytest.mark.parametrize("constant_points", [False, True], ids=["all_points_variable", "some_points_constant"])
def test_deterministic_solve_is_bit_identical_to_separate_passes(scene, monkeypatch, constant_points):
    prob = scene.copy()
    if constant_points:
        prob.point_const[::7] = 1
    so = _capi.default_ba_options(max_num_iterations=6, use_inner_iterations=1, deterministic=1)
    sa, pa = _solve(prob, so, monkeypatch, False)
    sb, pb = _solve(prob, so, monkeypatch, True)
    assert sa["num_inner_iteration_steps"] > 0
    assert _bits(sa, pa) == _bits(sb, pb)


def test_default_driver_follows_separate_passes(scene, monkeypatch):
    prob = scene.copy()
    prob.point_const[::11] = 1
    so = _capi.default_ba_options(max_num_iterations=8, use_inner_iterations=1)
    sa, pa = _solve(prob, so, monkeypatch, False)
    sb, pb = _solve(prob, so, monkeypatch, True)
    assert sa["num_inner_iteration_steps"] == sb["num_inner_iteration_steps"] > 0
    assert len(sa["iterations"]) == len(sb["iterations"])
    for x, y in zip(sa["iterations"], sb["iterations"]):
        assert x["step_is_successful"] == y["step_is_successful"] and x["step_is_valid"] == y["step_is_valid"]
        assert abs(x["cost"] - y["cost"]) <= 1e-6 * y["cost"]
    assert sa["iterations"][0]["cost"] == sb["iterations"][0]["cost"]
    assert abs(sa["final_cost"] - sb["final_cost"]) <= 1e-6 * sb["final_cost"]
    for k in ("xyz", "qvec", "tvec"):
        assert np.abs(getattr(pa, k) - getattr(pb, k)).max() < 1e-6, k


def test_windowed_run_matches_full_upload():
    """pxr_ba_run from pinned host patches with window residency: round 0's cost must come from the batch of rounds
    that reported no observation outside its window"""
    import os
    prob, _ = synthetic.make_ba_scene(n_cams=8, n_points=150, track_len=5, channels=128, seed=21)
    ic = _capi.default_interp()
    prob.refs, _ = O.refs_compute(prob, ic)
    so = _capi.default_ba_options(max_num_iterations=10, use_inner_iterations=1, deterministic=1)
    runs = []
    for window in (8, 0):
        pin = _engine.PinnedArray(prob.patches.shape, prob.patches.dtype)
        pin.array[...] = prob.patches
        q = prob.copy()
        q.patches = pin.array
        q._patches_ptr = pin.array.ctypes.data
        os.environ["PXR_RESIDENT_WINDOW"] = str(window)
        try:
            s = _engine.ba_run(q, ic, so)
        finally:
            os.environ.pop("PXR_RESIDENT_WINDOW", None)
        runs.append((s, _bits(s, q)))
        pin.close()
    (sw, bw), (sf, bf) = runs
    assert sw["resident_window"] == 8 and sf["resident_window"] == 0
    assert sw["num_inner_iteration_steps"] > 0
    assert bw == bf


def test_launches_fall_per_inner_iteration(scene, monkeypatch):
    """per LM iteration with inner iterations the separate trial pass (K0, K1 and the two-launch cost reduction) is
    gone, round 0 gains the reduction, and an accepted step no longer evaluates its point again (K0, K1, reduction).
    Without inner iterations only the latter differs, as it did before.
    The number of rounds depends on how far the host runs ahead of the device, so their three launches each are
    taken out before comparing."""
    so = _capi.default_ba_options(use_inner_iterations=1)

    def per_iteration(no_speculation):
        if no_speculation:
            monkeypatch.setenv("PXR_NO_SPECULATION", "1")
        h = _engine.BAHandle(scene.copy(), _capi.default_interp(), so)
        monkeypatch.delenv("PXR_NO_SPECULATION", raising=False)
        out, n_inner = [], 0
        for _ in range(6):
            s = h.iterate(1)
            ran_inner = s["num_inner_iteration_steps"] > n_inner
            n_inner = s["num_inner_iteration_steps"]
            rounds = len(h.debug_inner_rounds()[0]) if ran_inner else 0
            out.append((ran_inner, s["iterations"][-1]["step_is_successful"], s["kernel_launches"] - 3 * rounds))
        h.close()
        return out

    new, old = per_iteration(False), per_iteration(True)
    assert [r[:2] for r in new] == [r[:2] for r in old]
    assert any(r[0] and r[1] for r in new)
    for (ran_inner, accepted, n_new), (_, _, n_old) in zip(new, old):
        if not ran_inner:
            assert n_old - n_new == (4 if accepted else 0)   # the trial pass was already the linearisation
        elif accepted:
            assert n_old - n_new == 6      # -4 trial pass, -4 evaluation of the accepted point, +2 round 0's reduction
        else:
            assert n_old - n_new == 2      # -4 trial pass, +2 round 0's reduction
