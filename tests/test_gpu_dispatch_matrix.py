"""GPU parity over the assembly dispatch space: every scene of dispatch_scenes.SCENES under every row of its switch
matrices, against the CPU oracle and against the default GPU path.  test_dispatch_coverage.py checks on the CPU that
these rows reach every kernel the host can select."""
import ctypes as C

import numpy as np
import pytest

import dispatch_scenes as D
import oracle_lib as O
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

RADIUS = 1e3
_cache = {}


def _scene(name):
    if name not in _cache:
        ic = _capi.default_interp()
        prob = D.with_refs(D.SCENES[name](), ic)
        _cache[name] = (prob, ic)
    prob, ic = _cache[name]
    return prob.copy(), ic


def _cached(key, fn):
    if key not in _cache:
        _cache[key] = fn()
    return _cache[key]


def _set_env(monkeypatch, env):
    for k in ("PXR_SCHUR_KERNEL", "PXR_SCHUR_CTAS", "PXR_BUILD_ATOMIC", "PXR_BUILD_UNSTAGED", "PXR_PROJECT_UNSTAGED",
              "PXR_PCG_SPARSE", "PXR_BLOCK_ASSEMBLY", "PXR_NO_SPECULATION"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _oracle_lin(name, so_kw=()):
    def run():
        prob, ic = _scene(name)
        return O.ba_linearize(prob, ic, _capi.default_ba_options(use_inner_iterations=0, **dict(so_kw)), radius=RADIUS)
    return _cached(("oracle_lin", name, so_kw), run)


def _gpu_lin(name, dense=True, so_kw=()):
    prob, ic = _scene(name)
    ref = _oracle_lin(name, so_kw)
    h = _engine.BAHandle(prob, ic, _capi.default_ba_options(use_inner_iterations=0, **dict(so_kw)))
    return h.debug_linearize(ref["nc"], ref["nl"], radius=RADIUS, dense=dense)


def _close(got, ref, rtol, atol_rel):
    return np.allclose(got, ref, rtol=rtol, atol=atol_rel * np.abs(ref).max())


def _solve(name, runner, so):
    """(summary, refined problem) of a full solve of a catalogue scene"""
    p, ic = _scene(name)
    return runner(p, ic, so), p


def _compare_solutions(a, b, tol):
    for k in ("qvec", "tvec", "xyz"):
        assert np.abs(getattr(a, k) - getattr(b, k)).max() < tol, k
    assert (np.abs(a.cam_params - b.cam_params) / np.maximum(np.abs(b.cam_params), 1.0)).max() < tol


def _default_gpu_lin(name, monkeypatch):
    def run():
        _set_env(monkeypatch, {})
        return _gpu_lin(name)
    return _cached(("gpu_default", name), run)


@pytest.mark.parametrize("env", D.DENSE_ENVS, ids=D.env_id)
@pytest.mark.parametrize("name", list(D.SCENES))
def test_dense_assembly_matches_oracle_and_default_path(name, env, monkeypatch):
    ref = _oracle_lin(name)
    base = _default_gpu_lin(name, monkeypatch)
    _set_env(monkeypatch, env)
    got = _gpu_lin(name)
    tril = np.tril
    assert abs(got["cost"] - ref["cost"]) <= 1e-11 * ref["cost"]
    sc, ss = np.abs(ref["Hcc"]).max(), np.abs(ref["S"]).max()
    assert np.abs(tril(got["Hcc"]) - tril(ref["Hcc"])).max() <= 1e-9 * sc
    assert _close(got["gc"], ref["gc"], 1e-7, 1e-9)
    assert _close(got["Hpp"], ref["Hpp"], 1e-9, 1e-10)
    assert _close(got["gp"], ref["gp"], 1e-7, 1e-9)
    assert np.abs(tril(got["S"]) - tril(ref["S"])).max() <= 1e-9 * ss
    assert _close(got["rhs"], ref["rhs"], 1e-7, 1e-9)
    assert _close(got["delta"], ref["delta"], 1e-4, 1e-7)
    assert abs(got["model_cost_change"] - ref["model_cost_change"]) <= 1e-7 * abs(ref["model_cost_change"])
    # against the default kernels: the same sums in another order
    sb = np.abs(base["S"]).max()
    assert np.abs(tril(got["S"]) - tril(base["S"])).max() <= 1e-11 * sb
    assert np.abs(tril(got["Hcc"]) - tril(base["Hcc"])).max() <= 1e-11 * np.abs(base["Hcc"]).max()
    assert np.abs(got["gc"] - base["gc"]).max() <= 1e-11 * np.abs(base["gc"]).max()
    assert np.abs(got["rhs"] - base["rhs"]).max() <= 1e-11 * np.abs(base["rhs"]).max()
    assert np.abs(got["delta"] - base["delta"]).max() <= 1e-8 * np.abs(base["delta"]).max()


# LM iterations whose PCG trajectory is compared.  From its third iteration on, mixed_dc8's reduced system needs 24 CG
# iterations for 36 unknowns: there the inexact step moves with the summation order (the dense PCG path with one-CTA and
# with multi-CTA vector kernels ends 1.5e-4 apart in the poses and 2 CG iterations apart, as far as the dense path is
# from the oracle), so only its well-conditioned start is compared.
PCG_ITERATIONS = {"mixed_dc8": 2}


def _trajectory(s):
    return [(i["step_is_successful"], i["linear_solver_iterations"]) for i in s["iterations"][1:]]


@pytest.mark.parametrize("env", D.SPARSE_ENVS, ids=D.env_id)
@pytest.mark.parametrize("name", D.SPARSE_SCENES)
def test_block_sparse_assembly_matches_dense_and_oracle(name, env, monkeypatch):
    """the image-pair-block sink: ITERATIVE_SCHUR with PXR_PCG_SPARSE (compared with the dense PCG path and the oracle's
    PCG), and block mode with the exact solver (compared with the dense exact path and the oracle's step)"""
    pcg = "PXR_PCG_SPARSE" in env
    so_kw = (("linear_solver", 3),) if pcg else ()
    ref = _oracle_lin(name, so_kw)
    dense = _cached(("gpu_dense", name, so_kw), lambda: (_set_env(monkeypatch, {}), _gpu_lin(name, so_kw=so_kw))[1])
    _set_env(monkeypatch, env)
    got = _gpu_lin(name, dense=False, so_kw=so_kw)
    assert abs(got["cost"] - dense["cost"]) <= 1e-13 * dense["cost"]
    assert np.abs(got["gc"] - dense["gc"]).max() <= 1e-10 * np.abs(dense["gc"]).max()
    assert _close(got["gc"], ref["gc"], 1e-7, 1e-9)
    assert _close(got["gp"], ref["gp"], 1e-7, 1e-9)
    if pcg:    # inexact steps: the CG recurrences agree, not the rounding of every iterate
        assert np.abs(got["delta"] - dense["delta"]).max() <= 1e-6 * np.abs(dense["delta"]).max()
        assert np.abs(got["delta"] - ref["delta"]).max() <= 1e-4 * np.abs(ref["delta"]).max()
    else:
        assert np.abs(got["delta"] - dense["delta"]).max() <= 1e-9 * np.abs(dense["delta"]).max()
        assert _close(got["delta"], ref["delta"], 1e-4, 1e-7)
        assert abs(got["model_cost_change"] - dense["model_cost_change"]) <= 1e-10 * abs(dense["model_cost_change"])
    # the LM trajectory (with the block-diagonal preconditioner on the PCG path)
    iters = PCG_ITERATIONS.get(name, 6) if pcg else 6
    so = _capi.default_ba_options(use_inner_iterations=0, max_num_iterations=iters, **dict(so_kw))
    s_ref, p_ref = _cached(("oracle_solve", name, so_kw), lambda: _solve(name, O.ba_solve, so))
    s_dense, p_dense = _cached(("gpu_solve", name, so_kw),
                               lambda: (_set_env(monkeypatch, {}), _solve(name, _engine.ba_run, so))[1])
    _set_env(monkeypatch, env)
    s_got, p_got = _solve(name, _engine.ba_run, so)
    assert len(s_got["iterations"]) == len(s_dense["iterations"]) == len(s_ref["iterations"])
    for a, b in zip(_trajectory(s_got), _trajectory(s_dense)):
        assert a[0] == b[0] and abs(a[1] - b[1]) <= 2, (_trajectory(s_got), _trajectory(s_dense))
    assert abs(s_got["final_cost"] - s_dense["final_cost"]) <= 1e-6 * s_dense["final_cost"]
    assert abs(s_got["final_cost"] - s_ref["final_cost"]) <= 1e-5 * s_ref["final_cost"]
    _compare_solutions(p_got, p_dense, 1e-5 if pcg else 1e-9)
    _compare_solutions(p_got, p_ref, 1e-4 if pcg else 1e-6)


@pytest.mark.parametrize("name", ["dup_obs", "multi_chunk", "mixed_dc8"])
def test_full_solve_with_inner_iterations_matches_oracle(name, monkeypatch):
    """the whole LM loop, inner iterations included, on the scenes whose pair structure is unusual"""
    _set_env(monkeypatch, {})
    so = _capi.default_ba_options(use_inner_iterations=1, max_num_iterations=10)
    s_ref, p_ref = _cached(("oracle_full", name), lambda: _solve(name, O.ba_solve, so))
    s_gpu, p_gpu = _solve(name, _engine.ba_run, so)
    assert s_gpu["num_iterations"] == s_ref["num_iterations"]
    assert s_gpu["num_inner_iteration_steps"] > 0
    assert abs(s_gpu["initial_cost"] - s_ref["initial_cost"]) <= 1e-10 * s_ref["initial_cost"]
    for ig, ir in zip(s_gpu["iterations"], s_ref["iterations"]):
        assert ig["step_is_successful"] == ir["step_is_successful"]
        assert abs(ig["cost"] - ir["cost"]) <= 1e-6 * abs(ir["cost"])
    _compare_solutions(p_gpu, p_ref, 1e-6)


def test_inner_iterations_on_duplicate_observations(monkeypatch):
    """one coordinate-descent pass over the points when a point has two observations in one image"""
    prob, ic = _scene("dup_obs")
    prob.xyz += np.random.default_rng(6).normal(0, 0.004, prob.xyz.shape)
    so = _capi.default_ba_options(use_inner_iterations=1)
    p_ref = prob.copy()
    O.lib().orc_ba_inner_iterations(C.byref(p_ref.desc()), C.byref(ic), C.byref(so))
    assert np.abs(p_ref.xyz - prob.xyz).max() > 1e-5
    _set_env(monkeypatch, {})
    h = _engine.BAHandle(prob.copy(), ic, so)
    h.debug_inner_iterations()
    h.read_params()
    assert np.abs(h.problem.xyz - p_ref.xyz).max() < 1e-7


def _rejecting_scene():
    # large start perturbation and trust region, intrinsics constant: after ten accepted steps the oracle rejects two
    # (each would raise the cost by 0.14)
    prob, _ = synthetic.make_ba_scene(n_cams=5, n_points=40, track_len=4, channels=16, seed=1, dtype=np.float32,
                                      rot_sigma_deg=0.3, t_sigma=0.03, pt_sigma=0.05, refine_focal=False,
                                      refine_extra=False)
    ic = _capi.default_interp()
    return D.with_refs(prob, ic), ic


def test_speculative_jacobian_keeps_the_trajectory(monkeypatch):
    """The default driver evaluates the Jacobian at the trial point before it knows whether the step is accepted
    (and drops it on rejection).  With PXR_NO_SPECULATION=1 it does not; both must walk the oracle's trajectory."""
    prob, ic = _rejecting_scene()
    so = _capi.default_ba_options(use_inner_iterations=0, max_num_iterations=12, initial_trust_region_radius=1e8)
    p_ref, p_spec, p_plain = prob.copy(), prob.copy(), prob.copy()
    s_ref = O.ba_solve(p_ref, ic, so)
    _set_env(monkeypatch, {})
    s_spec = _engine.ba_run(p_spec, ic, so)
    _set_env(monkeypatch, {"PXR_NO_SPECULATION": "1"})
    s_plain = _engine.ba_run(p_plain, ic, so)
    ok = [i["step_is_successful"] for i in s_ref["iterations"][1:]]
    assert 0 in ok[ok.index(1):], ok          # a rejected step after an accepted one
    assert len(s_spec["iterations"]) == len(s_plain["iterations"]) == len(s_ref["iterations"])
    for a, b, r in zip(s_spec["iterations"], s_plain["iterations"], s_ref["iterations"]):
        assert a["step_is_successful"] == b["step_is_successful"] == r["step_is_successful"]
        assert abs(a["cost"] - b["cost"]) <= 1e-10 * abs(b["cost"])
        assert abs(a["cost"] - r["cost"]) <= 1e-6 * abs(r["cost"])
    _compare_solutions(p_spec, p_plain, 1e-9)
    _compare_solutions(p_spec, p_ref, 1e-6)
