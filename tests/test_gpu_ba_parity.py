"""GPU parity: the CUDA path (through the C-ABI of libpxr.so) against the CPU oracle on the same
seeded inputs.  Tolerances: the reference's own SIMD-vs-Ceres tolerance is 1e-5 on f/df
(interpolation_test.cc:352-354); because the kernels reproduce the reference's per-channel
operation order, much tighter bounds hold and are asserted here."""
import numpy as np
import pytest

import oracle_lib as O
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu


def _scene(**kw):
    args = dict(n_cams=6, n_points=60, track_len=4, channels=128, seed=0)
    args.update(kw)
    prob, gt = synthetic.make_ba_scene(**args)
    ic = _capi.default_interp()
    refs, _ = O.refs_compute(prob, ic)
    prob.refs = refs
    return prob, gt, ic


@pytest.mark.parametrize("channels,dtype", [(128, np.float16), (64, np.float16), (16, np.float16),
                                            (128, np.float32), (16, np.float64), (128, np.float64)])
def test_residual_blocks_match_oracle(channels, dtype):
    prob, gt, ic = _scene(channels=channels, dtype=dtype, n_points=40)
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_evaluate(prob, ic, so, residuals=True)
    h = _engine.BAHandle(prob, ic, so)
    got = h.evaluate(residuals=True)
    assert np.allclose(got["xy"], ref["xy"], rtol=0, atol=1e-9)
    assert np.abs(got["residuals"] - ref["residuals"]).max() < 1e-12
    assert np.allclose(got["sq_norm"], ref["sq_norm"], rtol=1e-10, atol=1e-15)
    assert np.allclose(got["gtr"], ref["gtr"], rtol=1e-9, atol=1e-13)
    assert np.allclose(got["gtg"], ref["gtg"], rtol=1e-10, atol=1e-14)
    assert abs(got["cost"] - ref["cost"]) <= 1e-11 * abs(ref["cost"])


def test_float_simd_mode_and_no_l2():
    prob, gt, _ = _scene(n_points=30)
    for l2, fs in ((True, True), (False, False), (False, True)):
        ic = _capi.default_interp(l2_normalize=l2, use_float_simd=fs)
        so = _capi.default_ba_options(use_inner_iterations=0)
        ref = O.ba_evaluate(prob, ic, so, residuals=True)
        got = _engine.BAHandle(prob, ic, so).evaluate(residuals=True)
        assert np.abs(got["residuals"] - ref["residuals"]).max() < 1e-12
        assert np.allclose(got["gtg"], ref["gtg"], rtol=1e-9, atol=1e-13)


def test_border_clamp_matches_oracle():
    # push projections to and beyond the patch border: per-tap clamp path (grid2d.h:29-35)
    prob, gt, ic = _scene(n_points=40)
    rng = np.random.default_rng(1)
    prob.corner[:] += rng.integers(-9, 10, prob.corner.shape).astype(np.int32)
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_evaluate(prob, ic, so, residuals=True)
    got = _engine.BAHandle(prob, ic, so).evaluate(residuals=True)
    assert np.abs(got["residuals"] - ref["residuals"]).max() < 1e-12
    assert np.allclose(got["gtr"], ref["gtr"], rtol=1e-9, atol=1e-13)


@pytest.mark.parametrize("shared_camera", [False, True])
def test_normal_equations_schur_and_step_match_oracle(shared_camera):
    prob, gt, ic = _scene(shared_camera=shared_camera)
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_linearize(prob, ic, so, radius=1e4)
    h = _engine.BAHandle(prob, ic, so)
    got = h.debug_linearize(ref["nc"], ref["nl"], radius=1e4)
    tril = lambda M: np.tril(M)
    assert abs(got["cost"] - ref["cost"]) <= 1e-11 * ref["cost"]
    scale = np.abs(ref["Hcc"]).max()
    assert np.abs(tril(got["Hcc"]) - tril(ref["Hcc"])).max() <= 1e-10 * scale
    assert np.allclose(got["gc"], ref["gc"], rtol=1e-8, atol=1e-10 * np.abs(ref["gc"]).max())
    assert np.allclose(got["Hpp"], ref["Hpp"], rtol=1e-9, atol=1e-10 * np.abs(ref["Hpp"]).max())
    assert np.allclose(got["gp"], ref["gp"], rtol=1e-8, atol=1e-10 * np.abs(ref["gp"]).max())
    assert np.abs(tril(got["S"]) - tril(ref["S"])).max() <= 1e-9 * np.abs(ref["S"]).max()
    assert np.allclose(got["rhs"], ref["rhs"], rtol=1e-7, atol=1e-9 * np.abs(ref["rhs"]).max())
    assert np.allclose(got["delta"], ref["delta"], rtol=1e-5, atol=1e-8 * np.abs(ref["delta"]).max())
    assert abs(got["model_cost_change"] - ref["model_cost_change"]) <= 1e-7 * abs(ref["model_cost_change"])


def test_constant_blocks_and_partial_masks():
    prob, gt, ic = _scene(n_cams=7, n_points=50, refine_pp=True)
    prob.point_const[::7] = 1
    prob.pose_const[3] = 1
    prob.tvec_const_mask[4] = 0b101
    prob.cam_const_mask[2] = 0xFFFFFFFF
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_linearize(prob, ic, so, radius=3e3)
    got = _engine.BAHandle(prob, ic, so).debug_linearize(ref["nc"], ref["nl"], radius=3e3)
    assert np.allclose(got["delta"], ref["delta"], rtol=1e-5, atol=1e-8 * np.abs(ref["delta"]).max())
    assert abs(got["model_cost_change"] - ref["model_cost_change"]) <= 1e-7 * abs(ref["model_cost_change"])


def _compare_solutions(a, b, tol):
    assert np.abs(a.qvec - b.qvec).max() < tol
    assert np.abs(a.tvec - b.tvec).max() < tol
    assert np.abs(a.xyz - b.xyz).max() < tol
    assert np.abs(a.cam_params[:, 1:] - b.cam_params[:, 1:]).max() < tol
    assert np.abs(a.cam_params[:, 0] / b.cam_params[:, 0] - 1).max() < tol


@pytest.mark.parametrize("inner", [0, 1])
def test_full_solve_matches_oracle(inner):
    prob, gt, ic = _scene()
    so = _capi.default_ba_options(use_inner_iterations=inner, max_num_iterations=15)
    p_ref = prob.copy(); p_gpu = prob.copy()
    s_ref = O.ba_solve(p_ref, ic, so)
    s_gpu = _engine.ba_run(p_gpu, ic, so)
    assert s_gpu["num_iterations"] == s_ref["num_iterations"]
    assert abs(s_gpu["initial_cost"] - s_ref["initial_cost"]) <= 1e-10 * s_ref["initial_cost"]
    assert abs(s_gpu["final_cost"] - s_ref["final_cost"]) <= 1e-6 * s_ref["final_cost"]
    for ig, ir in zip(s_gpu["iterations"], s_ref["iterations"]):
        assert ig["step_is_successful"] == ir["step_is_successful"]
        assert abs(ig["cost"] - ir["cost"]) <= 1e-6 * abs(ir["cost"])
    # the reference's own parameter tolerance for BA-vs-BA comparisons is 1e-4 (bundle_optimizer_test.cc:52)
    _compare_solutions(p_gpu, p_ref, 1e-6)
    assert s_gpu["kernel_launches"] > 0


def test_inner_iterations_kernel_matches_oracle_points():
    prob, gt, ic = _scene(n_points=30)
    prob.xyz += np.random.default_rng(5).normal(0, 0.004, prob.xyz.shape)
    so = _capi.default_ba_options(use_inner_iterations=1)
    h = _engine.BAHandle(prob.copy(), ic, so)
    h.debug_inner_iterations()
    h.read_params()
    # oracle: run ONLY the point coordinate descent = BA with everything but points constant, via
    # the public solve with max_num_iterations=0 is not possible; use the dedicated hook
    import ctypes as C
    p_ref = prob.copy()
    d = p_ref.desc()
    O.lib().orc_ba_inner_iterations(C.byref(d), C.byref(ic), C.byref(so))
    assert np.abs(h.problem.xyz - p_ref.xyz).max() < 1e-7
    assert np.abs(p_ref.xyz - prob.xyz).max() > 1e-5  # the points did move


def test_unsupported_channels_raise_value_error():
    prob, gt, ic = _scene(channels=16, n_points=10)
    bad = prob.copy()
    # 1/3/4 (cost maps) and 8..256 are built; anything else is refused like feature_reference_bundle_optimizer.h:12-18
    bad.patches = np.ascontiguousarray(prob.patches[..., :5])
    bad._patches_ptr = bad.patches.ctypes.data
    bad.channels = 5
    bad.refs = np.ascontiguousarray(prob.refs[:, :5])
    with pytest.raises(ValueError):
        _engine.BAHandle(bad, ic, _capi.default_ba_options())


def test_iterative_schur_pcg_matches_oracle():
    """ITERATIVE_SCHUR (bundle_optimizer.h:181-191 picks it above 1000 images): block-Jacobi PCG on the reduced
    camera system, Ceres' Q-based termination. Inexact steps -> compare at the reference's own 1e-4 BA tolerance."""
    prob, gt, ic = _scene()
    so = _capi.default_ba_options(use_inner_iterations=0, max_num_iterations=12, linear_solver=3)
    p_ref = prob.copy(); p_gpu = prob.copy()
    s_ref = O.ba_solve(p_ref, ic, so)
    s_gpu = _engine.ba_run(p_gpu, ic, so)
    assert abs(s_gpu["initial_cost"] - s_ref["initial_cost"]) <= 1e-10 * s_ref["initial_cost"]
    assert abs(s_gpu["final_cost"] - s_ref["final_cost"]) <= 1e-5 * s_ref["final_cost"]
    it_g = [i["linear_solver_iterations"] for i in s_gpu["iterations"][1:]]
    it_r = [i["linear_solver_iterations"] for i in s_ref["iterations"][1:]]
    assert min(it_g) >= 1 and len(it_g) == len(it_r)
    assert max(abs(a - b) for a, b in zip(it_g, it_r)) <= 2, (it_g, it_r)
    _compare_solutions(p_gpu, p_ref, 1e-4)
    # and the inexact path lands where the exact one does
    p_ex = prob.copy()
    s_ex = _engine.ba_run(p_ex, ic, _capi.default_ba_options(use_inner_iterations=0, max_num_iterations=12))
    assert abs(s_gpu["final_cost"] - s_ex["final_cost"]) <= 1e-3 * s_ex["final_cost"]


@pytest.mark.parametrize("n_cams,multikernel", [(45, False), (45, True), (150, False), (33, False), (45, "band"), (150, "band"),
                                                (33, "band"), (5, "band"), (9, "band")])
def test_reduced_system_cholesky_tile_dag(n_cams, multikernel, monkeypatch):
    """The exact reduced-camera-system solve (DENSE/SPARSE_SCHUR, bundle_optimizer.h:181-191) at sizes that span
    many 32x32 tiles with a ragged last tile: the persistent tile-DAG kernel (pxr_chol.cuh) and the older
    launch-per-panel path must both reproduce the oracle's step."""
    if multikernel == "band":
        monkeypatch.setenv("PXR_CHOL_BAND", "1")       # the band design (pxr_chol2.cuh), opt-in
    elif multikernel:
        monkeypatch.setenv("PXR_CHOL_MULTIKERNEL", "1")
    prob, gt, ic = _scene(n_cams=n_cams, n_points=12 * n_cams, track_len=min(6, n_cams), channels=16, seed=n_cams)
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_linearize(prob, ic, so, radius=1e4)
    assert ref["nc"] > 32 * 6 or n_cams < 33          # the small cases: one to three tiles (band kernel's start-up rows)
    h = _engine.BAHandle(prob, ic, so)
    for _ in range(2):       # twice: the second call replays the captured graph with re-zeroed flags
        got = h.debug_linearize(ref["nc"], ref["nl"], radius=1e4)
        assert np.allclose(got["delta"], ref["delta"], rtol=1e-5, atol=1e-8 * np.abs(ref["delta"]).max())
    assert abs(got["model_cost_change"] - ref["model_cost_change"]) <= 1e-7 * abs(ref["model_cost_change"])


@pytest.mark.parametrize("variant", ["per_image_cameras", "shared_camera", "constant_blocks"])
def test_iterative_schur_block_sparse_matches_dense_and_oracle(variant, monkeypatch):
    """The implicit block-sparse reduced system (pxr_sparse_schur.cuh; what config 5's 5 000 cameras need) against
    the dense PCG path and the oracle's PCG on the same problems: identical CG recurrences, different storage."""
    kw = dict(n_cams=12, n_points=150, track_len=5, channels=16, seed=5)
    if variant == "shared_camera":
        kw["shared_camera"] = True
    prob, gt, ic = _scene(**kw)
    if variant == "constant_blocks":
        prob.point_const[::9] = 1
        prob.pose_const[3] = 1
        prob.tvec_const_mask[4] = 0b101
        prob.cam_const_mask[2] = 0xFFFFFFFF
    so = _capi.default_ba_options(use_inner_iterations=0, max_num_iterations=10, linear_solver=3)
    p_ref, p_dense, p_sparse = prob.copy(), prob.copy(), prob.copy()
    s_ref = O.ba_solve(p_ref, ic, so)
    s_dense = _engine.ba_run(p_dense, ic, so)
    monkeypatch.setenv("PXR_PCG_SPARSE", "1")
    s_sparse = _engine.ba_run(p_sparse, ic, so)
    monkeypatch.delenv("PXR_PCG_SPARSE")
    it_s = [i["linear_solver_iterations"] for i in s_sparse["iterations"][1:]]
    it_d = [i["linear_solver_iterations"] for i in s_dense["iterations"][1:]]
    assert len(it_s) == len(it_d) and max(abs(a - b) for a, b in zip(it_s, it_d)) <= 2, (it_s, it_d)
    assert abs(s_sparse["final_cost"] - s_dense["final_cost"]) <= 1e-6 * s_dense["final_cost"]
    assert abs(s_sparse["final_cost"] - s_ref["final_cost"]) <= 1e-5 * s_ref["final_cost"]
    _compare_solutions(p_sparse, p_dense, 1e-5)
    _compare_solutions(p_sparse, p_ref, 1e-4)
    # the multi-CTA vector kernels (what runs from 4096 unknowns) give the same trajectory
    monkeypatch.setenv("PXR_CG_MULTI", "1")
    for sparse in (False, True):
        if sparse:
            monkeypatch.setenv("PXR_PCG_SPARSE", "1")
        p_m = prob.copy()
        s_m = _engine.ba_run(p_m, ic, so)
        it_m = [i["linear_solver_iterations"] for i in s_m["iterations"][1:]]
        assert len(it_m) == len(it_d) and max(abs(a - b) for a, b in zip(it_m, it_d)) <= 2, (it_m, it_d)
        assert abs(s_m["final_cost"] - s_dense["final_cost"]) <= 1e-6 * s_dense["final_cost"]
        _compare_solutions(p_m, p_dense, 1e-5)
