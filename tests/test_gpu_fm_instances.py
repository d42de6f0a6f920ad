"""GPU parity of every feature-metric kernel instance (K1 evaluation, both inner-iteration paths, reference
extraction, keypoint adjustment) against the oracle, at the patch geometries the kernels branch on: 16x16, 8x8 (the
reference's low_memory.yaml), a non-square patch and one smaller than the 4x4 interpolation tap window."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from ka_util import make_ka_problem
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

# (dtype, channels) of every K1 instance with C >= 8 that fm_supported (csrc/pxr_ba.cu) builds
FM_INSTANCES = [(np.float16, c) for c in (8, 16, 32, 64, 128, 256)] + \
               [(np.float32, c) for c in (16, 64, 128)] + [(np.float64, c) for c in (16, 128)]
# (ph, pw) cut out of the centre of a rendered 16x16 patch
PATCH_SHAPES = [(16, 16), (8, 8), (12, 8), (3, 3)]
# the instances pxr_ka.cu builds; fm_supported's f16 256 and f32 64 are not among them
KA_INSTANCES = [(np.float16, c) for c in (8, 16, 32, 64, 128)] + [(np.float32, c) for c in (16, 128)] + \
               [(np.float64, c) for c in (16, 128)]
KA_MISSING = [(np.float16, 256), (np.float32, 64)]


def _crop(patches, corner, ph, pw):
    """centred [ph, pw] window of every patch; the corner moves with it, so projections keep their pixel position"""
    r0, c0 = (patches.shape[1] - ph) // 2, (patches.shape[2] - pw) // 2
    corner = corner.copy()
    corner[:, 0] += c0
    corner[:, 1] += r0
    return np.ascontiguousarray(patches[:, r0:r0 + ph, c0:c0 + pw]), corner


def _ba_scene(dtype, channels, ph, pw):
    prob, _ = synthetic.make_ba_scene(n_cams=4, n_points=20, track_len=4, channels=channels, seed=channels + ph * 7 + pw,
                                      dtype=dtype)
    patches, corner = _crop(prob.patches, prob.corner, ph, pw)
    prob = prob.with_patches(patches)
    prob.corner = corner
    return prob


def _id(v):
    return v.__name__ if isinstance(v, type) else str(v)


@pytest.mark.parametrize("ph,pw", PATCH_SHAPES, ids=lambda v: str(v))
@pytest.mark.parametrize("dtype,channels", FM_INSTANCES, ids=_id)
def test_fm_instance_matches_oracle(dtype, channels, ph, pw):
    prob = _ba_scene(dtype, channels, ph, pw)
    ic = _capi.default_interp()
    assert (prob.ph, prob.pw) == (ph, pw)
    # reference extraction (the IRLS over each track's descriptors)
    r_cpu, s_cpu = O.refs_compute(prob, ic)
    r_gpu, s_gpu = _engine.refs_compute(prob, ic)
    assert np.array_equal(s_cpu, s_gpu)
    assert np.abs(r_gpu - r_cpu).max() < 1e-12
    prob.refs = r_cpu * 0.95 + 0.002
    # K1: residuals, the 2x2 normal-equation pieces and the cost
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_evaluate(prob, ic, so, residuals=True)
    got = _engine.BAHandle(prob, ic, so).evaluate(residuals=True)
    assert np.allclose(got["xy"], ref["xy"], rtol=0, atol=1e-9)
    assert np.abs(got["residuals"] - ref["residuals"]).max() < 1e-12
    assert np.allclose(got["sq_norm"], ref["sq_norm"], rtol=1e-10, atol=1e-15)
    assert np.allclose(got["gtr"], ref["gtr"], rtol=1e-9, atol=1e-13)
    assert np.allclose(got["gtg"], ref["gtg"], rtol=1e-10, atol=1e-14)
    assert abs(got["cost"] - ref["cost"]) <= 1e-11 * abs(ref["cost"])
    if min(ph, pw) < 4:
        # A patch smaller than the 4x4 interpolation stencil leaves the point's cost flat wherever the tap window is
        # clamped, and the per-point solve walks projections out of it (tens of pixels): where such an ill-posed solve
        # stops is not a property of the kernels.  The evaluation above covers these shapes.
        return
    # one inner-iteration pass over the points
    prob.xyz += np.random.default_rng(5).normal(0, 0.004, prob.xyz.shape)
    so = _capi.default_ba_options(use_inner_iterations=1)
    p_ref = prob.copy()
    O.lib().orc_ba_inner_iterations(C.byref(p_ref.desc()), C.byref(ic), C.byref(so))
    assert np.abs(p_ref.xyz - prob.xyz).max() > 1e-5
    h = _engine.BAHandle(prob.copy(), ic, so)
    h.debug_inner_iterations()
    h.read_params()
    assert np.abs(h.problem.xyz - p_ref.xyz).max() < 1e-7


def _ka(dtype, channels, ps):
    return make_ka_problem(n_images=5, n_tracks=12, track_len=4, channels=channels, ps=ps, seed=channels + ps,
                           kp_sigma=0.7, bound=4.0, max_per_problem=20, dtype=dtype)


@pytest.mark.parametrize("ps", [16, 8])
@pytest.mark.parametrize("dtype,channels", KA_INSTANCES, ids=_id)
def test_ka_instance_matches_oracle(dtype, channels, ps):
    prob, _, lab = _ka(dtype, channels, ps)
    ic = _capi.default_interp(); so = _capi.default_ka_options()
    _, c_start = O.ka_evaluate(prob, ic, so)
    p_cpu, p_gpu = prob.copy(), prob.copy()
    c0, c1 = O.ka_solve(p_cpu, ic, so)
    s = _engine.ka_run(p_gpu, ic, so)
    assert abs(s["initial_cost"] - c_start) <= 1e-9 * c_start
    assert abs(s["initial_cost"] - c0) <= 1e-9 * c0
    assert abs(s["final_cost"] - c1) <= 1e-6 * c1
    assert c1 < c0
    assert np.abs(p_gpu.keypoints - p_cpu.keypoints).max() < 1e-5
    moved = ~lab["roots"].astype(bool)
    assert np.abs(p_gpu.keypoints[moved] - prob.keypoints[moved]).max() > 1e-3


@pytest.mark.parametrize("dtype,channels", KA_MISSING, ids=_id)
def test_ka_refuses_an_instance_it_does_not_build(dtype, channels):
    """a shape bundle adjustment supports but keypoint adjustment does not build is refused before anything runs"""
    prob, _, _ = _ka(dtype, channels, 8)
    p = prob.copy()
    before = p.keypoints.copy()
    with pytest.raises((ValueError, _capi.PxrError)):
        _engine.ka_run(p, _capi.default_interp(), _capi.default_ka_options())
    assert np.array_equal(p.keypoints, before)
