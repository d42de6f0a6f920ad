"""Absolute pose estimation without a GPU: the host restatement's Lambda Twist, the written-down sample stream, the
pycolmap option mapping and the C-ABI's argument checks."""
import ctypes as C

import numpy as np
import pytest

import pnp_reference as P
from pixsfm._pixsfm import _capi, _localization as loc


def _triplet(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    R, t = P.quat_to_rot(q), rng.normal(size=3)
    Xc = np.column_stack([rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3), rng.uniform(2, 6, 3)])
    return R, t, (Xc - t) @ R, Xc[:, :2] / Xc[:, 2:]


def test_lambda_twist_recovers_the_ground_truth_pose():
    rng = np.random.default_rng(0)
    for _ in range(200):
        R, t, X, x = _triplet(rng)
        sols = P.p3p(x, X)
        assert 1 <= len(sols) <= 4
        err = min(max(np.abs(Rs - R).max(), np.abs(ts - t).max()) for Rs, ts in sols)
        assert err < 1e-9
        for Rs, ts in sols:                    # every solution is a rotation that reprojects the three points
            assert np.abs(Rs @ Rs.T - np.eye(3)).max() < 1e-9 and abs(np.linalg.det(Rs) - 1) < 1e-9
            Y = X @ Rs.T + ts
            assert np.abs(Y[:, :2] / Y[:, 2:] - x).max() < 1e-9


def test_sample_stream_known_answers():
    # splitmix64's first output from state 0 is the published 0xE220A8397B1DCDAF
    assert P.splitmix64(0) == 0xE220A8397B1DCDAF
    assert P.sample(1, 0, 10) == [3, 9, 7]
    assert P.sample(1, 1, 10) == [6, 7, 4]
    assert P.sample(12345, 7, 500) == [372, 72, 434]
    for trial in range(50):
        s = P.sample(2 ** 64 - 1, trial, 500)
        assert len(set(s)) == 3 and all(0 <= i < 500 for i in s)
    for seed, trial in ((0, 0), (7, 129), (99, 99999)):
        s = P.sample(seed, trial, 3)
        assert sorted(s) == [0, 1, 2]          # three correspondences: every trial draws all of them


def test_required_trials_is_colmaps_dynamic_count():
    # ceil(log(1 - confidence) / log(1 - ratio^3) * multiplier), clamped
    assert P.required_trials(70, 100, 0.9999, 3.0, 1000, 100000) == 1000
    assert P.required_trials(20, 100, 0.9999, 3.0, 0, 100000) == int(np.ceil(np.log(1e-4) / np.log(1 - 0.2 ** 3) * 3))
    assert P.required_trials(0, 100, 0.9999, 3.0, 1000, 100000) == 100000
    assert P.required_trials(100, 100, 0.9999, 3.0, 10, 100000) == 10


def test_options_take_pycolmap_names_and_reject_unknown_keys():
    o = loc.pnp_options({"ransac": {"max_error": 4.0, "min_num_trials": 200}}, {"refine_focal_length": True,
                                                                               "gradient_tolerance": 1e-3})
    assert o.max_error == 4.0 and o.min_num_trials == 200 and o.max_num_trials == 100000
    assert o.confidence == 0.9999 and o.dyn_num_trials_multiplier == 3.0 and o.min_inlier_ratio == 0.01
    assert o.refine_focal_length == 1 and o.refine_extra_params == 0 and o.gradient_tolerance == 1e-3
    assert o.max_num_iterations == 100 and o.loss_function_scale == 1.0 and o.refine == 1
    d = loc.pnp_options()
    assert d.max_error == 12.0 and d.gradient_tolerance == 1.0
    with pytest.raises(ValueError, match="unknown option 'max_eror'"):
        loc.pnp_options({"ransac": {"max_eror": 4.0}})
    with pytest.raises(ValueError, match="unknown option"):
        loc.pnp_options(None, {"refine_principal_point": True})
    with pytest.raises(ValueError, match="estimate_focal_length"):
        loc.pnp_options({"estimate_focal_length": True})


def _desc(begin, models, n_corr=None):
    nq = len(models)
    n_corr = int(begin[-1]) if n_corr is None else n_corr
    b = _capi.PnPBatch(begin, np.zeros((max(n_corr, 0), 2)), np.zeros((max(n_corr, 0), 3)), models,
                       np.ones((nq, 12)), np.zeros(nq, np.uint64))
    return b


def test_c_abi_rejects_malformed_descs_without_a_device():
    lib = _capi.load_lib()
    res = (_capi.PnPResult * 4)()
    o = _capi.default_pnp_options()
    assert lib.pxr_pnp_run(None, None, C.byref(o), res, None) == _capi.PXR_ERR_INVALID_ARGUMENT
    b = _desc([0, 5, 3], [0, 1], n_corr=5)
    d = b.desc()
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(o), res, None) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert b"non-decreasing" in lib.pxr_last_error()
    b = _desc([0, 4, 9], [1, 9])
    d = b.desc()
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(o), res, None) == _capi.PXR_ERR_UNSUPPORTED
    b = _desc([1, 4], [1])
    d = b.desc()
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(o), res, None) == _capi.PXR_ERR_INVALID_ARGUMENT
    b = _desc([0, 4], [1])
    d = b.desc()
    d.points2D = None
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(o), res, None) == _capi.PXR_ERR_INVALID_ARGUMENT
    d = b.desc()
    f = _capi.default_pnp_options(estimate_focal_length=1)
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(f), res, None) == _capi.PXR_ERR_UNSUPPORTED
    bad = _capi.default_pnp_options(min_num_trials=10, max_num_trials=5)
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(bad), res, None) == _capi.PXR_ERR_INVALID_ARGUMENT
    # a well-formed call reaches the context check
    assert lib.pxr_pnp_run(None, C.byref(d), C.byref(o), res, None) not in (_capi.PXR_OK, _capi.PXR_ERR_UNSUPPORTED)
    assert lib.pxr_pnp_debug_image_to_world(None, 7, None, 0, None, None) == _capi.PXR_ERR_UNSUPPORTED
