"""Host side of batched query bundle adjustment: packing, the wave plan and argument checks, without a GPU."""
import ctypes as C

import numpy as np
import pytest

from pixsfm._pixsfm import _capi, _engine, _features, _localization as loc
from pixsfm.util import colmap_types as ct

MODEL_PARAMS = {0: [500.0, 60.0, 50.0], 1: [500.0, 510.0, 60.0, 50.0], 2: [500.0, 60.0, 50.0, 0.01],
                3: [500.0, 60.0, 50.0, 0.01, -0.002], 4: [500.0, 510.0, 60.0, 50.0, 0.01, -0.002, 1e-4, -1e-4],
                5: [500.0, 510.0, 60.0, 50.0, 0.01, -0.002, 1e-3, -1e-3],
                6: [500.0, 510.0, 60.0, 50.0, 0.01, -0.002, 1e-4, -1e-4, 1e-3, 1e-4, 1e-5, 1e-6]}


def _query(seed, model, n=12, channels=16, dtype=np.float16, multi=False):
    rng = np.random.default_rng(seed)
    patches = rng.standard_normal((n, 8, 8, channels)).astype(dtype)
    fmap = _features.FeatureMap(patches, list(range(n)), rng.integers(0, 50, (n, 2)),
                                {"scale": [1.0, 1.0], "is_sparse": True})
    cam = ct.Camera(1, model, 120, 100, MODEL_PARAMS[model])
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    t = rng.normal(size=3)
    pts = [rng.normal(size=3) + [0, 0, 5] for _ in range(n)]
    refs = []
    for i in range(n):
        if multi and i % 3 == 0:
            refs.append([rng.normal(size=channels) for _ in range(2)])       # several descriptors: several blocks
        else:
            refs.append(rng.normal(size=channels))
    inliers = [i % 4 != 1 for i in range(n)]
    p2D = [(i * 5) % n for i in range(n)]
    return (q, t, cam, pts, fmap, refs, inliers, p2D)


@pytest.mark.parametrize("opts", [{}, {"refine_focal_length": True}, {"refine_principal_point": True, "refine_extra_params": True},
                                  {"refine_focal_length": True, "refine_principal_point": True, "refine_extra_params": True}])
def test_pack_batch_concatenates_build_problem(opts):
    qs = [_query(s, model, multi=bool(s % 2)) for s, model in enumerate(range(7))]
    qs.append(_query(9, 2)[:6])                       # no inliers / patch_idxs given
    qbo = loc.QueryBundleOptimizer(opts, {})
    batch = qbo.pack_batch(qs)
    assert batch.n_queries == len(qs)
    for k, q in enumerate(qs):
        prob = qbo.build_problem(*q[:6], *(q[6:] + (None,) * (8 - len(q)))[:2])
        b0, b1 = batch.obs_begin[k], batch.obs_begin[k + 1]
        assert b1 - b0 == prob.n_obs
        assert np.array_equal(batch.xyz[b0:b1], prob.xyz) and np.array_equal(batch.refs[b0:b1], prob.refs)
        assert np.array_equal(batch.obs_patch[b0:b1], prob.obs_patch)
        assert batch.cam_const_mask[k] == prob.cam_const_mask[0] and batch.cam_model[k] == prob.cam_model[0]
        assert np.array_equal(batch.cam_params[k], prob.cam_params[0])
        assert np.array_equal(batch.qvec[k], prob.qvec[0]) and np.array_equal(batch.tvec[k], prob.tvec[0])
        p0 = int(batch.patch_counts[:k].sum())
        n = int(batch.patch_counts[k])
        assert np.array_equal(batch.corner[p0:p0 + n], prob.corner) and np.array_equal(batch.scale[p0:p0 + n], prob.scale)


def _batch(sizes, channels=16):
    qs = [_query(s, 2, n=n, channels=channels) for s, n in enumerate(sizes)]
    return loc.QueryBundleOptimizer({}, {}).pack_batch(qs)


def _query_bytes(b, q):
    per_patch = b.ph * b.pw * b.channels * 2
    m = b.obs_begin[q + 1] - b.obs_begin[q]
    return b.patch_counts[q] * per_patch + m * (b.channels * 8 + 32) + b.patch_counts[q] * 16 + (19 * 8 + 32)


def test_wave_plan_respects_the_budget():
    b = _batch([12, 30, 5, 60, 8, 8, 8, 20])
    qb = [_query_bytes(b, q) for q in range(b.n_queries)]
    budget = 0.8 * max(qb)
    b.max_wave_bytes = budget
    begin, nbytes = _engine.qba_plan_waves(b)
    again = _engine.qba_plan_waves(b)
    assert np.array_equal(begin, again[0]) and np.array_equal(nbytes, again[1])          # deterministic
    assert begin[0] == 0 and begin[-1] == b.n_queries and np.all(np.diff(begin) >= 1)    # every query in one wave
    for w in range(len(nbytes)):
        q0, q1 = begin[w], begin[w + 1]
        assert abs(nbytes[w] - (8 + sum(qb[q0:q1]))) < 1e-6
        if q1 - q0 > 1:
            assert nbytes[w] <= budget
        if q1 < b.n_queries:          # greedy: the next query would not have fitted
            assert nbytes[w] + qb[q1] > budget
    big = int(np.argmax(qb))
    assert qb[big] + 8 > budget and big in begin and big + 1 in begin     # oversized: a wave of its own


def test_one_wave_when_everything_fits():
    b = _batch([4, 4, 4])
    b.max_wave_bytes = 1e12
    begin, nbytes = _engine.qba_plan_waves(b)
    assert list(begin) == [0, 3]


def _call(desc, opt=None, interp=None):
    lib = _capi.load_lib()
    res = (_capi.QBAResult * 8)()
    return lib.pxr_qba_run(None, C.byref(desc) if desc is not None else None, C.byref(interp) if interp else None,
                           C.byref(opt) if opt else None, res, None, 0, None, None)


def _no_device():
    lib = _capi.load_lib()
    h = C.c_void_p()
    return lib.pxr_ctx_create(-1, C.byref(h)) == _capi.PXR_ERR_NO_DEVICE


def test_argument_errors_come_before_the_device():
    b = _batch([6, 7])
    assert _call(None) == _capi.PXR_ERR_INVALID_ARGUMENT
    d = b.desc(); d.qvec = None
    assert _call(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    bad = b.obs_begin.copy(); bad[1] = bad[2] + 1
    d = b.desc(); d.obs_begin = bad.ctypes.data_as(C.c_void_p)
    assert _call(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    d = b.desc(); d.channels = 48
    assert _call(d) == _capi.PXR_ERR_UNSUPPORTED
    assert "Unsupported dimensions (CHANNELS,N_NODES)." in _capi.load_lib().pxr_last_error().decode()
    d = b.desc(); d.patch_dtype = 1; d.channels = 32          # fp32 32 channels: not a K1 instance
    assert _call(d) == _capi.PXR_ERR_UNSUPPORTED
    assert _call(b.desc(), _capi.default_ba_options(use_inner_iterations=1)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert _call(b.desc(), _capi.default_ba_options(use_inner_iterations=0, linear_solver=3)) == _capi.PXR_ERR_UNSUPPORTED
    bad_patch = b.obs_patch.copy(); bad_patch[0] = 10 ** 6
    d = b.desc(); d.obs_patch = bad_patch.ctypes.data_as(C.c_void_p)
    assert _call(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    if _no_device():
        rc = _call(b.desc(), _capi.default_ba_options(use_inner_iterations=0, deterministic=1))
        assert rc == _capi.PXR_ERR_NO_DEVICE


def test_run_still_rejects_device_feature_maps():
    q = _query(3, 2)

    class FakeDevice:
        def __init__(self, a):
            self.__cuda_array_interface__ = {"shape": a.shape, "typestr": "<f2", "data": (1 << 20, False), "version": 3,
                                             "strides": None}
    fm = q[4]
    dmap = _features.FeatureMap(FakeDevice(fm.patches), fm.point2D_ids, fm.corners, {"scale": fm.scale})
    with pytest.raises(ValueError, match="host"):
        loc.QueryBundleOptimizer({}, {}).run(*q[:4], dmap, q[5], q[6], q[7])
    batch = loc.QueryBundleOptimizer({}, {}).pack_batch([q[:4] + (dmap,) + q[5:]])    # run_batch takes them
    assert batch.patch_counts[0] == fm.size()
