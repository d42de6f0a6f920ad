"""Host side of batched query keypoint adjustment and nearest-candidate matching without a GPU: argument checks of
pxr_qka_run and pxr_query_match_run, their instance lists read from the sources, and QueryKeypointOptimizer.run_batch
with the oracle standing in for the device (the batch is also the pxr_ka_desc of the same problems)."""
import ctypes as C
import re

import numpy as np
import pytest

from pixsfm._pixsfm import _capi, _features, _localization as loc
from test_kernel_options_cpu import _body, _src, fm_instances, ka_instances
from test_mirror_with_oracle_solver import oracle_engine  # noqa: F401  (fixture)


def _queries(seed=0, n_queries=4, channels=16, multi=True):
    rng = np.random.default_rng(seed)
    qs = []
    for q in range(n_queries):
        n = [5, 8, 3, 6][q % 4]
        patches = rng.standard_normal((n, 16, 16, channels)).astype(np.float16)
        corners = rng.integers(0, 40, (n, 2))
        fmap = _features.FeatureMap(patches, list(range(n)), corners, {"scale": [1.0, 1.0], "is_sparse": True})
        kps = (corners + 0.5 + rng.uniform(5.0, 11.0, (n, 2))).astype(np.float64)
        refs = [[rng.standard_normal(channels) for _ in range(2)] if multi and i % 3 == 0 else rng.standard_normal(channels)
                for i in range(n)]
        qs.append((kps, fmap, refs, list(range(n)), [i % 4 != 1 for i in range(n)] if q % 2 else None))
    return qs


def _batch(**kw):
    return loc.QueryKeypointOptimizer({"bound": 4.0}, {}).pack_batch(_queries(**kw))[0]


def _qka(desc, interp=None):
    res = (_capi.QKAResult * 8)()
    return _capi.load_lib().pxr_qka_run(None, C.byref(desc) if desc is not None else None,
                                        C.byref(interp) if interp else None, None, res, None, None)


def _no_device():
    h = C.c_void_p()
    return _capi.load_lib().pxr_ctx_create(-1, C.byref(h)) == _capi.PXR_ERR_NO_DEVICE


def test_qka_argument_errors_come_before_the_device():
    b = _batch()
    assert _qka(None) == _capi.PXR_ERR_INVALID_ARGUMENT
    d = b.qka_desc(); d.kp_begin = None
    assert _qka(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    bad = b.kp_begin.copy(); bad[1] = bad[2] + 1
    d = b.qka_desc(); d.kp_begin = bad.ctypes.data_as(C.c_void_p)
    assert _qka(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    bad = b.desc_begin.copy(); bad[2] = bad[1] - 1
    d = b.qka_desc(); d.desc_begin = bad.ctypes.data_as(C.c_void_p)
    assert _qka(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    bad = b.kp_patch_local.copy(); bad[0] = 10 ** 6
    d = b.qka_desc(); d.kp_patch = bad.ctypes.data_as(C.c_void_p)
    assert _qka(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert "is not a patch of query 0" in _capi.load_lib().pxr_last_error().decode()
    d = b.qka_desc(); d.channels = 48
    assert _qka(d) == _capi.PXR_ERR_UNSUPPORTED
    d = b.qka_desc(); d.patch_dtype = 1; d.channels = 64          # fp32 64: not a query-mode instance
    assert _qka(d) == _capi.PXR_ERR_UNSUPPORTED
    assert _qka(b.qka_desc(), _capi.default_interp(use_float_simd=True)) == _capi.PXR_ERR_UNSUPPORTED
    if _no_device():
        assert _qka(b.qka_desc()) == _capi.PXR_ERR_NO_DEVICE


def test_run_batch_validation_names_the_query():
    qs = _queries()
    qs[2] = (qs[2][0], qs[2][1], qs[2][2][:-1]) + qs[2][3:]
    with pytest.raises(ValueError, match=r"query 2: references.size\(\) != keypoints.rows\(\)"):
        loc.QueryKeypointOptimizer({}, {}).pack_batch(qs)
    qs = _queries()
    qs.append(_queries(channels=32)[0])
    with pytest.raises(ValueError, match="query 4: every query of a batch must have the same channel count"):
        loc.QueryKeypointOptimizer({}, {}).pack_batch(qs)


def _match(n_queries=1, item_query=(0,), item_patch=(0,), begin=(0,), end=(1,), n_cand=1, channels=16, dtype=0):
    lib = _capi.load_lib()
    blk = np.zeros((2, 8, 8, channels), np.float16)
    ptrs = (C.c_void_p * 1)(blk.ctypes.data)
    counts = np.array([2], np.int64); corner = np.zeros((2, 2), np.int32); scale = np.ones((2, 2))
    iq = np.array(item_query, np.int32); ip = np.array(item_patch, np.int64); xy = np.full((len(iq), 2), 3.0)
    cb = np.array(begin, np.int64); ce = np.array(end, np.int64); cand = np.zeros((max(n_cand, 1), channels))
    best = np.zeros(len(iq), np.int64)
    p = _capi.ptr
    return lib.pxr_query_match_run(None, n_queries, C.cast(ptrs, C.c_void_p), p(counts), p(corner), p(scale), C.c_double(1.0),
                                   8, 8, channels, dtype, C.c_int64(len(iq)), p(iq), p(ip), p(xy), p(cb), p(ce), p(cand),
                                   C.c_int64(n_cand), 0, None, p(best), None, None)


def test_query_match_argument_errors_come_before_the_device():
    assert _match(item_query=(1,)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert _match(item_patch=(2,)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert _match(begin=(1,), end=(0,)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert _match(end=(2,)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert _match(channels=48) == _capi.PXR_ERR_UNSUPPORTED
    assert _match(n_queries=-1) == _capi.PXR_ERR_INVALID_ARGUMENT
    if _no_device():
        assert _match() == _capi.PXR_ERR_NO_DEVICE


def test_instance_lists_are_read_from_the_sources():
    src = _src("pxr_ka.cu")
    body = _body(src, "static bool ka_supported(int dtype, int C)")
    sup = set()
    for d, cs in re.findall(r"\(dtype == (PXR_F\d+) && \(((?:C == \d+(?: \|\| )?)+)\)\)", body):
        for c in re.findall(r"\d+", cs):
            sup.add(({"PXR_F16": "float16", "PXR_F32": "float32", "PXR_F64": "float64"}[d], int(c)))
    # pxr_qka_run accepts exactly the query-mode instances pxr_ka_run launches, and refuses float-SIMD first
    assert sup == {(d, c) for d, c, fs, ref in ka_instances() if ref and not fs}
    qka = _body(src, 'extern "C" int pxr_qka_run(')
    assert "ka_launch(ctx, &v.desc, false, ks[set])" in qka
    assert "use_float_simd is not built" in _body(src, "static int check_qka(")
    # the nearest-candidate kernel: one instance, behind fm_supported (the K1 instances of the descriptors)
    refs = _src("pxr_refs.cu")
    match = _body(refs, 'extern "C" int pxr_query_match_run(')
    assert "!fm_supported(patch_dtype, channels) || channels > kNCMaxC" in match
    assert len(re.findall(r"PXR_LAUNCH\(ctx, nearest_candidate_kernel,", refs)) == 1
    assert max(c for _, c in fm_instances()) <= 256


def test_run_batch_with_the_oracle(oracle_engine):  # noqa: F811
    """the batch is packed and written back as run() does: with the oracle solving the pxr_ka_desc view of the batch
    (one problem per query) the keypoints are those of a loop of run()"""
    qs = _queries()
    loop = []
    for q in qs:
        k = q[0].copy()
        loc.QueryKeypointOptimizer({"bound": 4.0}, {}).run(k, *q[1:])
        loop.append(k)
    cs = [(q[0].copy(),) + tuple(q[1:]) for q in qs]
    ok = loc.QueryKeypointOptimizer({"bound": 4.0}, {}).run_batch(cs)
    assert ok == [True] * len(qs)
    for a, c in zip(loop, cs):
        assert np.array_equal(a, c[0])


def test_observation_table_packs_every_point_once_in_order():
    rng = np.random.default_rng(1)
    refs = {}
    for pid in range(2000):
        r = _features.Reference(descriptor=rng.standard_normal(8))
        r.observations = [rng.standard_normal(8) for _ in range(1 + pid % 4)]
        refs[pid] = r
    ids = list(range(2000)) + [5, 7]                     # repeated ids are packed once
    rows, where = loc.observation_table(refs, ids)
    assert len(where) == 2000 and len(rows) == sum(1 + p % 4 for p in range(2000))
    for pid in (0, 1, 3, 1999):
        first, n = where[pid]
        assert n == len(refs[pid].observations)
        assert np.array_equal(rows[first:first + n], np.array(refs[pid].observations))
    refs[3].observations = []
    with pytest.raises(ValueError, match="Missing observations"):
        loc.observation_table(refs, [1, 3])


def test_query_match_checks_the_candidate_table_width():
    from pixsfm._pixsfm import _engine
    blk = np.zeros((2, 8, 8, 16), np.float16)
    args = ([blk], np.zeros((2, 2), np.int32), np.ones((2, 2)), [0], [0], [[3.0, 3.0]], [0], [1])
    with pytest.raises(ValueError, match=r"\[n, 16\]"):
        _engine.query_match_run(*args, np.zeros((4, 8)))

    class Dev:                                           # a device table of the wrong width / dtype
        def __init__(self, shape, typestr):
            self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (1 << 20, False), "version": 3,
                                             "strides": None}
    for bad in (Dev((4, 8), "<f8"), Dev((4, 16), "<f4"), Dev((64,), "<f8")):
        with pytest.raises(ValueError, match="C-contiguous"):
            _engine.query_match_run(*args, bad)
