"""Batched query refinement on the device: pxr_query_match_run (nearest candidate descriptor) against
pxr_interpolate_descriptors and an extended-precision arg-min, pxr_qka_run (QueryKeypointOptimizer.run_batch) against
pxr_ka_run per query, and QueryLocalizer.localize_batch against localize."""
import copy

import numpy as np
import pytest

from pixsfm._pixsfm import _capi, _engine, _features, _localization as loc
from test_kernel_options_cpu import fm_instances

pytestmark = pytest.mark.gpu

NP = {"float16": np.float16, "float32": np.float32, "float64": np.float64}
QKA_INSTANCES = [("float16", c) for c in (8, 16, 32, 64, 128)] + [(d, c) for d in ("float32", "float64") for c in (16, 128)]


def _device(a):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")


def _blocks(rng, n_queries, dtype, channels, sizes=(5, 9, 1, 12)):
    out = []
    for q in range(n_queries):
        n = sizes[q % len(sizes)]
        out.append((rng.standard_normal((n, 8, 8, channels)).astype(dtype), rng.integers(0, 40, (n, 2)).astype(np.int32),
                    np.tile(rng.uniform(0.5, 1.5, 2), (n, 1))))
    return out


@pytest.mark.parametrize("dtype,channels", sorted(fm_instances()))
@pytest.mark.parametrize("fs", [0, 1])
def test_query_match_descriptors_are_those_of_interpolate_descriptors(dtype, channels, fs):
    rng = np.random.default_rng(channels + 7 * fs)
    blocks = _blocks(rng, 3, NP[dtype], channels)
    iq, ip, xy = [], [], []
    for q, (p, c, s) in enumerate(blocks):
        for i in range(2 * len(p)):
            iq.append(q); ip.append(i % len(p))
            xy.append((c[i % len(p)] + rng.uniform(1.0, 7.0, 2)) / s[i % len(p)])
    ic = _capi.default_interp(use_float_simd=fs)
    n = len(iq)
    cb, ce = np.zeros(n, np.int64), np.zeros(n, np.int64)
    host = [b[0] for b in blocks]
    mixed = [host[0], _device(host[1]), host[2]]          # host and device blocks in one call
    for pb in (host, mixed):
        _, _, desc = _engine.query_match_run(pb, np.concatenate([b[1] for b in blocks]), np.concatenate([b[2] for b in blocks]),
                                             iq, ip, xy, cb, ce, np.zeros((0, channels)), ic, with_desc=True)
        for q, (p, c, s) in enumerate(blocks):
            sel = [k for k in range(n) if iq[k] == q]
            ref = _engine.interpolate_patches(p, c, s, [ip[k] for k in sel], [xy[k] for k in sel], ic)
            assert np.array_equal(desc[sel], ref), q


def _ld_argmin(q, rows):
    d = ((np.asarray(rows, np.longdouble) - np.asarray(q, np.longdouble)) ** 2).sum(1)
    return int(np.argmin(d)), d


def test_query_match_picks_the_first_nearest_candidate():
    rng = np.random.default_rng(3)
    channels = 128
    blocks = _blocks(rng, 2, np.float16, channels)
    lengths = [0, 1, 2, 4, 31, 32, 33, 70, 5, 3]
    iq, ip, xy, cb, ce, rows = [], [], [], [], [], []
    for k, m in enumerate(lengths):
        q = k % 2
        p, c, s = blocks[q]
        iq.append(q); ip.append(k % len(p)); xy.append((c[k % len(p)] + 4.0) / s[k % len(p)])
        cb.append(len(rows)); ce.append(len(rows) + m)
        r = rng.standard_normal((m, channels)) * 0.1
        if m >= 4:
            r[3] = r[1]                                   # an exact duplicate after the first one
        rows.extend(r)
    rows = np.array(rows)
    ic = _capi.default_interp()
    args = ([b[0] for b in blocks], np.concatenate([b[1] for b in blocks]), np.concatenate([b[2] for b in blocks]), iq, ip,
            xy, cb, ce)
    best, dmin, desc = _engine.query_match_run(*args, rows, ic, with_desc=True)
    best_d, dmin_d, _ = _engine.query_match_run(*args, _device(rows), ic)
    assert np.array_equal(best, best_d) and np.array_equal(dmin, dmin_d)      # device table: the same bits
    for k, m in enumerate(lengths):
        if m == 0:
            assert best[k] == -1 and np.isinf(dmin[k])
            continue
        # the duplicates are the nearest rows of the items whose own descriptor is planted there
        j, d = _ld_argmin(desc[k], rows[cb[k]:ce[k]])
        srt = np.sort(d)
        if len(d) > 1 and (srt[1] - srt[0]) <= 1e-12 * srt[0]:
            assert abs(dmin[k] - float(srt[0])) <= 1e-12 * float(srt[0])
        else:
            assert best[k] == cb[k] + j
            assert abs(dmin[k] - float(d[j])) <= 1e-12 * float(d[j])
    # duplicates at the minimum: the first one wins
    rows2 = rows.copy()
    for k, m in enumerate(lengths):
        if m >= 4:
            rows2[cb[k] + 1] = desc[k]; rows2[cb[k] + 3] = desc[k]
    best2, dmin2, _ = _engine.query_match_run(*args, rows2, ic)
    for k, m in enumerate(lengths):
        if m >= 4:
            assert best2[k] == cb[k] + 1 and dmin2[k] == 0.0
    # NaN distances: the first NaN row wins, as numpy's argmin (the per-query path) picks it
    rows3 = rows.copy()
    for k, m in enumerate(lengths):
        if m >= 4:
            rows3[cb[k] + 2, 0] = np.nan
    best3, dmin3, _ = _engine.query_match_run(*args, rows3, ic)
    for k, m in enumerate(lengths):
        if m >= 4:
            d = ((rows3[cb[k]:ce[k]] - desc[k]) ** 2).sum(1)
            assert best3[k] == cb[k] + int(np.argmin(d)) == cb[k] + 2 and np.isnan(dmin3[k])


def _qka_queries(rng, dtype, channels, n_queries=6, multi=False, sparse=True):
    qs = []
    for q in range(n_queries):
        n = [6, 11, 3, 9, 14, 5][q % 6]
        if sparse:
            patches = rng.standard_normal((n, 16, 16, channels)).astype(dtype)
            corners = rng.integers(0, 40, (n, 2))
            fmap = _features.FeatureMap(patches, list(range(n)), corners, {"scale": [1.0, 1.0], "is_sparse": True})
            kps = (corners + 0.5 + rng.uniform(5.0, 11.0, (n, 2))).astype(np.float64)
        else:                                            # one dense map: every keypoint reads the same patch
            patches = rng.standard_normal((1, 48, 48, channels)).astype(dtype)
            fmap = _features.FeatureMap(patches, [_features.kDenseId], np.zeros((1, 2), np.int64),
                                        {"scale": [1.0, 1.0], "is_sparse": False})
            kps = rng.uniform(8.0, 40.0, (n, 2))
        refs = []
        for i in range(n):
            if multi and i % 3 == 0:
                refs.append([rng.standard_normal(channels) for _ in range(2)])
            else:
                refs.append(rng.standard_normal(channels))
        inliers = [i % 4 != 2 for i in range(n)] if q % 2 else None
        qs.append((kps, fmap, refs, list(range(n)), inliers))
    return qs


def _single(opts, qs):
    out = []
    for q in qs:
        kps = q[0].copy()
        o = loc.QueryKeypointOptimizer(opts, {})
        ok = o.run(kps, *q[1:])
        out.append((ok, kps, o.summary()))
    return out


def _batch(opts, qs, **kw):
    cs = [(q[0].copy(),) + tuple(q[1:]) for q in qs]
    o = loc.QueryKeypointOptimizer(opts, {})
    ok = o.run_batch(cs, **kw)
    return ok, [c[0] for c in cs], o.summaries()


def _same(single, batch):
    ok, kps, sums = batch
    for (ok1, k1, s1), ok2, k2, s2 in zip(single, ok, kps, sums):
        assert ok1 == ok2
        assert np.array_equal(k1, k2)
        if ok1:
            assert s1.initial_cost == s2.initial_cost and s1.final_cost == s2.final_cost


@pytest.mark.parametrize("dtype,channels", QKA_INSTANCES)
def test_qka_batch_matches_single_query_path(dtype, channels):
    rng = np.random.default_rng(channels)
    for bound, sparse, multi in ((4.0, True, False), (-1.0, True, True), (-1.0, False, True), (4.0, False, False)):
        opts = {"bound": bound, "solver": {"max_num_iterations": 20}}
        qs = _qka_queries(rng, NP[dtype], channels, multi=multi, sparse=sparse)
        _same(_single(opts, qs), _batch(opts, qs))


def test_qka_batch_waves_and_edge_cases(monkeypatch):
    rng = np.random.default_rng(11)
    opts = {"bound": 4.0, "solver": {"max_num_iterations": 20}}
    qs = _qka_queries(rng, np.float16, 128, n_queries=8, multi=True)
    # a query without residual blocks (every correspondence an outlier) and one with a non-finite initial cost: the
    # first is not solved, the second gets what run() gives it (True, the keypoints as pxr_ka_run writes them)
    qs[2] = qs[2][:4] + ([False] * len(qs[2][0]),)
    bad = [r.copy() if isinstance(r, np.ndarray) else [x.copy() for x in r] for r in qs[5][2]]
    bad[1][0] = np.nan
    qs[5] = (qs[5][0], qs[5][1], bad) + qs[5][3:]
    single = _single(opts, qs)
    assert single[5][0] and np.isnan(single[5][2].initial_cost) and not single[2][0]
    for kw, one_buf in (({}, False), ({"max_wave_bytes": 1.0}, False), ({"max_wave_bytes": 1.0}, True),
                        ({"max_wave_bytes": 3e6}, False)):
        if one_buf:
            monkeypatch.setenv("PXR_QBA_WAVE_BUFFERS", "1")
        ok, kps, sums = _batch(opts, qs, **kw)
        assert ok == [s[0] for s in single]
        assert sums[2] is None and np.array_equal(kps[2], qs[2][0])
        assert np.isnan(sums[5].initial_cost)
        for (ok1, k1, s1), k2, s2 in zip(single, kps, sums):
            assert np.array_equal(k1, k2)
            if ok1 and k1 is not single[5][1]:
                assert s1.initial_cost == s2.initial_cost and s1.final_cost == s2.final_cost
        monkeypatch.delenv("PXR_QBA_WAVE_BUFFERS", raising=False)
    # results do not depend on the batch: reversed order, one query alone
    good = [q for k, q in enumerate(qs) if k != 5]
    gsingle = [x for k, x in enumerate(single) if k != 5]
    _same(gsingle[::-1], _batch(opts, good[::-1]))
    _same(gsingle[3:4], _batch(opts, good[3:4]))


def test_qka_batch_matches_oracle():
    """the oracle's query-mode solve of the same problems (the batch's pxr_ka_desc view, one problem per query), at the
    tolerances of test_gpu_localization.py::test_query_keypoint_adjuster_matches_oracle"""
    import oracle_lib as O
    from recon_util import make_reconstruction
    from pixsfm import bundle_adjustment as ba_pkg
    from pixsfm._pixsfm import _bundle_adjustment as ba
    rec, fm, _, _ = make_reconstruction(n_cams=6, n_points=60, track_len=4, channels=128, seed=15)
    refs = ba.ReferenceExtractor({"iters": 100, "keep_observations": True}, {}).run(ba_pkg.find_problem_labels(rec, 10),
                                                                                     rec, fm.fset(0))
    rng = np.random.default_rng(3)
    qs = []
    for k, (iid, img) in enumerate(sorted(rec.images.items())):
        p2D = [i for i, p in enumerate(img.points2D) if p.has_point3D()]
        p3D = [img.points2D[i].point3D_id for i in p2D]
        kps = np.array([img.points2D[i].xy for i in p2D], np.float64) + rng.normal(0, 1.0, (len(p2D), 2))
        if k % 2:
            r = [[o for o in refs[p].observations] for p in p3D]
        else:
            r = []
            for p in p3D:
                x = copy.copy(refs[p]); x.observations = []; r.append(x)
        qs.append((kps, fm.fset(0).fmap(img.name), r, p2D))
    o = loc.QueryKeypointOptimizer({"bound": 4.0}, {})
    batch, used = o.pack_batch(qs)
    cpu = batch.copy()
    c0, c1 = O.ka_solve(cpu, _capi.default_interp(), o.solver_options())
    ok, kps, sums = _batch({"bound": 4.0}, qs)
    assert all(ok)
    g0, g1 = sum(s.initial_cost for s in sums), sum(s.final_cost for s in sums)
    assert abs(g0 - c0) <= 1e-9 * c0 and abs(g1 - c1) <= 1e-6 * c1 and c1 < c0
    for k, (q, u) in enumerate(zip(qs, used)):
        kb, ke = batch.kp_begin[k], batch.kp_begin[k + 1]
        assert np.abs(kps[k][u] - cpu.keypoints[kb:ke]).max() < 1e-5
        assert np.abs(kps[k] - q[0]).max() > 1e-2


def test_qka_batch_refuses_float_simd():
    rng = np.random.default_rng(2)
    qs = _qka_queries(rng, np.float16, 16, n_queries=2)
    cs = [(q[0].copy(),) + tuple(q[1:]) for q in qs]
    with pytest.raises(ValueError, match="use_float_simd"):
        loc.QueryKeypointOptimizer({}, {"use_float_simd": True}).run_batch(cs)
    for c, q in zip(cs, qs):
        assert np.array_equal(c[0], q[0])


def test_qka_batch_device_patches_match_host_patches():
    rng = np.random.default_rng(5)
    opts = {"bound": 4.0, "solver": {"max_num_iterations": 20}}
    qs = _qka_queries(rng, np.float16, 64, n_queries=4)
    dev = []
    for k, q in enumerate(qs):
        fm = q[1]
        if k % 2:
            fm = _features.FeatureMap(_device(fm.patches), fm.point2D_ids, fm.corners, {"scale": fm.scale, "is_sparse": True})
        dev.append((q[0], fm) + tuple(q[2:]))
    _same(_single(opts, qs), _batch(opts, dev))


def _localizer(target, qka=None):
    import test_gpu_qba_batch as T
    from pixsfm import localization as loc_pkg
    rec, refs, qs, _ = T._localizer_scene()
    conf = {"target_reference": target, "QBA": {"optimizer": {"refine_focal_length": True}}}
    if qka:
        conf["QKA"] = qka
    return qs, lambda: loc_pkg.QueryLocalizer(rec, conf, references=[refs])


@pytest.mark.parametrize("target,qka", [("nearest", None), ("robust_mean", None), ("all_observations", None),
                                        ("full", None), ("nearest", {"stack_correspondences": True}),
                                        ("robust_mean", {"feature_inlier_thresh": 1.2})])
def test_localize_batch_matches_localize(target, qka):
    qs, make = _localizer(target, qka)
    loop = [make().localize(**dict(q, query_camera=copy.deepcopy(q["query_camera"]))) for q in qs]
    batch = make().localize_batch([dict(q, query_camera=copy.deepcopy(q["query_camera"])) for q in qs])
    for a, b in zip(loop, batch):
        assert a["success"] and b["success"]
        assert np.array_equal(a["keypoints"], b["keypoints"])
        assert np.abs(np.asarray(a["qvec"]) - np.asarray(b["qvec"])).max() < 1e-6
        assert np.abs(np.asarray(a["tvec"]) - np.asarray(b["tvec"])).max() < 1e-6
        assert a["inliers"] == b["inliers"]


def test_find_nearest_references_batch_matches_per_query():
    qs, make = _localizer("nearest")
    L = make()
    items = [(q["query_fmaps"][0], L.references[0], q["keypoints"][q["pnp_point2D_idxs"]], q["pnp_points3D_id"],
              q["pnp_point2D_idxs"]) for q in qs]
    got = loc.find_nearest_references_batch(items, {})
    for it, g in zip(items, got):
        want = loc.find_nearest_references(it[0], it[1], it[2], it[3], {}, it[4])
        assert len(g) == len(want) and all(np.array_equal(a, b) for a, b in zip(g, want))


def test_pybind_entry_points_match_ctypes():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pixel-perfect-sfm_b200",
                                    "bindings"))
    pb = pytest.importorskip("_pxr_pybind")
    rng = np.random.default_rng(9)
    qs = _qka_queries(rng, np.float16, 64, n_queries=4, multi=True)
    o = loc.QueryKeypointOptimizer({"bound": 4.0}, {})
    b1, _ = o.pack_batch([(q[0].copy(),) + tuple(q[1:]) for q in qs])
    b2, _ = o.pack_batch([(q[0].copy(),) + tuple(q[1:]) for q in qs])
    so = o.solver_options()
    _engine.ka_run(b1, _capi.default_interp(), so)
    prob = dict(kp_begin=b2.kp_begin, patch_blocks=[q[1].patches for q in qs], patches_are_sparse=b2.sparse,
                keypoints=b2.keypoints, kp_patch=b2.kp_patch_local, desc_begin=b2.desc_begin, descs=b2.ref_desc,
                corner=b2.corner, scale=b2.scale, bound=4.0)
    ctx = pb.Context(-1)
    out = pb.qka_run(ctx, prob, {}, {"loss_type": so.loss_type, "loss_scale": so.loss_scale,
                                     "parameter_tolerance": so.parameter_tolerance,
                                     "max_num_iterations": so.max_num_iterations})
    assert np.array_equal(b1.keypoints, b2.keypoints)
    for r1, r2 in zip(b1.results, out["results"]):
        assert r1["final_cost"] == r2["final_cost"] and r1["num_iterations"] == r2["num_iterations"]
    # nearest candidate: the same rows, distances and descriptors as _engine.query_match_run
    iq = [k % 4 for k in range(12)]
    ip = [k % len(qs[k % 4][0]) for k in range(12)]
    xy = [qs[q][0][i] for q, i in zip(iq, ip)]
    cand = rng.standard_normal((40, 64))
    cb = np.arange(12) * 3; ce = cb + 4
    best, dmin, desc = _engine.query_match_run([q[1].patches for q in qs], b2.corner, b2.scale, iq, ip, xy, cb, ce, cand,
                                               _capi.default_interp(), with_desc=True)
    m = pb.query_match_run(ctx, dict(patch_blocks=[q[1].patches for q in qs], corner=b2.corner, scale=b2.scale,
                                     item_query=np.array(iq, np.int32), item_patch=np.array(ip, np.int64),
                                     xy=np.array(xy), cand_begin=cb.astype(np.int64), cand_end=ce.astype(np.int64),
                                     cand=cand))
    assert np.array_equal(m["best"], best) and np.array_equal(m["d_min"], dmin) and np.array_equal(m["desc"], desc)
