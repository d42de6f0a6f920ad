"""Batched query bundle adjustment (pxr_qba_run, QueryBundleOptimizer.run_batch) against the single-query path
(pxr_ba_run per query) and the handle's linearisation: many queries in one launch, each with the decisions and results
it gets alone."""
import copy

import numpy as np
import pytest

from pixsfm import bundle_adjustment as ba_pkg
from pixsfm._pixsfm import _bundle_adjustment as ba
from pixsfm._pixsfm import _capi, _engine, _features, _localization as loc
from pixsfm.util import colmap_types as ct
from recon_util import make_reconstruction

pytestmark = pytest.mark.gpu

_CACHE = {}


def _scene(seed, n_cams=6, n_points=60, channels=128):
    key = (seed, n_cams, n_points, channels)
    if key not in _CACHE:
        rec, fm, _, _ = make_reconstruction(n_cams=n_cams, n_points=n_points, track_len=4, channels=channels, seed=seed)
        labels = ba_pkg.find_problem_labels(rec, 10)
        refs = ba.ReferenceExtractor({"iters": 100, "keep_observations": True}, {}).run(labels, rec, fm.fset(0))
        _CACHE[key] = (rec, fm, refs)
    return _CACHE[key]


def _queries(seeds=(15, 16), n_points=60, channels=128, models=("SIMPLE_RADIAL", "PINHOLE", "RADIAL", "OPENCV"), pert=1.0):
    """one query per image of several scenes: mixed camera models, inlier masks, robust-mean and all-observation
    references, perturbed poses"""
    qs = []
    for seed in seeds:
        rec, fm, refs = _scene(seed, n_points=n_points, channels=channels)
        rng = np.random.default_rng(seed)
        for k, (iid, img) in enumerate(sorted(rec.images.items())):
            fmap = fm.fset(0).fmap(img.name)
            p2D = [i for i, p in enumerate(img.points2D) if p.has_point3D()]
            p3D = [img.points2D[i].point3D_id for i in p2D]
            cam0 = rec.cameras[img.camera_id]
            f, cx, cy = cam0.params[:3]
            model = models[(k + seed) % len(models)]
            params = {"SIMPLE_RADIAL": [f, cx, cy, cam0.params[3]], "PINHOLE": [f, f, cx, cy],
                      "RADIAL": [f, cx, cy, cam0.params[3], 0.0], "OPENCV": [f, f, cx, cy, cam0.params[3], 0.0, 0.0, 0.0]}[model]
            cam = ct.Camera(cam0.camera_id, model, cam0.width, cam0.height, np.array(params, np.float64))
            qvec = img.qvec + rng.normal(0, 2e-4 * pert, 4); qvec /= np.linalg.norm(qvec)
            tvec = img.tvec + rng.normal(0, 2e-3 * pert, 3)
            pts = [rec.points3D[p].xyz.copy() for p in p3D]
            if k % 2:
                r = [[o for o in refs[p].observations] for p in p3D]
            else:
                r = []
                for p in p3D:
                    x = copy.copy(refs[p]); x.observations = []; r.append(x)
            inliers = [j % (3 + k % 3) != 0 for j in range(len(p3D))] if k % 3 else None
            qs.append((qvec, tvec, cam, pts, fmap, r, inliers, p2D))
    return qs


def _copy(q):
    return (q[0].copy(), q[1].copy(), copy.deepcopy(q[2])) + tuple(q[3:])


def _opt(**kw):
    o = {"solver": {"max_num_iterations": 30}}
    o.update(kw)
    return o


CASES = {
    "pose": _opt(),
    "focal": _opt(refine_focal_length=True),
    "pp_extra": _opt(refine_principal_point=True, refine_extra_params=True),
    "nonmonotonic": _opt(refine_focal_length=True, solver={"max_num_iterations": 30, "use_nonmonotonic_steps": True,
                                                           "max_consecutive_nonmonotonic_steps": 3}),
    "trivial": _opt(refine_focal_length=True, loss={"name": "trivial", "params": []}),
    "huber": _opt(refine_focal_length=True, loss={"name": "huber", "params": [0.1]}),
    "soft_l1": _opt(refine_focal_length=True, loss={"name": "soft_l1", "params": [0.1]}),
    "arctan": _opt(refine_focal_length=True, loss={"name": "arctan", "params": [0.1]}),
}


def _single(opts, interp, qs):
    out = []
    for q in qs:
        c = _copy(q)
        qbo = loc.QueryBundleOptimizer(opts, interp)
        ok = qbo.run(c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7])
        out.append((ok, c, qbo.summary()))
    return out


def _batch(opts, interp, qs, **kw):
    cs = [_copy(q) for q in qs]
    qbo = loc.QueryBundleOptimizer(opts, interp)
    ok = qbo.run_batch(cs, **kw)
    return ok, cs, qbo.summaries()


@pytest.mark.parametrize("case", sorted(CASES))
def test_batch_matches_single_query_path(case):
    qs = _queries(pert=5.0 if case in ("pose", "nonmonotonic") else 1.0)
    interp = {}
    single = _single(CASES[case], interp, qs)
    ok, cs, sums = _batch(CASES[case], interp, qs)
    assert any(s.num_successful_steps > 0 for _, _, s in single)          # the comparison covers LM steps
    for k, ((ok1, c1, s1), c2, s2) in enumerate(zip(single, cs, sums)):
        assert ok1 and ok[k]
        assert s2.num_iterations == s1.num_iterations, k
        assert (s2.num_successful_steps, s2.num_unsuccessful_steps, s2.termination_type) == \
            (s1.num_successful_steps, s1.num_unsuccessful_steps, s1.termination_type), k
        assert abs(s2.initial_cost - s1.initial_cost) <= 1e-12 * s1.initial_cost
        assert abs(s2.final_cost - s1.final_cost) <= 1e-6 * s1.final_cost
        assert np.abs(c2[0] - c1[0]).max() < 1e-6 and np.abs(c2[1] - c1[1]).max() < 1e-6
        assert np.all(np.abs(c2[2].params - c1[2].params) <= 1e-6 * np.maximum(1.0, np.abs(c1[2].params)))


def test_float_simd_matches_single_query_path():
    qs = _queries(seeds=(15,))
    interp = {"use_float_simd": True}
    single = _single(CASES["focal"], interp, qs)
    ok, cs, sums = _batch(CASES["focal"], interp, qs)
    for (ok1, c1, s1), c2, s2 in zip(single, cs, sums):
        assert s2.num_iterations == s1.num_iterations and abs(s2.final_cost - s1.final_cost) <= 1e-6 * s1.final_cost
        assert np.abs(c2[0] - c1[0]).max() < 1e-6 and np.abs(c2[1] - c1[1]).max() < 1e-6


@pytest.mark.parametrize("case", ["pose", "pp_extra"])
def test_linearisation_matches_single_query_handle(case):
    qs = _queries()
    qbo = loc.QueryBundleOptimizer(CASES[case], {})
    batch = qbo.pack_batch(qs)
    so = qbo.solver_options()
    ic = _capi.default_interp()
    lin = _engine.qba_debug_linearize(batch, ic, so)
    for k, q in enumerate(qs):
        prob = qbo.build_problem(*_copy(q)[:6], q[6], q[7])
        nc = 6 + bin(~int(batch.cam_const_mask[k]) & ((1 << _capi.CAMERA_NUM_PARAMS[int(batch.cam_model[k])]) - 1)).count("1")
        h = _engine.BAHandle(prob, ic, so)
        ref = h.debug_linearize(nc, nc)
        ev = h.evaluate()
        h.close()
        b0, b1 = batch.obs_begin[k], batch.obs_begin[k + 1]
        assert abs(lin["cost"][k] - ref["cost"]) <= 1e-12 * ref["cost"]
        H = np.tril(lin["H"][k, :nc, :nc]); Href = np.tril(ref["Hcc"])
        assert np.abs(H - Href).max() <= 1e-9 * np.abs(Href).max()
        assert np.abs(lin["g"][k, :nc] - ref["gc"]).max() <= 1e-9 * np.abs(ref["gc"]).max()
        rec = lin["rec"][b0:b1]
        # the records are K1's bit for bit; xy to 1e-12 (world_to_pixel may be contracted differently in the two kernels)
        assert np.array_equal(rec[:, 0], ev["sq_norm"]) and np.array_equal(rec[:, 1:3], ev["gtr"])
        assert np.array_equal(rec[:, 3:6], ev["gtg"])
        assert np.abs(lin["xy"][b0:b1] - ev["xy"]).max() <= 1e-12 * np.abs(ev["xy"]).max()


def _run_raw(qs, order, opts=CASES["focal"], max_wave_bytes=0.0):
    cs = [_copy(qs[i]) for i in order]
    qbo = loc.QueryBundleOptimizer(opts, {})
    batch = qbo.pack_batch(cs, max_wave_bytes)
    res, tot = _engine.qba_run(batch, _capi.default_interp(), qbo.solver_options())
    out = {}
    for j, i in enumerate(order):
        out[i] = (batch.qvec[j].copy(), batch.tvec[j].copy(), batch.cam_params[j].copy(), res[j]["final_cost"],
                  res[j]["num_iterations"])
    return out, tot


def test_query_results_do_not_depend_on_the_batch():
    qs = _queries()
    n = len(qs)
    full, tot = _run_raw(qs, list(range(n)))
    assert tot["n_waves"] == 1
    rev, _ = _run_raw(qs, list(range(n))[::-1])
    waves, tw = _run_raw(qs, list(range(n)), max_wave_bytes=1.0)      # every query a wave of its own
    assert tw["n_waves"] == n
    for i in range(n):
        alone, _ = _run_raw(qs, [i])
        for other in (rev, waves, alone):
            for a, b in zip(full[i], other[i]):
                assert np.array_equal(a, b), i


def test_device_patches_match_host_patches():
    torch = pytest.importorskip("torch")
    qs = _queries(seeds=(15,))
    dev = []
    for q in qs:
        fm = q[4]
        t = torch.from_numpy(np.ascontiguousarray(fm.patches)).cuda()
        dmap = _features.FeatureMap(t, fm.point2D_ids, fm.corners, {"scale": fm.scale, "is_sparse": fm.is_sparse})
        dev.append(q[:4] + (dmap,) + q[5:])
    host, th = _run_raw(qs, list(range(len(qs))))
    devr, td = _run_raw(dev, list(range(len(qs))))
    per_patch = int(np.prod(qs[0][4].patches.shape[1:])) * qs[0][4].patches.dtype.itemsize
    host_patch_bytes = sum(q[4].size() for q in qs) * per_patch
    assert th["h2d_bytes"] - td["h2d_bytes"] == host_patch_bytes       # device blocks are read in place
    for i in host:
        for a, b in zip(host[i], devr[i]):
            assert np.array_equal(a, b)
    with pytest.raises(ValueError):            # run() keeps taking host feature maps only
        c = _copy(dev[0])
        loc.QueryBundleOptimizer(CASES["pose"], {}).run(*c[:6], c[6], c[7])


def test_edge_cases_are_per_query():
    qs = _queries(seeds=(15,))
    empty = qs[1][:6] + ([False] * len(qs[1][3]), qs[1][7])             # every correspondence an outlier: no block
    one = qs[2][:6] + ([j == 0 for j in range(len(qs[2][3]))], qs[2][7])  # a single residual block
    bad_pts = [p.copy() for p in qs[3][3]]
    bad_pts[0][:] = np.nan
    bad = qs[3][:3] + (bad_pts,) + qs[3][4:]                            # non-finite initial cost
    batch = [qs[0], empty, one, bad, qs[4]]
    cs = [_copy(q) for q in batch]
    qbo = loc.QueryBundleOptimizer(CASES["pose"], {})
    with pytest.raises(_capi.PxrError, match="query 3"):
        qbo.run_batch(cs)
    assert np.array_equal(cs[1][0], batch[1][0]) and np.array_equal(cs[1][1], batch[1][1])    # untouched
    assert np.array_equal(cs[3][0], batch[3][0])
    sums = qbo.summaries()
    assert sums[1] is None and sums[3] is None and sums[2].num_residual_blocks == 1
    # the others are what they are without the odd ones
    ok = loc.QueryBundleOptimizer(CASES["pose"], {}).run_batch([_copy(qs[0]), _copy(qs[4]), _copy(one)])
    alone, _ = _run_raw([qs[0], qs[4], one], [0, 1, 2], CASES["pose"])
    assert ok == [True, True, True]
    for j, k in ((0, 0), (4, 1), (2, 2)):
        assert np.array_equal(cs[j][0], alone[k][0]) and np.array_equal(cs[j][1], alone[k][1])
    empty_only = loc.QueryBundleOptimizer(CASES["pose"], {}).run_batch([_copy(empty)])
    assert empty_only == [False]


@pytest.mark.parametrize("dtype,channels", [("float16", 8), ("float16", 16), ("float16", 32), ("float16", 64), ("float16", 256),
                                           ("float32", 16), ("float32", 64), ("float32", 128), ("float64", 16),
                                           ("float64", 128)])
def test_other_instances_match_single_query_path(dtype, channels):
    qs = _queries(seeds=(17,), n_points=40, channels=channels, models=("SIMPLE_RADIAL",))
    conv = []
    for q in qs:
        fm = q[4]
        f2 = _features.FeatureMap(np.ascontiguousarray(fm.patches.astype(dtype)), fm.point2D_ids, fm.corners,
                                  {"scale": fm.scale, "is_sparse": fm.is_sparse})
        conv.append(q[:4] + (f2,) + q[5:])
    single = _single(CASES["focal"], {}, conv)
    ok, cs, sums = _batch(CASES["focal"], {}, conv)
    for (ok1, c1, s1), c2, s2 in zip(single, cs, sums):
        assert s2.num_iterations == s1.num_iterations and abs(s2.final_cost - s1.final_cost) <= 1e-6 * s1.final_cost
        assert np.abs(c2[0] - c1[0]).max() < 1e-6 and np.abs(c2[1] - c1[1]).max() < 1e-6


def test_one_wave_buffer_over_many_waves(monkeypatch):
    """with one wave buffer every wave reuses the arena of the one before: each wave's outputs must be read back before
    the next upload overwrites them"""
    qs = _queries()
    full, _ = _run_raw(qs, list(range(len(qs))))
    monkeypatch.setenv("PXR_QBA_WAVE_BUFFERS", "1")
    waves, tw = _run_raw(qs, list(range(len(qs))), max_wave_bytes=1.0)
    assert tw["n_waves"] == len(qs)
    for i in full:
        for a, b in zip(full[i], waves[i]):
            assert np.array_equal(a, b), i


def test_pybind_qba_run_matches_ctypes():
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pixel-perfect-sfm_b200",
                                    "bindings"))
    pb = pytest.importorskip("_pxr_pybind")
    qs = _queries(seeds=(15,))
    qbo = loc.QueryBundleOptimizer(CASES["focal"], {})
    b1 = qbo.pack_batch([_copy(q) for q in qs])
    b2 = qbo.pack_batch([_copy(q) for q in qs])
    res, _ = _engine.qba_run(b1, _capi.default_interp(), qbo.solver_options())
    so = qbo.solver_options()
    prob = dict(cam_model=b2.cam_model, cam_params=b2.cam_params, cam_const_mask=b2.cam_const_mask, qvec=b2.qvec, tvec=b2.tvec,
                obs_begin=b2.obs_begin, xyz=b2.xyz, obs_patch=b2.obs_patch, refs=b2.refs,
                patch_blocks=[q[4].patches for q in qs], corner=b2.corner, scale=b2.scale)
    out = pb.qba_run(pb.Context(-1), prob, {}, {"loss_type": so.loss_type, "loss_scale": so.loss_scale,
                                                "parameter_tolerance": so.parameter_tolerance,
                                                "max_num_iterations": so.max_num_iterations})
    assert out["n_waves"] == 1
    assert np.array_equal(b1.qvec, b2.qvec) and np.array_equal(b1.tvec, b2.tvec) and np.array_equal(b1.cam_params, b2.cam_params)
    for r1, r2 in zip(res, out["results"]):
        assert r1["final_cost"] == r2["final_cost"] and r1["num_iterations"] == r2["num_iterations"]


def _localizer_scene():
    from pixsfm import localization as loc_pkg
    rec, fm, refs = _scene(21, n_cams=8)
    qs, pnp_poses = [], {}
    rng = np.random.default_rng(21)
    for k, (iid, img) in enumerate(sorted(rec.images.items())):
        p2D = [i for i, p in enumerate(img.points2D) if p.has_point3D()]
        p3D = [img.points2D[i].point3D_id for i in p2D]
        kps = np.array([img.points2D[i].xy for i in p2D]) + rng.normal(0, 0.5, (len(p2D), 2))
        all_kps = np.zeros((max(p2D) + 1, 2)); all_kps[p2D] = kps
        pose = dict(success=True, qvec=img.qvec.copy(), tvec=img.tvec + rng.normal(0, 2e-3, 3),
                    inliers=[j % 5 != 1 for j in range(len(p2D))])

        def pnp(points2D, points3D, camera, pose=pose):        # stands in for pycolmap.absolute_pose_estimation
            return dict(pose, qvec=pose["qvec"].copy(), tvec=pose["tvec"].copy(), inliers=list(pose["inliers"]))
        qs.append(dict(keypoints=all_kps, pnp_point2D_idxs=p2D, pnp_points3D_id=p3D,
                       query_camera=copy.deepcopy(rec.cameras[img.camera_id]), query_fmaps=[fm.fset(0).fmap(img.name)],
                       pose_estimator=pnp))
    conf = {"target_reference": "robust_mean", "QBA": {"optimizer": {"refine_focal_length": True}}}
    return rec, refs, qs, lambda: loc_pkg.QueryLocalizer(rec, conf, references=[refs])


def test_localize_batch_matches_localize():
    rec, refs, qs, make = _localizer_scene()
    loop = [make().localize(**dict(q, query_camera=copy.deepcopy(q["query_camera"]))) for q in qs]
    batch = make().localize_batch([dict(q, query_camera=copy.deepcopy(q["query_camera"])) for q in qs])
    assert len(loop) == len(batch) == 8
    for a, b in zip(loop, batch):
        assert a["success"] and b["success"]
        assert np.abs(np.asarray(a["qvec"]) - np.asarray(b["qvec"])).max() < 1e-6
        assert np.abs(np.asarray(a["tvec"]) - np.asarray(b["tvec"])).max() < 1e-6
        assert a["inliers"] == b["inliers"] and a["num_inliers"] == b["num_inliers"]
        assert np.array_equal(a["keypoints"], b["keypoints"])


def test_refine_multilevel_batch_matches_loop():
    from pixsfm import localization as loc_pkg
    qs = _queries(seeds=(15,))
    conf = {"optimizer": {"refine_focal_length": True, "solver": {"max_num_iterations": 20}}}
    two = [(q[0], q[1], q[2], q[3], [q[4], q[4]], [q[5], q[5]], q[6], q[7]) for q in qs]     # two feature levels
    loop = [_copy(q) for q in two]
    for c in loop:
        loc_pkg.QueryBundleAdjuster(conf).refine_multilevel(c[0], c[1], c[2], c[3], c[4], c[5], inliers=c[6], point2D_idxs=c[7])
    bat = [_copy(q) for q in two]
    loc_pkg.QueryBundleAdjuster(conf).refine_multilevel_batch(bat)
    for a, b in zip(loop, bat):
        assert np.abs(a[0] - b[0]).max() < 1e-6 and np.abs(a[1] - b[1]).max() < 1e-6
        assert np.all(np.abs(a[2].params - b[2].params) <= 1e-6 * np.abs(a[2].params))
