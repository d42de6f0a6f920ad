"""Absolute pose estimation on the GPU (csrc/pxr_pnp.cu) against the host restatement (tests/pnp_reference.py), a
float64 least-squares minimiser and the ground truth; the localizer's built-in PnP."""
import copy
import sys

import numpy as np
import pytest

import pnp_reference as P
from pixsfm._pixsfm import _capi, _engine, _localization as loc
from pixsfm.util import cameras, colmap_types as ct

pytestmark = pytest.mark.gpu

MODEL_PARAMS = {0: [500.0, 320.0, 240.0], 1: [500.0, 510.0, 320.0, 240.0], 2: [500.0, 320.0, 240.0, 0.01],
                3: [500.0, 320.0, 240.0, 0.01, -0.002], 4: [500.0, 510.0, 320.0, 240.0, 0.01, -0.002, 1e-4, -1e-4],
                5: [500.0, 510.0, 320.0, 240.0, 0.01, -0.002, 1e-3, -1e-3],
                6: [500.0, 510.0, 320.0, 240.0, 0.01, -0.002, 1e-4, -1e-4, 1e-3, 1e-4, 1e-5, 1e-6]}


def _cp(params):
    cp = np.zeros(12); cp[:len(params)] = params
    return cp


def _rot_deg(qa, qb):
    return np.degrees(2 * np.arccos(min(1.0, abs(float(np.dot(qa / np.linalg.norm(qa), qb / np.linalg.norm(qb)))))))


def scene(model, n, outlier_frac, seed, noise=0.5, far_outliers=36.0):
    """n correspondences seen by a random camera; a fraction are outliers at least `far_outliers` px from the true
    projection -> (points2D, points3D, params, qvec, tvec, is_outlier)"""
    rng = np.random.default_rng(seed)
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    if q[0] < 0:
        q = -q
    t = rng.normal(size=3)
    R = P.quat_to_rot(q)
    uv = rng.uniform(-0.5, 0.5, (n, 2))
    depth = rng.uniform(4.0, 8.0, n)
    Xc = np.column_stack([uv * depth[:, None], depth])
    X = (Xc - t) @ R
    params = np.asarray(MODEL_PARAMS[model], np.float64)
    xy = cameras.world_to_image(model, params, q, t, X) + rng.normal(0, noise, (n, 2))
    out = rng.random(n) < outlier_frac
    for i in np.nonzero(out)[0]:
        while True:
            cand = rng.uniform([0, 0], [640, 480])
            if np.linalg.norm(cand - xy[i]) > far_outliers:
                xy[i] = cand
                break
    return xy, X, params, q, t, out


def run(queries, **kw):
    """queries: (points2D, points3D, model, params, seed) -> (batch, results)"""
    begin = np.cumsum([0] + [len(q[0]) for q in queries])
    batch = _capi.PnPBatch(begin, np.concatenate([q[0] for q in queries]).reshape(-1, 2),
                           np.concatenate([q[1] for q in queries]).reshape(-1, 3), [q[2] for q in queries],
                           [_cp(q[3]) for q in queries], np.array([q[4] for q in queries], np.uint64))
    res, _ = _engine.pnp_run(batch, _capi.default_pnp_options(**kw))
    return batch, res


# ---- image to world
GRID = [(0, [655.123, 386.123, 511.123]), (1, [651.123, 655.123, 386.123, 511.123]),
        (2, [651.123, 386.123, 511.123, 0.0]), (2, [651.123, 386.123, 511.123, 0.1]),
        (3, [651.123, 386.123, 511.123, 0.0, 0.0]), (3, [651.123, 386.123, 511.123, 0.1, 0.0]),
        (3, [651.123, 386.123, 511.123, 0.05, 0.0]), (3, [651.123, 386.123, 511.123, 0.05, 0.03]),
        (4, MODEL_PARAMS[4]), (4, [651.123, 655.123, 386.123, 511.123, 0.1, 0.02, 1e-3, -2e-3]),
        (5, MODEL_PARAMS[5]), (5, [651.123, 655.123, 386.123, 511.123, 0.1, 0.02, 1e-2, -1e-3]),
        (6, MODEL_PARAMS[6]), (6, [651.123, 655.123, 386.123, 511.123, 0.1, 0.02, 1e-3, -2e-3, 1e-2, 1e-3, 1e-3, 1e-4])]


@pytest.mark.parametrize("model,params", GRID)
def test_image_to_world_round_trips_through_world_to_image(model, params):
    g = np.arange(-0.5, 0.5001, 0.1)
    uv = np.array([(u, v) for u in g for v in g])
    X = np.column_stack([uv, np.ones(len(uv))])
    q, t = np.array([1.0, 0, 0, 0]), np.zeros(3)
    xy = cameras.world_to_image(model, np.asarray(params), q, t, X)
    back = _engine.pnp_debug_image_to_world(model, params, xy)
    again = cameras.world_to_image(model, np.asarray(params), q, t, np.column_stack([back, np.ones(len(back))]))
    assert np.abs(again - xy).max() < 1e-9
    assert np.abs(back - uv).max() < 1e-9


# ---- P3P
def test_p3p_matches_the_restatement():
    rng = np.random.default_rng(1)
    xs, Xs = [], []
    for _ in range(500):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        R, t = P.quat_to_rot(q), rng.normal(size=3)
        Xc = np.column_stack([rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3), rng.uniform(2, 6, 3)])
        Xs.append((Xc - t) @ R); xs.append(Xc[:, :2] / Xc[:, 2:])
    poses, n_sol = _engine.pnp_debug_p3p(np.array(xs), np.array(Xs))
    for k in range(len(xs)):
        ref = P.p3p(xs[k], Xs[k])
        assert n_sol[k] == len(ref)
        for s in range(n_sol[k]):
            qd, td = poses[k, s, :4], poses[k, s, 4:]
            Y = Xs[k] @ P.quat_to_rot(qd).T + td
            assert np.abs(Y[:, :2] / Y[:, 2:] - xs[k]).max() < 1e-10
            assert min(max(np.abs(qd - P.rot_to_quat(Rr)).max(), np.abs(td - tr).max()) for Rr, tr in ref) < 1e-8


# ---- RANSAC against the restatement
@pytest.mark.parametrize("model", range(7))
@pytest.mark.parametrize("n", [3, 8, 50, 500, 5000])
@pytest.mark.parametrize("outliers", [0.0, 0.5, 0.8])
def test_ransac_matches_the_restatement(model, n, outliers):
    seed = 1000 * model + 10 * n + int(outliers * 10)
    xy, X, params, q, t, _ = scene(model, n, outliers, seed)
    batch, res = run([(xy, X, model, params, seed)], refine=0)
    r = res[0]
    uv = _engine.pnp_debug_image_to_world(model, params, xy)          # the kernel's normalised points
    f = params[0] if model in (0, 2, 3) else 0.5 * (params[0] + params[1])
    thr = 12.0 / f
    ref = P.ransac(uv, X, thr, seed)
    if ref is None:
        assert not r["success"] and r["num_trials"] == 0
        return
    assert r["num_trials"] == ref["num_trials"]
    assert (r["best_trial"], r["best_solution"]) == (ref["trial"], ref["solution"])
    if ref["count"] < 3:
        assert not r["success"]
        return
    assert r["success"] and bool(r["local_optimized"]) == ref["lo"]
    assert np.abs(batch.qvec[0] - P.rot_to_quat(ref["R"])).max() < 1e-9 and np.abs(batch.tvec[0] - ref["t"]).max() < 1e-9
    res2, front = P.residuals(ref["R"], ref["t"], uv, X)
    differ = (batch.inlier_mask.astype(bool) != ref["inliers"])
    assert np.all(np.abs(res2[differ] - thr * thr) <= 1e-9 * thr * thr)
    assert abs(r["num_inliers"] - ref["count"]) == differ.sum()


# ---- refinement against a float64 minimiser of the same objective
@pytest.mark.parametrize("model,focal,extra", [(1, False, False), (2, True, False), (4, True, True), (3, False, True)])
def test_refinement_minimises_the_cauchy_pixel_objective(model, focal, extra):
    from scipy.optimize import least_squares
    seed = 77 + model
    xy, X, params, q, t, _ = scene(model, 150, 0.2, seed, noise=1.0)
    b0, _ = run([(xy, X, model, params, seed)], refine=0)
    inl = b0.inlier_mask.astype(bool)
    # COLMAP's tolerances stop the solve near, not at, the minimum: switched off here to compare with the minimiser
    kw = dict(refine=1, gradient_tolerance=0.0, function_tolerance=0.0, parameter_tolerance=0.0, max_num_iterations=200,
              refine_focal_length=int(focal), refine_extra_params=int(extra))
    b, res = run([(xy, X, model, params, seed)], **kw)
    assert res[0]["success"] and res[0]["status"] == 0 and res[0]["final_cost"] < res[0]["initial_cost"]
    nf = 1 if model in (0, 2, 3) else 2
    free = [k for k in range(len(params)) if (k < nf and focal) or (k >= nf + 2 and extra)]
    q0 = b0.qvec[0]

    def unpack(z):
        w = z[:3]
        th = np.linalg.norm(w)
        dq = np.r_[np.cos(th), np.sinc(th / np.pi) * w] if th > 0 else np.array([1.0, 0, 0, 0])
        qq = np.array([dq[0] * q0[0] - dq[1:] @ q0[1:], *(dq[0] * q0[1:] + q0[0] * dq[1:] + np.cross(dq[1:], q0[1:]))])
        p = params.copy(); p[free] = z[6:]
        return qq, z[3:6], p

    def resid(z):        # one residual per correspondence: sqrt(rho(|r|^2)), Cauchy on the 2-vector as ceres applies it
        qq, tt, p = unpack(z)
        r = cameras.world_to_image(model, p, qq, tt, X[inl]) - xy[inl]
        return np.sqrt(np.log1p((r * r).sum(1)))

    z0 = np.r_[np.zeros(3), b0.tvec[0], params[free]]
    sol = least_squares(resid, z0, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15, max_nfev=5000)
    qs, ts, ps = unpack(sol.x)
    qs = qs * np.sign(qs[0])
    assert np.abs(b.qvec[0] - qs).max() < 1e-6
    assert np.abs(b.tvec[0] - ts).max() <= 1e-6 * max(1.0, np.abs(ts).max())
    # the objective is flat along the distortion coefficients: compare the minimum and what the intrinsics do to the
    # inliers' projections rather than each coefficient
    assert res[0]["final_cost"] <= sol.cost * (1 + 1e-9)
    nf_free = [k for k in free if k < nf]
    assert np.all(np.abs(b.cam_params[0, nf_free] - ps[nf_free]) <= 1e-6 * np.abs(ps[nf_free]))
    proj_dev = cameras.world_to_image(model, b.cam_params[0, :len(params)], b.qvec[0], b.tvec[0], X[inl])
    proj_ref = cameras.world_to_image(model, ps, qs, ts, X[inl])
    assert np.abs(proj_dev - proj_ref).max() < 1e-4
    if not free:
        assert np.array_equal(b.cam_params[0, :len(params)], params)


# ---- accuracy and failures
@pytest.mark.parametrize("model", range(7))
def test_pose_is_near_the_ground_truth_and_far_outliers_are_rejected(model):
    xy, X, params, q, t, out = scene(model, 1000, 0.4, 5 + model)
    b, res = run([(xy, X, model, params, 5)])
    assert res[0]["success"]
    assert _rot_deg(b.qvec[0], q) < 0.1
    c_gt, c = -P.quat_to_rot(q).T @ t, -P.quat_to_rot(b.qvec[0]).T @ b.tvec[0]
    scale = np.linalg.norm(X - c_gt, axis=1).mean()              # the scene's distance from the camera
    assert np.linalg.norm(c - c_gt) < 1e-3 * scale
    assert not np.any(b.inlier_mask.astype(bool) & out)          # every outlier is > 3 max_error from its projection
    assert res[0]["num_inliers"] == int(b.inlier_mask.sum())


def test_failures_leave_pose_and_camera_untouched():
    rng = np.random.default_rng(4)
    xy, X, params, q, t, _ = scene(1, 40, 0.0, 8)
    few = (xy[:2], X[:2], 1, params, 1)
    junk = (rng.uniform([0, 0], [640, 480], (40, 2)), rng.normal(size=(40, 3)) + [0, 0, 6], 1, params, 2)
    line = (xy[:20], np.outer(np.linspace(-1, 1, 20), [1.0, 0.5, 0.2]) + [0, 0, 5], 1, params, 3)
    b, res = run([few, junk, line], min_inlier_ratio=0.25, refine_focal_length=1)
    assert not res[0]["success"] and res[0]["num_trials"] == 0
    assert not res[1]["success"]                 # any minimal sample is its own three inliers: below the ratio asked
    assert not res[2]["success"] or (np.all(np.isfinite(b.qvec[2])) and np.all(np.isfinite(b.tvec[2])))
    for k in (0, 1):
        assert np.array_equal(b.qvec[k], [1.0, 0, 0, 0]) and np.array_equal(b.tvec[k], np.zeros(3))
        assert np.array_equal(b.cam_params[k], _cp(params))
    assert not b.inlier_mask[:2].any() and not b.inlier_mask[2:42].any()


def test_points_behind_the_camera_are_never_inliers():
    xy, X, params, q, t, _ = scene(0, 200, 0.0, 12)
    R = P.quat_to_rot(q)
    Xc = X @ R.T + t
    behind = np.arange(200) % 4 == 0
    Xb = X.copy()
    Xb[behind] = ((-Xc[behind]) - t) @ R        # the mirror point projects to the same pixel, behind the camera
    b, res = run([(xy, Xb, 0, params, 3)])
    assert res[0]["success"]
    assert not np.any(b.inlier_mask.astype(bool) & behind)
    assert _rot_deg(b.qvec[0], q) < 0.1


# ---- batch independence and determinism
def test_each_query_is_independent_of_its_batch_and_deterministic():
    rng = np.random.default_rng(21)
    qs = []
    for k in range(1000):
        model = int(rng.integers(0, 7))
        n = int(rng.choice([3, 5, 20, 80, 300, 600]))
        xy, X, params, _, _, _ = scene(model, n, float(rng.choice([0.0, 0.3, 0.6])), 5000 + k)
        qs.append((xy, X, model, params, int(rng.integers(0, 2 ** 63))))
    b1, r1 = run(qs)
    b2, r2 = run(qs)
    assert r1 == r2
    for f in ("qvec", "tvec", "cam_params", "inlier_mask"):
        assert np.array_equal(getattr(b1, f), getattr(b2, f))
    begin = np.cumsum([0] + [len(q[0]) for q in qs])
    for k in list(range(0, 1000, 50)) + [999]:
        b, r = run([qs[k]])
        assert r[0] == r1[k]
        assert np.array_equal(b.qvec[0], b1.qvec[k]) and np.array_equal(b.tvec[0], b1.tvec[k])
        assert np.array_equal(b.inlier_mask, b1.inlier_mask[begin[k]:begin[k + 1]])


def test_absolute_pose_estimation_returns_pycolmaps_dict():
    xy, X, params, q, t, out = scene(2, 120, 0.3, 31)
    cam = ct.Camera(1, 2, 640, 480, params)
    r = loc.absolute_pose_estimation(xy, X, cam, {"ransac": {"max_error": 12}}, {})
    assert set(r) == {"success", "qvec", "tvec", "num_inliers", "inliers"} and r["success"]
    assert len(r["inliers"]) == 120 and r["num_inliers"] == sum(r["inliers"])
    assert np.array_equal(cam.params, params)
    assert _rot_deg(r["qvec"], q) < 0.1
    r2 = loc.absolute_pose_estimation(xy, X, cam, None, {"refine_focal_length": True})
    assert r2["success"] and cam.params[0] != params[0] and np.array_equal(cam.params[1:], params[1:])
    assert loc.absolute_pose_estimation(xy[:2], X[:2], cam) == {"success": False}


# ---- the localizer with nothing but the built-in estimator
def test_localizer_uses_the_built_in_estimator_in_one_batched_call(monkeypatch):
    from pixsfm import bundle_adjustment as ba_pkg, localization as loc_pkg
    from pixsfm._pixsfm import _bundle_adjustment as ba
    from recon_util import make_reconstruction
    monkeypatch.setitem(sys.modules, "pycolmap", None)               # `import pycolmap` raises ImportError
    rec, fm, prob, gt = make_reconstruction(n_cams=6, n_points=60, track_len=4, channels=128, seed=15)
    labels = ba_pkg.find_problem_labels(rec, 10)
    refs = ba.ReferenceExtractor({"iters": 100, "keep_observations": True}, {}).run(labels, rec, fm.fset(0))
    rng = np.random.default_rng(2)
    qids = sorted(rec.images)[:4]
    queries = []
    for qid in qids:
        img = rec.images[qid]
        p2D_idxs = [i for i, p in enumerate(img.points2D) if p.has_point3D()]
        p3D_ids = [img.points2D[i].point3D_id for i in p2D_idxs]
        kps = np.array([p.xy for p in img.points2D], np.float64) + rng.normal(0, 0.3, (len(img.points2D), 2))
        queries.append(dict(keypoints=kps, pnp_point2D_idxs=p2D_idxs, pnp_points3D_id=p3D_ids,
                            query_camera=copy.deepcopy(rec.cameras[img.camera_id]), query_fmaps=[fm.fset(0).fmap(img.name)]))

    def fresh(qs):
        return [dict(q, query_camera=copy.deepcopy(q["query_camera"])) for q in qs]

    calls = []
    real = _engine.pnp_run
    monkeypatch.setattr(_engine, "pnp_run", lambda *a, **k: (calls.append(1), real(*a, **k))[1])
    # QBA off: what localize returns is the PnP pose, so batched and per-query PnP must agree bit for bit
    ql = loc_pkg.QueryLocalizer(rec, {"target_reference": "robust_mean", "QBA": {"apply": False}}, references=[refs])
    single = [ql.localize(**q) for q in fresh(queries)]
    assert len(calls) == len(queries)
    calls.clear()
    batch = ql.localize_batch(fresh(queries))
    assert len(calls) == 1
    for s, b in zip(single, batch):
        assert s["success"] and b["success"]
        assert np.array_equal(s["qvec"], b["qvec"]) and np.array_equal(s["tvec"], b["tvec"])
        assert s["inliers"] == b["inliers"] and np.array_equal(s["keypoints"], b["keypoints"])
    # the whole pipeline: QKA, built-in PnP, QBA
    calls.clear()
    full = loc_pkg.QueryLocalizer(rec, {"target_reference": "robust_mean"}, references=[refs]).localize_batch(fresh(queries))
    assert len(calls) == 1
    for qid, r, s in zip(qids, full, single):
        img = rec.images[qid]
        c_gt = -P.quat_to_rot(img.qvec).T @ img.tvec
        scale = np.linalg.norm(np.array([rec.points3D[p].xyz for p in rec.points3D]) - c_gt, axis=1).mean()
        for pose, deg, rel in ((r, 0.25, 1e-2), (s, 0.5, 2e-2)):    # after QBA, and the PnP pose QBA starts from
            assert pose["success"] and _rot_deg(pose["qvec"], img.qvec) < deg
            assert np.linalg.norm(-P.quat_to_rot(pose["qvec"]).T @ pose["tvec"] - c_gt) < rel * scale


def test_pybind_pnp_run_matches_the_ctypes_path():
    sys.path.insert(0, str(__import__("pathlib").Path(__file__).resolve().parents[1] / "pixel-perfect-sfm_b200" / "bindings"))
    pb = pytest.importorskip("_pxr_pybind")
    qs = [scene(m, 200, 0.3, 40 + m)[:3] for m in (1, 4)]
    b, res = run([(xy, X, m, p, 9) for (xy, X, p), m in zip(qs, (1, 4))])
    prob = dict(corr_begin=b.corr_begin, points2D=b.points2D, points3D=b.points3D, cam_model=b.cam_model,
                cam_params=np.array([_cp(q[2]) for q in qs]), seed=np.full(2, 9, np.uint64),
                qvec=np.tile([1.0, 0, 0, 0], (2, 1)), tvec=np.zeros((2, 3)), inlier_mask=np.zeros(400, np.uint8))
    out = pb.pnp_run(pb.Context(-1), prob, {"max_error": 12.0})
    assert [r["success"] for r in out["results"]] == [True, True]
    assert np.array_equal(prob["qvec"], b.qvec) and np.array_equal(prob["tvec"], b.tvec)
    assert np.array_equal(prob["inlier_mask"], b.inlier_mask)
    with pytest.raises(ValueError):
        pb.pnp_run(pb.Context(-1), prob, {"max_eror": 12.0})
