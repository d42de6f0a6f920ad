"""Triangulation from known poses on the GPU (csrc/pxr_tri.cu) against the numpy restatement
(tests/triangulation_reference.py): verification for every camera model, RANSAC tracks of every size class, determinism
and independence of the launch, evaluate mode, `triangulation.main` end to end on hloc files, and
`refine_hloc.PixSfM.triangulation` from rendered images without hloc."""
import numpy as np
import pytest

import triangulation_reference as T
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util.cameras import normalized_to_image

pytestmark = pytest.mark.gpu

MODELS = sorted(T.CAMERAS)


def _scene(model, n_images, seed=0):
    qv, tv = T.ring_poses(n_images, seed=seed)
    return dict(model=model, qvec=qv, tvec=tv, params=np.array(T.CAMERAS[model]), f=T.mean_focal(model, T.CAMERAS[model]))


def _tri_scene(S, track_begin=None, obs_img=None, obs_xy=None, track_key=None):
    n = len(S["qvec"])
    return _capi.TriScene([S["model"]], [T.padded(S["params"])], np.zeros(n, np.int32), S["qvec"], S["tvec"], track_begin,
                          obs_img, obs_xy, track_key)


# ---- verification
def _matches(S, n_points, rng, outlier_rate=0.2):
    """matches between every image pair: normalised points with 0.3 px noise, outliers 40..100 px off"""
    X = rng.uniform(-1, 1, (n_points, 3))
    out = dict(img=[], xn=[], xy=[])
    n = len(S["qvec"])
    for i in range(n):
        for j in range(i + 1, n):
            xs = []
            for k in (i, j):
                xn = T.project_normalised(S["qvec"][k], S["tvec"][k], X) + rng.normal(0, 0.3 / S["f"], (n_points, 2))
                bad = rng.random(n_points) < outlier_rate
                ang = rng.uniform(0, 2 * np.pi, bad.sum())
                xn[bad] += (rng.uniform(40, 100, bad.sum()) / S["f"])[:, None] * np.column_stack([np.cos(ang), np.sin(ang)])
                xs.append(xn)
            out["img"].append(np.tile([i, j], (n_points, 1)))
            out["xn"].append(np.hstack(xs))
            out["xy"].append(np.hstack([normalized_to_image(S["model"], S["params"], x) for x in xs]))
    return {k: np.concatenate(v) for k, v in out.items()}


@pytest.mark.parametrize("model", MODELS)
def test_verification_matches_the_reference(model):
    rng = np.random.default_rng(model)
    S = _scene(model, 4, seed=model)
    M = _matches(S, 300, rng)
    noise = np.column_stack([np.ones(len(M["img"])), np.full(len(M["img"]), 0.5)])
    keep, err, _ = _engine.tri_verify(_tri_scene(S), M["img"], M["xy"], noise, 4.0)
    ref = np.zeros_like(err)
    for i, j in {tuple(p) for p in M["img"].tolist()}:
        sel = (M["img"][:, 0] == i) & (M["img"][:, 1] == j)
        ref[sel] = np.column_stack(T.epipolar_errors(M["xn"][sel, :2], M["xn"][sel, 2:], S["qvec"][i], S["tvec"][i],
                                                     S["qvec"][j], S["tvec"][j]))
    # the device's ImageToWorld inverts the distortion to ~1e-14 in the normalised plane: relative 1e-9 with a floor
    np.testing.assert_array_less(np.abs(err - ref), 1e-9 * np.abs(ref) + 1e-12)
    thr = noise * 4.0 / S["f"]
    far = (np.abs(ref - thr) * S["f"] >= 0.5).all(axis=1)         # decisions at least half a pixel from the threshold
    assert far.mean() > 0.9
    np.testing.assert_array_equal(keep[far], (ref <= thr).all(axis=1)[far])
    assert 0.3 < keep.mean() < 0.9


# ---- tracks
def _tracks(length, n_tracks, model=1, seed=0, outlier_rate=0.15, n_images=None):
    """n_tracks tracks of `length` observations in distinct images of an arc of `n_images` (default `length`) cameras:
    0.3 px noise, outliers 40..100 px off (none on two-view tracks) -> (scene, track_begin, obs_img, obs_xy, normalised
    obs, truth)"""
    rng = np.random.default_rng(seed * 1000 + length)
    n_images = n_images or length
    S = _scene(model, n_images, seed=seed)
    X = rng.uniform(-1, 1, (n_tracks, 3))
    obs_img = np.concatenate([np.sort(rng.choice(n_images, length, replace=False)) for _ in range(n_tracks)]).astype(np.int32)
    xn = np.concatenate([T.project_normalised(S["qvec"][k], S["tvec"][k], X[o // length][None])
                         for o, k in enumerate(obs_img)])
    xn += rng.normal(0, 0.3 / S["f"], xn.shape)
    bad = (rng.random(len(xn)) < outlier_rate) if length > 2 else np.zeros(len(xn), bool)
    ang = rng.uniform(0, 2 * np.pi, bad.sum())
    xn[bad] += (rng.uniform(40, 100, bad.sum()) / S["f"])[:, None] * np.column_stack([np.cos(ang), np.sin(ang)])
    xy = normalized_to_image(model, S["params"], xn)
    begin = np.arange(n_tracks + 1, dtype=np.int64) * length
    return S, begin, obs_img, xy, xn, X


def _reference(S, begin, obs_img, xn, keys=None, **kw):
    out = []
    for t in range(len(begin) - 1):
        sl = slice(begin[t], begin[t + 1])
        d, c = zip(*[T.rays(xn[o:o + 1], S["qvec"][obs_img[o]], S["tvec"][obs_img[o]]) for o in range(sl.start, sl.stop)])
        d, c = np.concatenate(d), np.concatenate(c)
        r = T.triangulate_track(d, c, key=t if keys is None else int(keys[t]), **kw)
        e, front = T.errors(d, c, r["xyz"])
        r["margin"] = np.abs(e - np.radians(2.0)).min() / np.radians(2.0)
        out.append(r)
    return out


@pytest.mark.parametrize("length", [2, 3, 8, 32, 33, 45, 60])
def test_tracks_match_the_reference(length):
    n_tracks = 40 if length < 45 else 12
    S, begin, obs_img, xy, xn, X = _tracks(length, n_tracks, model=length % 7, seed=1)
    res = _engine.tri_run(_tri_scene(S, begin, obs_img, xy))
    ref = _reference(S, begin, obs_img, xn)
    assert min(r["margin"] for r in ref) > 0.05            # every inlier decision away from the threshold
    for t, r in enumerate(ref):
        sl = slice(begin[t], begin[t + 1])
        assert res["status"][t] == r["status"], t
        np.testing.assert_array_equal(res["obs_inlier"][sl], r["inliers"])
        assert res["n_inliers"][t] == r["n_inliers"]
        if r["status"] == T.TRI_OK:
            assert np.abs(res["xyz"][t] - r["xyz"]).max() <= 1e-9 * max(1.0, np.abs(r["xyz"]).max())
            assert abs(res["tri_angle"][t] - r["angle"]) <= 1e-9 * r["angle"]
            if length >= 8:                                 # a majority of true observations
                assert np.abs(r["xyz"] - X[t]).max() < 0.05
    assert np.mean([r["status"] == T.TRI_OK for r in ref]) > 0.9


def test_runs_are_deterministic_and_independent_of_the_launch():
    parts = [_tracks(n, 150, model=2, seed=2, n_images=50) for n in (3, 5, 12, 50)]
    S = parts[0][0]
    begin = np.concatenate([[0], np.cumsum(np.concatenate([np.diff(p[1]) for p in parts]))]).astype(np.int64)
    obs_img, xy = np.concatenate([p[2] for p in parts]), np.concatenate([p[3] for p in parts])
    opt = _capi.default_tri_options(tri_max_pairs=256, seed=11)
    a = _engine.tri_run(_tri_scene(S, begin, obs_img, xy), opt)
    b = _engine.tri_run(_tri_scene(S, begin, obs_img, xy), opt)
    for k in ("xyz", "status", "n_inliers", "tri_angle", "obs_inlier", "obs_error"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert (a["status"] == T.TRI_OK).mean() > 0.9
    # a shuffled subset, keyed by the tracks' original indices: every track's result is the same bits
    rng = np.random.default_rng(5)
    sub = rng.permutation(len(begin) - 1)[:200]
    sb = np.concatenate([[0], np.cumsum(np.diff(begin)[sub])]).astype(np.int64)
    osel = np.concatenate([np.arange(begin[t], begin[t + 1]) for t in sub])
    c = _engine.tri_run(_tri_scene(S, sb, obs_img[osel], xy[osel], track_key=sub), opt)
    for k in ("xyz", "status", "n_inliers", "tri_angle"):
        assert c[k].tobytes() == a[k][sub].tobytes(), k
    for k in ("obs_inlier", "obs_error"):
        assert c[k].tobytes() == a[k][osel].tobytes(), k
    assert (np.diff(begin)[sub] == 50).any()               # 1225 pairs > 256: sampled tracks are in the subset


def test_evaluate_matches_the_reference_and_flags_bad_points():
    S, begin, obs_img, xy, xn, X = _tracks(6, 60, model=4, seed=3)
    xyz = X + np.random.default_rng(0).normal(0, 0.01, X.shape)
    xyz[0] = 40.0 * X[0] + np.array([0, 0, 400.0])          # far away: a tiny triangulation angle
    c0 = -T.quat_to_rot(S["qvec"][0]).T @ S["tvec"][0]
    xyz[1] = 2 * c0 - X[1]                                  # behind camera 0
    err, ang, _ = _engine.tri_evaluate(_tri_scene(S, begin, obs_img, xy), xyz)
    for t in range(len(begin) - 1):
        sl = slice(begin[t], begin[t + 1])
        ref_err = np.concatenate([T.reprojection_errors(4, S["params"], S["qvec"][obs_img[o]], S["tvec"][obs_img[o]],
                                                        xyz[t:t + 1], xy[o:o + 1]) for o in range(sl.start, sl.stop)])
        fin = np.isfinite(ref_err)
        np.testing.assert_array_equal(np.isfinite(err[sl]), fin)
        np.testing.assert_array_less(np.abs(err[sl][fin] - ref_err[fin]), 1e-9 * ref_err[fin] + 1e-9)
        c = np.array([-T.quat_to_rot(S["qvec"][obs_img[o]]).T @ S["tvec"][obs_img[o]] for o in range(sl.start, sl.stop)])
        assert abs(ang[t] - np.degrees(T.max_tri_angle(c, xyz[t]))) <= 1e-9 * max(ang[t], 1.0)
    assert ang[0] < 1.5 and ang[2:].min() > 1.5
    assert np.isinf(err[begin[1]]) and np.isfinite(err[begin[2]:]).all()        # obs 0 of track 1 is in image 0


# ---- main on hloc files
def _write_hloc_scene(tmp_path, n_images=12, n_points=2000, noise_px=0.5, wrong=0.05, seed=0):
    from pixsfm.util import colmap_types as ct
    from pixsfm.util import h5lite, hloc
    rng = np.random.default_rng(seed)
    model, params = 1, np.array(T.CAMERAS[1])
    qv, tv = T.ring_poses(n_images, seed=seed)
    X = rng.uniform(-1.5, 1.5, (n_points, 3))
    rec = ct.Reconstruction()
    rec.add_camera(ct.Camera(1, "PINHOLE", 640, 480, params))
    names = ["img%02d.jpg" % k for k in range(n_images)]
    kp = [[] for _ in range(n_images)]
    owner = [[] for _ in range(n_images)]
    tracks = []
    for p in range(n_points):
        L = rng.integers(3, 9)
        imgs = np.sort(rng.choice(n_images, L, replace=False))
        el = []
        for k in imgs:
            x = normalized_to_image(model, params, T.project_normalised(qv[k], tv[k], X[p:p + 1]))[0]
            el.append((k, len(kp[k])))
            kp[k].append(x + rng.normal(0, noise_px, 2))
            owner[k].append(p)
        tracks.append(el)
    for k in range(n_images):                                # unmatched keypoints
        for _ in range(50):
            kp[k].append(rng.uniform([0, 0], [640, 480])); owner[k].append(-1)
    kp = [np.array(a) for a in kp]
    owner = [np.array(a) for a in owner]
    for k in range(n_images):
        rec.add_image(ct.Image(k + 1, names[k], 1, qv[k], tv[k]))
    rec.write(str(tmp_path / "ref"))
    with h5lite.File(str(tmp_path / "feats.h5"), "w") as f:
        for k, n in enumerate(names):
            f.create_group(n).create_dataset("keypoints", data=kp[k] - 0.5)        # hloc convention
    pm = {}
    for el in tracks:
        for a in range(len(el)):
            for b in range(a + 1, len(el)):
                (i, ki), (j, kj) = el[a], el[b]
                pm.setdefault((i, j), []).append((ki, kj))
    n_wrong = 0
    with h5lite.File(str(tmp_path / "matches.h5"), "w") as f:
        for (i, j), ms in sorted(pm.items()):
            m0 = np.full(len(kp[i]), -1, np.int32)
            for ki, kj in ms:
                if rng.random() < wrong:                 # a keypoint at least 20 px from the right one
                    far = np.flatnonzero(np.linalg.norm(kp[j] - kp[j][kj], axis=1) > 20)
                    kj = int(far[rng.integers(len(far))]); n_wrong += 1
                m0[ki] = kj
            g = f.create_group(names[i] + "/" + names[j])
            g.create_dataset("matches0", data=m0)
            g.create_dataset("matching_scores0", data=rng.uniform(0.5, 1.0, len(m0)).astype(np.float32))
    hloc.write_image_pairs(tmp_path / "pairs.txt", [(names[i], names[j]) for i, j in sorted(pm)])
    return rec, X, owner, names, n_wrong


def test_main_triangulates_a_synthetic_model(tmp_path):
    from pixsfm.triangulation import main
    from pixsfm.util.cameras import world_to_image
    from pixsfm.util.colmap_types import Reconstruction
    ref, X, owner, names, n_wrong = _write_hloc_scene(tmp_path)
    assert n_wrong > 100
    out = main(tmp_path / "sfm", tmp_path / "ref", None, tmp_path / "pairs.txt", tmp_path / "feats.h5",
               tmp_path / "matches.h5")
    assert sorted(out.images) == sorted(ref.images) and sorted(out.cameras) == sorted(ref.cameras)
    for i, im in ref.images.items():
        o = out.images[i]
        assert o.name == im.name and o.camera_id == im.camera_id
        assert np.array_equal(o.qvec, im.qvec) and np.array_equal(o.tvec, im.tvec)
    for c, cam in ref.cameras.items():
        assert out.cameras[c].model_id == cam.model_id and np.array_equal(out.cameras[c].params, cam.params)
    assert sorted(out.points3D) == list(range(1, len(out.points3D) + 1))
    found, errs = set(), []
    for pid, p in out.points3D.items():
        gt = {int(owner[e.image_id - 1][e.point2D_idx]) for e in p.track.elements}
        assert len(gt) == 1 and -1 not in gt, (pid, gt)          # no wrong match in a track
        found |= gt
        errs.append(np.linalg.norm(p.xyz - X[gt.pop()]))
        for e in p.track.elements:
            im = out.images[e.image_id]
            assert im.points2D[e.point2D_idx].point3D_id == pid
            px = world_to_image(1, out.cameras[1].params, im.qvec, im.tvec, p.xyz)[0]
            assert np.linalg.norm(px - im.points2D[e.point2D_idx].xy) <= 4.0
    assert len(found) >= 0.95 * len(X), len(found)
    # 0.5 px at f = 500 and depth ~6 is 6e-3 laterally; three or more views from 30 degrees apart and more
    assert np.median(errs) < 0.01, np.median(errs)
    back = Reconstruction.read(tmp_path / "sfm")
    assert sorted(back.points3D) == sorted(out.points3D)
    assert all(np.array_equal(back.points3D[p].xyz, out.points3D[p].xyz) for p in out.points3D)


def test_pixsfm_triangulation_from_images_without_hloc(tmp_path, monkeypatch):
    from test_gpu_dsift import _build, _conf
    from pixsfm import refine_hloc
    from pixsfm.util import h5lite, hloc
    from pixsfm.util.colmap_types import Reconstruction

    def no_hloc():
        raise ImportError("No module named 'hloc'")
    monkeypatch.setattr(refine_hloc, "_HlocBackend", no_hloc)
    scene, rec, truth, xyz, params = _build(tmp_path, n_images=4, n_points=60)
    rec.write(str(tmp_path / "ref"))
    names = sorted(truth)
    rng = np.random.default_rng(2)
    with h5lite.File(str(tmp_path / "feats.h5"), "w") as f:
        for n in names:
            f.create_group(n).create_dataset("keypoints", data=truth[n] + rng.normal(0, 1.0, truth[n].shape) - 0.5)
    with h5lite.File(str(tmp_path / "matches.h5"), "w") as f:
        for i, a in enumerate(names):
            for b in names[i + 1:]:
                g = f.create_group(a + "/" + b)
                g.create_dataset("matches0", data=np.arange(len(xyz), dtype=np.int32))
                g.create_dataset("matching_scores0", data=np.ones(len(xyz), np.float32))
    hloc.write_image_pairs(tmp_path / "pairs.txt", [(a, b) for i, a in enumerate(names) for b in names[i + 1:]])
    sfm = refine_hloc.PixSfM(_conf())
    assert sfm.sfm_backend is None
    out, data = sfm.triangulation(tmp_path / "out", tmp_path / "ref", tmp_path / "images", tmp_path / "pairs.txt",
                                  tmp_path / "feats.h5", tmp_path / "matches.h5")
    assert all(s.final_cost < s.initial_cost for s in data["KA"]["summary"])
    assert all(s.final_cost < s.initial_cost for s in data["BA"]["summary"])
    assert len(out.points3D) >= 0.9 * len(xyz)
    tri = Reconstruction.read(tmp_path / "out" / "hloc")                # the built-in triangulator's model
    assert len(tri.points3D) == len(out.points3D)
    on_disk = Reconstruction.read(tmp_path / "out")
    assert sorted(on_disk.points3D) == sorted(out.points3D) and sorted(on_disk.images) == sorted(rec.images)
    err = np.median([np.linalg.norm(p.xyz - xyz[int(np.argmin(np.linalg.norm(xyz - p.xyz, axis=1)))])
                     for p in out.points3D.values()])
    assert err < 0.05, err
