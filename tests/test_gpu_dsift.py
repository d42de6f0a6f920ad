"""Dense SIFT on the GPU (csrc/pxr_dsift.cu): the map against oracle (a) within the fp32 bound derived in
dsift_oracle.fp32_bound, slab windows bit for bit equal to the map, host / device input and output, a slab past 2^31
elements, the argument errors, and PixSfM / QueryLocalizer run from rendered images with the `dsift` preset."""
import copy

import numpy as np
import pytest

import dsift_oracle as D
from pixsfm._pixsfm import _capi, _engine

pytestmark = pytest.mark.gpu

AS = [(4, 2), (4, 4), (8, 2), (8, 4)]


def _image(h, w, seed):
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(seed)
    img = gaussian_filter(rng.random((h, w)), 1.0) * 255 * 3 - 255
    img = np.clip(img, 0, 255).astype(np.uint8)
    img[: h // 3, : w // 3] = 77                           # flat: zero gradients
    img[h // 2, :] = 200                                   # gy only
    return img


def _cases():
    out = []
    for A, S in AS:
        for b in (3, 4, 5):
            for k, (h, w) in enumerate([(13, 9), (37, 50)]):
                out.append((A, S, b, h, w, (b + k) % 2 == 0, (A + b + k) % 3 != 0))
    out += [(8, 4, 4, 70, 45, r, l) for r in (True, False) for l in (True, False)]
    return out


@pytest.mark.parametrize("A,S,b,h,w,rootsift,l2", _cases())
def test_dense_map_matches_the_oracle_within_the_fp32_bound(A, S, b, h, w, rootsift, l2):
    img = _image(h, w, A * 100 + S * 10 + b + h)
    ref, extra = D.dsift_conv(img, A, S, b, 0.2, rootsift, l2, intermediates=True)
    for dtype in (np.float32, np.float16):
        got = _engine.dsift(img, None, 16, A, S, b, 0.2, rootsift, l2, dtype, to_host=True)
        assert got.shape == (1,) + ref.shape and got.dtype == dtype
        err = np.abs(got[0].astype(np.float64) - ref)
        bound = D.fp32_bound(ref, extra, A, S, b, rootsift, l2, dtype)
        assert (err <= bound).all(), (dtype, float(err.max()), float((err / bound).max()))


@pytest.mark.parametrize("ps", [5, 8, 16, 32])
@pytest.mark.parametrize("A,S,b", [(8, 4, 4), (4, 2, 3), (8, 2, 5)])
def test_slab_windows_equal_the_dense_map_bit_for_bit(ps, A, S, b):
    img = _image(71, 93, ps + A + b)
    hm, wm = D.map_size(71, 93, S, b)
    rng = np.random.default_rng(ps)
    corners = [(0, 0), (wm - ps, 0), (0, hm - ps), (wm - ps, hm - ps), (0, 17), (wm - ps, 9), (11, 0), (23, hm - ps)]
    corners += [(int(rng.integers(0, wm - ps + 1)), int(rng.integers(0, hm - ps + 1))) for _ in range(20)]
    corners = np.array(corners, np.int32)
    for dtype in (np.float16, np.float32, np.float64):
        full = _engine.dsift(img, None, ps, A, S, b, 0.2, True, True, dtype, to_host=True)[0]
        slab = _engine.dsift(img, corners, ps, A, S, b, 0.2, True, True, dtype, to_host=True)
        for k, (x, y) in enumerate(corners):
            assert slab[k].tobytes() == full[y:y + ps, x:x + ps].tobytes(), (dtype, k)


def test_host_and_device_input_and_output_give_the_same_bytes():
    import torch
    img = _image(120, 160, 3)
    corners = np.array([[0, 0], [100, 50], [144, 104]], np.int32)
    dev = torch.from_numpy(img).cuda().contiguous()
    for c in (corners, None):
        host = _engine.dsift(img, c, 16, to_host=True)
        for src in (img, dev):
            a = _engine.dsift(src, c, 16, to_host=True)
            slab = _engine.dsift(src, c, 16)
            b = torch.as_tensor(slab, device="cuda").cpu().numpy()
            assert a.tobytes() == host.tobytes() and b.tobytes() == host.tobytes()


def test_slab_past_2_to_the_31_elements_gets_its_last_window_right():
    ps, C = 16, 128
    n = (1 << 31) // (ps * ps * C) + 3                    # n * ps * ps * C > 2^31
    img = _image(64, 80, 5)
    rng = np.random.default_rng(0)
    corners = np.stack([rng.integers(0, 80 - ps + 1, n), rng.integers(0, 64 - ps + 1, n)], 1).astype(np.int32)
    corners[-1] = (80 - ps, 64 - ps)
    corners[-2] = (3, 7)
    full = _engine.dsift(img, None, ps, to_host=True)[0]
    slab = _engine.dsift(img, corners, ps)
    assert n * ps * ps * C > (1 << 31) and slab.shape == (n, ps, ps, C)
    win = ps * ps * C * 2
    for k in (n - 2, n - 1):
        out = np.empty((ps, ps, C), np.float16)
        _engine.memcpy_d2h(out, slab.ptr + k * win, win)
        x, y = corners[k]
        assert out.tobytes() == full[y:y + ps, x:x + ps].tobytes()
    del slab


def test_errors_launch_nothing():
    ctx = _capi.default_context()
    img = _image(40, 50, 1)
    before = ctx.kernel_launches()
    for bad in ([[-1, 0]], [[0, -1]], [[50 - 16 + 1, 0]], [[0, 40 - 16 + 1]]):
        with pytest.raises(ValueError, match="leaves the"):
            _engine.dsift(img, np.array(bad, np.int32), 16, to_host=True)
    for A, S, b in ((6, 4, 4), (8, 3, 4), (8, 4, 9), (8, 4, 0)):
        with pytest.raises(ValueError, match="supports"):
            _engine.dsift(img, None, 16, A, S, b, to_host=True)
    assert ctx.kernel_launches() == before


# ------------------------------------------------------------------------------------------------ end to end
W_IMG, H_IMG, F = 320, 240, 300.0


def _rot(axis_angle):
    from scipy.spatial.transform import Rotation
    q = Rotation.from_rotvec(axis_angle).as_quat()                   # x, y, z, w
    return np.array([q[3], q[0], q[1], q[2]]), Rotation.from_rotvec(axis_angle).as_matrix()


class Scene:
    """Two textured planes (a square of z = 0 and a tilted plane behind it) seen by pinhole cameras 4 units away; pixel centres at
    +0.5 (COLMAP).  The texture is smooth random noise, bilinearly sampled."""

    def __init__(self, seed=0):
        from scipy.ndimage import gaussian_filter
        rng = np.random.default_rng(seed)
        self.tex = [gaussian_filter(rng.random((512, 512)), 2.5) for _ in range(2)]
        self.tex = [(t - t.min()) / (t.max() - t.min()) for t in self.tex]
        self.rng = rng

    def _planes(self):
        n1, d1 = np.array([0.0, 0.0, 1.0]), 0.0                     # z = 0
        n2 = np.array([0.3, 0.0, 1.0]) / np.linalg.norm([0.3, 0.0, 1.0])
        return [(n1, d1), (n2, 0.8)]                                # n . X = d

    def render(self, qvec, R, t):
        from scipy.ndimage import map_coordinates
        jj, ii = np.meshgrid(np.arange(W_IMG) + 0.5, np.arange(H_IMG) + 0.5)
        d_cam = np.stack([(jj - W_IMG / 2) / F, (ii - H_IMG / 2) / F, np.ones_like(jj)], -1)
        d = d_cam @ R                                               # R^T d_cam, row vectors
        c = -R.T @ t
        best = np.full(jj.shape, np.inf)
        value = np.zeros(jj.shape)
        for k, (n, dd) in enumerate(self._planes()):
            lam = (dd - c @ n) / (d @ n)
            X = c + lam[..., None] * d
            u, v = (X[..., 0] + 1.5) * 150, (X[..., 1] + 1.5) * 150
            val = map_coordinates(self.tex[k], [v.ravel(), u.ravel()], order=1, mode="reflect").reshape(jj.shape)
            closer = (lam > 0) & (lam < best)
            if k == 0:
                closer &= (np.abs(X[..., 0]) <= 1.2) & (np.abs(X[..., 1]) <= 1.2)      # a square, the other plane behind
            value = np.where(closer, val, value)
            best = np.where(closer, lam, best)
        return (value * 220 + 20).astype(np.uint8)

    def points(self, n):
        xy = self.rng.uniform(-0.9, 0.9, (n, 2))
        return np.concatenate([xy, np.zeros((n, 1))], 1)             # on z = 0, in front of the tilted plane

    def camera(self, k):
        aa = np.array([0.05 * np.sin(k), 0.05 * np.cos(k), 0.02 * k])
        qvec, R = _rot(aa)
        C = np.array([0.4 * np.cos(k), 0.3 * np.sin(k), -4.0])
        return qvec, R, -R @ C


def _build(tmp_path, n_images=4, n_points=60, seed=0):
    from PIL import Image
    from pixsfm.util import cameras
    from pixsfm.util import colmap_types as ct
    scene = Scene(seed)
    xyz = scene.points(n_points)
    rec = ct.Reconstruction()
    params = np.array([F, F, W_IMG / 2, H_IMG / 2])
    rec.add_camera(ct.Camera(1, "PINHOLE", W_IMG, H_IMG, params))
    (tmp_path / "images").mkdir()
    truth = {}
    for i in range(n_images):
        qvec, R, t = scene.camera(i)
        name = "image%03d.png" % i
        Image.fromarray(scene.render(qvec, R, t), "L").save(str(tmp_path / "images" / name))
        xy = cameras.world_to_image(1, params, qvec, t, xyz)
        truth[name] = xy
        rec.add_image(ct.Image(i + 1, name, 1, qvec, t, [ct.Point2D(p) for p in xy]))
    for p in range(n_points):
        rec.add_point3D(p + 1, xyz[p])
        for i in range(n_images):
            rec.add_observation(p + 1, i + 1, p)
    return scene, rec, truth, xyz, params


def _conf(**dense):
    from pixsfm.configs import parse_config_path
    conf = parse_config_path("dsift")
    for block in (conf["mapping"]["dense_features"], conf["localization"]["dense_features"]):
        block.update(dict(max_edge=W_IMG, **dense))
    conf["mapping"]["KA"]["optimizer"]["solver"] = {"max_num_iterations": 50}
    return conf


def test_pixsfm_from_images_refines_keypoints_and_points(tmp_path):
    from pixsfm.features.extractor import FeatureExtractor
    from pixsfm.refine_colmap import PixSfM
    scene, rec, truth, xyz, params = _build(tmp_path)
    names = sorted(truth)
    rng = np.random.default_rng(1)
    noisy = {n: truth[n] + rng.normal(0, 1.0, truth[n].shape) for n in names}
    pairs = [(a, b) for i, a in enumerate(names) for b in names[i + 1:]]
    idx = np.arange(len(xyz), dtype=np.uint32)
    matches = [np.stack([idx, idx], 1) for _ in pairs]
    runs = {}
    for on_device in (False, True):
        sfm = PixSfM(_conf(on_device=on_device))
        assert isinstance(sfm.extractor, FeatureExtractor)
        kps = copy.deepcopy(noisy)
        out, _, _ = sfm.run_ka(kps, tmp_path / "images", pairs, (matches, None))
        runs[on_device] = out
    # the patches of the two runs are the same bytes; the refined keypoints agree to far below a pixel (the adjuster's
    # device reductions need not add in the same order for device-resident and uploaded patches)
    import torch
    host = PixSfM(_conf()).extractor.features_from_image_list(tmp_path / "images", names, noisy)
    dev = PixSfM(_conf(on_device=True)).extractor.features_from_image_list(tmp_path / "images", names, noisy)
    for n in names:
        a, b = host.fset(0).fmap(n), dev.fset(0).fmap(n)
        assert a.is_sparse and b.is_sparse and np.array_equal(a.corners, b.corners)
        assert torch.as_tensor(b.patches.owner, device="cuda").cpu().numpy().tobytes() == np.asarray(a.patches).tobytes()
        assert np.abs(runs[False][n] - runs[True][n]).max() < 1e-6
    # KA has no absolute anchor (it aligns the keypoints of a track with each other, one of them held fixed), so the
    # truth it can reach is the true projections up to a shift common to the track: compare with that
    def spread(kps):
        err = np.stack([kps[n] - truth[n] for n in names])                 # [images, points, 2]
        return np.linalg.norm(err - err.mean(0, keepdims=True), axis=-1).mean()
    before, after = spread(noisy), spread(runs[False])
    assert after < 0.5 * before, (before, after)

    # BA from perturbed points: lower cost, points closer to the truth
    rec_noisy = copy.deepcopy(rec)
    for pid, p in rec_noisy.points3D.items():
        p.xyz = p.xyz + rng.normal(0, 0.01, 3)
    err0 = np.mean([np.linalg.norm(rec_noisy.points3D[p].xyz - xyz[p - 1]) for p in rec_noisy.points3D])
    out_rec, ba_data, _ = PixSfM(_conf()).run_ba(rec_noisy, tmp_path / "images")
    assert all(s.final_cost < s.initial_cost for s in ba_data["summary"])
    err1 = np.mean([np.linalg.norm(out_rec.points3D[p].xyz - xyz[p - 1]) for p in out_rec.points3D])
    assert err1 < 0.9 * err0, (err0, err1)          # depth is weakly constrained by the short baselines


def test_query_localizer_from_images_refines_the_pose(tmp_path):
    from PIL import Image
    from pixsfm.localization.main import QueryLocalizer
    from pixsfm.util import cameras
    from pixsfm.util import colmap_types as ct
    scene, rec, truth, xyz, params = _build(tmp_path, n_images=3, seed=2)
    qvec, R, t = scene.camera(7)
    path = tmp_path / "query.png"
    Image.fromarray(scene.render(qvec, R, t), "L").save(str(path))
    kps = cameras.world_to_image(1, params, qvec, t, xyz)
    rng = np.random.default_rng(3)
    start_t = t + rng.normal(0, 0.02, 3)

    def pnp(points2D, points3D, camera):          # stands in for pycolmap.absolute_pose_estimation
        return {"success": True, "qvec": qvec.copy(), "tvec": start_t.copy(), "inliers": [True] * len(points2D)}

    loc = QueryLocalizer(rec, _conf(), image_dir=tmp_path / "images", pose_estimator=pnp)
    cam = ct.Camera(1, "PINHOLE", W_IMG, H_IMG, params)
    ids = list(range(len(xyz)))
    out = loc.localize(kps + rng.normal(0, 0.5, kps.shape), ids, [i + 1 for i in ids], cam, image_path=path)
    assert out["success"]
    assert np.linalg.norm(out["tvec"] - t) < 0.5 * np.linalg.norm(start_t - t), (start_t - t, out["tvec"] - t)
