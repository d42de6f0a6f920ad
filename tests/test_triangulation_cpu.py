"""Triangulation from known poses without a GPU: the numpy restatement on exact data, the sample stream, the mapper
options, the C-ABI's argument checks and the input plumbing from hloc's files up to the first device call."""
import ctypes as C

import numpy as np
import pytest

import triangulation_reference as T
from pixsfm import triangulation as tri
from pixsfm._pixsfm import _capi
from pixsfm.util import colmap_types as ct
from pixsfm.util import h5lite, hloc


def _track(n, seed=0, outlier=None):
    rng = np.random.default_rng(seed)
    qv, tv = T.ring_poses(n, seed=seed)
    X = rng.uniform(-1, 1, 3)
    d, c = [], []
    for k in range(n):
        xn = T.project_normalised(qv[k], tv[k], X[None])
        if k == outlier:
            xn = xn + 0.2                                     # about 11 degrees off
        dk, ck = T.rays(xn, qv[k], tv[k])
        d.append(dk[0]); c.append(ck[0])
    return np.array(d), np.array(c), X


@pytest.mark.parametrize("n", [2, 3, 8, 33, 60])
def test_reference_recovers_exact_points(n):
    d, c, X = _track(n, seed=n)
    r = T.triangulate_track(d, c, key=n)
    assert r["status"] == T.TRI_OK and r["n_inliers"] == n and r["inliers"].all()
    assert np.abs(r["xyz"] - X).max() < 1e-9 * max(1.0, np.abs(X).max())
    assert r["angle"] > 1.5


def test_reference_rejects_a_planted_outlier():
    d, c, X = _track(8, seed=3, outlier=5)
    r = T.triangulate_track(d, c)
    assert r["status"] == T.TRI_OK and r["n_inliers"] == 7 and not r["inliers"][5]
    assert np.abs(r["xyz"] - X).max() < 1e-9


def test_reference_parallel_rays_have_no_hypothesis():
    d = np.tile([0.0, 0.0, 1.0], (4, 1))
    c = np.array([[0.0, 0.0, 0.0], [1e-3, 0, 0], [0, 1e-3, 0], [1e-3, 1e-3, 0]])
    assert T.triangulate_track(d, c)["status"] == T.TRI_ANGLE_TOO_SMALL


def test_sample_stream_known_answers():
    assert T.pair_sample(0, 7, 0, 60) == (36, 57)
    assert [T.pair_sample(0, 7, h, 60) for h in range(1, 6)] == [(1, 24), (24, 32), (38, 20), (52, 47), (47, 26)]
    assert [T.pair_sample(12345, 2 ** 40 + 3, h, 1000) for h in range(4)] == [(439, 931), (747, 819), (675, 320), (876, 451)]
    # 45 observations: 990 pairs, all taken in order; 46: 1035 > 1024, so 1024 sampled ones
    assert len(T.hypothesis_pairs(45, 1024, 0, 0)) == 990 and T.hypothesis_pairs(45, 1024, 0, 0)[44] == (1, 2)
    pairs = T.hypothesis_pairs(60, 1024, 9, 4)
    assert len(pairs) == 1024 and all(p is not None and p[0] != p[1] and max(p) < 60 for p in pairs)


def test_mapper_options_reject_unknown_keys_and_two_view_geometries(tmp_path):
    assert tri.mapper_options_from({"min_angle": 3.0})["min_angle"] == 3.0
    with pytest.raises(ValueError, match="ba_refine_focal_length.*accepted: ba_max_num_iterations"):
        tri.mapper_options_from({"ba_refine_focal_length": True})
    with pytest.raises(ValueError, match="estimate_two_view_geometries"):
        tri.main(tmp_path, tmp_path, None, None, None, None, estimate_two_view_geometries=True)
    with pytest.raises(ValueError, match="unknown mapper option 'foo'"):
        tri.main(tmp_path, tmp_path, None, None, None, None, mapper_options={"foo": 1})


def _scene(n_tracks=3, n_obs=6):
    tb = np.array([0, 2, 4, 6][:n_tracks + 1], np.int64)
    return _capi.TriScene([1], [T.padded(T.CAMERAS[1])], [0, 0, 0], np.tile([1.0, 0, 0, 0], (3, 1)), np.zeros((3, 3)),
                          tb, np.array([0, 1, 0, 2, 1, 2][:n_obs]), np.zeros((n_obs, 2)))


def test_c_abi_rejects_malformed_descs_without_a_device():
    lib = _capi.load_lib()
    o = _capi.default_tri_options()
    assert (o.min_angle, o.create_max_angle_error, o.tri_max_pairs, o.seed) == (1.5, 2.0, 1024, 0)
    out = [np.zeros((3, 3)), np.zeros(3, np.int32), np.zeros(3, np.int32), np.zeros(3), np.zeros(6, np.uint8), np.zeros(6)]
    P = [_capi.ptr(a) for a in out]

    def run(d, opt=o):
        return lib.pxr_tri_run(None, C.byref(d) if d is not None else None, C.byref(opt), *P, None)

    def evaluate(d):
        return lib.pxr_tri_evaluate(None, C.byref(d), _capi.ptr(out[0]), _capi.ptr(out[5]), _capi.ptr(out[3]), None)

    assert run(None) == _capi.PXR_ERR_INVALID_ARGUMENT
    s = _scene()
    d = s.desc(); d.n_tracks = -1
    assert run(d) == _capi.PXR_ERR_INVALID_ARGUMENT and b"negative" in lib.pxr_last_error()
    d = s.desc(); d.n_images = -2
    assert run(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    s.cam_model[0] = 9
    assert run(s.desc()) == _capi.PXR_ERR_UNSUPPORTED and evaluate(s.desc()) == _capi.PXR_ERR_UNSUPPORTED
    s = _scene()
    s.track_begin[:] = [0, 2, 3, 6]                     # one observation in track 1
    assert run(s.desc()) == _capi.PXR_ERR_INVALID_ARGUMENT and b">= 2" in lib.pxr_last_error()
    s.track_begin[:] = [0, 4, 2, 6]                     # not monotone
    assert run(s.desc()) == _capi.PXR_ERR_INVALID_ARGUMENT and evaluate(s.desc()) == _capi.PXR_ERR_INVALID_ARGUMENT
    s.track_begin[:] = [1, 3, 5, 6]
    assert run(s.desc()) == _capi.PXR_ERR_INVALID_ARGUMENT
    s = _scene()
    d = s.desc(); d.obs_xy = None
    assert run(d) == _capi.PXR_ERR_INVALID_ARGUMENT and b"NULL" in lib.pxr_last_error()
    d = s.desc(); d.qvec = None
    assert run(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    d = s.desc(); d.track_begin = None
    assert run(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    s.obs_img[3] = 3
    assert run(s.desc()) == _capi.PXR_ERR_INVALID_ARGUMENT and b"out of range" in lib.pxr_last_error()
    s = _scene()
    assert run(s.desc(), _capi.default_tri_options(tri_max_pairs=0)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert run(s.desc(), _capi.default_tri_options(create_max_angle_error=0.0)) == _capi.PXR_ERR_INVALID_ARGUMENT
    # verification: a negative count, an image index out of range, NULL arrays
    mi, mx, mn = np.array([[0, 1]], np.int32), np.zeros((1, 4)), np.ones((1, 2))
    keep, err = np.zeros(1, np.uint8), np.zeros((1, 2))

    def verify(d, n=1, img=mi, max_error=4.0):
        return lib.pxr_tri_verify(None, C.byref(d), C.c_int64(n), _capi.ptr(img), _capi.ptr(mx), _capi.ptr(mn),
                                  C.c_double(max_error), _capi.ptr(keep), _capi.ptr(err), None)
    assert verify(s.desc(), n=-1) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert verify(s.desc(), img=np.array([[0, 5]], np.int32)) == _capi.PXR_ERR_INVALID_ARGUMENT
    assert verify(s.desc(), max_error=0.0) == _capi.PXR_ERR_INVALID_ARGUMENT
    d = s.desc(); d.img_cam = None
    assert verify(d) == _capi.PXR_ERR_INVALID_ARGUMENT
    # well-formed calls reach the context check
    assert run(s.desc()) not in (_capi.PXR_OK, _capi.PXR_ERR_UNSUPPORTED)
    assert verify(s.desc()) not in (_capi.PXR_OK, _capi.PXR_ERR_UNSUPPORTED)


def _hloc_files(tmp_path, with_uncertainty=True):
    """three images, a reference model with one stale 3D point, hloc keypoints (one image with an uncertainty) and
    matches for pairs (a, b), (b, a) (a repeat) and (b, c)"""
    rec = ct.Reconstruction()
    rec.add_camera(ct.Camera(3, "PINHOLE", 640, 480, T.CAMERAS[1]))
    names = ["a.jpg", "sub/b.jpg", "c.jpg"]
    rng = np.random.default_rng(0)
    kps = {n: rng.uniform(0, 400, (5 + k, 2)) for k, n in enumerate(names)}
    for k, n in enumerate(names):
        rec.add_image(ct.Image(10 + k, n, 3, [1, 0, 0, 0], [k, 0, 0], [ct.Point2D(p) for p in kps[n]]))
    rec.add_point3D(1, [0, 0, 5])
    rec.add_observation(1, 10, 0)
    rec.write(str(tmp_path / "ref"))
    with h5lite.File(str(tmp_path / "feats.h5"), "w") as f:
        for n in names:
            ds = f.create_group(n).create_dataset("keypoints", data=kps[n])
            if with_uncertainty and n == "c.jpg":
                ds.attrs["uncertainty"] = 0.25
    with h5lite.File(str(tmp_path / "matches.h5"), "w") as f:
        def put(n0, n1, m0, s0):
            g = f.create_group(n0.replace("/", "-") + "/" + n1.replace("/", "-"))
            g.create_dataset("matches0", data=np.asarray(m0, np.int32))
            g.create_dataset("matching_scores0", data=np.asarray(s0, np.float32))
        put("a.jpg", "sub/b.jpg", [0, -1, 2, 3, 1], [0.9, 0, 0.3, 0.6, 0.7])
        put("sub/b.jpg", "c.jpg", [4, 3, -1, -1, -1, 0], [0.8, 0.2, 0, 0, 0, 0.95])
    hloc.write_image_pairs(tmp_path / "pairs.txt", [("a.jpg", "sub/b.jpg"), ("sub/b.jpg", "a.jpg"), ("sub/b.jpg", "c.jpg")])
    return rec, kps, names


def test_inputs_from_hloc_files_are_packed_without_the_device(tmp_path):
    rec, kps, names = _hloc_files(tmp_path)
    ref, keypoints, noise, pairs, m, s = tri.read_inputs(tmp_path / "ref", tmp_path / "pairs.txt",
                                                               tmp_path / "feats.h5", tmp_path / "matches.h5")
    assert ref.points3D == {} and sorted(ref.images) == [10, 11, 12]
    assert pairs == [("a.jpg", "sub/b.jpg"), ("sub/b.jpg", "c.jpg")]           # the repeat in reverse order is skipped
    for n in names:
        np.testing.assert_array_equal(keypoints[n], kps[n] + 0.5)
    assert noise == {"a.jpg": None, "sub/b.jpg": None, "c.jpg": 0.25}
    P = tri.pack_matches(ref, keypoints, pairs, m, s, keypoint_noise=noise)
    assert P["n_pairs"] == 2 and P["kp_begin"].tolist() == [0, 5, 11, 18]
    np.testing.assert_array_equal(P["noise"], [1.0, 1.0, 0.25])
    assert P["kp"].tolist() == [[0, 0], [2, 2], [3, 3], [4, 1], [0, 4], [1, 3], [5, 0]]
    assert P["img"].tolist() == [[0, 1]] * 4 + [[1, 2]] * 3 and P["pair"].tolist() == [0, 0, 0, 0, 1, 1, 1]
    np.testing.assert_allclose(P["score"], [0.9, 0.3, 0.6, 0.7, 0.8, 0.2, 0.95], rtol=1e-6)
    # the same pair list with repeats: packed once
    P2 = tri.pack_matches(ref, keypoints, [pairs[0], pairs[0][::-1], pairs[1]], [m[0], m[0], m[1]], [s[0], s[0], s[1]])
    assert P2["kp"].tolist() == P["kp"].tolist()
    # min_match_score keeps scores > the threshold
    P3 = tri.pack_matches(ref, keypoints, pairs, m, s, min_match_score=0.65)
    assert P3["kp"].tolist() == [[0, 0], [4, 1], [0, 4], [5, 0]]
    # no scores: similarity 1
    assert tri.pack_matches(ref, keypoints, pairs, m)["score"].tolist() == [1.0] * 7
    # a keypoint index out of range, an image outside the model
    with pytest.raises(ValueError, match="out of range"):
        tri.pack_matches(ref, keypoints, pairs[:1], [np.array([[0, 6]])])
    with pytest.raises(ValueError, match="not in the model"):
        tri.pack_matches(ref, keypoints, [("a.jpg", "zz.jpg")], [np.zeros((0, 2))])


def test_an_image_missing_from_the_keypoint_file_raises(tmp_path):
    rec, kps, names = _hloc_files(tmp_path, with_uncertainty=False)
    with h5lite.File(str(tmp_path / "feats2.h5"), "w") as f:
        for n in names[:2]:
            f.create_group(n).create_dataset("keypoints", data=kps[n])
    with pytest.raises(ValueError, match="c.jpg"):
        tri.read_inputs(tmp_path / "ref", tmp_path / "pairs.txt", tmp_path / "feats2.h5", tmp_path / "matches.h5")
    with pytest.raises(ValueError, match="no keypoints for 1 image"):
        tri.pack_matches(rec, {n: kps[n] for n in names[:2]}, [], [])
