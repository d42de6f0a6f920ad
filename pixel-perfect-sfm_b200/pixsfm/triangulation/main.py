"""pixsfm.triangulation — points of a model with known poses, from hloc's keypoint and match files: COLMAP's
point_triangulator as `hloc.triangulation.main` drives it, so `PixSfM.triangulation` runs without hloc.

The chain: keypoints and matches are packed into flat arrays (one Python iteration per image pair, none per match);
matches are verified against the known poses on the GPU (pxr_tri_verify, hloc's geometric_verification with
max_error 4 px); the verified matches are joined into tracks by the track rule of the keypoint adjustment
(pxr_graph_track_labels, which never puts two keypoints of one image in a track); every track is triangulated on the
GPU (pxr_tri_run: RANSAC over observation pairs with COLMAP's angular error, then an N-view refit); a points-only
geometric bundle adjustment refines them (GeometricBundleOptimizer with every pose and camera constant); and one filter
pass (pxr_tri_evaluate) drops observations that reproject too far and points whose triangulation angle is too small.
Cameras, image ids, names and poses are the reference model's, unchanged.

Deliberate deviations, as far as hloc and COLMAP are recalled (not checked against an installed copy):
 - verification uses COLMAP-convention keypoints (+0.5) throughout; recent hloc passes hloc-convention keypoints to its
   verification, a half-pixel shift.  The essential matrix of a pair is not stored.
 - one bundle adjustment and one filter pass; COLMAP's track completion, track merging and re-triangulation are not run.
 - relative poses are not estimated (`estimate_two_view_geometries=True` raises)."""
import time
from pathlib import Path

import numpy as np

from .. import logger
from .._pixsfm import _bundle_adjustment as ba
from .._pixsfm import _capi, _engine
from ..util.colmap_types import ArrayReconstruction, Camera, Image, Point2D, Reconstruction
from ..util.hloc import list_h5_names, read_image_pairs, read_keypoint_uncertainty, read_keypoints_hloc, read_matches_hloc

# names follow COLMAP's IncrementalTriangulator::Options / IncrementalMapper::Options as best known (unverified);
# tri_max_pairs and seed are this module's RANSAC budget and sample-stream seed
DEFAULT_MAPPER_OPTIONS = dict(min_angle=1.5, create_max_angle_error=2.0, ignore_two_view_tracks=True,
                              filter_max_reproj_error=4.0, filter_min_tri_angle=1.5, ba_max_num_iterations=50,
                              tri_max_pairs=1024, seed=0)
VERIFY_MAX_ERROR = 4.0          # hloc's geometric_verification default, pixels


def mapper_options_from(mapper_options=None):
    """DEFAULT_MAPPER_OPTIONS updated by a flat dict; an unknown key raises ValueError"""
    out = dict(DEFAULT_MAPPER_OPTIONS)
    for k, v in dict(mapper_options or {}).items():
        if k not in out:
            raise ValueError("unknown mapper option '%s'; accepted: %s" % (k, ", ".join(sorted(out))))
        out[k] = v
    return out


def unique_pairs(pairs):
    """the pairs in order, a pair already seen in either order skipped (hloc's import_matches)"""
    seen, out = set(), []
    for n0, n1 in pairs:
        if (n0, n1) in seen or (n1, n0) in seen:
            continue
        seen.add((n0, n1))
        out.append((n0, n1))
    return out


def pack_matches(reconstruction, keypoints, pairs, matches, scores=None, min_match_score=None, keypoint_noise=None):
    """Flat arrays of the inputs (host, no device): per image of the model (ascending id) its keypoints, back to back
    (`kp_begin`, `kp_xy`) and its keypoint noise (`noise`, 1 px unless given); per match its pair, image indices and
    keypoint indices and its score (1 when there is none).  `keypoints` are COLMAP-convention pixels by image name;
    `matches[p]` [m, 2] and `scores[p]` [m] belong to `pairs[p]`.  A pair already seen in either order is skipped;
    with `min_match_score` a match is kept when its score is > the threshold (hloc's rule as recalled, unverified)."""
    image_ids = np.array(sorted(reconstruction.images), np.int64)
    names = [reconstruction.images[int(i)].name for i in image_ids]
    missing = [n for n in names if n not in keypoints]
    if missing:
        raise ValueError("no keypoints for %d image(s) of the model: %s" % (len(missing), ", ".join(missing[:10])))
    index = {n: k for k, n in enumerate(names)}
    kps = [np.asarray(keypoints[n], np.float64).reshape(-1, 2) for n in names]
    counts = np.array([len(k) for k in kps], np.int64)
    kp_begin = np.zeros(len(names) + 1, np.int64)
    np.cumsum(counts, out=kp_begin[1:])
    noise_of = keypoint_noise or {}
    noise = np.array([1.0 if noise_of.get(n) is None else float(noise_of[n]) for n in names])
    seen = set()
    pair_idx, img, kp, score = [], [], [], []
    for p, (n0, n1) in enumerate(pairs):
        if n0 not in index or n1 not in index:
            raise ValueError("pair %s %s names an image that is not in the model" % (n0, n1))
        i0, i1 = index[n0], index[n1]
        if (i0, i1) in seen or (i1, i0) in seen:
            continue
        seen.add((i0, i1))
        m = np.asarray(matches[p]).reshape(-1, 2).astype(np.int64)
        s = None if scores is None or scores[p] is None else np.asarray(scores[p], np.float64).reshape(-1)
        if s is not None and min_match_score is not None:
            keep = s > min_match_score
            m, s = m[keep], s[keep]
        if len(m) and (m.min() < 0 or m[:, 0].max() >= counts[i0] or m[:, 1].max() >= counts[i1]):
            raise ValueError("pair %s %s has a keypoint index out of range" % (n0, n1))
        pair_idx.append(np.full(len(m), len(seen) - 1, np.int64))
        img.append(np.broadcast_to(np.array([i0, i1], np.int32), (len(m), 2)))
        kp.append(m)
        score.append(np.ones(len(m)) if s is None else s)
    cat = lambda a, shape, dt: np.concatenate(a).astype(dt) if a else np.zeros(shape, dt)    # noqa: E731
    return dict(image_ids=image_ids, names=names, kp_begin=kp_begin,
                kp_xy=np.concatenate(kps) if kps else np.zeros((0, 2)), noise=noise, n_pairs=len(seen),
                pair=cat(pair_idx, 0, np.int64), img=cat(img, (0, 2), np.int32), kp=cat(kp, (0, 2), np.int64),
                score=cat(score, 0, np.float64))


def _select(track_begin, obs_keep, track_keep):
    """tracks with track_keep and >= 2 kept observations -> (their indices, new track_begin, kept observation indices)"""
    counts = np.add.reduceat(obs_keep.astype(np.int64), track_begin[:-1]) if len(obs_keep) else np.zeros(0, np.int64)
    tsel = np.flatnonzero(track_keep & (counts >= 2))
    obs_track = np.repeat(np.arange(len(track_begin) - 1), np.diff(track_begin))
    osel = np.flatnonzero(obs_keep & np.isin(obs_track, tsel))
    begin = np.zeros(len(tsel) + 1, np.int64)
    np.cumsum(counts[tsel], out=begin[1:])
    return tsel, begin, osel


def triangulate_points(reconstruction, keypoints, pairs, matches, scores=None, options=None, min_match_score=None,
                       keypoint_noise=None, skip_geometric_verification=False, timings=None):
    """The in-memory core of `main`: a new Reconstruction with the cameras and images (ids, names, poses) of
    `reconstruction`, every keypoint as a Point2D of its image, and the triangulated points (ids 1..N in ascending
    track-label order).  `options`: mapper options (see DEFAULT_MAPPER_OPTIONS); `keypoint_noise`: {name: pixels};
    `timings`: a dict that receives the seconds of each stage (host clock; `*_kernels` entries are device time)."""
    tm = timings if timings is not None else {}
    t0 = time.perf_counter()
    opts = mapper_options_from(options)
    P = pack_matches(reconstruction, keypoints, pairs, matches, scores, min_match_score, keypoint_noise)
    rec = reconstruction
    image_ids, kp_begin, kp_xy = P["image_ids"], P["kp_begin"], P["kp_xy"]
    images = [rec.images[int(i)] for i in image_ids]
    cam_ids = np.array(sorted(rec.cameras), np.int64)
    cam_index = {int(c): k for k, c in enumerate(cam_ids)}
    cam_model = np.array([int(rec.cameras[int(c)].model_id) for c in cam_ids], np.int32)
    cam_params = np.zeros((len(cam_ids), _capi.PXR_MAX_CAM_PARAMS))
    for k, c in enumerate(cam_ids):
        prm = np.asarray(rec.cameras[int(c)].params, np.float64)
        cam_params[k, :len(prm)] = prm
    img_cam = np.array([cam_index[int(im.camera_id)] for im in images], np.int32)
    qvec = np.array([im.qvec for im in images], np.float64).reshape(-1, 4)
    tvec = np.array([im.tvec for im in images], np.float64).reshape(-1, 3)
    cams = (cam_model, cam_params, img_cam, qvec, tvec)
    tm["pack"] = time.perf_counter() - t0

    # geometric verification against the known poses
    g = kp_begin[P["img"]] + P["kp"]                                      # [M, 2] global keypoint indices
    if skip_geometric_verification or len(g) == 0:
        keep = np.ones(len(g), bool)
    else:
        keep, _, t = _engine.tri_verify(_capi.TriScene(*cams), P["img"], kp_xy[g].reshape(-1, 4), P["noise"][P["img"]],
                                        VERIFY_MAX_ERROR)
        tm["verify_kernels"] = t["solve_time_s"]
    t0 = time.perf_counter()
    # tracks: nodes are (image, keypoint) in ascending order, verified matches the edges
    e = g[keep]
    nodes, inv = np.unique(e.reshape(-1), return_inverse=True)
    inv = inv.reshape(-1, 2)
    node_img = (np.searchsorted(kp_begin, nodes, side="right") - 1).astype(np.int32)
    labels = _engine.graph_labels(node_img, inv[:, 0], inv[:, 1], P["score"][keep])[0] if len(nodes) else np.zeros(0, np.int64)
    degree = np.bincount(inv.reshape(-1), minlength=len(nodes))
    length = np.bincount(labels) if len(labels) else np.zeros(0, np.int64)
    track_ok = length >= 2
    if opts["ignore_two_view_tracks"] and len(labels):
        # COLMAP's IsTwoViewObservation: a two-node track whose nodes have one correspondence each
        max_degree = np.zeros(len(length), np.int64)
        np.maximum.at(max_degree, labels, degree)
        track_ok &= ~((length == 2) & (max_degree == 1))
    sel = np.flatnonzero(track_ok[labels]) if len(labels) else np.zeros(0, np.int64)
    order = sel[np.argsort(labels[sel], kind="stable")]
    t_label = np.flatnonzero(track_ok)
    track_begin = np.zeros(len(t_label) + 1, np.int64)
    np.cumsum(length[t_label], out=track_begin[1:])
    obs_node, obs_img = nodes[order], node_img[order]
    tm["tracks"] = time.perf_counter() - t0

    # robust triangulation
    xyz = np.zeros((0, 3))
    if len(t_label):
        scene = _capi.TriScene(*cams, track_begin, obs_img, kp_xy[obs_node], track_key=t_label)
        res = _engine.tri_run(scene, _capi.default_tri_options(
            min_angle=float(opts["min_angle"]), create_max_angle_error=float(opts["create_max_angle_error"]),
            tri_max_pairs=int(opts["tri_max_pairs"]), seed=int(opts["seed"])))
        tsel, track_begin, osel = _select(track_begin, res["obs_inlier"], res["status"] == _capi.TRI_OK)
        t_label, xyz, obs_node, obs_img = t_label[tsel], res["xyz"][tsel], obs_node[osel], obs_img[osel]
        tm["triangulate_kernels"] = res["timing"]["solve_time_s"]

    # points-only bundle adjustment, then one filter pass
    t0 = time.perf_counter()
    if len(t_label) and int(opts["ba_max_num_iterations"]) > 0:
        xyz = _refine_points(rec, P, cam_ids, qvec, tvec, track_begin, obs_node, obs_img, xyz,
                             int(opts["ba_max_num_iterations"]))
    tm["ba"] = time.perf_counter() - t0
    err = np.zeros(0)
    if len(t_label):
        err, _, t = _engine.tri_evaluate(_capi.TriScene(*cams, track_begin, obs_img, kp_xy[obs_node]), xyz)
        tm["evaluate_kernels"] = t["solve_time_s"]
        tsel, track_begin, osel = _select(track_begin, err <= float(opts["filter_max_reproj_error"]),
                                          np.ones(len(t_label), bool))
        t_label, xyz, obs_node, obs_img = t_label[tsel], xyz[tsel], obs_node[osel], obs_img[osel]
    if len(t_label):
        err, angle, _ = _engine.tri_evaluate(_capi.TriScene(*cams, track_begin, obs_img, kp_xy[obs_node]), xyz)
        tsel, track_begin, osel = _select(track_begin, np.ones(len(obs_node), bool),
                                          angle >= float(opts["filter_min_tri_angle"]))
        t_label, xyz, obs_node, obs_img, err = t_label[tsel], xyz[tsel], obs_node[osel], obs_img[osel], err[osel]

    out = _assemble(rec, P, cam_ids, xyz, track_begin, obs_node, obs_img)
    n_obs = len(obs_node)
    logger.info("Triangulation: %d pairs, %d matches, %d verified, %d tracks, %d points, %d observations, "
                "mean track length %.3f, mean reprojection error %.3f px.", P["n_pairs"], len(g), int(keep.sum()),
                len(length), len(t_label), n_obs, n_obs / max(len(t_label), 1), float(err.mean()) if n_obs else 0.0)
    return out


def _refine_points(rec, P, cam_ids, qvec, tvec, track_begin, obs_node, obs_img, xyz, max_iterations):
    """GeometricBundleOptimizer over the points alone (poses and cameras constant, trivial loss) on an array-backed
    copy of the model -> refined xyz"""
    image_ids, kp_begin = P["image_ids"], P["kp_begin"]
    n_pts = len(track_begin) - 1
    pid = np.arange(1, n_pts + 1, dtype=np.int64)
    obs_pid = np.repeat(pid, np.diff(track_begin))
    p2d_pid = np.full(int(kp_begin[-1]), -1, np.int64)
    p2d_pid[obs_node] = obs_pid
    cams = [rec.cameras[int(c)] for c in cam_ids]
    arec = ArrayReconstruction(image_ids, P["names"], [rec.images[int(i)].camera_id for i in image_ids], qvec.copy(),
                               tvec.copy(), kp_begin, p2d_pid, cam_ids, [int(c.model_id) for c in cams],
                               [np.asarray(c.params, np.float64) for c in cams], pid, xyz.copy(), track_begin,
                               image_ids[obs_img], obs_node - kp_begin[obs_img])
    arec.p2d_xy = P["kp_xy"]
    setup = ba.BundleAdjustmentSetup()
    setup.add_images(image_ids.tolist())
    options = ba.BundleOptimizerOptions(refine_focal_length=False, refine_principal_point=False, refine_extra_params=False,
                                        refine_extrinsics=False, print_summary=False,
                                        loss={"name": "trivial", "params": []},
                                        solver={"max_num_iterations": max_iterations})
    ba.GeometricBundleOptimizer(options, setup).run(arec)
    return arec.xyz


def _assemble(rec, P, cam_ids, xyz, track_begin, obs_node, obs_img):
    """the output Reconstruction: the model's cameras and images, every keypoint a Point2D, points 1..N"""
    out = Reconstruction()
    for c in cam_ids:
        cam = rec.cameras[int(c)]
        out.add_camera(Camera(int(c), int(cam.model_id), cam.width, cam.height, np.array(cam.params, np.float64)))
    kp_begin, kp_xy = P["kp_begin"], P["kp_xy"]
    for k, i in enumerate(P["image_ids"]):
        im = rec.images[int(i)]
        out.add_image(Image(int(i), im.name, im.camera_id, np.array(im.qvec, np.float64), np.array(im.tvec, np.float64),
                            [Point2D(xy) for xy in kp_xy[kp_begin[k]:kp_begin[k + 1]]]))
    image_id = P["image_ids"][obs_img].tolist()
    p2d_idx = (obs_node - kp_begin[obs_img]).tolist()
    for t in range(len(track_begin) - 1):
        pid = t + 1
        out.add_point3D(pid, xyz[t])
        for o in range(int(track_begin[t]), int(track_begin[t + 1])):
            out.add_observation(pid, image_id[o], p2d_idx[o])
    return out


def read_inputs(reference_model, pairs, features, matches):
    """hloc's files -> (reference Reconstruction without its points3D, keypoints in COLMAP convention, keypoint noise,
    pairs without repeats, matches, scores).  An image of the model missing from the keypoint file raises ValueError."""
    rec = Reconstruction.read(str(reference_model))
    rec.points3D = {}
    names = [rec.images[i].name for i in sorted(rec.images)]
    available = set(list_h5_names(features))
    missing = [n for n in names if n not in available]
    if missing:
        raise ValueError("image(s) of the model missing from %s: %s" % (features, ", ".join(missing[:10])))
    keypoints = read_keypoints_hloc(features, names)
    for n in names:
        keypoints[n] += 0.5                    # hloc -> COLMAP pixel convention
    noise = read_keypoint_uncertainty(features, names)
    pair_list = unique_pairs(tuple(p) for p in read_image_pairs(pairs))
    m, s = read_matches_hloc(matches, pair_list)
    return rec, keypoints, noise, pair_list, m, s


def main(sfm_dir, reference_model, image_dir, pairs, features, matches, skip_geometric_verification=False,
         estimate_two_view_geometries=False, min_match_score=None, verbose=False, mapper_options=None):
    """hloc.triangulation.main's signature: triangulates the model at `reference_model` (binary or text) from hloc's
    pairs / keypoint / match files, writes it to `sfm_dir` as a binary COLMAP model and returns it.  `image_dir` and
    `verbose` are accepted for the signature and not used; `mapper_options` takes the keys of DEFAULT_MAPPER_OPTIONS."""
    if estimate_two_view_geometries:
        raise ValueError("estimate_two_view_geometries=True is not supported: relative poses are not estimated")
    options = mapper_options_from(mapper_options)
    rec, keypoints, noise, pair_list, m, s = read_inputs(reference_model, pairs, features, matches)
    out = triangulate_points(rec, keypoints, pair_list, m, s, options, min_match_score=min_match_score,
                             keypoint_noise=noise, skip_geometric_verification=skip_geometric_verification)
    sfm_dir = Path(sfm_dir)
    sfm_dir.mkdir(parents=True, exist_ok=True)
    out.write(str(sfm_dir))
    return out
