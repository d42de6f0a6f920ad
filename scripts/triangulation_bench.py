"""Triangulation from known poses (pixsfm.triangulation.triangulate_points) on synthetic models: one JSON line.

Workloads (0.5 px keypoint noise, 5 % of the matches sent to a random keypoint, every pair of a track's images matched):
  eth3d   38 images, 100 000 points, tracks of 3-12 observations (the size of an ETH3D triangulation scene)
  large   300 images, 300 000 points, tracks of 3-12 observations
For each: the device time (CUDA events) of pxr_tri_verify, of pxr_tri_run (ray, track and error kernels) and of the first
pxr_tri_evaluate, and the host-clock time of packing the inputs, the track labels, the points-only bundle adjustment and
triangulate_points end to end: the median of three runs after one warm-up run.  The numpy restatement
(tests/triangulation_reference.py) is timed on a 10 000-track sample of `eth3d`: it is the test oracle, not a tuned CPU
baseline.  Run from the repository root on a machine with a GPU:  python scripts/triangulation_bench.py"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "pixel-perfect-sfm_b200"), os.path.join(ROOT, "tests")]

import triangulation_reference as T  # noqa: E402
from pixsfm.triangulation import triangulate_points  # noqa: E402
from pixsfm.util import colmap_types as ct  # noqa: E402
from pixsfm.util.cameras import normalized_to_image  # noqa: E402


def make_workload(n_images, n_points, seed=0, noise_px=0.5, wrong=0.05, max_len=12):
    rng = np.random.default_rng(seed)
    params = np.array(T.CAMERAS[1])
    qv, tv = T.ring_poses(n_images, seed=seed)
    X = rng.uniform(-1.5, 1.5, (n_points, 3))
    L = rng.integers(3, max_len + 1, n_points)
    # distinct images per track: increasing offsets whose sum stays below n_images
    step = rng.integers(1, max(2, n_images // max_len), (n_points, max_len))
    imgs = np.sort((rng.integers(0, n_images, n_points)[:, None] + np.cumsum(step, 1)) % n_images, axis=1)
    valid = np.arange(max_len)[None] < L[:, None]
    imgs = np.sort(np.where(valid, imgs, n_images), axis=1)              # invalid slots last
    valid = imgs < n_images
    obs_p, obs_slot = np.nonzero(valid)
    obs_i = imgs[obs_p, obs_slot]
    order = np.argsort(obs_i, kind="stable")
    start = np.searchsorted(obs_i[order], np.arange(n_images))
    kp_idx = np.empty(len(obs_i), np.int64)
    kp_idx[order] = np.arange(len(obs_i)) - np.repeat(start, np.bincount(obs_i, minlength=n_images))
    rec = ct.Reconstruction()
    rec.add_camera(ct.Camera(1, "PINHOLE", 640, 480, params))
    names = ["img%03d.jpg" % k for k in range(n_images)]
    keypoints = {}
    for k in range(n_images):
        sel = order[start[k]:start[k] + np.count_nonzero(obs_i == k)]
        kp = np.zeros((len(sel), 2))
        kp[kp_idx[sel]] = normalized_to_image(1, params, T.project_normalised(qv[k], tv[k], X[obs_p[sel]]))
        keypoints[names[k]] = kp + rng.normal(0, noise_px, kp.shape)
        rec.add_image(ct.Image(k + 1, names[k], 1, qv[k], tv[k]))
    slot_kp = np.full(imgs.shape, -1, np.int64)
    slot_kp[obs_p, obs_slot] = kp_idx
    src, dst = [], []
    for a in range(max_len):
        for b in range(a + 1, max_len):
            m = valid[:, b]
            src.append(np.column_stack([imgs[m, a], slot_kp[m, a]]))
            dst.append(np.column_stack([imgs[m, b], slot_kp[m, b]]))
    src, dst = np.concatenate(src), np.concatenate(dst)
    counts = np.bincount(obs_i, minlength=n_images)
    bad = rng.random(len(dst)) < wrong
    dst[bad, 1] = (rng.random(bad.sum()) * counts[dst[bad, 0]]).astype(np.int64)
    key = src[:, 0] * n_images + dst[:, 0]
    o = np.argsort(key, kind="stable")
    uk, first = np.unique(key[o], return_index=True)
    bounds = np.append(first, len(o))
    pairs, matches, scores = [], [], []
    for q, k in enumerate(uk):
        sel = o[bounds[q]:bounds[q + 1]]
        pairs.append((names[k // n_images], names[k % n_images]))
        matches.append(np.column_stack([src[sel, 1], dst[sel, 1]]))
        scores.append(rng.uniform(0.5, 1.0, len(sel)))
    return rec, keypoints, pairs, matches, scores, len(obs_i)


def gpu_card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def bench(name, n_images, n_points, runs=3):
    t0 = time.perf_counter()
    rec, keypoints, pairs, matches, scores, n_obs = make_workload(n_images, n_points)
    gen = time.perf_counter() - t0
    results = []
    for r in range(runs + 1):
        tm = {}
        t0 = time.perf_counter()
        out = triangulate_points(rec, keypoints, pairs, matches, scores, timings=tm)
        tm["end_to_end"] = time.perf_counter() - t0
        if r:
            results.append(tm)
    med = {k: float(np.median([t[k] for t in results])) * 1e3 for k in results[0]}
    return dict(workload=name, images=n_images, points=n_points, observations=n_obs,
                matches=int(sum(len(m) for m in matches)), pairs=len(pairs), generate_s=round(gen, 2),
                triangulated_points=len(out.points3D), observations_kept=out.num_observations(),
                verify_kernel_ms=med["verify_kernels"], tri_run_kernels_ms=med["triangulate_kernels"],
                evaluate_kernels_ms=med["evaluate_kernels"], pack_ms=med["pack"], track_labels_ms=med["tracks"],
                points_only_ba_ms=med["ba"], end_to_end_ms=med["end_to_end"]), rec, keypoints


def oracle_time(n_tracks=10000, seed=1):
    """the numpy restatement over n_tracks tracks of 3-12 observations (ETH3D-shaped geometry)"""
    rng = np.random.default_rng(seed)
    qv, tv = T.ring_poses(38)
    t0 = time.perf_counter()
    for _ in range(n_tracks):
        L = int(rng.integers(3, 13))
        imgs = np.sort(rng.choice(38, L, replace=False))
        X = rng.uniform(-1.5, 1.5, 3)
        d, c = zip(*[T.rays(T.project_normalised(qv[k], tv[k], X[None]) + rng.normal(0, 1e-3, 2), qv[k], tv[k])
                     for k in imgs])
        T.triangulate_track(np.concatenate(d), np.concatenate(c))
    return (time.perf_counter() - t0) * 1e3


def main():
    card = gpu_card()
    rows = [bench("eth3d", 38, 100_000)[0], bench("large", 300, 300_000)[0]]
    print(json.dumps(dict(card=card, workloads=rows, numpy_oracle_10k_tracks_ms=oracle_time(),
                          note="kernel times are CUDA-event medians of 3 runs after a warm-up; the numpy oracle is the "
                               "test restatement, not a tuned CPU baseline")))


if __name__ == "__main__":
    main()
