"""Batched localization (QueryLocalizer.localize_batch) against a loop of localize on one synthetic workload.

Workload: N queries x M correspondences, every 3D point with 4 stored observations, C = 128 fp16 16x16 patches made
on the device, the default QueryLocalizer configuration (target_reference 'nearest', QKA and QBA on) and a stand-in
pose estimator that returns the ground-truth pose with every correspondence an inlier (PnP is a user callable; this
keeps its cost out of the comparison).  The loop arm runs localize on the first --loop-queries queries (host copies of
their patches: localize takes host maps) and is extrapolated to N queries; the output says so.

The batched time is split into the device calls it makes (host clock around each call; every call ends with a device
synchronise, so each includes its uploads), the pose estimator, and the rest (Python packing).  The kernel times
pxr_qka_run and pxr_qba_run report (CUDA events) are printed beside them.  One JSON line; the card's name and power
limit are read in the same run."""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "pixel-perfect-sfm_b200"))

from pixsfm import localization as loc_pkg  # noqa: E402
from pixsfm._pixsfm import _engine, _features  # noqa: E402
from pixsfm.util import colmap_types as ct  # noqa: E402


class _Point:
    def __init__(self, xyz):
        self.xyz = xyz


class _Rec:
    def __init__(self, points3D):
        self.points3D = points3D


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:                      # the numbers are still printed, without the card
        return "unknown (%s)" % e, "unknown"


def make_workload(n_queries, n_corr, n_points, channels, seed):
    rng = np.random.default_rng(seed)
    W, H, f = 1024, 768, 800.0
    cam = ct.Camera(1, "PINHOLE", W, H, np.array([f, f, W / 2, H / 2]))
    # points and their stored observations (unit descriptors, as L2-normalised features)
    xyz = rng.uniform([-4, -3, 6], [4, 3, 12], (n_points, 3))
    refs = {}
    for pid in range(n_points):
        obs = rng.standard_normal((4, channels)); obs /= np.linalg.norm(obs, axis=1, keepdims=True)
        r = _features.Reference(descriptor=obs[0].reshape(1, -1))
        r.observations = [o.reshape(1, -1) for o in obs]
        refs[pid] = r
    rec = _Rec({pid: _Point(xyz[pid]) for pid in range(n_points)})
    queries, poses = [], []
    for q in range(n_queries):
        pids = rng.choice(n_points, n_corr, replace=False)
        tvec = rng.normal(0, 0.05, 3)
        qvec = np.array([1.0, 0.0, 0.0, 0.0])
        cam_pts = xyz[pids] + tvec
        uv = cam_pts[:, :2] / cam_pts[:, 2:3] * f + [W / 2, H / 2]
        kps = uv + rng.normal(0, 0.5, uv.shape)
        corners = np.floor(kps).astype(np.int32) - 8
        # the patches are made on the device: one smooth field per point, its centre at the true projection
        uv0 = (uv - corners - 0.5)
        dptr = _engine.synth_patches_device(n_corr, 16, channels, uv0, pids, seed=seed + q, noise=0.01)
        slab = _engine.DeviceSlab(dptr, (n_corr, 16, 16, channels), np.float16, _engine._capi.default_context())
        fmap = _features.FeatureMap(slab, list(range(n_corr)), corners, {"scale": [1.0, 1.0], "is_sparse": True})
        pose = dict(success=True, qvec=qvec, tvec=tvec, inliers=[True] * n_corr)
        queries.append(dict(keypoints=kps, pnp_point2D_idxs=list(range(n_corr)), pnp_points3D_id=[int(p) for p in pids],
                            query_camera=cam, query_fmaps=[fmap]))
        poses.append(pose)
    return rec, refs, queries, poses


def host_maps(query):
    fm = query["query_fmaps"][0]
    shape = tuple(fm.patches.shape)
    host = np.empty(shape, np.float16)
    _engine.memcpy_d2h(host, fm.patches.ptr, host.nbytes)
    return [_features.FeatureMap(host, fm.point2D_ids, fm.corners, {"scale": fm.scale, "is_sparse": True})]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--corr", type=int, default=500)
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--channels", type=int, default=128)
    ap.add_argument("--loop-queries", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    name, power = card()
    t = time.perf_counter()
    rec, refs, queries, poses = make_workload(a.queries, a.corr, a.points, a.channels, a.seed)
    setup_s = time.perf_counter() - t

    times = {"query_match_run": 0.0, "qka_run": 0.0, "qba_run": 0.0, "pose_estimator": 0.0}
    kernel = {"qka_run": 0.0, "qba_run": 0.0}
    calls = {k: 0 for k in times}

    def timed(key, fn, kern=None):
        def run(*args, **kw):
            t0 = time.perf_counter()
            out = fn(*args, **kw)
            times[key] += time.perf_counter() - t0
            calls[key] += 1
            if kern == "qka" and isinstance(out, dict) and "n_waves" in out:
                kernel["qka_run"] += out["solve_time_s"]
            if kern == "qba":
                kernel["qba_run"] += out[1]["solve_time_s"]
            return out
        return run

    orig = (_engine.query_match_run, _engine.ka_run, _engine.qba_run)
    _engine.query_match_run = timed("query_match_run", orig[0])
    _engine.ka_run = timed("qka_run", orig[1], "qka")
    _engine.qba_run = timed("qba_run", orig[2], "qba")
    for qd, pose in zip(queries, poses):
        qd["pose_estimator"] = timed("pose_estimator", lambda p2, p3, cam, pose=pose: dict(
            pose, qvec=pose["qvec"].copy(), tvec=pose["tvec"].copy(), inliers=list(pose["inliers"])))
    L = loc_pkg.QueryLocalizer(rec, {}, references=[refs])
    t = time.perf_counter()
    out = L.localize_batch(queries)
    batch_s = time.perf_counter() - t
    _engine.query_match_run, _engine.ka_run, _engine.qba_run = orig
    ok = sum(bool(o.get("success")) for o in out)

    n_loop = min(a.loop_queries, a.queries)
    loop_q = [dict(qd, query_fmaps=host_maps(qd)) for qd in queries[:n_loop]]
    L2 = loc_pkg.QueryLocalizer(rec, {}, references=[refs])
    t = time.perf_counter()
    for qd in loop_q:
        L2.localize(**qd)
    loop_s = time.perf_counter() - t
    loop_per_query = loop_s / max(n_loop, 1)

    device_calls = times["query_match_run"] + times["qka_run"] + times["qba_run"]
    res = {
        "metric": "localize_batch queries/s", "value": a.queries / batch_s, "unit": "queries/s",
        "card": name, "power_limit": power,
        "workload": "%d queries x %d correspondences, %d points x 4 stored observations, C=%d fp16 16x16 device patches, "
                    "default QueryLocalizer conf, ground-truth stand-in PnP" % (a.queries, a.corr, a.points, a.channels),
        "batched_seconds": batch_s, "queries_localized": ok,
        "split_seconds": {"pxr_query_match_run (calls, host clock)": times["query_match_run"],
                          "pxr_qka_run (calls, host clock)": times["qka_run"],
                          "pxr_qba_run (calls, host clock)": times["qba_run"],
                          "pose estimator (PnP stand-in)": times["pose_estimator"],
                          "rest (Python packing and glue)": batch_s - device_calls - times["pose_estimator"]},
        "kernel_seconds": {"qka solve kernels (CUDA events)": kernel["qka_run"],
                           "qba solve kernels (CUDA events)": kernel["qba_run"]},
        "calls": calls,
        "loop_of_localize": {"queries_run": n_loop, "seconds": loop_s, "queries_per_s": 1.0 / loop_per_query,
                             "extrapolated_seconds_for_all": loop_per_query * a.queries,
                             "note": "extrapolated from the first %d queries (host patch copies)" % n_loop},
        "speedup_vs_loop_extrapolated": loop_per_query * a.queries / batch_s,
        "setup_seconds": setup_s,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
