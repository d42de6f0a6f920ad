"""Batched absolute pose estimation (pxr_pnp_run) on one synthetic workload, beside the host restatement and the
batched localizer with the built-in PnP.

Workload: N queries x M correspondences (default 1000 x 500), PINHOLE f = 800, points 4-8 units in front of the camera,
0.5 px noise, 30 % outliers placed at least 36 px (3 x max_error) from their true projection, pycolmap's default
options (max_error 12 px, min 1000 trials, confidence 0.9999, refinement on).

  pxr_pnp_run   CUDA events around the RANSAC and refinement kernels (the call's solve time), median of three runs
                after one warm-up, plus the host clock around the whole call (uploads and copies back included)
  host          tests/pnp_reference.ransac (numpy / Python, one core) on the first --host-queries queries, per query
  localize      QueryLocalizer.localize_batch on localize_batch_bench.make_workload with the built-in PnP in place of
                the ground-truth stand-in (pycolmap made unimportable), host clock

One JSON line; the card's name and power limit are read in the same run."""
import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT / "pixel-perfect-sfm_b200"))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "scripts"))

from pixsfm._pixsfm import _capi, _engine  # noqa: E402
from pixsfm.util import cameras  # noqa: E402
import localize_batch_bench as lbb  # noqa: E402
import pnp_reference as P  # noqa: E402


def make_pnp_workload(n_queries, n_corr, outliers, seed):
    rng = np.random.default_rng(seed)
    params = np.array([800.0, 800.0, 512.0, 384.0])
    p2, p3, truth = [], [], []
    for _ in range(n_queries):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        t = rng.normal(size=3)
        R = P.quat_to_rot(q)
        uv = rng.uniform([-0.6, -0.45], [0.6, 0.45], (n_corr, 2))
        d = rng.uniform(4.0, 8.0, n_corr)
        X = (np.column_stack([uv * d[:, None], d]) - t) @ R
        xy = cameras.world_to_image(1, params, q, t, X) + rng.normal(0, 0.5, (n_corr, 2))
        for i in np.nonzero(rng.random(n_corr) < outliers)[0]:
            while True:
                c = rng.uniform([0, 0], [1024, 768])
                if np.linalg.norm(c - xy[i]) > 36.0:
                    xy[i] = c
                    break
        p2.append(xy); p3.append(X); truth.append((q, t))
    return params, p2, p3, truth


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--corr", type=int, default=500)
    ap.add_argument("--outliers", type=float, default=0.3)
    ap.add_argument("--host-queries", type=int, default=3)
    ap.add_argument("--localize-queries", type=int, default=1000)
    ap.add_argument("--points", type=int, default=100000)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    name, power = lbb.card()
    params, p2, p3, truth = make_pnp_workload(a.queries, a.corr, a.outliers, a.seed)
    cp = np.zeros(12); cp[:4] = params
    begin = np.arange(a.queries + 1) * a.corr

    def batch():
        return _capi.PnPBatch(begin, np.concatenate(p2), np.concatenate(p3), [1] * a.queries, [cp] * a.queries,
                              np.arange(a.queries, dtype=np.uint64))

    _engine.pnp_run(batch())                                   # warm-up: module load, first launches
    kern, wall = [], []
    for _ in range(3):
        b = batch()
        t0 = time.perf_counter()
        res, info = _engine.pnp_run(b)
        wall.append(time.perf_counter() - t0)
        kern.append(info["solve_time_s"])
    ok = sum(r["success"] for r in res)
    trials = [r["num_trials"] for r in res]
    rot_err = [np.degrees(2 * np.arccos(min(1.0, abs(float(b.qvec[k] @ truth[k][0]))))) for k in range(a.queries)]

    n_host = min(a.host_queries, a.queries)
    t0 = time.perf_counter()
    for k in range(n_host):
        uv = _engine.pnp_debug_image_to_world(1, params, p2[k])
        P.ransac(uv, p3[k], 12.0 / 800.0, k)
    host_per_query = (time.perf_counter() - t0) / max(n_host, 1)

    sys.modules["pycolmap"] = None                             # the localizer falls back to the built-in estimator
    from pixsfm import localization as loc_pkg
    rec, refs, queries, _ = lbb.make_workload(a.localize_queries, a.corr, a.points, 128, a.seed)
    L = loc_pkg.QueryLocalizer(rec, {}, references=[refs])
    t0 = time.perf_counter()
    out = L.localize_batch(queries)
    loc_s = time.perf_counter() - t0

    med = statistics.median(kern)
    print(json.dumps({
        "metric": "pxr_pnp_run queries/s", "value": a.queries / med, "unit": "queries/s",
        "card": name, "power_limit": power,
        "workload": "%d queries x %d correspondences, %.0f %% outliers, PINHOLE, pycolmap default options" %
                    (a.queries, a.corr, 100 * a.outliers),
        "pnp_kernel_seconds_median_of_3 (CUDA events)": med, "pnp_kernel_seconds_runs": kern,
        "pnp_call_seconds_runs (host clock)": wall,
        "queries_succeeded": ok, "trials_per_query": {"median": statistics.median(trials), "max": max(trials),
                                                      "mean": float(np.mean(trials))},
        "rotation_error_deg": {"median": float(np.median(rot_err)), "max": float(np.max(rot_err))},
        "host_restatement_seconds_per_query": host_per_query, "host_queries_run": n_host,
        "host_vs_device_per_query": host_per_query / (med / a.queries),
        "localize_batch": {"queries": a.localize_queries, "seconds": loc_s,
                           "queries_per_s": a.localize_queries / loc_s,
                           "localized": sum(bool(o.get("success")) for o in out),
                           "workload": "localize_batch_bench.make_workload, default QueryLocalizer conf, built-in PnP"},
    }))


if __name__ == "__main__":
    main()
