"""Keypoint adjustment of problems with more than 80 variable keypoints, on one GPU.  Prints one JSON line.

    python scripts/ka_large_problems_bench.py [--tracks 25000] [--repeats 3] [--workloads abc]

Every workload has the shape of the `low_memory` preset's KA step: topological-reference edges (one unit-weight edge
from every non-root keypoint to its track's root, which stays constant), tracks of 4, 8x8 fp16 patches of 128
channels, bound 2, Cauchy(0.25) loss, parameter tolerance 1e-5:
  a  the whole scene (4 x tracks keypoints) in problems of <= 1000 keypoints, the preset's max_kps_per_problem:
     about 750 variable keypoints per problem, each its own 2x2 block, solved on chip;
  b  the same scene in problems of <= 50 keypoints, sizes that also run where problems were limited to 80 variable
     keypoints;
  c  one problem over the first 20 000 keypoints (split_in_subproblems: False).  Its workspace does not fit in shared
     memory, so it lives in global memory; one problem is one CTA, so this runs on one SM by design.
Per workload: end-to-end seconds of pxr_ka_run (host packing, upload, solve, download; the smallest and the median of
the repeats), the solve kernel's time from the run's summary, keypoints per second end to end, and the number of
problems whose workspace was off chip."""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "pixel-perfect-sfm_b200"))

CHUNK = 2500          # tracks per generated piece of the scene (bounds the generator's float32 temporaries)


def make_scene(n_tracks, seed=11):
    """tracks of 4 in 40 images, generated in pieces; -> list of (keypoints, roots, track labels, patches, corner,
    scale) per piece, track labels already global"""
    from pixsfm._pixsfm import _engine
    from pixsfm.util import synthetic
    pieces, t0 = [], 0
    for k, start in enumerate(range(0, n_tracks, CHUNK)):
        nt = min(CHUNK, n_tracks - start)
        sc = synthetic.make_ka_scene(n_images=40, n_tracks=nt, track_len=4, channels=128, ps=8, seed=seed + k,
                                     kp_sigma=1.0, dtype=np.float16)
        tl, _, roots = _engine.graph_labels(sc["node_image"], sc["edge_src"], sc["edge_dst"], sc["edge_sim"])
        pieces.append((sc["keypoints"], roots, tl + t0, sc["patches"], sc["corner"], sc["scale"]))
        t0 += int(tl.max()) + 1
    return pieces


def ka_problem(pieces, max_per_problem):
    """the topological-reference IR over the given pieces, packed first-fit decreasing (max_per_problem <= 0: one
    problem)"""
    from pixsfm._pixsfm import _capi, _engine
    kps, roots, tl = (np.concatenate([p[i] for p in pieces]) for i in range(3))
    if max_per_problem > 0:
        plabels, n_prob = _engine.ka_problem_labels(tl, max_per_problem)
    else:
        plabels, n_prob = np.zeros(len(tl), np.int64), 1
    root_of = np.full(int(tl.max()) + 1, -1, np.int64)
    root_of[tl[roots == 1]] = np.nonzero(roots == 1)[0]
    src = np.nonzero(roots == 0)[0]
    dst = root_of[tl[src]]
    order = np.argsort(plabels[src], kind="stable")
    src, dst = src[order], dst[order]
    return _capi.KAProblem(keypoints=kps, kp_const=roots, edge_src=src, edge_dst=dst, edge_weight=np.ones(len(src)),
                           edge_problem=plabels[src], n_problems=n_prob,
                           patches=np.ascontiguousarray(np.concatenate([p[3] for p in pieces])),
                           corner=np.concatenate([p[4] for p in pieces]), scale=np.concatenate([p[5] for p in pieces]),
                           bound=2.0, patches_are_sparse=True)


def run(prob, repeats):
    from pixsfm._pixsfm import _capi, _engine
    ic = _capi.default_interp()
    so = _capi.default_ka_options(parameter_tolerance=1e-5)
    e2e, kms = [], []
    for _ in range(repeats):
        p = prob.copy()
        t0 = time.perf_counter()
        s = _engine.ka_run(p, ic, so)       # returns after the keypoints are back on the host
        e2e.append(time.perf_counter() - t0)
        kms.append(float(re.search(r"solve kernel ([0-9.]+) ms", s["message"]).group(1)))
    roots = prob.kp_const == 1
    assert np.array_equal(p.keypoints[roots], prob.keypoints[roots])
    off = re.search(r"(\d+) with an off-chip workspace", s["message"])
    return {"keypoints": len(prob.keypoints), "variable_keypoints": int(np.sum(~roots)), "edges": len(prob.edge_src),
            "problems": prob.n_problems, "seconds_e2e_min": min(e2e), "seconds_e2e_median": float(np.median(e2e)),
            "solve_kernel_ms_min": min(kms), "solve_kernel_ms_median": float(np.median(kms)),
            "keypoints_per_s_e2e": len(prob.keypoints) / min(e2e), "offchip_problems": int(off.group(1)) if off else None,
            "initial_cost": s["initial_cost"], "final_cost": s["final_cost"], "message": s["message"]}


def gpu_info():
    """name and power limit of the card the numbers were taken on"""
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True, timeout=60, check=True)
    name, power = [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tracks", type=int, default=25000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--workloads", default="abc")
    args = ap.parse_args()
    t0 = time.time()
    pieces = make_scene(args.tracks)
    gen = time.time() - t0
    run(ka_problem(pieces[:1], 50), 1)           # warm-up: context, module load
    out = {"workload": "KA, low_memory shape: topological-reference edges, 8x8 fp16 128-ch patches, bound 2, "
                       "%d keypoints" % (4 * args.tracks)}
    if "a" in args.workloads:
        out["a_bins_of_1000"] = run(ka_problem(pieces, 1000), args.repeats)
    if "b" in args.workloads:
        out["b_bins_of_50"] = run(ka_problem(pieces, 50), args.repeats)
    if "c" in args.workloads:
        out["c_one_problem_20k"] = run(ka_problem(pieces[:20000 // (4 * CHUNK)], 0), args.repeats)
    out["gpu"], out["power_limit"] = gpu_info()
    out["scene_generation_s"] = gen
    print(json.dumps(out))


if __name__ == "__main__":
    main()
