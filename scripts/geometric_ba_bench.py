"""Geometric (reprojection-error) BA on the benchmark scene: time per LM iteration on the GPU, the stages of it, and
the CPU restatement's time for the same solve.

Scene: bench.py's configs[2] geometry (200 cameras / 50 000 points / 500 000 observations, SIMPLE_RADIAL, the gauge of
bench.make_problem) with keypoints = the true projections + seeded N(0, 0.5 px) noise; the solve starts from bench's
perturbed parameters.  Per run: 3 warm-up LM iterations, pxr_ba_reset, then 5 iterations from iteration zero (timed)
and the 5 after them (steady state), CUDA events on the library stream.  Then the geometric-evaluation stage and K0
(pxr_ba_time_stage 0 and 3), and the CPU restatement's -O3 build (oracle_geo/liboracle_geo_fast.so) on the same solve
from iteration zero.  The card name and its power limit are printed with the numbers.

    python scripts/geometric_ba_bench.py [--runs 3] [--no-cpu] [--no-inner]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pixel-perfect-sfm_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as e:      # noqa: BLE001
        return {"gpu": "unknown", "power_limit": "unknown (%s)" % e}


def problem(seed=0):
    import bench
    from pixsfm._pixsfm import _capi
    saved = sys.argv
    sys.argv = [saved[0]]
    try:
        bargs = bench.parse()
    finally:
        sys.argv = saved
    g = bench.geometry(bargs, 0)
    xy = g["uv0"] + 0.5 + g["corners"]                      # the true projections (scale 1)
    kp = xy + np.random.default_rng(seed + 7).normal(0, 0.5, xy.shape)
    n_cams, n_models = bargs.cams, len(g["cam_params"])
    pose_const = np.zeros(n_cams, np.uint8); pose_const[0] = 1
    tmask = np.zeros(n_cams, np.uint8); tmask[1] = 1
    _, pp, _ = _capi.CAMERA_PARAM_GROUPS[2]
    return _capi.BAProblem(cam_model=np.full(n_models, 2, np.int32), cam_params=g["cam_params"],
                           cam_const_mask=np.full(n_models, pp, np.uint32), qvec=g["qvec"], tvec=g["tvec"],
                           img_cam=g["img_cam"], pose_const=pose_const, tvec_const_mask=tmask, xyz=g["xyz"],
                           point_const=np.zeros(len(g["xyz"]), np.uint8), obs_img=g["obs_img"], obs_pt=g["obs_pt"],
                           patches=None, corner=None, scale=None, obs_xy=kp)


def gpu_run(prob, so, steps, warmup):
    from pixsfm._pixsfm import _capi, _engine
    ctx = _capi.default_context()
    h = _engine.BAHandle(prob.copy(), options=so, ctx=ctx)
    try:
        h.iterate(warmup)
        h.reset(prob.cam_params, prob.qvec, prob.tvec, prob.xyz)
        l0 = ctx.kernel_launches()
        ctx.timer_start(); s1 = h.iterate(steps); ms1 = ctx.timer_stop()
        launches = ctx.kernel_launches() - l0
        ctx.timer_start(); s2 = h.iterate(steps); ms2 = ctx.timer_stop()
        n1 = len(s1["iterations"]) - 1
        n2 = len(s2["iterations"]) - 1 - n1
        return {"ms_per_iteration": ms1 / max(n1, 1), "iterations": n1, "launches_per_iteration": launches / max(n1, 1),
                "steady_ms_per_iteration": ms2 / max(n2, 1) if n2 > 0 else None, "steady_iterations": n2,
                "geometric_eval_ms": h.time_stage(0, 20), "k0_ms": h.time_stage(3, 20),
                "cost": [s1["iterations"][0]["cost"], s1["iterations"][-1]["cost"]]}
    finally:
        h.close()


def cpu_run(prob, so, steps):
    import geo_oracle_lib as GO
    o = type(so).from_buffer_copy(so)
    o.max_num_iterations = steps
    p = prob.copy()
    t0 = time.perf_counter()
    s = GO.ba_solve_geometric(p, o, fast=True)
    dt = time.perf_counter() - t0
    return {"cpu_s": dt, "cpu_ms_per_iteration": 1e3 * dt / max(len(s["iterations"]) - 1, 1),
            "cpu_threads": os.cpu_count(), "cost": [s["iterations"][0]["cost"], s["iterations"][-1]["cost"]]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--no-inner", action="store_true")
    args = ap.parse_args()
    from pixsfm._pixsfm import _capi
    info = card()
    print(json.dumps(info), flush=True)
    prob = problem()
    so = _capi.default_ba_options(use_inner_iterations=0 if args.no_inner else 1)
    print(json.dumps({"n_images": len(prob.qvec), "n_points": len(prob.xyz), "n_obs": prob.n_obs,
                      "inner_iterations": not args.no_inner}), flush=True)
    for r in range(args.runs):
        out = dict(info, run=r, **gpu_run(prob, so, args.steps, args.warmup))
        print(json.dumps(out), flush=True)
    if not args.no_cpu:
        print(json.dumps(dict(info, **cpu_run(prob, so, args.steps))), flush=True)


if __name__ == "__main__":
    main()
