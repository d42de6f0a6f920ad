#!/usr/bin/env python
"""Where the inner-iteration time of the benchmark goes, round by round.

    python scripts/inner_rounds_profile.py [--steps 5] [--warmup 3] [--out FILE]

Runs bench.py's workload (BASELINE configs[2]: the same geometry, seeds and options, inner iterations on) and, like
bench.py, times the first `steps` LM iterations from iteration zero after `warmup` iterations and a reset.  It walks
that trajectory twice from the same start:
  1. with the stage timers on: per LM iteration the "inner iterations" (stage 9) and "K1 residual/Jacobian" (stage 1)
     device time, the same CUDA-event stages bench.py reports;
  2. with the round timers on (pxr_ba_debug_inner_rounds): per LM iteration the rounds of its inner iterations, each
     with its active points, active observations and stream time.  That is the time between two events recorded
     around the round's launches, so it includes any time the device sat idle waiting for the host to enqueue them
     (the host runs ahead of the device and only waits on a round two behind): it is not kernel time.  The extra
     events make this pass slightly slower.  Each round is also split at the ends of its three launches
     (pxr_ba_debug_inner_round_split): K0 (the projection), K1 (fm_eval_kernel) and the step kernel, each part with
     the launch gap in front of it, reported per round and summed per LM iteration.
It prints one JSON object, with the card name and power limit read in the same process, and the share of the inner
rounds whose list is shorter than 32 items per K1 warp (--short-list, default 32 x 132 SMs x 16 warps = 67 584).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "pixel-perfect-sfm_b200"))

import numpy as np  # noqa: E402

import bench  # noqa: E402  (geometry and problem set-up of the benchmark workload)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, plim, smax = [x.strip() for x in r.stdout.strip().split(",")[:3]]
        return {"name": name, "power_limit": plim, "sm_max_clock": smax}
    except Exception as ex:   # report, never guess
        return {"error": repr(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--short-list", type=int, default=32 * 132 * 16)
    ap.add_argument("--out", default=None)
    own = ap.parse_args()
    sys.argv = [sys.argv[0], "--steps", str(own.steps), "--warmup", str(own.warmup)]
    args = bench.parse()
    args.points_per_rank = args.points

    from pixsfm._pixsfm import _capi, _engine
    ctx = _capi.Context(0)
    g = bench.geometry(args, 0)
    n_obs = len(g["obs_pt"])
    d_patches = _engine.synth_patches_device(n_obs, args.ps, args.channels, g["uv0"], g["obs_pt"],
                                             seed=args.seed * 7919, noise=0.01, ctx=ctx)
    prob = bench.make_problem(args, g, d_patches, True)
    ic = _capi.default_interp()
    prob.refs, _ = _engine.refs_compute(prob, ic, ctx=ctx)
    x0 = [np.array(a, np.float64, copy=True) for a in (prob.cam_params, prob.qvec, prob.tvec, prob.xyz)]
    so = _capi.default_ba_options(use_inner_iterations=1, max_num_iterations=10 ** 6, linear_solver=args.linear_solver)
    h = _engine.BAHandle(prob, ic, so, ctx=ctx)
    h.iterate(max(args.warmup, 0))
    ctx.sync()

    # pass 1: stage times per LM iteration
    h.reset(*x0)
    stages, n_inner_prev = [], 0
    for it in range(args.steps):
        h.kernel_timing(enable=1, read=False)
        s = h.iterate(1)
        inner_ms, _ = h.kernel_timing(enable=-1, which=9)
        k1_ms, k1_n = h.kernel_timing(enable=-1, which=1)
        ran = s["num_inner_iteration_steps"] > n_inner_prev
        n_inner_prev = s["num_inner_iteration_steps"]
        stages.append({"inner_iterations_ms": inner_ms, "k1_jacobian_ms": k1_ms, "k1_jacobian_launches": k1_n,
                       "inner_iterations_ran": bool(ran)})
    h.kernel_timing(enable=0, read=False)

    # pass 2: the rounds of every LM iteration, same trajectory
    h.reset(*x0)
    h.debug_inner_rounds(enable_timing=1)
    per_it, n_inner_prev = [], 0
    for it in range(args.steps):
        s = h.iterate(1)
        ran = s["num_inner_iteration_steps"] > n_inner_prev
        n_inner_prev = s["num_inner_iteration_steps"]
        rounds = []
        if ran:
            counts, ms = h.debug_inner_rounds()
            split = h.debug_inner_round_split()
            rounds = [{"active_obs": int(c[0]), "active_points": int(c[1]), "ms": float(t),
                       "k0_ms": float(sp[0]), "k1_ms": float(sp[1]), "step_ms": float(sp[2])}
                      for c, t, sp in zip(counts, ms, split)]
        short = [r for r in rounds if r["active_obs"] < own.short_list]
        per_it.append(dict(stages[it], iteration=it, rounds=len(rounds),
                           rounds_ms=sum(r["ms"] for r in rounds),
                           rounds_k0_ms=sum(r["k0_ms"] for r in rounds),
                           rounds_k1_ms=sum(r["k1_ms"] for r in rounds),
                           rounds_step_ms=sum(r["step_ms"] for r in rounds),
                           short_rounds=len(short), short_rounds_ms=sum(r["ms"] for r in short),
                           round_list=rounds))
    h.debug_inner_rounds(enable_timing=0)
    h.close()
    res = {"workload": "bench.py configs[2]: %d cams / %d points / %d observations, %d-ch fp16 %dx%d patches, inner iterations on"
                       % (args.cams, args.points, n_obs, args.channels, args.ps, args.ps),
           "card": card(), "steps": args.steps, "warmup": args.warmup, "short_list_threshold": own.short_list,
           "iterations": per_it}
    line = json.dumps(res)
    print(line)
    if own.out:
        with open(own.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
