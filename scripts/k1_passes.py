#!/usr/bin/env python
"""K1 (fm_eval_kernel) on its own, at the benchmark's shape.

    python scripts/k1_passes.py [--iters 20] [--warmup 3] [--channels 128] [--dump DIR] [--out FILE]

Builds bench.py's workload (BASELINE configs[2]: 200 cameras, 50 000 points, 500 000 observations of 16x16 fp16
patches with 128 channels, feature references; --channels picks another fp16 instance) the way
scripts/inner_rounds_profile.py does, and times with CUDA events over `iters` launches after `warmup`
(pxr_ba_time_stage):
  - a full pass in Jacobian mode (stage 0) and in cost-only mode (stage 1); each includes the small cost-sum kernel
    that follows K1;
  - K1 in Jacobian mode over a list of every second observation (stage 6): a list pass of the size of the large inner
    rounds.  It is a proxy: an inner round's list holds the observations of its active points instead.
It prints one JSON object: ms per pass, the algorithmic bytes (4 736 B per observation at 128 channels: 16 taps x C x
2 B, the 4 C B fp32-equivalent reference and 128 B of metadata) over that time, their share of the H100 SXM data sheet's
3.35 TB/s, and the card name and power limit read in the same process.

--dump DIR writes DIR/k1_jacobian.npy ([n_obs, 8] records of one Jacobian pass: s, G^T r, G^T G) and DIR/k1_cost.npy
([n_obs] s of one cost-only pass), so that two builds can be compared array for array.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "pixel-perfect-sfm_b200"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

import bench  # noqa: E402  (geometry and problem set-up of the benchmark workload)
from inner_rounds_profile import card  # noqa: E402

HBM_PEAK = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--channels", type=int, default=None)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--out", default=None)
    own = ap.parse_args()
    sys.argv = [sys.argv[0]]
    args = bench.parse()
    args.points_per_rank = args.points
    if own.channels:
        args.channels = own.channels
    bytes_per_obs = 16 * args.channels * 2 + 4 * args.channels + 128

    from pixsfm._pixsfm import _capi, _engine
    ctx = _capi.Context(0)
    g = bench.geometry(args, 0)
    n_obs = len(g["obs_pt"])
    d_patches = _engine.synth_patches_device(n_obs, args.ps, args.channels, g["uv0"], g["obs_pt"],
                                             seed=args.seed * 7919, noise=0.01, ctx=ctx)
    prob = bench.make_problem(args, g, d_patches, True)
    ic = _capi.default_interp()
    prob.refs, _ = _engine.refs_compute(prob, ic, ctx=ctx)
    so = _capi.default_ba_options(use_inner_iterations=0, linear_solver=args.linear_solver)
    h = _engine.BAHandle(prob, ic, so, ctx=ctx)

    passes = {}
    for name, stage, n in (("jacobian_full", 0, n_obs), ("cost_full", 1, n_obs), ("jacobian_list_half", 6, n_obs // 2)):
        h.time_stage(stage, max(own.warmup, 1))
        ms = h.time_stage(stage, own.iters)
        gbs = bytes_per_obs * n / (ms * 1e-3) / 1e9
        passes[name] = {"items": n, "ms": ms, "algorithmic_GB_per_s": gbs, "share_of_3_35_TB_per_s": gbs * 1e9 / HBM_PEAK}
    if own.dump:
        os.makedirs(own.dump, exist_ok=True)
        np.save(os.path.join(own.dump, "k1_jacobian.npy"), h.debug_eval_records(1))
        np.save(os.path.join(own.dump, "k1_cost.npy"), h.debug_eval_records(0)[:, 0].copy())
    h.close()
    res = {"workload": "bench.py configs[2]: %d cams / %d points / %d observations, %d-ch fp16 %dx%d patches, refs"
                       % (args.cams, args.points, n_obs, args.channels, args.ps, args.ps),
           "card": card(), "iters": own.iters, "warmup": own.warmup, "passes": passes}
    line = json.dumps(res)
    print(line)
    if own.out:
        with open(own.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
