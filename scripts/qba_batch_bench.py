"""Batched query bundle adjustment throughput: many localization queries per launch (pxr_qba_run) against the
single-query path (pxr_ba_run per query).  Prints one JSON line.

Workload (defaults): 1000 queries x 500 correspondences, one descriptor each (500 k residual blocks), C = 128 fp16
16 x 16 patches made on the device by pxr_synth_patches_device, SIMPLE_RADIAL cameras, poses perturbed by a few pixels.
Arms:
  batched_device  run_batch on feature maps wrapping the device slab (read in place): end to end (packing included,
                  like the single arm), and packing / pxr_qba_run timed apart
  batched_host    run_batch on the first --host-queries queries with patches in pinned host memory (waves of
                  --host-wave-gb), reporting waves and H2D bytes
  single          QueryBundleOptimizer.run per query on the first --single-queries queries (host patches); the time for
                  all queries is extrapolated from them and labelled as such
The solve kernel's algorithmic bandwidth counts 4736 B per residual-block evaluation (one K1 Jacobian record, DESIGN §3)
times the evaluations the kernel reports, over the summed kernel time (CUDA events), against 3.35 TB/s."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "pixel-perfect-sfm_b200"))

from pixsfm._pixsfm import _capi, _engine, _features, _localization as loc   # noqa: E402
from pixsfm.util import colmap_types as ct                                     # noqa: E402

BYTES_PER_EVAL = 4736
HBM_BPS = 3.35e12


class DeviceView:
    """[n, ps, ps, C] fp16 window of the device slab (CUDA array interface, no ownership)"""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f2", "data": (int(ptr), False),
                                         "version": 3, "strides": None}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:      # reported, not guessed
        return "unknown (%s)" % e, "unknown"


def scene(nq, m, ps, seed):
    rng = np.random.default_rng(seed)
    f, cx, cy = 800.0, 500.0, 500.0
    Q = []
    for q in range(nq):
        z = rng.uniform(4.0, 10.0, m)
        xy = rng.uniform(40.0, 960.0, (m, 2))
        Xc = np.stack([(xy[:, 0] - cx) / f * z, (xy[:, 1] - cy) / f * z, z], 1)
        t = rng.normal(0, 0.5, 3) + [0.0, 0.0, 7.0]      # points around the world origin: ceres' ||x|| counts them
        Xw = Xc - t                                      # identity rotation: Xc = Xw + t
        corner = np.floor(xy - 0.5 - (ps / 2 - 0.5)).astype(np.int32)
        uv0 = xy - 0.5 - corner
        Q.append(dict(xy=xy, Xw=Xw, t=t, corner=corner, uv0=uv0))
    return Q, (f, cx, cy)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--blocks", type=int, default=500)
    ap.add_argument("--channels", type=int, default=128)
    ap.add_argument("--ps", type=int, default=16)
    ap.add_argument("--host-queries", type=int, default=150)
    ap.add_argument("--host-wave-gb", type=float, default=1.0)
    ap.add_argument("--single-queries", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    name, power = gpu_info()
    ctx = _capi.default_context()
    nq, m, ps, Cn = args.queries, args.blocks, args.ps, args.channels
    Q, (f, cx, cy) = scene(nq, m, ps, args.seed)
    n = nq * m
    uv0 = np.concatenate([q["uv0"] for q in Q])
    field = np.arange(n, dtype=np.int64)
    t0 = time.time()
    dptr = _engine.synth_patches_device(n, ps, Cn, uv0, field, seed=args.seed, noise=0.01, ctx=ctx)
    per_patch = ps * ps * Cn * 2
    # reference descriptors: the patches' descriptors at the true projections (one BA problem over every query)
    cams = np.tile([f, cx, cy, 0.0], (nq, 1))
    prob = _capi.BAProblem(cam_model=np.full(nq, 2), cam_params=cams, cam_const_mask=np.zeros(nq), qvec=np.tile([1.0, 0, 0, 0], (nq, 1)),
                           tvec=np.array([q["t"] for q in Q]), img_cam=np.arange(nq), pose_const=np.zeros(nq),
                           tvec_const_mask=np.zeros(nq), xyz=np.concatenate([q["Xw"] for q in Q]), point_const=np.zeros(n),
                           obs_img=np.repeat(np.arange(nq), m), obs_pt=np.arange(n), patches=dptr,
                           corner=np.concatenate([q["corner"] for q in Q]), scale=np.ones((n, 2)), patches_on_device=True,
                           patch_shape=(n, ps, ps, Cn), patch_dtype=0)
    refs = _engine.obs_descriptors(prob, _capi.default_interp(), ctx=ctx)
    setup_s = time.time() - t0
    rng = np.random.default_rng(args.seed + 1)

    def queries(fmaps, idx):
        out = []
        for i in idx:
            q = Q[i]
            rv = rng_q[i]
            cam = ct.Camera(1, "SIMPLE_RADIAL", 1000, 1000, [f, cx, cy, 0.0])
            out.append((rv[0].copy(), rv[1].copy(), cam, list(q["Xw"]), fmaps[i], list(refs[i * m:(i + 1) * m]), None,
                        list(range(m))))
        return out

    rng_q = []
    for i in range(nq):             # a few pixels: ~2.5e-3 rad of rotation (2 px at f = 800) and 2e-2 of translation
        dq = np.concatenate([[1.0], rng.normal(0, 2.5e-3 / 2, 3)]); dq /= np.linalg.norm(dq)
        rng_q.append((dq, Q[i]["t"] + rng.normal(0, 2e-2, 3)))
    meta = {"scale": [1.0, 1.0], "is_sparse": True}
    dev_maps = [_features.FeatureMap(DeviceView(dptr + i * m * per_patch, (m, ps, ps, Cn)), list(range(m)), Q[i]["corner"], meta)
                for i in range(nq)]
    opts = {"solver": {"max_num_iterations": 100}}
    out = {"gpu": name, "power_limit": power, "queries": nq, "blocks_per_query": m, "channels": Cn, "patch": ps,
           "dtype": "f16", "patch_gb": n * per_patch / 1e9, "setup_s": setup_s}

    def run_arm(maps, idx, max_wave_bytes=0.0):
        """run_batch end to end (packing, solve, write-back: the like-for-like figure against run() per query), then the
        same queries again as pack_batch and pxr_qba_run timed apart (kernel time, waves, bytes)"""
        qbo = loc.QueryBundleOptimizer(opts, {})
        qs = queries(maps, idx)
        ctx.sync()
        t = time.time()
        qbo.run_batch(qs, max_wave_bytes)
        e2e = time.time() - t
        qs = queries(maps, idx)
        t = time.time()
        batch = qbo.pack_batch(qs, max_wave_bytes)
        pack = time.time() - t
        so = qbo.solver_options()
        ctx.sync()
        t = time.time()
        res, tot = _engine.qba_run(batch, _capi.default_interp(), so, ctx=ctx)
        solve = time.time() - t
        evals = sum(r["block_evaluations"] for r in res)
        n = len(qs)
        arm = {"queries": n, "queries_per_s_end_to_end": n / e2e, "end_to_end_s": e2e, "pack_s": pack,
               "pack_us_per_block": 1e6 * pack / max(1, int(batch.obs_begin[-1])), "solve_call_s": solve,
               "queries_per_s_solve_call": n / solve, "kernel_s": tot["solve_time_s"], "waves": tot["n_waves"],
               "h2d_gb": tot["h2d_bytes"] / 1e9, "kernel_ms_per_wave": 1e3 * tot["solve_time_s"] / max(1, tot["n_waves"]),
               "block_evaluations": evals,
               "algorithmic_tb_per_s": evals * BYTES_PER_EVAL / tot["solve_time_s"] / 1e12,
               "share_of_3_35_tb_per_s": evals * BYTES_PER_EVAL / tot["solve_time_s"] / HBM_BPS,
               "iterations_mean": float(np.mean([r["num_iterations"] for r in res])),
               "cost_decreased": int(sum(r["final_cost"] < r["initial_cost"] for r in res))}
        return batch, arm

    run_arm(dev_maps, range(min(8, nq)))            # warm-up (module load, first launch)
    batch_d, out["batched_device"] = run_arm(dev_maps, range(nq))
    # host arm: pinned host copies of the first host-queries blocks
    nh = min(args.host_queries, nq)
    pins, host_maps = [], []
    for i in range(nh):
        p = _engine.PinnedArray((m, ps, ps, Cn), np.float16, ctx=ctx)
        _engine.memcpy_d2h(p.array, dptr + i * m * per_patch, m * per_patch, ctx=ctx)
        pins.append(p)
        host_maps.append(_features.FeatureMap(p.array, list(range(m)), Q[i]["corner"], meta))
    _, out["batched_host"] = run_arm(host_maps, range(nh), max_wave_bytes=args.host_wave_gb * 1e9)
    # single-query path on the first queries (host patches, as QueryBundleOptimizer.run takes them)
    ns = min(args.single_queries, nh)
    qs = queries(host_maps, range(ns))
    qbo = loc.QueryBundleOptimizer(opts, {})
    t = time.time()
    for q in qs:
        qbo.run(*q[:6], q[6], q[7])
    wall_s = time.time() - t
    dq = max(float(np.abs(np.asarray(qs[i][0]) - batch_d.qvec[i]).max()) for i in range(ns))
    dt = max(float(np.abs(np.asarray(qs[i][1]) - batch_d.tvec[i]).max()) for i in range(ns))
    out["single"] = {"queries": ns, "queries_per_s": ns / wall_s, "wall_s": wall_s,
                     "extrapolated_wall_s_all_queries": wall_s / ns * nq,
                     "extrapolated": True}
    out["max_abs_diff_vs_single"] = {"qvec": dq, "tvec": dt}
    out["speedup_end_to_end_batched_device_vs_single"] = (out["batched_device"]["queries_per_s_end_to_end"] /
                                                          out["single"]["queries_per_s"])
    for p in pins:
        p.close()
    _engine.device_free(dptr, ctx=ctx)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
