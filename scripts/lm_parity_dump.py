"""Dumps what the LM loops compute, to compare two builds bit for bit: `python scripts/lm_parity_dump.py OUT` writes .npy
files under OUT, and `python scripts/lm_parity_dump.py --compare A B` compares two such directories.

- ba_det_*: deterministic BA solves (block-mode driver): iteration records and parameters, inner iterations on and off,
  non-monotonic steps on and off, and ITERATIVE_SCHUR.  Compared with np.array_equal.
- ba_default_*: the default single-GPU driver.  It sums with fp64 atomics, so it is not bit-reproducible from run to
  run: compared are the accept/reject sequence (exactly) and the parameters (reported as a max difference).
- qba_*: one pxr_qba_run batch (focal length refined, non-monotonic steps): parameters, results and iteration records.
- ka_*: one keypoint-adjustment solve: keypoints and the summary costs."""
import argparse
import glob
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "pixel-perfect-sfm_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

REC_FIELDS = ("iteration", "cost", "cost_change", "gradient_max_norm", "step_norm", "relative_decrease",
              "trust_region_radius", "step_is_valid", "step_is_successful", "linear_solver_iterations")


def _records(its):
    return np.array([[float(i[k]) for k in REC_FIELDS] for i in its], np.float64).reshape(-1, len(REC_FIELDS))


def dump(out):
    import oracle_lib as O
    from ka_util import make_ka_problem
    from pixsfm._pixsfm import _capi, _engine
    from pixsfm.util import synthetic

    os.makedirs(out, exist_ok=True)
    save = lambda name, a: np.save(os.path.join(out, name + ".npy"), np.asarray(a))   # noqa: E731

    prob, _ = synthetic.make_ba_scene(n_cams=12, n_points=400, track_len=6, channels=32, seed=31, rot_sigma_deg=0.3,
                                      pt_sigma=0.03)
    ic = _capi.default_interp()
    prob.refs, _ = O.refs_compute(prob, ic)
    for inner in (0, 1):
        for nm in (0, 1):
            for solver in (0, 3):
                kw = dict(max_num_iterations=25, use_inner_iterations=inner, linear_solver=solver,
                          use_nonmonotonic_steps=nm, max_consecutive_nonmonotonic_steps=2)
                tag = "i%d_nm%d_s%d" % (inner, nm, solver)
                p = prob.copy()
                s = _engine.ba_run(p, ic, _capi.default_ba_options(deterministic=1, **kw))
                save("ba_det_%s_records" % tag, _records(s["iterations"]))
                save("ba_det_%s_params" % tag, np.concatenate([p.qvec.ravel(), p.tvec.ravel(), p.xyz.ravel(), p.cam_params.ravel()]))
                save("ba_det_%s_summary" % tag, [s["initial_cost"], s["final_cost"], s["termination_type"],
                                                  s["num_successful_steps"], s["num_unsuccessful_steps"],
                                                  s["num_inner_iteration_steps"]])
                if solver == 0:
                    p = prob.copy()
                    s = _engine.ba_run(p, ic, _capi.default_ba_options(**kw))
                    save("ba_default_%s_accept" % tag, [int(i["step_is_successful"]) for i in s["iterations"]])
                    save("ba_default_%s_params" % tag, np.concatenate([p.qvec.ravel(), p.tvec.ravel(), p.xyz.ravel(),
                                                                       p.cam_params.ravel()]))

    from test_gpu_qba_batch import CASES, _copy, _queries, loc
    cs = [_copy(q) for q in _queries()]
    qbo = loc.QueryBundleOptimizer(CASES["nonmonotonic"], {})
    batch = qbo.pack_batch(cs, 0.0)
    res, _ = _engine.qba_run(batch, _capi.default_interp(), qbo.solver_options(), capacity=40)
    save("qba_params", np.concatenate([batch.qvec.ravel(), batch.tvec.ravel(), batch.cam_params.ravel()]))
    save("qba_results", [[r[k] for k in ("status", "initial_cost", "final_cost", "num_iterations", "num_successful_steps",
                                         "num_unsuccessful_steps", "termination_type", "block_evaluations")] for r in res])
    save("qba_records", np.concatenate([_records(r["iterations"]) for r in res]))

    for nm in (0, 1):
        kp, _, _ = make_ka_problem(n_images=6, n_tracks=40, track_len=4, channels=128, seed=2, kp_sigma=2.5, bound=1.0,
                                   max_per_problem=20)
        so = _capi.default_ka_options()
        so.use_nonmonotonic_steps = nm
        s = _engine.ka_run(kp, ic, so)
        save("ka_nm%d_keypoints" % nm, kp.keypoints)
        save("ka_nm%d_summary" % nm, [s["initial_cost"], s["final_cost"], s["num_successful_steps"], s["num_unsuccessful_steps"]])
    print("wrote", len(glob.glob(os.path.join(out, "*.npy"))), "arrays to", out)


def compare(a, b):
    bad = 0
    names = sorted(os.path.basename(f) for f in glob.glob(os.path.join(a, "*.npy")))
    assert names == sorted(os.path.basename(f) for f in glob.glob(os.path.join(b, "*.npy"))), "different file sets"
    for n in names:
        x, y = np.load(os.path.join(a, n)), np.load(os.path.join(b, n))
        if n.startswith("ba_default_") and n.endswith("_params.npy"):
            print("%-34s max |diff| %.3e" % (n, np.abs(x - y).max() if x.shape == y.shape else np.inf))
            continue
        ok = x.shape == y.shape and np.array_equal(x, y, equal_nan=True)
        bad += not ok
        print("%-34s %s" % (n, "identical" if ok else "DIFFERS"))
    print("%d of %d arrays differ" % (bad, len(names)))
    return bad


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("out", nargs="?")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(1 if compare(*args.compare) else 0)
    dump(args.out)
