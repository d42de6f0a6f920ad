"""Batched query refinement against the long-double reference (query_reference.py) and the oracle at real query
sizes: pxr_qba_debug_linearize and pxr_qba_run (csrc/pxr_qba.cu) on queries of 1 .. 2 500 residual blocks (so each
warp of qba_evaluate runs several batches of 32, partial last batches and uneven warps), every camera model and
intrinsic set up to the 18-column FULL_OPENCV system, every loss, a dense query map, clamped tap windows and a fisheye
query on the optical axis; the BA camera block of every model against the same reference; and batched query
keypoint adjustment at 1 000+ keypoints against the oracle."""
import copy

import numpy as np
import pytest

import oracle_lib as O
import query_reference as R
from pixsfm._pixsfm import _capi, _engine, _features, _localization as loc
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

KAPPA = R.KAPPA
MAX_IT = 30
# Above this condition number of the scaled, damped first system the solve is compared by its decisions (iteration
# count, step outcomes, termination) and its final cost to 1e-4 only: with k3..k6 of FULL_OPENCV (or the fisheye
# terms on the optical axis, or a dense map's flat directions) free, the minimum is a long valley, and 30 steps along
# it carry the last-bit differences of two double-precision solvers up by the condition number (measured on an H100:
# 2e-6 .. 2e-5 relative in the final cost, up to 4e-4 in the least observable parameters, every decision equal).
WELL_POSED = 1e8

# name -> make_query arguments (and the loss).  Block counts around the warp batch (32) and the CTA stride (256)
SCENES = {
    "b1_simple_pinhole_pose": dict(blocks=1, model=0, iset="pose"),
    "b2_pinhole_focal": dict(blocks=2, model=1, iset="focal"),
    "b31_simple_radial_pp": dict(blocks=31, model=2, iset="pp"),
    "b32_radial_extra": dict(blocks=32, model=3, iset="extra"),
    "b33_opencv_all": dict(blocks=33, model=4, iset="all"),
    "b255_fisheye_all": dict(blocks=255, model=5, iset="all"),
    "b256_full_opencv_extra": dict(blocks=256, model=6, iset="extra"),
    "b257_full_opencv_all": dict(blocks=257, model=6, iset="all"),
    "b513_opencv_focal": dict(blocks=513, model=4, iset="focal"),
    "b1126_full_opencv_all_multiref": dict(blocks=1126, model=6, iset="all", refs_per_point=3),
    "b2500_full_opencv_all": dict(blocks=2500, model=6, iset="all"),
    "b300_full_opencv_all_trivial": dict(blocks=300, model=6, iset="all", loss="trivial"),
    "b300_full_opencv_all_huber": dict(blocks=300, model=6, iset="all", loss="huber"),
    "b300_full_opencv_all_soft_l1": dict(blocks=300, model=6, iset="all", loss="soft_l1"),
    "b300_full_opencv_all_arctan": dict(blocks=300, model=6, iset="all", loss="arctan"),
    "dense_map_full_opencv_all": dict(blocks=400, model=6, iset="all", kind="dense"),
    "border_8x8_simple_radial_focal": dict(blocks=64, model=2, iset="focal", kind="border"),
    "axis_fisheye_all": dict(blocks=40, model=5, iset="all", kind="axis"),
}


def _query(name, seed=11):
    kw = dict(SCENES[name])
    loss = kw.pop("loss", "cauchy")
    q, m = R.make_query(seed=seed, **kw)
    return q, m, loss


def _options(loss):
    return {"refine_focal_length": True, "loss": {"name": loss, "params": [R.LOSSES[loss][1]]},
            "solver": {"max_num_iterations": MAX_IT}}


def _check_linearisation(batch, k, lin, ic, so):
    """query k of a qba_debug_linearize output against the reference and the oracle's records -> the reference"""
    prob = R.query_problem(batch, k)
    ref = R.normal_equations(prob, ic, so.loss_type, so.loss_scale)
    n = R.n_columns(batch, k)
    assert ref["nc"] == n
    L = lin["H"][k, :n, :n]
    H = np.tril(L) + np.tril(L, -1).T
    assert np.all(lin["H"][k][n:] == 0) and np.all(lin["H"][k][:, n:] == 0) and np.all(lin["g"][k][n:] == 0)
    eh, eg = R.scaled_error(H, ref), R.scaled_error(lin["g"][k, :n], ref, "g")
    assert eh <= KAPPA and eg <= KAPPA, (eh, eg)
    cost = float(ref["cost"])
    assert abs(lin["cost"][k] - cost) <= 1e-12 * cost
    b0, b1 = int(batch.obs_begin[k]), int(batch.obs_begin[k + 1])
    ev = O.ba_evaluate(prob, ic, so)
    rec = lin["rec"][b0:b1]
    for key, got, tol in (("xy", lin["xy"][b0:b1], 1e-9), ("sq_norm", rec[:, 0], 1e-12), ("gtr", rec[:, 1:3], 1e-11),
                          ("gtg", rec[:, 3:6], 1e-10)):
        assert np.abs(got - ev[key]).max() <= tol * max(1.0, np.abs(ev[key]).max()), key
    return ref, H


@pytest.mark.parametrize("name", sorted(SCENES))
def test_linearisation_matches_the_long_double_reference(name):
    q, m, loss = _query(name)
    batch, o = R.pack([(q, m)], _options(loss))
    so, ic = o.solver_options(), _capi.default_interp()
    lin = _engine.qba_debug_linearize(batch, ic, so)
    _check_linearisation(batch, 0, lin, ic, so)


@pytest.mark.parametrize("iset", R.INTRINSIC_SETS)
@pytest.mark.parametrize("model", sorted(R.MODEL_PARAMS))
def test_every_model_and_intrinsic_set(model, iset):
    """one batch per model and intrinsic set; its queries end mid-batch, on a warp stride and past it"""
    qs = [R.make_query(b, model=model, iset=iset, channels=128, seed=21) for b in (97, 256, 300)]
    batch, o = R.pack(qs, _options("cauchy"))
    so, ic = o.solver_options(), _capi.default_interp()
    lin = _engine.qba_debug_linearize(batch, ic, so)
    for k in range(len(qs)):
        _check_linearisation(batch, k, lin, ic, so)


INSTANCES = [("float16", c) for c in (8, 16, 32, 64, 128, 256)] + [("float32", c) for c in (16, 64, 128)] + \
            [("float64", c) for c in (16, 128)]


@pytest.mark.parametrize("fs,l2", [(0, 1), (1, 1), (0, 0)])
@pytest.mark.parametrize("dtype,channels", INSTANCES)
def test_every_kernel_instance(dtype, channels, fs, l2):
    """a 300-block FULL_OPENCV query with every intrinsic free through each (dtype, C) instance launch_qba builds"""
    q, m = R.make_query(300, model=6, iset="all", channels=channels, dtype=np.dtype(dtype), seed=31)
    interp = {"use_float_simd": bool(fs), "l2_normalize": bool(l2)}
    batch, o = R.pack([(q, m)], _options("cauchy"), interp)
    so, ic = o.solver_options(), _capi.default_interp(bool(l2), bool(fs))
    lin = _engine.qba_debug_linearize(batch, ic, so)
    _check_linearisation(batch, 0, lin, ic, so)


def _solve_case(name):
    q, m, loss = _query(name)
    batch, o = R.pack([(q, m)], _options(loss))
    return batch, o.solver_options(), _capi.default_interp()


@pytest.mark.parametrize("name", sorted(SCENES))
def test_solve_matches_the_oracle(name):
    batch, so, ic = _solve_case(name)
    lin = _engine.qba_debug_linearize(batch, ic, so)
    ref, H = _check_linearisation(batch, 0, lin, ic, so)
    prob = R.query_problem(batch, 0)
    n = R.n_columns(batch, 0)
    step = R.first_step(ref, n, batch.qvec[0], batch.tvec[0], batch.cam_params[0], int(batch.cam_model[0]),
                        int(batch.cam_const_mask[0]), so)
    res, _ = _engine.qba_run(batch, ic, so, capacity=MAX_IT + 1)
    s = O.ba_solve(prob, ic, so)
    r = res[0]
    assert r["status"] == _capi.PXR_OK
    assert (r["num_iterations"], r["num_successful_steps"], r["num_unsuccessful_steps"], r["termination_type"]) == \
        (s["num_iterations"], s["num_successful_steps"], s["num_unsuccessful_steps"], s["termination_type"])
    assert abs(r["initial_cost"] - float(ref["cost"])) <= 1e-12 * float(ref["cost"])
    if step["cond"] < WELL_POSED:
        assert abs(r["final_cost"] - s["final_cost"]) <= 1e-6 * s["final_cost"]
        assert np.abs(batch.qvec[0] - prob.qvec[0]).max() < 1e-6 and np.abs(batch.tvec[0] - prob.tvec[0]).max() < 1e-6
        assert np.all(np.abs(batch.cam_params[0] - prob.cam_params[0]) <= 1e-6 * np.maximum(1.0, np.abs(prob.cam_params[0])))
    else:
        assert abs(r["final_cost"] - s["final_cost"]) <= 1e-4 * s["final_cost"]
    # iteration 1's step against the long-double step: the perturbation bound of the scaled damped system, with
    # the kernel's measured scaled errors in H and g and its own double-precision solve
    it1 = r["iterations"][1]
    if step["step_norm"] is None:
        assert it1["step_is_valid"] == 0
        return
    S = 1.0 / np.sqrt(np.asarray(np.diag(ref["H"]), np.float64))
    Hs_ref = np.asarray(ref["H"], np.float64) * np.outer(S, S)
    eM = np.abs((H - np.asarray(ref["H"], np.float64)) * np.outer(S, S)).max() / np.abs(Hs_ref).max()
    gs = np.asarray(ref["g"], np.float64) * S
    eb = np.abs((lin["g"][0, :n] - np.asarray(ref["g"], np.float64)) * S).max() / np.abs(gs).max()
    tol = 4.0 * step["cond"] * (eM + eb + 1e-15) + 1e-13
    assert abs(it1["step_norm"] - step["step_norm"]) <= tol * step["step_norm"], (it1["step_norm"], step, tol)


def test_every_scene_gives_the_same_bits_in_one_batch():
    """all the scenes of one patch shape in one batch (one loss) against each alone"""
    ic = _capi.default_interp()

    def run(sub):
        batch, o = R.pack([(_copy(q), m) for q, m in sub], _options("cauchy"))
        res, tot = _engine.qba_run(batch, ic, o.solver_options())
        return batch, res, tot

    groups = {}
    for name in sorted(SCENES):
        q, m, _ = _query(name)
        groups.setdefault(q[4].patches.shape[1:], []).append((q, m))
    assert max(len(g) for g in groups.values()) == len(SCENES) - 2      # all but the dense map and the 8x8 patches
    for qs in groups.values():
        full, fres, tot = run(qs)
        assert tot["n_waves"] == 1
        for k, qm in enumerate(qs):
            one, ores, _ = run([qm])
            for key in ("qvec", "tvec", "cam_params"):
                assert np.array_equal(getattr(full, key)[k], getattr(one, key)[0]), (k, key)
            for key in ("final_cost", "initial_cost", "num_iterations", "num_successful_steps", "termination_type"):
                assert fres[k][key] == ores[0][key], (k, key)


def _copy(q):
    return (q[0].copy(), q[1].copy(), copy.deepcopy(q[2])) + tuple(q[3:])


@pytest.mark.parametrize("model", sorted(R.MODEL_PARAMS))
def test_ba_camera_block_matches_the_long_double_reference(model):
    """BAHandle.debug_linearize on a 5-image scene with every intrinsic free: Hcc / gc and the point blocks Hpp / gp
    against the reference over all local columns"""
    prob, _ = synthetic.make_ba_scene(n_cams=5, n_points=40, track_len=4, channels=16, seed=40 + model, dtype=np.float32)
    prob.cam_model[:] = model
    prob.cam_params[:] = 0
    prob.cam_params[:, :len(R.MODEL_PARAMS[model])] = R.MODEL_PARAMS[model]
    prob.cam_const_mask[:] = 0
    ic = _capi.default_interp()
    refs, _ = O.refs_compute(prob, ic)
    prob.refs = refs * 0.95 + 0.002
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = R.normal_equations(prob, ic, so.loss_type, so.loss_scale)
    nc, nl, _, _, point_off = O.ba_layout(prob)
    h = _engine.BAHandle(prob, ic, so)
    got = h.debug_linearize(nc, nl)
    h.close()
    L = got["Hcc"]
    Hcc = np.tril(L) + np.tril(L, -1).T
    assert R.scaled_error(Hcc, ref) <= KAPPA
    assert R.scaled_error(got["gc"], ref, "g") <= KAPPA
    # the free points' 3 x 3 blocks and gradients, under the same elementwise bound
    for p, off in enumerate(point_off):
        if off >= 0:
            blk = slice(off, off + 3)
            assert np.all(np.abs(got["Hpp"][p] - np.asarray(ref["H"][blk, blk], np.float64)) <=
                          KAPPA * np.asarray(ref["A"][blk, blk], np.float64)), p
            assert np.all(np.abs(got["gp"][p] - np.asarray(ref["g"][blk], np.float64)) <=
                          KAPPA * np.asarray(ref["a"][blk], np.float64)), p
    assert abs(got["cost"] - float(ref["cost"])) <= 1e-12 * float(ref["cost"])


# ---- batched query keypoint adjustment at real sizes
def _qka_queries(kind):
    rng = np.random.default_rng(41)
    if kind == "dense":        # 1 000 keypoints on one dense 256 x 256 map at a quarter of the image's resolution
        dense = R.smooth_map(256, 256, 128, np.float16, 41)
        dmap = _features.FeatureMap(dense[None], [_features.kDenseId], np.zeros((1, 2), np.int32),
                                    {"scale": np.array([0.25, 0.25]), "is_sparse": False})
        kps = rng.uniform(40, 960, (1000, 2))
        at = (np.clip((kps[:, 1] * 0.25 + rng.normal(0, 1.0, 1000)).astype(int), 0, 255),
              np.clip((kps[:, 0] * 0.25 + rng.normal(0, 1.0, 1000)).astype(int), 0, 255))
        return [(kps, dmap, list(dense[at].astype(np.float64)), None)]
    sc = R._base_scene(1200, 128, np.float16, 16, 41)
    kps = sc["xy"] + rng.normal(0, 1.0, sc["xy"].shape)
    fmap = _features.FeatureMap(sc["patches"], list(range(1200)), sc["corners"], {"scale": sc["scale"], "is_sparse": True})
    multi = [[r, r * 0.97 + rng.normal(0, 0.01, 128), r * 1.02] for r in sc["refs"][:1100]]   # three references each
    return [(kps.copy(), fmap, list(sc["refs"]), list(range(1200))), (kps[:1100].copy(), fmap, multi, list(range(1100)))]


@pytest.mark.parametrize("kind,sizes", [("sparse", [1200, 1100]), ("dense", [1000])])
def test_qka_batch_at_real_sizes_matches_oracle(kind, sizes):
    """sparse queries of 1 200 keypoints and of 1 100 keypoints with three references each, and a dense-map query of
    1 000 keypoints, against the oracle's query-mode solve at the tolerances of test_qka_batch_matches_oracle"""
    qs = _qka_queries(kind)
    opts = {"bound": 4.0}
    o = loc.QueryKeypointOptimizer(opts, {})
    batch, used = o.pack_batch(qs)
    assert list(np.diff(batch.kp_begin)) == sizes
    cpu = batch.copy()
    c0, c1 = O.ka_solve(cpu, _capi.default_interp(), o.solver_options())
    cs = [(q[0].copy(),) + tuple(q[1:]) for q in qs]
    ob = loc.QueryKeypointOptimizer(opts, {})
    ok = ob.run_batch(cs)
    sums = ob.summaries()
    assert all(ok)
    g0, g1 = sum(s.initial_cost for s in sums), sum(s.final_cost for s in sums)
    assert abs(g0 - c0) <= 1e-9 * c0 and abs(g1 - c1) <= 1e-6 * c1 and c1 < c0
    for k, (q, u) in enumerate(zip(qs, used)):
        kb, ke = batch.kp_begin[k], batch.kp_begin[k + 1]
        assert np.abs(cs[k][0][u] - cpu.keypoints[kb:ke]).max() < 1e-5, k
        assert np.abs(cs[k][0] - q[0]).max() > 1e-2
