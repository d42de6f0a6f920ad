"""The damped Schur system, its right-hand side, the LM step and the model cost change of feature-metric bundle
adjustment (BAHandle.debug_linearize) against the block-sparse long-double reference (ba_schur_reference), entry by
entry against its derived error scales:
  * small scenes: every camera model x intrinsic set, every loss, shared cameras, partial tvec masks, constant poses and
    points, single-observation tracks, duplicate observations and images of more than 8 camera columns; every dispatch
    row of dispatch_scenes.DENSE_ENVS; block assembly and deterministic assembly (step and model cost change only);
  * a 1 000-image scene, the largest that still takes the exact (Cholesky) solve, with nc just under 8 000;
  * bench.py's configs[2] at full size (200 images, 50 000 points, 500 000 observations), from the per-observation
    factors of BAHandle.evaluate_jacobians after pinning a fresh random sample of 200 whole points to the oracle's Jets.
The large cases print their wall times and the process's peak host memory."""
import resource
import sys
import time

import numpy as np
import pytest

import ba_schur_reference as R
import dispatch_scenes as D
import query_reference as Q
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

_cache = {}
_ENV_KEYS = ("PXR_SCHUR_KERNEL", "PXR_SCHUR_CTAS", "PXR_BUILD_ATOMIC", "PXR_BUILD_UNSTAGED", "PXR_PROJECT_UNSTAGED",
             "PXR_PCG_SPARSE", "PXR_BLOCK_ASSEMBLY", "PXR_NO_SPECULATION")


def _peak_gb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20       # ru_maxrss is in KiB on Linux


def _set_env(monkeypatch, env):
    for k in _ENV_KEYS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _reference(key, prob, ic, so):
    """the reference at the largest radius of 1e4, 1e3, 1e2, 10 whose damped S is conditioned well enough for the
    step's bound (ba_schur_reference.linearize_at_largest_radius); the GPU runs at the same radius"""
    if key not in _cache:
        _cache[key] = R.linearize_at_largest_radius(prob, R.oracle_blocks(prob, ic, so.loss_type, so.loss_scale), so)
    return _cache[key]


def _check(prob, ic, so, ref, dense=True, label=""):
    got = _engine.BAHandle(prob, ic, so).debug_linearize(ref["nc"], ref["nl"], radius=ref["radius"], dense=dense)
    errs = R.all_errors(got, ref, dense=dense)
    if not dense:
        errs = {k: errs[k] for k in ("delta", "model_cost_change")}
    print("%s (radius %g) worst error / scale: %s" % (label, ref["radius"],
                                                       " ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    assert max(errs.values()) <= 1.0, errs
    return errs


# ---- small scenes ----------------------------------------------------------------------------------------------------
FREE = {"pose": "", "focal": "f", "pp": "p", "extra": "e", "all": "fpe"}


def _model_scene(model, iset):
    prob = D._base(seed=50 + model)
    n = len(prob.img_cam)
    return D.with_refs(D._with_cameras(prob, [model] * n, np.arange(n), [FREE[iset]] * n))


@pytest.mark.parametrize("iset", Q.INTRINSIC_SETS)
@pytest.mark.parametrize("model", list(Q.MODEL_NAMES))
def test_every_camera_model_and_intrinsic_set(model, iset, monkeypatch):
    _set_env(monkeypatch, {})
    ic, so = _capi.default_interp(), R.default_options()
    prob = _model_scene(model, iset)
    _check(prob, ic, so, _reference(("model", model, iset), prob, ic, so), label="%s/%s" % (Q.MODEL_NAMES[model], iset))


@pytest.mark.parametrize("loss", list(Q.LOSSES))
def test_every_loss(loss, monkeypatch):
    _set_env(monkeypatch, {})
    lt, ls = Q.LOSSES[loss]
    ic, so = _capi.default_interp(), R.default_options(loss_type=lt, loss_scale=ls)
    prob = D.with_refs(D._base(n_cams=6, n_points=50, seed=60))
    _check(prob, ic, so, _reference(("loss", loss), prob, ic, so), label=loss)


def _single_observation_tracks(seed=61):
    """every third point keeps only its first observation: its V_p is rank 2 plus the damping, so the error scale of
    its inverse grows as radius^2 and _reference picks a small radius for it"""
    prob = D._base(n_cams=6, n_points=60, seed=seed)
    keep = np.ones(len(prob.obs_pt), bool)
    for p in range(0, len(prob.xyz), 3):
        keep[np.flatnonzero(prob.obs_pt == p)[1:]] = False
    return D._rebuild(prob, obs_img=prob.obs_img[keep], obs_pt=prob.obs_pt[keep],
                      patches=np.ascontiguousarray(prob.patches[keep]), corner=prob.corner[keep],
                      scale=prob.scale[keep])


def _constant_blocks(seed=62):
    prob = D._base(n_cams=7, n_points=50, seed=seed)
    prob = D._with_cameras(prob, [2] * 7, np.arange(7), ["fe"] * 7)
    prob.point_const[::7] = 1
    prob.pose_const[3] = 1
    prob.tvec_const_mask[4] = 0b101
    prob.tvec_const_mask[5] = 0b010
    prob.cam_const_mask[2] = 0xFFFFFFFF
    return prob


STRUCTURES = {
    "shared_camera": lambda: synthetic.make_ba_scene(n_cams=6, n_points=50, channels=16, seed=63, dtype=np.float32,
                                                     shared_camera=True)[0],
    "shared_and_per_image": lambda: D._mixed("fe", seed=64),
    "constant_blocks_and_tvec_masks": _constant_blocks,
    "single_observation_tracks": _single_observation_tracks,
    "duplicate_observations": lambda: D._duplicate_observations(seed=65, every=2),
    "full_opencv_all_free": lambda: D._one_model(6, "fpe", 66),        # 18 camera columns per image
    "shared_full_opencv_all_free": lambda: D._with_cameras(D._base(n_cams=6, n_points=50, seed=67), [6, 6],
                                                           [0, 1, 0, 1, 0, 1], ["fpe", "fpe"]),
}


@pytest.mark.parametrize("name", list(STRUCTURES))
def test_problem_structures(name, monkeypatch):
    _set_env(monkeypatch, {})
    ic, so = _capi.default_interp(), R.default_options()
    if ("structure", name) not in _cache:
        _cache[("structure", name)] = D.with_refs(STRUCTURES[name](), ic)
    prob = _cache[("structure", name)]
    _check(prob, ic, so, _reference(("structure_ref", name), prob, ic, so), label=name)


def _dispatch_scene(name, ic):
    if ("dispatch", name) not in _cache:
        _cache[("dispatch", name)] = D.with_refs(D.SCENES[name](), ic)
    return _cache[("dispatch", name)]


@pytest.mark.parametrize("env", D.DENSE_ENVS, ids=D.env_id)
@pytest.mark.parametrize("name", list(D.SCENES))
def test_every_dense_dispatch_row(name, env, monkeypatch):
    ic, so = _capi.default_interp(), R.default_options()
    prob = _dispatch_scene(name, ic)
    ref = _reference(("dispatch_ref", name), prob, ic, so)
    _set_env(monkeypatch, env)
    _check(prob, ic, so, ref, label="%s/%s" % (name, D.env_id(env)))


@pytest.mark.parametrize("mode", ["block_assembly", "deterministic"])
@pytest.mark.parametrize("name", D.SPARSE_SCENES)
def test_block_and_deterministic_assembly_step(name, mode, monkeypatch):
    """these paths never form the dense S: their step and model cost change are checked"""
    ic = _capi.default_interp()
    prob = _dispatch_scene(name, ic)
    ref = _reference(("dispatch_ref", name), prob, ic, R.default_options())
    _set_env(monkeypatch, {"PXR_BLOCK_ASSEMBLY": "1"} if mode == "block_assembly" else {})
    so = R.default_options(deterministic=1 if mode == "deterministic" else 0)
    _check(prob, ic, so, ref, dense=False, label="%s/%s" % (name, mode))


# ---- the largest exact-solve scene -----------------------------------------------------------------------------------
def test_thousand_image_scene(monkeypatch):
    """1 000 images (AUTO stays on the Cholesky path up to 1 000), per-image SIMPLE_RADIAL cameras with focal and k
    free: nc = 1000 x 8 - 7 (the gauge) = 7 993, under the 8 192-column ceiling of the exact solve; 6 000 points in
    tracks of 6, 36 observations per image on average; C = 16 fp16 on 8 x 8 patches"""
    _set_env(monkeypatch, {})
    t0 = time.perf_counter()
    prob, _ = synthetic.make_ba_scene(n_cams=1000, n_points=6000, track_len=6, channels=16, ps=8, seed=71,
                                      dtype=np.float16)
    ic, so = _capi.default_interp(), R.default_options()
    per_image = np.bincount(prob.obs_img, minlength=1000)
    assert per_image.min() >= 12, per_image.min()
    t1 = time.perf_counter()
    ref = R.linearize_at_largest_radius(prob, R.oracle_blocks(prob, ic, so.loss_type, so.loss_scale), so)
    t2 = time.perf_counter()
    assert 7900 < ref["nc"] < 8192
    _check(prob, ic, so, ref, label="1000 images")
    t3 = time.perf_counter()
    print("1000 images: scene %.1f s, reference %.1f s, GPU + comparison %.1f s, peak host memory %.1f GB"
          % (t1 - t0, t2 - t1, t3 - t2, _peak_gb()))


# ---- bench.py configs[2] at full size --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    """built exactly as test_gpu_full_size builds it: bench.parse, bench.geometry, synth_patches_device, make_problem;
    the 32.8 GB device slab is freed on teardown"""
    import bench
    argv, sys.argv = sys.argv, ["bench.py"]
    try:
        args = bench.parse()
    finally:
        sys.argv = argv
    assert (args.cams, args.points, args.channels, args.ps) == (200, 50000, 128, 16)
    ctx = _capi.default_context()
    g = bench.geometry(args, 0)
    n_obs = len(g["obs_pt"])
    d_patches = _engine.synth_patches_device(n_obs, args.ps, args.channels, g["uv0"], g["obs_pt"],
                                             seed=args.seed * 7919, noise=0.01, ctx=ctx)
    h = None
    try:
        prob = bench.make_problem(args, g, d_patches, True)
        ic = _capi.default_interp()
        refs, _ = _engine.refs_compute(prob, ic, ctx=ctx)
        prob.refs = refs
        so = R.default_options()
        h = _engine.BAHandle(prob, ic, so, ctx=ctx)
        yield dict(args=args, g=g, prob=prob, d_patches=d_patches, ic=ic, so=so, refs=refs, handle=h, ctx=ctx)
    finally:
        if h is not None:
            h.close()
        _engine.device_free(d_patches, ctx)


def test_full_size_schur_system_step_and_cost_change(full):
    """SIMPLE_RADIAL per image with focal and k free (nc = 1 593), every point variable.  The reference takes its
    per-observation factors from evaluate_jacobians, so a fresh random sample of 200 whole points (2 000 observations)
    pins those factors to the oracle's Jets first: the blocks w J^T J and w J^T r must agree within KAPPA of their sums
    of absolute terms.  After that the reference checks what the GPU does downstream of the factors: build, Schur pair
    walk, damping, Cholesky and back-substitution, for S, rhs, the step of every camera column and all 50 000 points,
    and the model cost change."""
    args, g, prob, h, ic, so = full["args"], full["g"], full["prob"], full["handle"], full["ic"], full["so"]
    t0 = time.perf_counter()
    jac = h.evaluate_jacobians()
    L = min(args.track, args.cams)
    seed = int(np.random.SeedSequence().entropy % 2 ** 32)
    pts = np.sort(np.random.default_rng(seed).choice(args.points, 200, replace=False))
    obs = (pts[:, None] * L + np.arange(L)[None, :]).reshape(-1)
    pbytes = args.ps * args.ps * args.channels * 2
    host = np.empty((len(obs), args.ps, args.ps, args.channels), np.float16)
    for k, o in enumerate(obs):          # pull exactly the sampled patches out of the device slab
        _engine.memcpy_d2h(host[k], full["d_patches"] + int(o) * pbytes, pbytes, full["ctx"])
    small = _capi.BAProblem(cam_model=prob.cam_model, cam_params=prob.cam_params, cam_const_mask=prob.cam_const_mask,
                            qvec=prob.qvec, tvec=prob.tvec, img_cam=prob.img_cam, pose_const=prob.pose_const,
                            tvec_const_mask=prob.tvec_const_mask, xyz=g["xyz"][pts],
                            point_const=np.zeros(len(pts), np.uint8), obs_img=g["obs_img"][obs],
                            obs_pt=np.repeat(np.arange(len(pts), dtype=np.int64), L), patches=host,
                            corner=g["corners"][obs], scale=g["scale"][obs],
                            refs=np.ascontiguousarray(full["refs"][pts]))
    lay_s, lay_f = R.layout(small), R.layout(prob)
    assert lay_s["DC"] == lay_f["DC"]
    Mo, Mao, vo, vao, _ = R.oracle_blocks(small, ic, so.loss_type, so.loss_scale)(lay_s, np.arange(len(obs)))
    Mf, _, vf, _, _ = R.factored_blocks(prob, jac, so.loss_type, so.loss_scale)(lay_f, obs)
    pin = dict(M=R._ratio(Mf - Mo, R.KAPPA * np.asarray(Mao, np.float64)),
               v=R._ratio(vf - vo, R.KAPPA * np.asarray(vao, np.float64)))
    print("full size: sample seed %d, factor pin worst error / scale: M %.2e v %.2e" % (seed, pin["M"], pin["v"]))
    assert max(pin.values()) <= 1.0, (seed, pin)
    t1 = time.perf_counter()
    ref = R.linearize_at_largest_radius(prob, R.factored_blocks(prob, jac, so.loss_type, so.loss_scale), so)
    del jac
    t2 = time.perf_counter()
    assert ref["nc"] == 200 * 8 - 7
    got = h.debug_linearize(ref["nc"], ref["nl"], radius=ref["radius"])
    errs = R.all_errors(got, ref)
    t3 = time.perf_counter()
    print("full size (radius %g) worst error / scale: %s" % (ref["radius"],
                                                           " ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    print("full size: factors + pin %.1f s, reference %.1f s, GPU + comparison %.1f s, peak host memory %.1f GB"
          % (t1 - t0, t2 - t1, t3 - t2, _peak_gb()))
    assert max(errs.values()) <= 1.0, errs
