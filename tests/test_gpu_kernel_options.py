"""GPU parity, against the oracle, of every feature-metric kernel instance under the interpolation and loss options the
Python layer passes through (`use_float_simd`, `l2_normalize`, the solver's loss), and at the size limits of keypoint
adjustment and reference extraction:

- K1 and one inner-iteration pass, every fm_supported instance x use_float_simd x l2_normalize;
- keypoint adjustment, every (dtype, C) x {plain, float-SIMD} x l2_normalize, the other solver options on two
  instances, every query-mode instance, and the 80-variable-keypoint problem size;
- batched query BA, every float-SIMD instance, against the single-query path and the oracle's solve;
- reference extraction (IRLS) on tracks up to 256 observations, under every loss.

test_kernel_options_cpu.py checks that these rows are exactly the instances the CUDA sources build."""
import numpy as np
import pytest

import oracle_lib as O
from ka_util import make_ka_problem, make_query_ka_problem
from pixsfm._pixsfm import _capi, _engine, _features, _localization as loc
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

# (dtype, C) of every instance fm_supported (csrc/pxr_ba.cu) accepts with C >= 8; batched query BA builds the same set
FM_INSTANCES = [(np.float16, c) for c in (8, 16, 32, 64, 128, 256)] + \
               [(np.float32, c) for c in (16, 64, 128)] + [(np.float64, c) for c in (16, 128)]
# the 1/3/4-channel maps (cost maps), one thread per item
SMALL_INSTANCES = [(dt, c) for dt in (np.float16, np.float32, np.float64) for c in (1, 3, 4)]
# (dtype, C) pairs pxr_ka.cu builds
KA_INSTANCES = [(np.float16, c) for c in (8, 16, 32, 64, 128)] + [(np.float32, c) for c in (16, 128)] + \
               [(np.float64, c) for c in (16, 128)]
IRLS_CHANNELS = (8, 16, 32, 64, 128, 256)
# one warp holds 32 observations per register slot, eight slots
IRLS_LENGTHS = (1, 2, 31, 32, 33, 64, 65, 128, 129, 255, 256)
LOSSES = {0: 1.0, 1: 0.25, 2: 0.1, 3: 0.1, 4: 0.2}       # loss id -> scale


def _id(v):
    return v.__name__ if isinstance(v, type) else str(v)


# ---- K1 and the inner iterations

def _ba_scene(dtype, channels, ph, pw):
    import test_gpu_fm_instances as F
    return F._ba_scene(dtype, channels, ph, pw)


def _k1_and_inner(prob, ic):
    refs, _ = O.refs_compute(prob, ic)
    prob.refs = refs * 0.95 + 0.002
    so = _capi.default_ba_options(use_inner_iterations=0)
    ref = O.ba_evaluate(prob, ic, so, residuals=True)
    got = _engine.BAHandle(prob, ic, so).evaluate(residuals=True)
    assert np.allclose(got["xy"], ref["xy"], rtol=0, atol=1e-9)
    assert np.abs(got["residuals"] - ref["residuals"]).max() < 1e-12
    assert np.allclose(got["sq_norm"], ref["sq_norm"], rtol=1e-10, atol=1e-15)
    assert np.allclose(got["gtr"], ref["gtr"], rtol=1e-9, atol=1e-13)
    assert np.allclose(got["gtg"], ref["gtg"], rtol=1e-10, atol=1e-14)
    assert abs(got["cost"] - ref["cost"]) <= 1e-11 * abs(ref["cost"])
    prob.xyz += np.random.default_rng(5).normal(0, 0.004, prob.xyz.shape)
    so = _capi.default_ba_options(use_inner_iterations=1)
    p_ref = prob.copy()
    import ctypes as C
    O.lib().orc_ba_inner_iterations(C.byref(p_ref.desc()), C.byref(ic), C.byref(so))
    assert np.abs(p_ref.xyz - prob.xyz).max() > 1e-5
    h = _engine.BAHandle(prob.copy(), ic, so)
    h.debug_inner_iterations()
    h.read_params()
    assert np.abs(h.problem.xyz - p_ref.xyz).max() < 1e-7


@pytest.mark.parametrize("ph,pw", [(16, 16), (8, 8)], ids=str)
@pytest.mark.parametrize("l2", [1, 0])
@pytest.mark.parametrize("fs", [0, 1])
@pytest.mark.parametrize("dtype,channels", FM_INSTANCES, ids=_id)
def test_k1_and_inner_options(dtype, channels, fs, l2, ph, pw):
    prob = _ba_scene(dtype, channels, ph, pw)
    _k1_and_inner(prob, _capi.default_interp(l2_normalize=l2, use_float_simd=fs))


@pytest.mark.parametrize("dtype,channels", SMALL_INSTANCES, ids=_id)
def test_k1_and_inner_small_channels_float_simd(dtype, channels):
    """the first C channels of a 16-channel scene: smooth, unnormalised maps as the cost maps are"""
    prob = _ba_scene(np.float64, 16, 16, 16)
    prob = prob.with_patches(np.ascontiguousarray(prob.patches[..., :channels].astype(dtype)))
    _k1_and_inner(prob, _capi.default_interp(l2_normalize=0, use_float_simd=1))


# ---- keypoint adjustment

def _ka(dtype, channels, ps=16):
    import test_gpu_fm_instances as F
    return F._ka(dtype, channels, ps)


def _ka_compare(prob, ic, so, lab=None, moved_min=1e-3):
    _, c_start = O.ka_evaluate(prob, ic, so)
    p_cpu, p_gpu = prob.copy(), prob.copy()
    c0, c1 = O.ka_solve(p_cpu, ic, so)
    s = _engine.ka_run(p_gpu, ic, so)
    assert abs(s["initial_cost"] - c_start) <= 1e-9 * c_start
    assert abs(s["initial_cost"] - c0) <= 1e-9 * c0
    assert abs(s["final_cost"] - c1) <= 1e-6 * c1
    assert c1 < c0
    assert np.abs(p_gpu.keypoints - p_cpu.keypoints).max() < 1e-5
    if lab is not None:
        roots = lab["roots"].astype(bool)
        assert np.array_equal(p_gpu.keypoints[roots], prob.keypoints[roots])
        assert np.abs(p_gpu.keypoints[~roots] - prob.keypoints[~roots]).max() > moved_min
    return p_cpu, c_start


@pytest.mark.parametrize("l2", [1, 0])
@pytest.mark.parametrize("fs", [0, 1])
@pytest.mark.parametrize("dtype,channels", KA_INSTANCES, ids=_id)
def test_ka_instance_options(dtype, channels, fs, l2):
    prob, _, lab = _ka(dtype, channels)
    ic = _capi.default_interp(l2_normalize=l2, use_float_simd=fs)
    so = _capi.default_ka_options()
    _, c_start = _ka_compare(prob, ic, so, lab)
    # the two interpolations differ by more than twice the initial-cost bound (5e-9 relative and up on these scenes):
    # a kernel that interpolates the other way cannot pass it
    _, c_other = O.ka_evaluate(prob, _capi.default_interp(l2_normalize=l2, use_float_simd=1 - fs), so)
    assert abs(c_other - c_start) > 2e-9 * c_start


KA_VARIANTS = ["loss%d" % k for k in sorted(LOSSES)] + ["no_edge_weight", "no_jacobi_scaling", "unbounded_dense",
                                                         "tight_bound"]


@pytest.mark.parametrize("variant", KA_VARIANTS)
@pytest.mark.parametrize("dtype,channels,fs", [(np.float16, 128, 1), (np.float64, 16, 0)], ids=_id)
def test_ka_solver_options(dtype, channels, fs, variant):
    prob, _, lab = _ka(dtype, channels)
    ic = _capi.default_interp(use_float_simd=fs)
    so = _capi.default_ka_options()
    if variant.startswith("loss"):
        k = int(variant[4:])
        so = _capi.default_ka_options(loss_type=k, loss_scale=LOSSES[k])
    elif variant == "no_edge_weight":
        prob.edge_weight = None
    elif variant == "no_jacobi_scaling":
        so = _capi.default_ka_options(jacobi_scaling=0)
    elif variant == "unbounded_dense":
        prob.bound = -1.0
        prob.patches_are_sparse = False     # dense maps and bound <= 0: no box constraint at all
    elif variant == "tight_bound":
        prob.bound = 0.3
    p_cpu, _ = _ka_compare(prob, ic, so, lab, moved_min=1e-3 if variant != "tight_bound" else 0.1)
    if variant == "tight_bound":            # the box is active at the solution
        assert np.isclose(np.abs(p_cpu.keypoints - prob.keypoints), 0.3, rtol=0, atol=1e-9).any()


def _query_ka(dtype, channels):
    prob, _ = make_query_ka_problem(n_queries=1, n_images=6, n_tracks=44, track_len=4, channels=channels, seed=6,
                                    kp_sigma=1.0, dtype=dtype)
    assert len(prob.keypoints) == 176 > 160 and prob.n_problems == 1     # more than the dense in-smem path holds
    return prob


@pytest.mark.parametrize("dtype,channels", KA_INSTANCES, ids=_id)
def test_query_ka_instance(dtype, channels):
    prob = _query_ka(dtype, channels)
    ic = _capi.default_interp(); so = _capi.default_ka_options()
    p_cpu, p_gpu = prob.copy(), prob.copy()
    c0, c1 = O.ka_solve(p_cpu, ic, so)
    s = _engine.ka_run(p_gpu, ic, so)
    assert abs(s["initial_cost"] - c0) <= 1e-9 * c0
    assert abs(s["final_cost"] - c1) <= 1e-6 * c1
    assert c1 < 0.9 * c0
    assert np.abs(p_gpu.keypoints - p_cpu.keypoints).max() < 1e-5
    assert np.abs(p_gpu.keypoints - prob.keypoints).max() > 1e-2


@pytest.mark.parametrize("dtype,channels", KA_INSTANCES, ids=_id)
def test_query_ka_refuses_float_simd(dtype, channels):
    """float-SIMD is not built for the query mode: refused before anything runs"""
    p = _query_ka(dtype, channels)
    before = p.keypoints.copy()
    with pytest.raises((ValueError, _capi.PxrError), match="use_float_simd"):
        _engine.ka_run(p, _capi.default_interp(use_float_simd=1), _capi.default_ka_options())
    assert np.array_equal(p.keypoints, before)


def _one_track(n_images, dtype, channels):
    """one track seen in every image: a single root, every other keypoint variable and in one component"""
    return make_ka_problem(n_images=n_images, n_tracks=1, track_len=n_images, channels=channels, ps=16, seed=n_images,
                           kp_sigma=0.7, bound=4.0, max_per_problem=1000, dtype=dtype, extra_edge_prob=0.05)


@pytest.mark.parametrize("dtype,channels,fs", [(np.float64, 128, 0), (np.float16, 128, 1)], ids=_id)
def test_ka_one_track_of_80_variable_keypoints(dtype, channels, fs):
    """80 variable keypoints (the per-problem limit) in one component of 160 scalars: the widest dense system, 219 040 B
    of shared memory, and a Cholesky block five times a warp wide"""
    prob, _, lab = _one_track(81, dtype, channels)
    assert prob.n_problems == 1 and int(lab["roots"].sum()) == 1 and len(prob.keypoints) - 1 == 80
    _ka_compare(prob, _capi.default_interp(use_float_simd=fs), _capi.default_ka_options(), lab)


def test_ka_refuses_81_variable_keypoints():
    prob, _, lab = _one_track(82, np.float64, 128)
    assert prob.n_problems == 1 and len(prob.keypoints) - int(lab["roots"].sum()) == 81
    before = prob.keypoints.copy()
    with pytest.raises((ValueError, _capi.PxrError), match="80 supported"):
        _engine.ka_run(prob, _capi.default_interp(), _capi.default_ka_options())
    assert np.array_equal(prob.keypoints, before)


@pytest.mark.parametrize("dtype,channels,fs", [(np.float64, 128, 0), (np.float16, 128, 1)], ids=_id)
def test_ka_many_small_components_at_the_size_limit(dtype, channels, fs):
    """40 tracks of three in one problem: 80 variable keypoints again, as 40 components of 4 scalars"""
    prob, _, lab = make_ka_problem(n_images=3, n_tracks=40, track_len=3, channels=channels, ps=16, seed=9, kp_sigma=0.7,
                                   bound=4.0, max_per_problem=1000, dtype=dtype)
    assert prob.n_problems == 1 and len(prob.keypoints) - int(lab["roots"].sum()) == 80
    _ka_compare(prob, _capi.default_interp(use_float_simd=fs), _capi.default_ka_options(), lab)


def test_ka_degenerate_problem():
    """only constant keypoints, one edge from a keypoint to itself: nothing to solve, the cost is still the oracle's"""
    prob, _, _ = _ka(np.float64, 16)
    prob.kp_const = np.ones(len(prob.keypoints), np.uint8)
    k = int(prob.edge_src[0])
    prob.edge_src = np.concatenate([prob.edge_src, [k]]).astype(np.int64)
    prob.edge_dst = np.concatenate([prob.edge_dst, [k]]).astype(np.int64)
    prob.edge_weight = np.concatenate([prob.edge_weight, [0.7]])
    prob.edge_problem = np.concatenate([prob.edge_problem, [prob.n_problems - 1]]).astype(np.int32)
    ic = _capi.default_interp(); so = _capi.default_ka_options()
    _, c_start = O.ka_evaluate(prob, ic, so)
    p_cpu, p_gpu = prob.copy(), prob.copy()
    c0, c1 = O.ka_solve(p_cpu, ic, so)
    s = _engine.ka_run(p_gpu, ic, so)
    assert c_start > 0 and abs(s["initial_cost"] - c_start) <= 1e-9 * c_start
    assert abs(s["final_cost"] - c1) <= 1e-9 * c1 and abs(c1 - c0) <= 1e-12 * c0
    assert np.array_equal(p_gpu.keypoints, prob.keypoints) and np.array_equal(p_cpu.keypoints, prob.keypoints)


# ---- batched query BA

def _qba_queries(dtype, channels):
    import test_gpu_qba_batch as Q
    out = []
    for q in Q._queries(seeds=(17,), n_points=40, channels=channels, models=("SIMPLE_RADIAL",)):
        fm = q[4]
        f2 = _features.FeatureMap(np.ascontiguousarray(fm.patches.astype(dtype)), fm.point2D_ids, fm.corners,
                                  {"scale": fm.scale, "is_sparse": fm.is_sparse})
        out.append(q[:4] + (f2,) + q[5:])
    return out


@pytest.mark.parametrize("dtype,channels,l2", [(dt, c, 1) for dt, c in FM_INSTANCES] + [(np.float16, 128, 0)], ids=_id)
def test_qba_float_simd_instance(dtype, channels, l2):
    import test_gpu_qba_batch as Q
    qs = _qba_queries(dtype, channels)
    interp = {"use_float_simd": True, "l2_normalize": bool(l2)}
    opts = Q.CASES["focal"]
    single = Q._single(opts, interp, qs)
    ok, cs, sums = Q._batch(opts, interp, qs)
    ic = _capi.default_interp(l2_normalize=l2, use_float_simd=1)
    for (ok1, c1, s1), c2, s2, q in zip(single, cs, sums, qs):
        assert ok1 and s2.num_iterations == s1.num_iterations and abs(s2.final_cost - s1.final_cost) <= 1e-6 * s1.final_cost
        assert np.abs(c2[0] - c1[0]).max() < 1e-6 and np.abs(c2[1] - c1[1]).max() < 1e-6
        # the oracle's solve of the problem the single-query path builds
        qbo = loc.QueryBundleOptimizer(opts, interp)
        c = Q._copy(q)
        prob = qbo.build_problem(c[0], c[1], c[2], c[3], c[4], c[5], q[6], q[7])
        s_ref = O.ba_solve(prob, ic, qbo.solver_options())
        assert s2.num_iterations == s_ref["num_iterations"]
        assert abs(s2.initial_cost - s_ref["initial_cost"]) <= 1e-10 * s_ref["initial_cost"]
        assert abs(s2.final_cost - s_ref["final_cost"]) <= 1e-6 * s_ref["final_cost"]
        assert np.abs(c2[0] - prob.qvec[0]).max() < 1e-6 and np.abs(c2[1] - prob.tvec[0]).max() < 1e-6
        assert abs(c2[2].params[0] / prob.cam_params[0, 0] - 1) < 1e-6
        assert np.abs(c2[2].params[1:] - prob.cam_params[0, 1:len(c2[2].params)]).max() < 1e-6


# ---- reference extraction

def irls_scene(channels, lengths, dtype=np.float16, seed=3, noise=0.01):
    """one point per track length, every observation in another image, plus two tracks with a repeated observation
    (identical descriptors): one of just the pair, one of five.  -> (BAProblem, ids of the two repeated-pair points)"""
    lengths = list(lengths)
    n = len(lengths) + 2
    L = max(lengths + [5])
    prob, _ = synthetic.make_ba_scene(n_cams=L, n_points=n, track_len=L, channels=channels, ps=8, seed=seed, dtype=dtype,
                                      noise=noise)
    rng = np.random.default_rng(seed)
    sel = []
    for p, k in enumerate(lengths):
        idx = np.where(prob.obs_pt == p)[0]
        sel.append(np.sort(rng.choice(idx, k, replace=False)))
    a = np.where(prob.obs_pt == n - 2)[0]
    sel.append(a[[0, 0]])
    b = np.where(prob.obs_pt == n - 1)[0]
    sel.append(b[[0, 0, 1, 2, 3]])
    obs_pt = np.repeat(np.arange(n, dtype=np.int64), [len(s) for s in sel])
    sel = np.concatenate(sel)
    sub = _capi.BAProblem(cam_model=prob.cam_model, cam_params=prob.cam_params, cam_const_mask=prob.cam_const_mask,
                          qvec=prob.qvec, tvec=prob.tvec, img_cam=prob.img_cam, pose_const=prob.pose_const,
                          tvec_const_mask=prob.tvec_const_mask, xyz=prob.xyz, point_const=prob.point_const,
                          obs_img=prob.obs_img[sel], obs_pt=obs_pt, patches=np.ascontiguousarray(prob.patches[sel]),
                          corner=prob.corner[sel], scale=prob.scale[sel])
    return sub, [n - 2, n - 1]


def oracle_descriptors(prob, ic):
    """[n_obs, C]: the oracle's interpolation of every observation at its projection"""
    q = prob.copy()
    q.refs = np.zeros((len(prob.xyz), prob.channels))
    xy = O.ba_evaluate(q, ic, _capi.default_ba_options())["xy"]
    out = np.zeros((prob.n_obs, prob.channels))
    for o in range(prob.n_obs):
        uv = (xy[o] * prob.scale[o] - 0.5 - prob.corner[o]) * prob.upsampling_factor
        out[o] = O.pixel_interp(prob.patches[o], uv[1], uv[0], bool(ic.l2_normalize), bool(ic.use_float_simd))[0]
    return out


def _irls_compare(prob, dup, ic, loss_type, scale):
    r_cpu, s_cpu = O.refs_compute(prob, ic, loss_type, scale, 100)
    r_gpu, s_gpu = _engine.refs_compute(prob, ic, loss_type, scale, 100)
    tl = np.bincount(prob.obs_pt, minlength=len(prob.xyz))
    first = np.concatenate([[0], np.cumsum(tl)])[:-1]
    # a 2-observation track of two different descriptors is an exact tie (test_gpu_models_losses.py)
    pinned = (tl != 2) | np.isin(np.arange(len(tl)), dup)
    assert np.array_equal(s_gpu[pinned], s_cpu[pinned]), [(int(tl[p]), int(s_gpu[p] - first[p]), int(s_cpu[p] - first[p]))
                                                          for p in np.where(pinned & (s_gpu != s_cpu))[0]]
    assert all(first[p] <= s_gpu[p] < first[p] + 2 for p in np.where(tl == 2)[0])
    assert np.abs(r_gpu[pinned] - r_cpu[pinned]).max() <= 1e-12
    assert s_gpu[dup[0]] == first[dup[0]]               # the first of the identical pair


@pytest.mark.parametrize("l2", [1, 0])
@pytest.mark.parametrize("loss", sorted(LOSSES))
def test_irls_lengths_and_losses(loss, l2):
    prob, dup = irls_scene(16, IRLS_LENGTHS)
    _irls_compare(prob, dup, _capi.default_interp(l2_normalize=l2), loss, LOSSES[loss])


@pytest.mark.parametrize("channels", IRLS_CHANNELS)
def test_irls_every_channel_count(channels):
    # low noise: the descriptors of a track spread along the smooth field, so where the IRLS ends depends on the
    # weights of every round, not just on the first (equal-weight) mean
    prob, dup = irls_scene(channels, (33, 65, 129, 255, 256), seed=channels, noise=0.002)
    _irls_compare(prob, dup, _capi.default_interp(), 1, 0.25)
