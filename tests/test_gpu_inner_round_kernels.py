"""The kernels of a batched inner-iteration round other than K1.  K0 in a round is the point-only projection: it must
give the uv and the point columns of the full projection's Jacobian bit for bit, on every camera model and for lists
that cover part of the observations.  The step kernel appends the points that stay active, and their observations,
to the next round's lists a warp at a time, and the rounds size their grids from the lengths published two rounds
back: every round's lists, read back, must hold exactly the points that are still active and their observations, in
warp-ordered chunks, down to a single point, and the result must not depend on round timing."""
import numpy as np
import pytest

from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

MODELS = {
    0: [1200.0, 500.0, 500.0],                                              # SIMPLE_PINHOLE
    1: [1200.0, 1190.0, 500.0, 502.0],                                      # PINHOLE
    2: None,                                                                # SIMPLE_RADIAL (the scene's own)
    3: [1200.0, 500.0, 500.0, 0.02, -0.01],                                 # RADIAL
    4: [1200.0, 1195.0, 500.0, 501.0, 0.02, -0.01, 1e-3, -2e-3],            # OPENCV
    5: [1200.0, 1195.0, 500.0, 501.0, 0.01, -0.005, 0.002, -0.001],         # OPENCV_FISHEYE
    6: [1200.0, 1195.0, 500.0, 501.0, 0.02, -0.01, 1e-3, -2e-3, 0.003, 0.01, -0.004, 0.002],  # FULL_OPENCV
}


def _scene(model):
    prob, _ = synthetic.make_ba_scene(n_cams=6, n_points=300, track_len=5, channels=16, seed=60 + model, dtype=np.float32)
    if MODELS[model] is not None:
        prob.cam_model[:] = model
        prob.cam_params[:] = 0
        prob.cam_params[:, :len(MODELS[model])] = MODELS[model]
    prob.refs, _ = _engine.refs_compute(prob, _capi.default_interp())
    return prob


@pytest.mark.parametrize("count_on_device", [False, True], ids=["host_count", "device_count"])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_point_projection_matches_full_projection(model, count_on_device):
    prob = _scene(model)
    h = _engine.BAHandle(prob.copy(), _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=1))
    full = h.evaluate_jacobians()["juv"]                   # [n_obs, 2, W]: 6 pose | 3 point | K intrinsics columns
    rng = np.random.default_rng(model)
    n_obs = prob.n_obs
    for n in (1, n_obs // 3, n_obs):
        items = rng.permutation(n_obs)[:n]
        got = h.debug_project_point(items, count_on_device=count_on_device)
        listed = np.zeros(n_obs, bool)
        listed[items] = True
        assert np.array_equal(got["jpt"][listed], full[listed, :, 6:9]), "model %d, list length %d" % (model, n)
        assert np.array_equal(got["uv"][listed], got["uv_full"][listed]), "model %d, list length %d" % (model, n)
        assert np.isnan(got["jpt"][~listed]).all() and np.isnan(got["uv"][~listed]).all()
    h.close()


def _until_empty(counts):
    """the rows of debug_inner_rounds up to and including the first round with no points: how many empty rounds the host
    enqueues after that depends on how far it ran ahead of the device"""
    empty = np.flatnonzero(counts[:, 1] == 0)
    return counts[: empty[0] + 1] if len(empty) else counts


def _runs(keys):
    """start offsets of the runs of equal values in keys"""
    return np.flatnonzero(np.r_[True, keys[1:] != keys[:-1]])


@pytest.fixture(scope="module")
def big_scene():
    """70 000 observations, more than 32 W = 67 584 (one 16-warp K1 CTA per SM of an H100), a few constant points, and
    one point started far off so that it keeps going after the others have stopped"""
    prob, _ = synthetic.make_ba_scene(n_cams=40, n_points=7000, track_len=10, channels=16, ps=8, seed=1, dtype=np.float32)
    prob.refs, _ = _engine.refs_compute(prob, _capi.default_interp())
    rng = np.random.default_rng(2)
    prob.xyz += rng.normal(0, 0.004, prob.xyz.shape)
    prob.xyz[1234] += np.array([0.02, -0.015, 0.01])
    prob.point_const[::997] = 1
    return prob


def test_round_lists_restate_the_active_points(big_scene):
    """Every round's lists, read back: the points are the variable ones (round 0) or those the previous round's step
    kernel kept active, the observations are exactly theirs, a warp's points keep their order and its observations
    follow them point by point, and the lists shrink from the whole problem to a single point."""
    prob = big_scene
    assert prob.n_obs >= 32 * 132 * 16
    ic, so = _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=1)
    h = _engine.BAHandle(prob.copy(), ic, so)
    h.debug_inner_capture(True)
    h.debug_inner_iterations()
    counts, _ = h.debug_inner_rounds()
    rounds = h.debug_inner_round_lists()
    h.close()
    pt_begin = np.searchsorted(prob.obs_pt, np.arange(len(prob.xyz) + 1))
    n_per = np.diff(pt_begin)
    assert len(rounds) == len(counts)
    prev_pos = None
    for r, rd in enumerate(rounds):
        pts, obs = rd["points"], rd["obs"]
        assert len(obs) == counts[r, 0] and len(pts) == counts[r, 1], "round %d" % r
        if r == 0:
            want = np.flatnonzero((prob.point_const == 0) & (n_per > 0))
        else:
            want = np.sort(rounds[r - 1]["points"][rounds[r - 1]["active"]])
        assert np.array_equal(np.sort(pts), want), "round %d" % r
        ranges = [np.arange(pt_begin[p], pt_begin[p + 1]) for p in np.sort(pts)]
        assert np.array_equal(np.sort(obs), np.concatenate(ranges) if ranges else obs), "round %d" % r
        if len(pts) == 0:
            break
        # the warp that appended a point: round 0's list kernel runs one thread per point, a later round's step kernel
        # one thread per position of the previous round's list
        src = pts if r == 0 else prev_pos[pts]
        key = src // 32
        starts = _runs(key)
        assert len(starts) == len(np.unique(key)), "round %d: a warp's points are not contiguous" % r
        same = key[1:] == key[:-1]
        assert (np.diff(src)[same] > 0).all(), "round %d: a warp's points are out of order" % r
        want_obs = {}
        for k, p in zip(key, pts):
            want_obs.setdefault(k, []).append(np.arange(pt_begin[p], pt_begin[p + 1]))
        okey = np.empty(len(prob.xyz), np.int64)
        okey[pts] = key
        okeys = okey[prob.obs_pt[obs]]
        ostarts = _runs(okeys)
        assert len(ostarts) == len(want_obs), "round %d: a warp's observations are not contiguous" % r
        for a, b in zip(ostarts, np.r_[ostarts[1:], len(obs)]):
            assert np.array_equal(obs[a:b], np.concatenate(want_obs[okeys[a]])), "round %d" % r
        prev_pos = np.full(len(prob.xyz), -1, np.int64)
        prev_pos[pts] = np.arange(len(pts))
    live = counts[:, 1][counts[:, 1] > 0]
    assert live.min() == 1, "the lists never got down to one point: %s" % counts[:, 1]


def test_round_timing_and_capture_do_not_change_the_rounds(big_scene):
    """Round timing adds events and list capture makes the host wait for every round; the rounds that do work, and the
    points they leave, must be the same as without either."""
    ic, so = _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=1)
    out = []
    for mode in ("plain", "timed", "captured"):
        h = _engine.BAHandle(big_scene.copy(), ic, so)
        h.debug_inner_rounds(enable_timing=1 if mode == "timed" else 0)
        h.debug_inner_capture(mode == "captured")
        h.debug_inner_iterations()
        counts, ms = h.debug_inner_rounds()
        if mode == "timed":
            split = h.debug_inner_round_split()
            assert (ms >= 0).all() and (split >= 0).all() and len(split) == len(ms)
        h.read_params()
        out.append((_until_empty(counts.astype(np.int64)), h.problem.xyz.copy()))
        h.close()
    (c0, x0), (c1, x1), (c2, x2) = out
    assert c0[-1, 1] == 0, "the rounds ran out before the lists emptied: %s" % c0[:, 1]
    assert np.array_equal(c0, c1) and np.array_equal(c0, c2)
    assert np.array_equal(x0, x1) and np.array_equal(x0, x2)
    obs, pts = c0[:, 0], c0[:, 1]
    n_per = np.bincount(big_scene.obs_pt, minlength=len(big_scene.xyz))
    assert obs[0] == n_per[big_scene.point_const == 0].sum() and obs[0] >= 32 * 132 * 16
    assert (np.diff(obs) <= 0).all() and (np.diff(pts) <= 0).all()
