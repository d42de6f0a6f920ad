"""K1 evaluates one observation per half-warp, and the two halves of a warp run different observations in step.  Every
record must be the one a full-range pass computes, bit for bit, whatever the list length and whatever the other half
of the warp is doing: list lengths straddle the half-warp count W2 of a long fp16 128-channel launch and 32 W2, where
the batch size and the number of batches per half-warp change; warps mix in-range, clamped border and far-off windows;
and the cost-only pass reduces ||r||^2 with the same tree as the Jacobian pass."""
import numpy as np
import pytest

from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

FM_INSTANCES = [(np.float16, c) for c in (8, 16, 32, 64, 128, 256)] + \
               [(np.float32, c) for c in (16, 64, 128)] + [(np.float64, c) for c in (16, 128)]


def _k1_half_warps():
    """half-warps of one K1 launch over a long list of the fp16 128-channel instance, as the library sizes it"""
    W2 = _engine.k1_half_warps(np.float16, 128, 10 ** 7)
    per_cta = _engine.k1_half_warps(np.float16, 128, 1)      # a one-item launch is one CTA
    assert per_cta >= 2 and W2 % per_cta == 0
    return W2


def _records(h):
    full = h.evaluate()
    return np.concatenate([full["sq_norm"][:, None], full["gtr"], full["gtg"]], axis=1)


@pytest.fixture(scope="module")
def scene():
    """110 000 observations (more than 32 W2 + 1) of 8x8 patches, with feature references"""
    prob, _ = synthetic.make_ba_scene(n_cams=40, n_points=11000, track_len=10, channels=128, ps=8, seed=5)
    prob.refs, _ = _engine.refs_compute(prob, _capi.default_interp())
    return prob


@pytest.mark.parametrize("count_on_device", [False, True], ids=["host_count", "device_count"])
def test_list_lengths_around_half_warp_counts(scene, count_on_device):
    W2 = _k1_half_warps()
    n_obs = scene.n_obs
    assert n_obs > 32 * W2 + 1
    h = _engine.BAHandle(scene.copy(), _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=0))
    ref = _records(h)
    rng = np.random.default_rng(11)
    for n in (1, 2, 3, W2 - 1, W2, W2 + 1, 32 * W2 - 1, 32 * W2, 32 * W2 + 1, n_obs):
        items = rng.permutation(n_obs)[:n]
        out = h.debug_eval_list(items, count_on_device=count_on_device)
        listed = np.zeros(n_obs, bool)
        listed[items] = True
        assert np.array_equal(out[listed, :6], ref[listed]), "list length %d" % n
        assert np.isnan(out[~listed]).all(), "list length %d wrote outside the list" % n
    h.close()


def _mixed_scene(n_points, seed):
    """observations cycling through three kinds of window: 0 in range, 1 clamped at the border, 2 far off the patch"""
    prob, _ = synthetic.make_ba_scene(n_cams=40, n_points=n_points, track_len=10, channels=128, ps=8, seed=seed)
    prob.refs, _ = _engine.refs_compute(prob, _capi.default_interp())
    kind = np.arange(prob.n_obs) % 3
    corner = prob.corner.copy()
    corner[kind == 1, 0] += 4                    # the projection lands left of column 0
    corner[kind == 1, 1] -= 3                    # and below the last row
    corner[kind == 2] += 100000
    prob.corner = corner
    return prob, kind


def test_halves_mixing_border_and_far_off_windows():
    """short lists put item k on half-warp k, so items 2m and 2m + 1 share a warp: every pair of kinds, both orders"""
    prob, kind = _mixed_scene(300, 9)
    n = prob.n_obs
    h = _engine.BAHandle(prob, _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=0))
    rng = np.random.default_rng(4)
    by_kind = [rng.permutation(np.flatnonzero(kind == k)) for k in range(3)]
    pairs = [(a, b) for a in range(3) for b in range(3)]
    mixed = np.array([by_kind[k][i] for i, (a, b) in enumerate(pairs) for k in (a, b)])
    alone = {o: h.debug_eval_list(np.array([o]))[o] for o in mixed}
    assert all(np.isfinite(r[:6]).all() for r in alone.values())
    full = _records(h)
    for items in (mixed, mixed[:-1]):
        out = h.debug_eval_list(items)
        for o in items:
            assert np.array_equal(out[o], alone[o], equal_nan=True)
            assert np.array_equal(full[o], alone[o][:6])
    h.close()


def test_mixed_windows_through_the_ring():
    """more than 32 W2 observations of mixed kinds in random order: every half-warp walks batches of close to 32 items,
    so border and far-off windows go through the ring refill of both halves; every record must be the full-range one
    and the one of the observation evaluated alone"""
    W2 = _k1_half_warps()
    prob, kind = _mixed_scene(8000, 13)
    n = prob.n_obs
    assert n > 32 * W2
    h = _engine.BAHandle(prob, _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=0))
    full = _records(h)
    assert np.isfinite(full).all()
    rng = np.random.default_rng(6)
    for count_on_device in (False, True):
        items = rng.permutation(n)
        out = h.debug_eval_list(items, count_on_device=count_on_device)
        assert np.array_equal(out[:, :6], full)
    for o in rng.choice(n, 60, replace=False):
        assert np.array_equal(h.debug_eval_list(np.array([o]))[o, :6], full[o])
    h.close()


@pytest.mark.parametrize("with_refs", [False, True], ids=["no_refs", "refs"])
@pytest.mark.parametrize("float_simd", [0, 1], ids=["f64_vertical", "float_simd"])
@pytest.mark.parametrize("dtype,channels", FM_INSTANCES, ids=lambda v: v.__name__ if isinstance(v, type) else str(v))
def test_cost_only_sq_norm_equals_jacobian_mode(dtype, channels, float_simd, with_refs):
    prob, _ = synthetic.make_ba_scene(n_cams=5, n_points=60, track_len=4, channels=channels, seed=channels, dtype=dtype)
    ic = _capi.default_interp()
    ic.use_float_simd = float_simd
    prob.refs = _engine.refs_compute(prob, ic)[0] if with_refs else None
    h = _engine.BAHandle(prob, ic, _capi.default_ba_options(use_inner_iterations=0))
    jac = h.debug_eval_records(1)
    cost = h.debug_eval_records(0)
    h.close()
    assert np.isfinite(jac[:, :6]).all()
    assert np.array_equal(cost[:, 0], jac[:, 0])
    assert np.isnan(cost[:, 1:]).all()
