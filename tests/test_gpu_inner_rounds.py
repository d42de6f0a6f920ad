"""K1 spreads the items of a pass evenly over all its warps: whatever the length of the observation list, every
observation's record must be the one a full-range evaluation computes, bit for bit.  The list lengths straddle the
warp count W of the fp16 128-channel instance and 32 W, where the number of batches per warp and the batch size
change.  The batched inner iterations, whose rounds (K0, K1 and the step kernel that builds the next round's lists)
evaluate ever shorter lists, must stop every point where the oracle's per-point solve stops it."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu


def _k1_warps():
    """warps of one K1 launch over a long list of the fp16 128-channel instance: one 16-warp CTA per SM"""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 16


@pytest.fixture(scope="module")
def scene():
    """70 000 observations (more than 32 W + 1) of 8x8 patches, with feature references"""
    prob, _ = synthetic.make_ba_scene(n_cams=40, n_points=7000, track_len=10, channels=128, ps=8, seed=1)
    prob.refs, _ = _engine.refs_compute(prob, _capi.default_interp())
    return prob


@pytest.mark.parametrize("count_on_device", [False, True], ids=["host_count", "device_count"])
def test_k1_list_lengths_match_full_range(scene, count_on_device):
    W = _k1_warps()
    n_obs = scene.n_obs
    assert n_obs > 32 * W + 1
    assert n_obs % 32 != 0 and n_obs % W != 0            # the full range ends in a partial batch
    h = _engine.BAHandle(scene.copy(), _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=0))
    full = h.evaluate()
    ref = np.concatenate([full["sq_norm"][:, None], full["gtr"], full["gtg"]], axis=1)
    rng = np.random.default_rng(3)
    for n in (1, W - 1, W, W + 1, 32 * W - 1, 32 * W, 32 * W + 1, n_obs):
        items = rng.permutation(n_obs)[:n]
        out = h.debug_eval_list(items, count_on_device=count_on_device)
        listed = np.zeros(n_obs, bool)
        listed[items] = True
        assert np.array_equal(out[listed, :6], ref[listed]), "list length %d" % n
        assert np.isnan(out[~listed, 0]).all(), "list length %d wrote outside the list" % n
    h.close()


def test_device_counted_list_longer_than_the_problem_is_refused(scene):
    h = _engine.BAHandle(scene.copy(), _capi.default_interp(), _capi.default_ba_options(use_inner_iterations=0))
    with pytest.raises((ValueError, _capi.PxrError)):
        h.debug_eval_list(np.zeros(scene.n_obs + 1, np.int64), count_on_device=True)
    h.close()


def test_inner_rounds_match_oracle(scene):
    W = _k1_warps()
    ic = _capi.default_interp()
    so = _capi.default_ba_options(use_inner_iterations=1)
    prob = scene.copy()
    prob.xyz += np.random.default_rng(2).normal(0, 0.004, prob.xyz.shape)
    p_ref = prob.copy()
    O.lib().orc_ba_inner_iterations(C.byref(p_ref.desc()), C.byref(ic), C.byref(so))
    assert np.abs(p_ref.xyz - prob.xyz).max() > 1e-3
    h = _engine.BAHandle(prob.copy(), ic, so)
    h.debug_inner_iterations()
    counts, _ = h.debug_inner_rounds()
    h.read_params()
    xyz = h.problem.xyz.copy()
    h.close()
    obs = counts[:, 0].astype(np.int64)
    # the active list starts at every observation and shrinks round by round, through 32 W
    assert obs[0] == prob.n_obs
    assert (np.diff(obs) <= 0).all()
    assert obs[obs > 0].min() < 32 * W
    assert np.abs(xyz - p_ref.xyz).max() < 1e-7
