"""The block-sparse long-double reference of bundle adjustment's damped Schur system and LM step (ba_schur_reference)
checked on the CPU: the float64 oracle (orc_ba_linearize) falls inside its error bounds, its camera blocks equal the
dense long-double normal equations (query_reference.normal_equations), and its comparators reject small, structural
mistakes applied to the oracle's output."""
import numpy as np
import pytest

import ba_schur_reference as R
import dispatch_scenes as D
import oracle_lib as O
import query_reference as Q
from pixsfm._pixsfm import _capi
from pixsfm.util import synthetic

_cache = {}


def _parity_scene(variant):
    """the scenes of test_gpu_ba_parity: per-image and shared cameras, constant blocks and partial masks"""
    kw = dict(n_cams=6, n_points=60, track_len=4, channels=128, seed=0)
    if variant == "shared_camera":
        kw["shared_camera"] = True
    if variant == "constant_blocks":
        kw.update(n_cams=7, n_points=50, refine_pp=True)
    prob, _ = synthetic.make_ba_scene(**kw)
    if variant == "constant_blocks":
        prob.point_const[::7] = 1
        prob.pose_const[3] = 1
        prob.tvec_const_mask[4] = 0b101
        prob.cam_const_mask[2] = 0xFFFFFFFF
    return prob


SCENES = {"per_image": lambda: _parity_scene("per_image"), "shared_camera": lambda: _parity_scene("shared_camera"),
          "constant_blocks": lambda: _parity_scene("constant_blocks")}
SCENES.update({"model_%s" % Q.MODEL_NAMES[m]: (lambda m=m: D._one_model(m, "fpe", 40 + m)) for m in Q.MODEL_NAMES})


def _case(name):
    if name not in _cache:
        ic = _capi.default_interp()
        prob = SCENES[name]()
        if prob.refs is None:
            prob = D.with_refs(prob, ic)
        so = R.default_options()
        # small point chunks: several chunks per scene, with tracks ending at the chunk boundaries
        ref = R.linearize_at_largest_radius(prob, R.oracle_blocks(prob, ic, so.loss_type, so.loss_scale), so,
                                            chunk_points=17)
        orc = O.ba_linearize(prob, ic, so, radius=ref["radius"])
        _cache[name] = (prob, ic, so, ref, orc)
    return _cache[name]


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_falls_within_the_reference_bounds(name):
    prob, ic, so, ref, orc = _case(name)
    assert (ref["nc"], ref["nl"]) == (orc["nc"], orc["nl"])
    errs = R.all_errors(orc, ref)
    assert max(errs.values()) <= 1.0, errs


@pytest.mark.parametrize("name", ["per_image", "shared_camera", "constant_blocks", "model_FULL_OPENCV"])
def test_camera_blocks_equal_the_dense_reference(name):
    """Hcc and gc against query_reference.normal_equations: both are long-double sums of the same terms in another
    order, apart by at most (n_terms x 5.4e-20) of the sum of absolute terms, i.e. under 1e-6 of KAPPA for n_terms
    below 1e4"""
    prob, ic, so, ref, orc = _case(name)
    dense = Q.normal_equations(prob, ic, so.loss_type, so.loss_scale)
    nc = ref["nc"]
    assert R.hcc_error(dense["H"][:nc, :nc], ref) <= 1e-6
    assert R.gc_error(dense["g"][:nc], ref) <= 1e-6
    assert abs(dense["cost"] - ref["cost"]) <= 1e-15 * dense["cost"]


def _two_image_point(ref):
    """a variable point with observations in two images whose column blocks are both non-empty"""
    lay = ref["layout"]
    for p in np.nonzero(lay["point_off"] >= 0)[0]:
        o0, o1 = lay["start"][p], lay["start"][p + 1]
        imgs = ref["obs_img"][lay["order"][o0:o1]]
        ok = [i for i in np.unique(imgs) if (lay["cols_img"][i] < lay["nc"]).any()]
        if len(ok) >= 2:
            return p, ok[0], ok[1]
    raise AssertionError("no point seen by two images with camera columns")


def test_mutations_are_rejected():
    prob, ic, so, ref, orc = _case("per_image")
    assert max(R.all_errors(orc, ref).values()) <= 1.0
    lay = ref["layout"]
    nc, ci = lay["nc"], lay["cols_img"]
    p, i, j = _two_image_point(ref)
    term, rterm, _ = R.point_terms(ref, p)
    ri, rj = ci[i][ci[i] < nc], ci[j][ci[j] < nc]
    # one point's pair term removed from one off-diagonal camera block (and its mirror)
    S = np.array(orc["S"])
    blk = np.ix_(ri, rj)
    S[blk] += np.asarray(term[blk], np.float64)
    S[np.ix_(rj, ri)] += np.asarray(term[np.ix_(rj, ri)], np.float64)
    assert R.s_error(S, ref) > 1.0
    # one point's term removed from rhs
    assert R.rhs_error(orc["rhs"] - np.asarray(rterm, np.float64), ref) > 1.0
    # two camera columns of delta swapped
    d = np.array(orc["delta"])
    a, b = ri[0], rj[0]
    assert abs(d[a] - d[b]) > 0
    d[a], d[b] = d[b], d[a]
    assert R.delta_error(d, ref) > 1.0
    # one entry of one W_p changed by 1e-6 relative
    o0 = lay["start"][p]
    Wp = np.array(ref["W"][o0:lay["start"][p + 1]])
    k = int(np.argmax(np.abs(Wp[0, 0])))
    Wp[0, 0, k] *= 1 + 1e-6
    mterm, _, _ = R.point_terms(ref, p, W=Wp)
    S = np.array(orc["S"]) - np.asarray(mterm - term, np.float64)
    assert R.s_error(S, ref) > 1.0
