"""The long-double reference of a query's normal equations (query_reference.py) and the query scenes the batched
query refinement is tested on, without a device: the reference against the oracle's own linearisation for every
camera model and intrinsic set, the PlusJacobian against a central difference, and the measured size of the smallest
columns the old max|H|-relative comparison could not see."""
import numpy as np
import pytest

import oracle_lib as O
import query_reference as R
from pixsfm._pixsfm import _capi


def test_plus_jacobian_is_the_derivative_of_quaternion_plus():
    rng = np.random.default_rng(1)
    for _ in range(5):
        q = rng.normal(size=4); q /= np.linalg.norm(q)
        P = R.plus_jacobian(q)
        h = 1e-6
        for a in range(3):
            d = np.zeros(3); d[a] = h
            qp, qm = np.zeros(4), np.zeros(4)
            O.lib().orc_quaternion_plus(O.p(q), O.p(d), O.p(qp))
            O.lib().orc_quaternion_plus(O.p(q), O.p(-d), O.p(qm))
            assert np.abs((qp - qm) / (2 * h) - P[:, a]).max() < 1e-9
        assert np.abs(P.T @ q).max() < 1e-15           # tangent columns are orthogonal to q
    # the long-double Plus is the oracle's
    d = np.array([0.3, -0.2, 0.1]); out = np.zeros(4)
    O.lib().orc_quaternion_plus(O.p(q), O.p(d), O.p(out))
    assert np.abs(np.asarray(R.quaternion_plus(q, d), np.float64) - out).max() < 1e-15


def _oracle_case(model, iset, loss="cauchy", blocks=40):
    q, m = R.make_query(blocks, model=model, iset=iset, channels=16, seed=3)
    lt, ls = R.LOSSES[loss]
    batch, o = R.pack([(q, m)], {"refine_focal_length": True, "loss": {"name": loss, "params": [ls]}})
    prob = R.query_problem(batch, 0)
    so = o.solver_options()
    assert (so.loss_type, so.loss_scale) == (lt, ls)
    ic = _capi.default_interp()
    return batch, prob, so, ic, R.normal_equations(prob, ic, lt, ls)


@pytest.mark.parametrize("iset", R.INTRINSIC_SETS)
@pytest.mark.parametrize("model", sorted(R.MODEL_PARAMS))
def test_reference_matches_oracle_linearisation(model, iset):
    batch, prob, so, ic, ref = _oracle_case(model, iset)
    lin = O.ba_linearize(prob, ic, so)
    n = R.n_columns(batch, 0)
    assert lin["nc"] == ref["nc"] == n
    assert R.scaled_error(lin["Hcc"], ref) <= R.KAPPA
    assert R.scaled_error(lin["gc"], ref, "g") <= R.KAPPA
    assert abs(lin["cost"] - float(ref["cost"])) <= 1e-12 * lin["cost"]


@pytest.mark.parametrize("loss", sorted(R.LOSSES))
def test_reference_matches_oracle_linearisation_under_each_loss(loss):
    batch, prob, so, ic, ref = _oracle_case(6, "all", loss)
    lin = O.ba_linearize(prob, ic, so)
    assert R.scaled_error(lin["Hcc"], ref) <= R.KAPPA and R.scaled_error(lin["gc"], ref, "g") <= R.KAPPA
    assert abs(lin["cost"] - float(ref["cost"])) <= 1e-12 * lin["cost"]


def test_first_step_matches_the_oracle_step():
    """the long-double step of iteration 1 is the oracle's (ba_linearize's delta at the initial radius)"""
    batch, prob, so, ic, ref = _oracle_case(6, "all")
    lin = O.ba_linearize(prob, ic, so, radius=so.initial_trust_region_radius)
    n = R.n_columns(batch, 0)
    st = R.first_step(ref, n, batch.qvec[0], batch.tvec[0], batch.cam_params[0], 6, int(batch.cam_const_mask[0]), so)
    d = np.asarray(st["delta"], np.float64)
    assert np.abs(d - lin["delta"][:n]).max() <= 1e-12 * st["cond"] * np.abs(d).max()


@pytest.mark.parametrize("blocks,refs_per_point,kind", [(1, 1, "sparse"), (2, 1, "sparse"), (31, 1, "sparse"),
                                                        (32, 1, "sparse"), (33, 1, "sparse"), (257, 1, "sparse"),
                                                        (1126, 3, "sparse"), (300, 1, "dense"), (64, 1, "border"),
                                                        (40, 1, "axis")])
def test_query_scenes_have_the_blocks_and_columns_they_promise(blocks, refs_per_point, kind):
    qs = [R.make_query(blocks, model=m, iset=i, channels=16, seed=5, kind=kind, refs_per_point=refs_per_point)
          for m, i in ((6, "all"), (5, "extra"), (0, "pose"), (2, "focal"))]
    batch, _ = R.pack(qs)
    assert list(np.diff(batch.obs_begin)) == [blocks] * 4
    assert [R.n_columns(batch, k) for k in range(4)] == [18, 10, 6, 7]
    if kind == "dense":
        assert (batch.obs_patch == 0).all() and batch.patch_blocks[0].shape[1:3] == (192, 256)
    if kind == "border":           # projections before, on and past the patch's first and last rows and columns
        prob = R.query_problem(batch, 2)
        ev = O.ba_evaluate(prob, _capi.default_interp(), _capi.default_ba_options())
        u = ev["xy"][:, 0] * prob.scale[prob.obs_patch, 0] - 0.5 - prob.corner[prob.obs_patch, 0]
        assert u.min() < -1 and u.max() > 8 and ((u > 6) & (u < 8)).any()
    if kind == "axis":
        prob = R.query_problem(batch, 1)
        ev = O.ba_evaluate(prob, _capi.default_interp(), _capi.default_ba_options())
        assert np.abs(ev["xy"] - np.array(R.MODEL_PARAMS[5][2:4])).max() < 1e-3


def test_small_columns_are_far_below_the_max_h_scale():
    """min diag(H) / max|H| at the synthetic scenes' field of view (measured, printed): the high-order distortion
    columns of OPENCV_FISHEYE and FULL_OPENCV sit many orders of magnitude below 1e-9 * max|H|.  Applied to the
    reference itself, every swap of two distortion columns and the loss of the last free intrinsic are far outside
    the scaled bound; the printed max|H|-relative size of the same changes shows how close they come to a
    1e-9 * max|H| tolerance (their cross terms with the pose columns scale like sqrt(diag), which keeps swaps visible
    to it, while a dropped last column is at its edge)."""
    for model in (5, 6):
        batch, prob, so, ic, ref = _oracle_case(model, "all")
        H = np.asarray(ref["H"], np.float64)
        n, mx = H.shape[0], np.abs(H).max()
        ratio = np.diag(H).min() / mx
        print("model %d (%s), every intrinsic free: min diag(H) / max|H| = %.3g" % (model, R.MODEL_NAMES[model], ratio))
        assert ratio < 1e-9
        extra = [6 + k for k in R.free_params(model, 0) if k >= 4]
        old = []
        for i in extra:
            for j in extra:
                if i < j:
                    perm = np.arange(n); perm[[i, j]] = perm[[j, i]]
                    Hs = H[np.ix_(perm, perm)]
                    old.append(np.abs(Hs - H).max() / mx)
                    assert R.scaled_error(Hs, ref) > 1.0, (i, j)
        Hd = H.copy(); Hd[-1, :] = 0; Hd[:, -1] = 0
        assert R.scaled_error(Hd, ref) >= 1.0
        print("  swapped distortion columns: smallest change %.2g of max|H|; last column dropped: %.2g of max|H|"
              % (min(old), np.abs(Hd - H).max() / mx))
