"""ctypes loader for the CPU oracle (oracle/liboracle.so) and the verbatim-reference shim
(oracle/_ref/libpxref.so).  TEST INFRASTRUCTURE: imported by tests/, smoke() and bench.py's
cpu_baseline / --impl reference legs only."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")

_lib = None
_ref = None


def build():
    subprocess.check_call(["make", "-C", ORACLE_DIR, "-s"])


def lib():
    global _lib
    if _lib is None:
        p = os.path.join(ORACLE_DIR, "liboracle.so")
        if not os.path.exists(p):
            build()
        _lib = C.CDLL(p)
        _lib.orc_ka_problem_labels.restype = C.c_int
    return _lib


def ref():
    """libpxref.so or None (it only exists where a reference checkout was present at build time)."""
    global _ref
    if _ref is None:
        p = os.path.join(ORACLE_DIR, "_ref", "libpxref.so")
        if not os.path.exists(p):
            return None
        _ref = C.CDLL(p)
    return _ref


def p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def pixel_interp(grid, r, c, l2_normalize=True, use_float_simd=False):
    """PixelInterpolator::Evaluate on a [H,W,C] grid -> f, dfdr, dfdc"""
    from pixsfm._pixsfm._capi import DTYPE_IDS
    grid = np.ascontiguousarray(grid)
    h, w, ch = grid.shape
    f = np.zeros(ch); dr = np.zeros(ch); dc = np.zeros(ch)
    lib().orc_pixel_interp(p(grid), DTYPE_IDS[grid.dtype], h, w, ch, C.c_double(r), C.c_double(c),
                           int(l2_normalize), int(use_float_simd), p(f), p(dr), p(dc))
    return f, dr, dc


def bicubic_ceres(grid, r, c):
    from pixsfm._pixsfm._capi import DTYPE_IDS
    grid = np.ascontiguousarray(grid)
    h, w, ch = grid.shape
    f = np.zeros(ch); dr = np.zeros(ch); dc = np.zeros(ch)
    lib().orc_bicubic_ceres(p(grid), DTYPE_IDS[grid.dtype], h, w, ch, C.c_double(r), C.c_double(c),
                            p(f), p(dr), p(dc))
    return f, dr, dc


def ba_evaluate(prob, interp, opts, residuals=False):
    d = prob.desc()
    n = prob.n_obs
    out = dict(sq_norm=np.zeros(n), gtr=np.zeros((n, 2)), gtg=np.zeros((n, 3)), xy=np.zeros((n, 2)))
    res = np.zeros((n, prob.channels)) if residuals else None
    cost = C.c_double()
    lib().orc_ba_evaluate(C.byref(d), C.byref(interp), C.byref(opts), p(out["sq_norm"]), p(out["gtr"]),
                          p(out["gtg"]), p(out["xy"]), p(res), C.byref(cost))
    out["cost"] = cost.value
    if residuals:
        out["residuals"] = res
    return out


def ba_block_jacobians(prob, interp):
    """per residual block: r [n,C] and the ambient ceres Jacobian [n,C,10+PXR_MAX_CAM_PARAMS] (q4|t3|X3|cam) by Jets"""
    from pixsfm._pixsfm._capi import PXR_MAX_CAM_PARAMS
    d = prob.desc()
    n = prob.n_obs
    res = np.zeros((n, prob.channels)); J = np.zeros((n, prob.channels, 10 + PXR_MAX_CAM_PARAMS))
    rc = lib().orc_ba_block_jacobians(C.byref(d), C.byref(interp), p(res), p(J))
    assert rc == 0
    return res, J


def ba_layout(prob):
    d = prob.desc()
    nc = C.c_int(); nl = C.c_int()
    pose_off = np.zeros(d.n_images, np.int32); intr_off = np.zeros(d.n_cameras, np.int32)
    point_off = np.zeros(d.n_points, np.int64)
    lib().orc_ba_layout(C.byref(d), C.byref(nc), C.byref(nl), p(pose_off), p(intr_off), p(point_off))
    return nc.value, nl.value, pose_off, intr_off, point_off


PCG_STOP_ZETA, PCG_STOP_NONPOSITIVE_CURVATURE, PCG_STOP_MAX_ITERATIONS, PCG_STOP_FAILURE = range(4)


def schur_jacobi_pcg(S, b, blk_off, blk_dim, max_iter, eta=0.1):
    """SchurJacobiPCG (orc_ba.h) on S x = b, S symmetric [n, n] -> (x, iterations, stop reason PCG_STOP_*, ok)"""
    S = np.ascontiguousarray(S, np.float64); b = np.ascontiguousarray(b, np.float64)
    blk_off = np.ascontiguousarray(blk_off, np.int32); blk_dim = np.ascontiguousarray(blk_dim, np.int32)
    n = len(b)
    x = np.zeros(n); it = C.c_int(); stop = C.c_int()
    rc = lib().orc_schur_jacobi_pcg(n, p(S), p(b), len(blk_off), p(blk_off), p(blk_dim), int(max_iter), C.c_double(eta),
                                    p(x), C.byref(it), C.byref(stop))
    return x, it.value, stop.value, rc == 0


def ba_linearize(prob, interp, opts, radius=1e4):
    d = prob.desc()
    nc, nl, _, _, _ = ba_layout(prob)
    npts = d.n_points
    out = dict(Hcc=np.zeros((nc, nc)), gc=np.zeros(nc), Hpp=np.zeros((npts, 3, 3)), gp=np.zeros((npts, 3)),
               S=np.zeros((nc, nc)), rhs=np.zeros(nc), delta=np.zeros(nl))
    cost = C.c_double(); mcc = C.c_double()
    rc = lib().orc_ba_linearize(C.byref(d), C.byref(interp), C.byref(opts), C.c_double(radius), C.byref(cost),
                                p(out["Hcc"]), p(out["gc"]), p(out["Hpp"]), p(out["gp"]), p(out["S"]),
                                p(out["rhs"]), p(out["delta"]), C.byref(mcc))
    if rc != 0:
        raise RuntimeError("orc_ba_linearize failed: %d" % rc)
    out["cost"] = cost.value; out["model_cost_change"] = mcc.value
    out["nc"] = nc; out["nl"] = nl
    return out


def ba_solve(prob, interp, opts, verbose=False):
    """Runs the oracle LM on prob IN PLACE (prob arrays are updated). Returns summary dict."""
    from pixsfm._pixsfm import _capi
    d = prob.desc()
    s = _capi.make_summary(512)
    lib().orc_ba_solve(C.byref(d), C.byref(interp), C.byref(opts), C.byref(s), int(verbose))
    return _capi.summary_to_dict(s)


def refs_compute(prob, interp, loss_type=1, loss_scale=0.25, iters=100):
    d = prob.desc()
    refs = np.zeros((d.n_points, prob.channels)); src = np.zeros(d.n_points, np.int64)
    lib().orc_refs_compute(C.byref(d), C.byref(interp), loss_type, C.c_double(loss_scale), iters, p(refs), p(src))
    return refs, src


def costmaps_compute(prob, loss_type=0, loss_scale=1.0, as_gradientfield=True, apply_sqrt=False):
    """orc_costmaps_compute (costmap_extractor.h:230-358); prob.refs must be set."""
    d = prob.desc()
    oc = 3 if as_gradientfield else 1
    n_patches = d.n_patches if d.n_patches else d.n_obs
    out = np.zeros((n_patches, prob.ph, prob.pw, oc), prob.patch_np_dtype)
    rc = lib().orc_costmaps_compute(C.byref(d), int(loss_type), C.c_double(loss_scale), int(as_gradientfield),
                                    int(apply_sqrt), p(out))
    assert rc == 0
    return out


def ka_solve(kaprob, interp, opts):
    """Oracle KA on kaprob IN PLACE (keypoints updated). Returns (initial_cost, final_cost)."""
    from pixsfm._pixsfm import _capi
    d = kaprob.desc()
    s = _capi.make_summary(0)
    lib().orc_ka_solve(C.byref(d), C.byref(interp), C.byref(opts), C.byref(s))
    return s.initial_cost, s.final_cost


def ka_evaluate(kaprob, interp, opts):
    d = kaprob.desc()
    sq = np.zeros(len(kaprob.edge_src)); cost = C.c_double()
    lib().orc_ka_evaluate(C.byref(d), C.byref(interp), C.byref(opts), p(sq), C.byref(cost))
    return sq, cost.value
