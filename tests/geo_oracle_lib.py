"""ctypes loader for the CPU restatement of geometric bundle adjustment (oracle_geo/liboracle_geo.so).  TEST
INFRASTRUCTURE: imported by the geometric tests and scripts/geometric_ba_bench.py.  Every function takes a BAProblem
with obs_xy (a geometric problem: no patches)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEO_DIR = os.path.join(ROOT, "oracle_geo")

_libs = {}


def lib(fast=False):
    """the parity build, or with fast=True the -O3 build that is only ever timed"""
    name = "liboracle_geo_fast.so" if fast else "liboracle_geo.so"
    if name not in _libs:
        p = os.path.join(GEO_DIR, name)
        if not os.path.exists(p):
            subprocess.check_call(["make", "-C", GEO_DIR, "-s"])
        _libs[name] = C.CDLL(p)
    return _libs[name]


def p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ba_evaluate_geometric(prob, opts, residuals=False):
    d = prob.desc()
    n = prob.n_obs
    out = dict(sq_norm=np.zeros(n), gtr=np.zeros((n, 2)), gtg=np.zeros((n, 3)), xy=np.zeros((n, 2)))
    res = np.zeros((n, 2)) if residuals else None
    cost = C.c_double()
    lib().orc_geo_evaluate(C.byref(d), C.byref(opts), p(prob.obs_xy), p(out["sq_norm"]), p(out["gtr"]), p(out["gtg"]),
                           p(out["xy"]), p(res), C.byref(cost))
    out["cost"] = cost.value
    if residuals:
        out["residuals"] = res
    return out


def ba_block_jacobians_geometric(prob):
    """per residual block: r [n,2] and the ambient ceres Jacobian [n,2,10+PXR_MAX_CAM_PARAMS] (q4|t3|X3|cam) by Jets"""
    from pixsfm._pixsfm._capi import PXR_MAX_CAM_PARAMS
    d = prob.desc()
    n = prob.n_obs
    res = np.zeros((n, 2)); J = np.zeros((n, 2, 10 + PXR_MAX_CAM_PARAMS))
    assert lib().orc_geo_block_jacobians(C.byref(d), p(prob.obs_xy), p(res), p(J)) == 0
    return res, J


def ba_linearize_geometric(prob, opts, radius=1e4):
    import oracle_lib as O
    d = prob.desc()
    nc, nl, _, _, _ = O.ba_layout(prob)
    npts = d.n_points
    out = dict(Hcc=np.zeros((nc, nc)), gc=np.zeros(nc), Hpp=np.zeros((npts, 3, 3)), gp=np.zeros((npts, 3)),
               S=np.zeros((nc, nc)), rhs=np.zeros(nc), delta=np.zeros(nl))
    cost = C.c_double(); mcc = C.c_double()
    rc = lib().orc_geo_linearize(C.byref(d), C.byref(opts), p(prob.obs_xy), C.c_double(radius), C.byref(cost),
                                 p(out["Hcc"]), p(out["gc"]), p(out["Hpp"]), p(out["gp"]), p(out["S"]), p(out["rhs"]),
                                 p(out["delta"]), C.byref(mcc))
    if rc != 0:
        raise RuntimeError("orc_geo_linearize failed: %d" % rc)
    out["cost"] = cost.value; out["model_cost_change"] = mcc.value
    out["nc"] = nc; out["nl"] = nl
    return out


def ba_solve_geometric(prob, opts, fast=False):
    """the trust-region solve of the geometric problem IN PLACE -> summary dict"""
    from pixsfm._pixsfm import _capi
    d = prob.desc()
    s = _capi.make_summary(512)
    lib(fast).orc_geo_solve(C.byref(d), C.byref(opts), p(prob.obs_xy), C.byref(s))
    return _capi.summary_to_dict(s)


def ba_inner_iterations_geometric(prob, opts):
    d = prob.desc()
    lib().orc_geo_inner_iterations(C.byref(d), C.byref(opts), p(prob.obs_xy))
