"""The reduced camera solve S x = rhs on its own (pxr_ba_debug_reduced_solve), against extended-precision references.

Cholesky paths: the persistent tile-DAG kernel (default), the band kernel (PXR_CHOL_BAND) and the launch-per-panel
kernels (PXR_CHOL_MULTIKERNEL, also the bail-out's fall-back).  Every solution is held to LAPACK on the same matrix:
normwise backward error ||b - S x||inf / (||S||inf ||x||inf + ||b||inf) with the residual in long double, and forward
error against LAPACK's solution refined twice with long-double residuals (checked against mpmath at 50 digits up to
n = 64).  A backward-stable Cholesky has backward error O(u sqrt(n)) and forward error O(kappa u sqrt(n)) (Higham,
Accuracy and Stability of Numerical Algorithms, 2nd ed., Thm 10.3 and 7.2); the GPU is allowed 8x LAPACK's measured
errors, with those first-order terms as floors.

The dense PCG (linear_solver = ITERATIVE_SCHUR) is compared with orc_schur_jacobi_pcg, the oracle's restatement of
ceres' ConjugateGradientsSolver with the SCHUR_JACOBI preconditioner: iteration count, stop and x.

Handles of a chosen size nc come from geometric problems with one constant point: variable poses (6 columns, fewer
with a tvec mask) and free intrinsics set the column count."""
import contextlib
import os

import numpy as np
import pytest
import scipy.linalg as sla

import oracle_lib as O
from pixsfm._pixsfm import _capi, _engine
from pixsfm.util import synthetic

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
TB = 32
PATHS = {"persistent": {}, "band": {"PXR_CHOL_BAND": "1"}, "panel": {"PXR_CHOL_MULTIKERNEL": "1"}}
SIMPLE_RADIAL = 2


@contextlib.contextmanager
def _env(env):
    """the path switches are read when the handle is created and at its first solve: keep them set around both"""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# ------------------------------------------------------------------------------------------------ handles of size nc
def _problem(pose_free_t, cam_free, img_cam):
    """pose_free_t[i]: free tvec components of image i (-1: constant pose); cam_free[c]: free SIMPLE_RADIAL parameters
    of camera c (the leading ones).  One constant point observed once: the reduced system is all there is."""
    ni, ncam = len(pose_free_t), len(cam_free)
    pose_const = np.array([k < 0 for k in pose_free_t], np.uint8)
    tmask = np.array([7 & ~((1 << max(k, 0)) - 1) for k in pose_free_t], np.uint8)
    cmask = np.array([15 & ~((1 << k) - 1) for k in cam_free], np.uint32)
    q = np.tile([1.0, 0.0, 0.0, 0.0], (ni, 1)); t = np.tile([0.0, 0.0, 10.0], (ni, 1))
    cams = np.tile([1200.0, 500.0, 500.0, 0.0], (ncam, 1))
    return _capi.BAProblem(np.full(ncam, SIMPLE_RADIAL, np.int32), cams, cmask, q, t, np.asarray(img_cam, np.int32),
                           pose_const, tmask, np.zeros((1, 3)), np.ones(1, np.uint8), np.zeros(1, np.int32),
                           np.zeros(1, np.int64), None, None, None, obs_xy=np.full((1, 2), 500.0))


def _problem_nc(nc):
    """nc columns: full poses, one image with a partial tvec mask or free intrinsics of one shared camera for the rest"""
    if nc < 3:
        return _problem([-1], [nc], [0])
    full, rem = divmod(nc, 6)
    poses = [3] * full + ([rem - 3] if rem >= 3 else [])
    return _problem(poses, [rem if rem in (1, 2) else 0], [0] * len(poses))


def _problem_images(n_images, intr_free):
    """n_images variable poses, each with its own camera of intr_free free parameters"""
    return _problem([3] * n_images, [intr_free] * n_images, range(n_images))


def _blocks(prob):
    """the SCHUR_JACOBI blocks, as pcg_setup_blocks forms them from the layout"""
    nc, _, pose_off, intr_off, _ = O.ba_layout(prob)
    off = np.sort(np.concatenate([pose_off[pose_off >= 0], intr_off[intr_off >= 0]])).astype(np.int32)
    return nc, off, np.diff(np.append(off, nc)).astype(np.int32)


_HANDLES = {}


def _handle(path, nc=None, prob=None, cg=False, max_iter=200, fresh=False):
    """a handle per (path, size), kept for the module: every later solve also replays the earlier ones' state"""
    prob = prob if prob is not None else _problem_nc(nc)
    n = O.ba_layout(prob)[0]
    assert nc is None or n == nc
    key = (path, n, cg, max_iter, id(prob) if fresh else None)
    if key in _HANDLES and not fresh:
        return _HANDLES[key], prob
    so = _capi.default_ba_options(use_inner_iterations=0, linear_solver=3 if cg else 1, max_linear_solver_iterations=max_iter)
    with _env(_path_env(path)):
        h = _engine.BAHandle(prob, options=so)
    if n < 2048 and not fresh:            # large handles are not kept: device memory
        _HANDLES[key] = h
    return h, prob


def _path_env(path):
    return {"cg_multi": {"PXR_CG_MULTI": "1"}, "cg": {}}.get(path, PATHS.get(path, {}))


def _solve(path, h, S, b, factor=False):
    with _env(_path_env(path)):
        return h.debug_reduced_solve(S, b, factor=factor)


# ------------------------------------------------------------------------------------------------ matrices
def _sym(S):
    return (S + S.T) / 2


def spd_kappa(n, kappa, rng):
    """SPD with 2-norm condition number kappa: Q diag(logspace) Q^T, or above 2000 unknowns G G^T + log-spaced diagonal
    (O(n^2 m), condition number about 2 kappa)"""
    ev = np.logspace(0, -np.log10(kappa), n)
    if n <= 2000:
        Q, _ = np.linalg.qr(rng.standard_normal((n, n)))
        return _sym((Q * ev) @ Q.T)
    G = rng.standard_normal((n, 48)) / np.sqrt(n)
    rng.shuffle(ev)
    S = G @ G.T
    S[np.diag_indices(n)] += ev
    return _sym(S)


def lowrank(n, kappa, rng, hi=3.0, m=64):
    """G diag(logspace(-1, hi)) G^T + log-spaced diagonal (1 .. 1/kappa): a spectrum the block-Jacobi preconditioner
    barely helps; the larger hi, the more CG iterations"""
    G = rng.standard_normal((n, m)) / np.sqrt(n)
    d = np.logspace(0, -np.log10(kappa), n); rng.shuffle(d)
    S = G @ (G.T * np.logspace(-1 if hi < 3 else 0, hi, m)[:, None])
    S[np.diag_indices(n)] += d
    return _sym(S)


def scaled(n, rng):
    """D S D with D log-uniform over 1e-8 .. 1e8: badly row/column-scaled, well conditioned once equilibrated"""
    d = 10.0 ** rng.uniform(-8, 8, n)
    return d[:, None] * spd_kappa(n, 10.0, rng) * d[None, :]


def arrowhead(n, rng):
    """one camera block (the last min(3, n) columns) coupled to every image block of 6: what a shared camera gives"""
    k = min(3, n); m = n - k
    S = np.zeros((n, n))
    cam = list(range(m, n))
    for o in range(0, max(m, 1), 6):
        cols = list(range(o, min(o + 6, m))) + cam
        W = rng.standard_normal((2 * len(cols), len(cols)))
        S[np.ix_(cols, cols)] += W.T @ W
    S[np.diag_indices(n)] += 1e-3
    return S


def blockdiag(n, rng):
    S = np.zeros((n, n))
    for o in range(0, n, 6):
        e = min(o + 6, n)
        S[o:e, o:e] = spd_kappa(e - o, 10.0 ** rng.uniform(0, 8), rng)
    return S


FAMILIES = {
    "kappa1e1": lambda n, rng: spd_kappa(n, 1e1, rng),
    "kappa1e6": lambda n, rng: spd_kappa(n, 1e6, rng),
    "kappa1e10": lambda n, rng: spd_kappa(n, 1e10, rng),
    "kappa1e14": lambda n, rng: spd_kappa(n, 1e14, rng),
    "scaled": scaled,
    "arrowhead": arrowhead,
    "blockdiag": blockdiag,
    "identity": lambda n, rng: np.eye(n),
}


def _system(n, family, seed):
    rng = np.random.default_rng([n, seed, sorted(FAMILIES).index(family) if family in FAMILIES else 99])
    S = FAMILIES[family](n, rng) if family in FAMILIES else family(n, rng)
    b = S @ rng.standard_normal(n)            # a solution of ordinary size, whatever the scaling
    return S, b


def _with_upper_garbage(S):
    """only the lower triangle may be read: poison the strict upper one"""
    G = S.copy()
    G[np.triu_indices(len(S), 1)] = np.nan
    return G


# ------------------------------------------------------------------------------------------------ references
assert np.finfo(np.longdouble).eps < 1e-18, "long double must be the x87 80-bit type for the residuals"


def residual_ld(S, b, x):
    """b - S x in long double, in row blocks (S is symmetric: use the full matrix)"""
    xl = x.astype(np.longdouble)
    r = np.empty(len(b), np.longdouble)
    for i in range(0, len(b), 512):
        r[i:i + 512] = b[i:i + 512].astype(np.longdouble) - S[i:i + 512].astype(np.longdouble) @ xl
    return r


def backward_error(S, b, x):
    r = residual_ld(S, b, x)
    den = np.abs(S).sum(1).max() * np.abs(x).max() + np.abs(b).max()
    return float(np.abs(r).max() / den) if den > 0 else float(np.abs(r).max())


def _kappa_est(S, cf):
    """2-norm condition number: 30 power steps on S and on S^-1 (LAPACK factor)"""
    rng = np.random.default_rng(0)
    v = rng.standard_normal(len(S)); w = v.copy()
    lmax = lmin_inv = 0.0
    for _ in range(30):
        v = S @ v; lmax = np.linalg.norm(v); v /= lmax
        w = sla.cho_solve(cf, w, check_finite=False); lmin_inv = np.linalg.norm(w); w /= lmin_inv
    return lmax * lmin_inv


def reference(S, b):
    """LAPACK (potrf/potrs) + two steps of iterative refinement with long-double residuals"""
    cf = sla.cho_factor(S, lower=True, check_finite=False)
    x0 = sla.cho_solve(cf, b, check_finite=False)
    x = x0.copy()
    for _ in range(2):
        x = x + sla.cho_solve(cf, residual_ld(S, b, x).astype(np.float64), check_finite=False)
    n = len(b)
    ref = dict(x=x, cf=cf, bw_lapack=backward_error(S, b, x0), fw_lapack=_fw(x0, x), kappa=_kappa_est(S, cf))
    if n <= 64:
        import mpmath
        with mpmath.workdps(50):
            xm = mpmath.lu_solve(mpmath.matrix(S.tolist()), mpmath.matrix(b.tolist()))
            xm = [xm[i] for i in range(n)]
            err = float(max(abs(mpmath.mpf(float(x[i])) - xm[i]) for i in range(n)) / max(abs(v) for v in xm))
        xm_f = np.array([float(v) for v in xm])
        # the refined solution is u-accurate, or at least 100x more accurate than the unrefined one
        assert float(err) <= max(16 * U, 1e-2 * _fw(x0, xm_f)), ("refined reference off mpmath", float(err), _fw(x0, xm_f))
    return ref


def _fw(x, xref):
    return float(np.abs(x - xref).max() / np.abs(xref).max())


def _worst_tile(factor, S, b, cf):
    """the 32x32 tile of [L; y^T] furthest from LAPACK's, relative to the largest entry of L in that tile column"""
    n = len(b)
    L = np.tril(cf[0])
    y = sla.solve_triangular(L, b, lower=True)
    got = np.vstack([np.tril(factor[:n]), factor[n:n + 1]])
    want = np.vstack([L, y[None, :]])
    nb = -(-n // TB)
    worst = (0.0, None)
    for j in range(nb):
        scale = np.abs(want[j * TB:, j * TB:(j + 1) * TB]).max() or 1.0
        for i in range(j, nb + 1):
            r0, r1 = (i * TB, min((i + 1) * TB, n)) if i < nb else (n, n + 1)
            d = np.abs(got[r0:r1, j * TB:(j + 1) * TB] - want[r0:r1, j * TB:(j + 1) * TB]).max() / scale
            if not d <= worst[0]:
                worst = (d, (i, j))
    return "worst tile (row tile, column tile) %s of %d (row tile %d = rhs row): relative error %.3g" % (worst[1], nb, nb, worst[0])


def check_chol(path, S, b, got, ref, what=""):
    """-> None, or a message naming the path, the errors and the worst factor tile"""
    n = len(b)
    x = got["x"]
    bw_bound = max(8 * ref["bw_lapack"], 4 * U * np.sqrt(n))
    fw_bound = max(8 * ref["fw_lapack"], U * np.sqrt(n) * ref["kappa"], 4 * U * np.sqrt(n))
    msg = None
    if got["status"] != _capi.REDUCED_SOLVE_OK:
        msg = "status %d" % got["status"]
    elif not np.all(np.isfinite(x)):
        msg = "non-finite solution"
    else:
        bw, fw = backward_error(S, b, x), _fw(x, ref["x"])
        if not (bw <= bw_bound and fw <= fw_bound):
            msg = "backward error %.3g (bound %.3g, LAPACK %.3g), forward error %.3g (bound %.3g, LAPACK %.3g)" % (
                bw, bw_bound, ref["bw_lapack"], fw, fw_bound, ref["fw_lapack"])
    if msg and "factor" in got:
        msg += "; " + _worst_tile(got["factor"], S, b, ref["cf"])
    return None if msg is None else "%s n=%d %s: %s" % (path, n, what, msg)


def _run_all_paths(S, b, nc=None, prob=None, what="", upper_garbage=True):
    ref = reference(S, b)
    Sin = _with_upper_garbage(S) if upper_garbage else S
    errs = []
    for path in PATHS:
        h, _ = _handle(path, nc=nc, prob=prob)
        got = _solve(path, h, Sin, b, factor=True)
        e = check_chol(path, S, b, got, ref, what)
        if e:
            errs.append(e)
    assert not errs, "\n".join(errs)


# ------------------------------------------------------------------------------------------------ Cholesky: sizes x families
TILE_EDGES = [1, 2, 5, 6, 8, 31, 32, 33, 63, 64, 65, 95, 96, 97, 255, 256, 257]


@pytest.mark.parametrize("family", sorted(FAMILIES))
@pytest.mark.parametrize("n", TILE_EDGES)
def test_cholesky_tile_edges(n, family):
    S, b = _system(n, family, 0)
    _run_all_paths(S, b, nc=n, what=family)


@pytest.mark.parametrize("family", ["kappa1e6", "kappa1e14", "scaled"])
@pytest.mark.parametrize("n", [700, 2048, 4095, 4096, 4097])
def test_cholesky_many_tiles_per_cta(n, family):
    S, b = _system(n, family, 1)
    _run_all_paths(S, b, nc=n, what=family)


@pytest.mark.parametrize("n,prob", [(6000, "poses"), (8192, None), (8193, None), (9000, "intrinsics")])
def test_cholesky_exact_solve_ceiling(n, prob):
    """1000 pose-only images, 1000 images with per-image intrinsics, and the tile counts around 8192"""
    p = {"poses": lambda: _problem_images(1000, 0), "intrinsics": lambda: _problem_images(1000, 3), None: lambda: None}[prob]()
    S, b = _system(n, "kappa1e10", 2)
    _run_all_paths(S, b, nc=n, prob=p, what="kappa1e10")


def _ba_scene(shared_camera, constant_blocks, seed=0, n_images=1000):
    g = synthetic.make_geometry(n_images, 4 * n_images, 6, seed=seed, shared_camera=shared_camera)
    ncam = len(g["cam_params"])
    xy = np.empty((len(g["obs_pt"]), 2))
    for i in range(n_images):
        sel = np.flatnonzero(g["obs_img"] == i)
        xy[sel] = synthetic.project_simple_radial(g["cam_params"][g["img_cam"][i]], g["qvec"][i], g["tvec"][i], g["xyz"][g["obs_pt"][sel]])
    rng = g["rng"]
    xy += rng.normal(0, 0.5, xy.shape)
    pose_const = np.zeros(n_images, np.uint8); pose_const[0] = 1
    tmask = np.zeros(n_images, np.uint8); tmask[1] = 1
    cmask = np.full(ncam, 0b0110, np.uint32)                 # focal length and radial distortion free
    if constant_blocks:
        pose_const[rng.choice(n_images, n_images // 10, replace=False)] = 1
        tmask[rng.choice(n_images, n_images // 10, replace=False)] = 5
        cmask[rng.choice(ncam, max(ncam // 3, 1), replace=False)] = 0b1111
    return _capi.BAProblem(np.full(ncam, SIMPLE_RADIAL, np.int32), g["cam_params"], cmask, g["qvec"], g["tvec"], g["img_cam"],
                           pose_const, tmask, g["xyz"], np.zeros(len(g["xyz"]), np.uint8), g["obs_img"], g["obs_pt"],
                           None, None, None, obs_xy=xy)


@pytest.mark.parametrize("scene", ["per_image_cameras", "shared_camera", "constant_blocks"])
def test_cholesky_on_assembled_ba_systems(scene):
    """S / rhs as debug_linearize assembles them on 1000-image geometric scenes, fed back through every path"""
    prob = _ba_scene(shared_camera=scene == "shared_camera", constant_blocks=scene == "constant_blocks")
    nc, nl = O.ba_layout(prob)[:2]
    so = _capi.default_ba_options(use_inner_iterations=0, linear_solver=1)
    lin = _engine.BAHandle(prob, options=so).debug_linearize(nc, nl, radius=1e4)
    S = np.tril(lin["S"]) + np.tril(lin["S"], -1).T
    _run_all_paths(S, lin["rhs"].copy(), prob=prob, what=scene)


# ------------------------------------------------------------------------------------------------ Cholesky: failure and recovery
def _indefinite_at(n, col, rng):
    """SPD up to column col, whose pivot is then -1: S[col, col] set to its Schur complement minus 1"""
    S = spd_kappa(n, 10.0, rng)
    if col > 0:
        s = S[:col, col]
        S[col, col] = s @ np.linalg.solve(S[:col, :col], s) - 1.0
    else:
        S[0, 0] = -1.0
    return S


FAILURES = {
    "pivot_tile0": lambda n, rng: _indefinite_at(n, 5, rng),
    "pivot_col31": lambda n, rng: _indefinite_at(n, 31, rng),
    "pivot_col32": lambda n, rng: _indefinite_at(n, 32, rng),
    "pivot_middle_tile": lambda n, rng: _indefinite_at(n, 70, rng),
    "pivot_ragged_last_tile": lambda n, rng: _indefinite_at(n, n - 3, rng),
    "nan_offdiagonal": lambda n, rng: _poke(spd_kappa(n, 10.0, rng), (77, 40), np.nan),
    "inf_offdiagonal": lambda n, rng: _poke(spd_kappa(n, 10.0, rng), (120, 3), np.inf),
    "zero_matrix": lambda n, rng: np.zeros((n, n)),
}


def _poke(S, ij, v):
    S[ij] = v
    return S


@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("case", sorted(FAILURES))
def test_cholesky_failure_then_recovery(case, path):
    n = 150                                      # tiles 0..4, the last one ragged (22 columns)
    rng = np.random.default_rng(sorted(FAILURES).index(case))
    S = FAILURES[case](n, rng)
    b = rng.standard_normal(n)
    h, _ = _handle(path, nc=n)
    got = _solve(path, h, S, b)
    assert got["status"] == _capi.REDUCED_SOLVE_FAILED, "%s: status %d (1 = numerical failure, 2 = bail-out)" % (case, got["status"])
    S2, b2 = _system(n, "kappa1e6", 5)
    got2 = _solve(path, h, S2, b2, factor=True)
    e = check_chol(path, S2, b2, got2, reference(S2, b2), "after " + case)
    assert e is None, e


# ------------------------------------------------------------------------------------------------ Cholesky: replay and determinism
@pytest.mark.parametrize("path", sorted(PATHS))
@pytest.mark.parametrize("n", [97, 1000])
def test_cholesky_replay_and_determinism(path, n):
    """three matrices in turn on one fresh handle, then the first again: all accurate; the tile-DAG and per-panel paths
    repeat bit for bit, the band path (whose band tiles count commuting updates) is only reported"""
    h, _ = _handle(path, prob=_problem_nc(n), fresh=True)
    systems = [_system(n, f, 7) for f in ("kappa1e10", "scaled", "arrowhead")]
    first = None
    errs = []
    for k, (S, b) in enumerate(systems + systems[:1]):
        got = _solve(path, h, S, b, factor=True)
        e = check_chol(path, S, b, got, reference(S, b), "replay %d" % k)
        if e:
            errs.append(e)
        if k == 0:
            first = got
    assert not errs, "\n".join(errs)
    same = np.array_equal(first["x"].view(np.uint64), got["x"].view(np.uint64)) and \
        np.array_equal(np.nan_to_num(first["factor"]).view(np.uint64), np.nan_to_num(got["factor"]).view(np.uint64))
    if path == "band":
        print("band path n=%d: repeat bit-identical: %s" % (n, same))
    else:
        assert same, "%s: the repeated solve of the same matrix is not bit-identical" % path


# ------------------------------------------------------------------------------------------------ dense PCG
# CG's iteration count and iterate depend on rounding once it has run long enough to lose orthogonality, so a count and
# an x that must match the oracle's exactly need systems where that has not happened: the capped runs stop after at
# most 11 iterations on a slow spectrum (hi = 2: tens of iterations to converge, condition numbers 1e3 .. 1e5), the
# uncapped ones converge in a few to ~20 on a faster one (hi = 1, condition number below 1e3)
ITERS = [1, 7, 8, 9, 10, 11, 200]


def _pcg_case(path, n, kappa, max_iter, seed=0, prob=None):
    prob = prob if prob is not None else _problem_nc(n)
    nc, off, dim = _blocks(prob)
    assert nc == n
    h, _ = _handle(path, prob=prob, cg=True, max_iter=max_iter)
    rng = np.random.default_rng([n, seed, int(np.log10(kappa))])
    S = lowrank(n, kappa, rng, hi=2.0 if max_iter <= 11 else 1.0)
    b = rng.standard_normal(n)
    return h, S, b, off, dim


def _check_pcg(got, ref, what):
    x_ref, it_ref, stop_ref, ok_ref = ref
    assert ok_ref, "oracle failed"
    assert got["status"] == _capi.REDUCED_SOLVE_OK, what
    assert got["linear_iterations"] == it_ref, "%s: %d iterations, oracle %d (stop %d)" % (what, got["linear_iterations"], it_ref, stop_ref)
    err = np.abs(got["x"] - x_ref).max() / np.abs(x_ref).max()
    assert err <= 1e-9, "%s: x differs from the oracle by %.3g relative" % (what, err)


@pytest.mark.parametrize("kappa,max_iter", [(k, m) for m in ITERS[:-1] for k in (1e2, 1e4)] + [(1e2, ITERS[-1])])
@pytest.mark.parametrize("path,n", [("cg", 97), ("cg", 4095), ("cg_multi", 61), ("cg_multi", 97), ("cg", 4096)])
def test_pcg_against_oracle(path, n, kappa, max_iter):
    """single-CTA vector kernels below 4096 unknowns, multi-CTA ones from 4096 (and under PXR_CG_MULTI); the caps around
    the host's poll every 8 iterations and the residual refresh every 10; repeats bit-identical"""
    h, S, b, off, dim = _pcg_case(path, n, kappa, max_iter)
    ref = O.schur_jacobi_pcg(S, b, off, dim, max_iter)
    what = "%s n=%d kappa=%g max_iter=%d" % (path, n, kappa, max_iter)
    got = _solve(path, h, _with_upper_garbage(S), b)
    _check_pcg(got, ref, what)
    again = _solve(path, h, _with_upper_garbage(S), b)
    assert np.array_equal(again["x"].view(np.uint64), got["x"].view(np.uint64)) and again["linear_iterations"] == got["linear_iterations"], what


@pytest.mark.parametrize("max_iter", [10, 200])
@pytest.mark.parametrize("n", [4097, 9000])
def test_pcg_multi_cta_at_default_sizes(n, max_iter):
    prob = _problem_images(1000, 3) if n == 9000 else None
    h, S, b, off, dim = _pcg_case("cg", n, 1e4 if max_iter <= 11 else 1e2, max_iter, prob=prob)
    _check_pcg(_solve("cg", h, S, b), O.schur_jacobi_pcg(S, b, off, dim, max_iter), "cg n=%d max_iter=%d" % (n, max_iter))


@pytest.mark.parametrize("path,n", [("cg", 97), ("cg", 4096)])
def test_pcg_zero_rhs(path, n):
    h, S, _, _, _ = _pcg_case(path, n, 1e2, 200)
    got = _solve(path, h, S, np.zeros(n))
    assert got["status"] == _capi.REDUCED_SOLVE_OK and got["linear_iterations"] == 0
    assert np.array_equal(got["x"], np.zeros(n))


def _indefinite_for_cg(n, off, dim):
    """symmetric indefinite with positive-definite diagonal blocks, and a b for which the oracle's CG meets p.q <= 0
    after at least one step"""
    for seed in range(200):
        rng = np.random.default_rng(seed)
        S = lowrank(n, 1e2, rng)
        for o, d in zip(off, dim):
            S[o:o + d, o + d:] *= 4.0
            S[o + d:, o:o + d] *= 4.0
        b = rng.standard_normal(n)
        x, it, stop, ok = O.schur_jacobi_pcg(S, b, off, dim, 200)
        if ok and stop == O.PCG_STOP_NONPOSITIVE_CURVATURE and it >= 2:
            assert np.linalg.eigvalsh(S)[0] < 0
            return S, b, (x, it, stop, ok)
    raise AssertionError("no indefinite test system found")


@pytest.mark.parametrize("path,n", [("cg", 97), ("cg_multi", 97)])
def test_pcg_stops_on_nonpositive_curvature(path, n):
    prob = _problem_nc(n)
    _, off, dim = _blocks(prob)
    S, b, ref = _indefinite_for_cg(n, off, dim)
    h, _ = _handle(path, prob=prob, cg=True)
    got = _solve(path, h, S, b)
    assert got["status"] == _capi.REDUCED_SOLVE_OK, "p.q <= 0 keeps x and is not a failure"
    assert got["linear_iterations"] == ref[1]
    np.testing.assert_allclose(got["x"], ref[0], rtol=0, atol=1e-9 * np.abs(ref[0]).max())


@pytest.mark.parametrize("path,n", [("cg", 97), ("cg_multi", 97), ("cg", 4096)])
def test_pcg_failed_preconditioner_then_recovery(path, n):
    """a diagonal block that is not positive definite, on a fresh handle: failure before any CG iteration (ceres'
    LINEAR_SOLVER_FAILURE, the oracle's false); the next solve on the handle is right"""
    prob = _problem_nc(n)
    _, off, dim = _blocks(prob)
    h, _ = _handle(path, prob=prob, cg=True, fresh=True)
    rng = np.random.default_rng(3)
    S = lowrank(n, 1e2, rng)
    k = len(off) // 2
    S[off[k] + 1, off[k] + 1] = -1.0
    b = rng.standard_normal(n)
    assert not O.schur_jacobi_pcg(S, b, off, dim, 200)[3]
    got = _solve(path, h, S, b)
    assert got["status"] == _capi.REDUCED_SOLVE_FAILED and got["linear_iterations"] == 0
    S2 = lowrank(n, 1e2, rng, hi=1.0)
    _check_pcg(_solve(path, h, S2, b), O.schur_jacobi_pcg(S2, b, off, dim, 200), "after the failed preconditioner")


def test_block_sparse_and_block_mode_handles_are_refused():
    prob = _problem_nc(12)
    so = _capi.default_ba_options(use_inner_iterations=0, deterministic=1)
    h = _engine.BAHandle(prob, options=so)
    with pytest.raises(ValueError):
        h.debug_reduced_solve(np.eye(12), np.ones(12))
