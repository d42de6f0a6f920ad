"""Extended-precision reference for the normal equations of feature-metric bundle adjustment, and the query scenes
the batched query refinement (csrc/pxr_qba.cu) is checked on.

The reference takes every residual block's residual and ambient Jacobian from the oracle's forward-mode Jets
(oracle_lib.ba_block_jacobians: q4 | t3 | X3 | cam), maps them to the tangent columns the solvers use (3 rotation
columns through ceres' QuaternionManifold PlusJacobian, the free translation components, the free intrinsics in
parameter order, the free points) and accumulates in long double:
  H = sum rho' J^T J,   g = sum rho' J^T r,   cost = 1/2 sum rho,
  A = sum |rho'| |J|^T |J|,   a = sum |rho'| |J|^T |r|      (error scales: what the same sums of absolute values give)
For every supported loss rho'' <= 0, so ceres' corrector reduces to sqrt(rho') (pxr_device.cuh loss_eval) and the
loss enters only through rho'."""
import ctypes as C

import numpy as np

import oracle_lib as O
from pixsfm import features
from pixsfm._pixsfm import _capi
from pixsfm._pixsfm._features import kDenseId
from pixsfm.util import synthetic

LD = np.longdouble

# elementwise bound of a linearisation against the reference: |H - H_ref| <= KAPPA * A and |g - g_ref| <= KAPPA * a.
# The per-block records (||r||^2, G^T r, G^T G) the kernels accumulate agree with the oracle's to 1e-12 .. 1e-10 of
# their scale and the projections to 1e-9 of theirs (test_gpu_full_size), and H / g are sums of products of those
# with the projection Jacobian, each term bounded by the corresponding term of A / a.  1e-9 leaves an order of
# magnitude over the record-level agreement; a wrong, missing or swapped column is off by O(1) of its scaled entries.
KAPPA = 1e-9

MODEL_NAMES = {0: "SIMPLE_PINHOLE", 1: "PINHOLE", 2: "SIMPLE_RADIAL", 3: "RADIAL", 4: "OPENCV", 5: "OPENCV_FISHEYE",
               6: "FULL_OPENCV"}
MODEL_PARAMS = {
    0: [1200.0, 500.0, 500.0],
    1: [1200.0, 1190.0, 500.0, 502.0],
    2: [1200.0, 500.0, 500.0, 0.02],
    3: [1200.0, 500.0, 500.0, 0.02, -0.01],
    4: [1200.0, 1195.0, 500.0, 501.0, 0.02, -0.01, 1e-3, -2e-3],
    5: [1200.0, 1195.0, 500.0, 501.0, 0.01, -0.005, 0.002, -0.001],
    6: [1200.0, 1195.0, 500.0, 501.0, 0.02, -0.01, 1e-3, -2e-3, 0.003, 0.01, -0.004, 0.002],
}
INTRINSIC_SETS = ("pose", "focal", "pp", "extra", "all")
LOSSES = {"trivial": (0, 1.0), "cauchy": (1, 0.25), "huber": (2, 0.1), "soft_l1": (3, 0.1), "arctan": (4, 0.1)}


def const_mask(model, iset):
    """cam_const_mask of QueryBundleOptimizer's refine_* flags: `iset` names the free intrinsic group"""
    focal, pp, extra = _capi.CAMERA_PARAM_GROUPS[model]
    return {"pose": 0xFFFFFFFF, "focal": pp | extra, "pp": focal | extra, "extra": focal | pp, "all": 0}[iset]


def free_params(model, mask):
    return [k for k in range(_capi.CAMERA_NUM_PARAMS[model]) if not (mask >> k) & 1]


def plus_jacobian(q):
    """d QuaternionPlus(q, d) / d d at d = 0 (ceres QuaternionManifold::PlusJacobian, w first), [4, 3]"""
    w, x, y, z = q
    return np.array([[-x, -y, -z], [w, z, -y], [-z, w, x], [y, -x, w]])


def quaternion_plus(q, d):
    """QuaternionPlus in long double"""
    q = np.asarray(q, LD); d = np.asarray(d, LD)
    nd = np.sqrt((d * d).sum())
    if nd == 0:
        return q.copy()
    s = np.sin(nd) / nd
    z = np.array([np.cos(nd), s * d[0], s * d[1], s * d[2]], LD)
    return np.array([z[0] * q[0] - z[1] * q[1] - z[2] * q[2] - z[3] * q[3],
                     z[0] * q[1] + z[1] * q[0] + z[2] * q[3] - z[3] * q[2],
                     z[0] * q[2] - z[1] * q[3] + z[2] * q[0] + z[3] * q[1],
                     z[0] * q[3] + z[1] * q[2] - z[2] * q[1] + z[3] * q[0]], LD)


def loss(loss_type, scale, s):
    """(rho, rho', rho'') of the oracle's loss at the squared norm s"""
    rho = np.zeros(3)
    O.lib().orc_loss(C.c_int(int(loss_type)), C.c_double(scale), C.c_double(1.0), C.c_double(float(s)), O.p(rho))
    return rho


def query_problem(batch, k):
    """query k of a QBABatch as the per-query BAProblem QueryBundleOptimizer.build_problem makes: one image, constant
    points, the batch's refs, obs_patch, corner and scale"""
    b0, b1 = int(batch.obs_begin[k]), int(batch.obs_begin[k + 1])
    p0 = int(np.sum(batch.patch_counts[:k]))
    n = int(batch.patch_counts[k])
    m = b1 - b0
    return _capi.BAProblem(cam_model=[batch.cam_model[k]], cam_params=batch.cam_params[k:k + 1],
                           cam_const_mask=[batch.cam_const_mask[k]], qvec=batch.qvec[k:k + 1], tvec=batch.tvec[k:k + 1],
                           img_cam=[0], pose_const=[0], tvec_const_mask=[0], xyz=batch.xyz[b0:b1],
                           point_const=np.ones(m, np.uint8), obs_img=np.zeros(m, np.int32),
                           obs_pt=np.arange(m, dtype=np.int64), patches=np.ascontiguousarray(batch.patch_blocks[k]),
                           corner=batch.corner[p0:p0 + n], scale=batch.scale[p0:p0 + n], refs=batch.refs[b0:b1],
                           obs_patch=batch.obs_patch[b0:b1])


def normal_equations(prob, interp, loss_type, loss_scale):
    """the long-double reference of prob's linearisation over all of its local columns (cameras first, in
    oracle_lib.ba_layout's order, then the free points) -> dict(H, g, A, a [long double], cost, nc, nl)"""
    nc, nl, pose_off, intr_off, point_off = O.ba_layout(prob)
    r, J = O.ba_block_jacobians(prob, interp)
    nb = prob.n_obs
    dmax = 6 + 12 + 3
    Jl = np.zeros((nb, r.shape[1], dmax), LD)
    cols = np.full((nb, dmax), -1, np.int64)
    for o in range(nb):
        img, pt = int(prob.obs_img[o]), int(prob.obs_pt[o])
        cam = int(prob.img_cam[img])
        c = 0
        if pose_off[img] >= 0:
            Jl[o, :, 0:3] = np.asarray(J[o, :, 0:4], LD) @ np.asarray(plus_jacobian(prob.qvec[img]), LD)
            cols[o, 0:3] = pose_off[img] + np.arange(3)
            c = 3
            tfree = [a for a in range(3) if not (int(prob.tvec_const_mask[img]) >> a) & 1]
            for j, a in enumerate(tfree):
                Jl[o, :, c] = J[o, :, 4 + a]; cols[o, c] = pose_off[img] + 3 + j; c += 1
        if intr_off[cam] >= 0:
            for j, k in enumerate(free_params(int(prob.cam_model[cam]), int(prob.cam_const_mask[cam]))):
                Jl[o, :, c] = J[o, :, 10 + k]; cols[o, c] = intr_off[cam] + j; c += 1
        if point_off[pt] >= 0:
            Jl[o, :, c:c + 3] = J[o, :, 7:10]; cols[o, c:c + 3] = point_off[pt] + np.arange(3)
    rl = np.asarray(r, LD)
    s = (rl * rl).sum(1)
    rho = np.array([loss(loss_type, loss_scale, x) for x in s])
    w = np.asarray(rho[:, 1], LD)
    Jt = Jl.transpose(0, 2, 1)
    M = np.matmul(Jt, Jl) * w[:, None, None]
    Ma = np.matmul(np.abs(Jt), np.abs(Jl)) * np.abs(w)[:, None, None]
    v = np.matmul(Jt, rl[:, :, None])[:, :, 0] * w[:, None]
    va = np.matmul(np.abs(Jt), np.abs(rl)[:, :, None])[:, :, 0] * np.abs(w)[:, None]
    H = np.zeros((nl, nl), LD); A = np.zeros((nl, nl), LD); g = np.zeros(nl, LD); a = np.zeros(nl, LD)
    ok = cols >= 0
    bi, ci = np.nonzero(ok)
    np.add.at(g, cols[bi, ci], v[bi, ci]); np.add.at(a, cols[bi, ci], va[bi, ci])
    pair = ok[:, :, None] & ok[:, None, :]
    bb, ii, jj = np.nonzero(pair)
    np.add.at(H, (cols[bb, ii], cols[bb, jj]), M[bb, ii, jj])
    np.add.at(A, (cols[bb, ii], cols[bb, jj]), Ma[bb, ii, jj])
    cost = (np.asarray(rho[:, 0], LD) * LD(0.5)).sum()
    return dict(H=H, g=g, A=A, a=a, cost=cost, nc=nc, nl=nl, residuals=r)


def scaled_error(got, ref, key="H"):
    """Jacobi-scaled comparison with S = diag(H_ref)^-1/2: max over entries of |S (got - ref) S| / (S A S) (for g:
    |S (got - ref)| / (S a)); entries whose error scale is zero must agree exactly"""
    d = np.sqrt(np.asarray(np.diag(ref["H"]), np.float64))
    S = np.where(d > 0, 1.0 / np.where(d > 0, d, 1.0), 1.0)
    if key == "H":
        n = got.shape[0]
        diff = (np.asarray(got, LD) - ref["H"][:n, :n]) * np.outer(S[:n], S[:n])
        scale = ref["A"][:n, :n] * np.outer(S[:n], S[:n])
    else:
        n = len(got)
        diff = (np.asarray(got, LD) - ref["g"][:n]) * S[:n]
        scale = ref["a"][:n] * S[:n]
    diff = np.abs(np.asarray(diff, np.float64)); scale = np.asarray(scale, np.float64)
    if np.any(diff[scale == 0] != 0):
        return np.inf
    return float(np.max(np.where(scale > 0, diff / np.where(scale > 0, scale, 1.0), 0.0)))


def _cholesky_solve(M, b):
    n = len(b)
    L = np.zeros((n, n), LD)
    for j in range(n):
        djj = M[j, j] - (L[j, :j] ** 2).sum()
        if not djj > 0:
            return None
        L[j, j] = np.sqrt(djj)
        for i in range(j + 1, n):
            L[i, j] = (M[i, j] - (L[i, :j] * L[j, :j]).sum()) / L[j, j]
    y = np.zeros(n, LD)
    for i in range(n):
        y[i] = (b[i] - (L[i, :i] * y[:i]).sum()) / L[i, i]
    x = np.zeros(n, LD)
    for i in range(n - 1, -1, -1):
        x[i] = (y[i] - (L[i + 1:, i] * x[i + 1:]).sum()) / L[i, i]
    return x


def first_step(ref, n, qvec, tvec, cam_params, model, mask, so):
    """iteration 1 of the LM loop in long double: Jacobi scaling from this linearisation, the LM damping at
    initial_trust_region_radius (pxr_lm.cuh jacobi_scale / lm_damping), the exact solve, Plus -> dict(step_norm,
    delta, cond: condition number of the scaled damped system)"""
    H = ref["H"][:n, :n]; g = ref["g"][:n]
    diag = np.diag(H)
    s = LD(1) / (LD(1) + np.sqrt(diag)) if so.jacobi_scaling else np.ones(n, LD)
    s2 = s * s
    D = np.minimum(np.maximum(diag * s2, LD(so.min_lm_diagonal)), LD(so.max_lm_diagonal)) / (LD(so.initial_trust_region_radius) * s2)
    M = H + np.diag(D)
    d = _cholesky_solve(M, -g)
    Ms = np.asarray(M * np.outer(s, s), np.float64)
    out = dict(cond=float(np.linalg.cond(Ms)), delta=d, step_norm=None)
    if d is None:
        return out
    qn = quaternion_plus(qvec, d[:3])
    dn = ((qn - np.asarray(qvec, LD)) ** 2).sum() + (d[3:6] ** 2).sum() + (d[6:n] ** 2).sum()
    out["step_norm"] = float(np.sqrt(dn))
    return out


# ---- query scenes -------------------------------------------------------------------------------------------------
_SCENES = {}


def _base_scene(n_points, channels, dtype, ps, seed, refs_per_point=1):
    """one image of a two-camera synthetic scene (synthetic.make_ba_scene, the scene recon_util.make_reconstruction
    wraps) seen as a query: its pose, the true 3D points, its observations' patches and the oracle's IRLS reference
    descriptors of the two-view tracks (refs_per_point > 1: the reference and perturbed copies of it, one residual
    block each)"""
    key = (n_points, channels, np.dtype(dtype).name, ps, seed, refs_per_point)
    if key not in _SCENES:
        prob, gt = synthetic.make_ba_scene(n_cams=2, n_points=n_points, track_len=2, channels=channels, ps=ps, seed=seed,
                                           dtype=dtype)
        refs, _ = O.refs_compute(prob, _capi.default_interp())
        sel = np.nonzero(prob.obs_img == 0)[0]
        pts = prob.obs_pt[sel]
        rng = np.random.default_rng(seed + 17)
        r = []
        for p in pts:
            rr = [refs[p]] + [refs[p] * (1.0 - 0.02 * j) + rng.normal(0, 0.01, channels) for j in range(1, refs_per_point)]
            r.append(rr if refs_per_point > 1 else refs[p])
        _SCENES[key] = dict(qvec=prob.qvec[0].copy(), tvec=prob.tvec[0].copy(), xyz=gt["xyz"][pts].copy(),
                            patches=np.ascontiguousarray(prob.patches[sel]), corners=prob.corner[sel].copy(),
                            scale=prob.scale[sel[0]].copy(), refs=r, xy=gt["xy_true"][sel].copy())
    return _SCENES[key]


def make_query(blocks, model=6, iset="all", channels=128, dtype=np.float16, ps=16, seed=0, kind="sparse",
               refs_per_point=1):
    """one query of QueryBundleOptimizer.pack_batch's argument form with exactly `blocks` residual blocks ->
    (query tuple, cam_const_mask).  kind:
      sparse  one patch per correspondence (the usual sparse query map)
      dense   one large non-square patch read by every block (obs_patch all 0)
      border  8x8 patches placed so that the projections sit at and beyond their border (the tap window clamps)
      axis    points within 1e-7 of the optical axis (for OPENCV_FISHEYE's theta / r at r -> 0)"""
    npts = -(-blocks // refs_per_point)
    sc = _base_scene(npts, channels, dtype, 8 if kind == "border" else ps, seed, refs_per_point)
    qvec, tvec = sc["qvec"].copy(), sc["tvec"].copy()
    xyz = [x.copy() for x in sc["xyz"]]
    refs = list(sc["refs"])
    patches, corners, scale = sc["patches"], sc["corners"].copy(), sc["scale"]
    if kind == "border":       # shift the patches: the projection sits before, on or past the first / last row and column
        t = np.array([-3, 0, 7, 9])
        i = np.arange(npts)
        off = np.stack([t[i % 4], t[(i // 4) % 4]], 1)
        corners = (np.floor(sc["xy"] * scale).astype(np.int64) - off).astype(np.int32)
    if kind == "axis":         # move the points onto the optical axis: camera-frame x, y of 1e-8 .. 1e-7
        R = synthetic.quat_to_R(qvec)
        rng = np.random.default_rng(seed + 5)
        for i, X in enumerate(xyz):
            pc = R @ X + tvec
            pc[:2] = rng.uniform(-1e-7, 1e-7, 2) * pc[2]
            xyz[i] = R.T @ (pc - tvec)
        corners = np.full_like(corners, 500 - ps // 2)
    if kind == "dense":        # one 192 x 256 map of the image at a quarter of its resolution: every block reads it
        dense = smooth_map(192, 256, channels, dtype, seed)[None]
        scale = np.array([0.25, 0.25])
        fmap = features.FeatureMap(dense, [kDenseId], np.zeros((1, 2), np.int32), {"scale": scale, "is_sparse": False})
        idx = [0] * npts
    else:
        fmap = features.FeatureMap(np.ascontiguousarray(patches[:npts]), list(range(npts)), corners[:npts],
                                   {"scale": scale, "is_sparse": True})
        idx = list(range(npts))
    if refs_per_point > 1:     # trim the last point's references so that the query has exactly `blocks` blocks
        extra = npts * refs_per_point - blocks
        refs = refs[:npts]
        if extra:
            refs[-1] = refs[-1][:refs_per_point - extra]
    cam = _camera(model)
    q = (qvec, tvec, cam, xyz[:npts], fmap, refs[:npts], None, idx)
    return q, const_mask(model, iset)


def smooth_map(h, w, channels, dtype, seed):
    """a dense [h, w, C] feature map: per channel a plane wave of a few pixels' wavelength"""
    rng = np.random.default_rng(seed + 9)
    k = rng.uniform(0.2, 0.8, (2, channels)) * rng.choice([-1, 1], (2, channels))
    ph = rng.uniform(0, 2 * np.pi, channels)
    y, x = np.mgrid[0:h, 0:w]
    return np.sin(x[..., None] * k[0] + y[..., None] * k[1] + ph).astype(dtype)


def _camera(model):
    from pixsfm.util import colmap_types as ct
    return ct.Camera(1, MODEL_NAMES[model], 1000, 1000, np.array(MODEL_PARAMS[model], np.float64))


def pack(queries, options=None, interp=None):
    """QueryBundleOptimizer.pack_batch of (query, mask) pairs, each query keeping its own constancy mask"""
    from pixsfm._pixsfm import _localization as loc
    o = loc.QueryBundleOptimizer(options or {"refine_focal_length": True}, interp or {})
    batch = o.pack_batch([q for q, _ in queries])
    for k, (_, m) in enumerate(queries):
        batch.cam_const_mask[k] = m
    return batch, o


def n_columns(batch, k):
    return 6 + len(free_params(int(batch.cam_model[k]), int(batch.cam_const_mask[k])))
