"""Block-sparse long-double reference for one linearisation and LM step of feature-metric bundle adjustment: what
BAHandle.debug_linearize returns (Hcc, gc, Hpp, gp, the damped Schur system S / rhs, delta and the model cost change),
with a componentwise error scale for every output.

Definitions (taken from the code they check)
  Per residual block o with residual r_o, local Jacobian J_o = [Jc_o | Jp_o] (camera columns of the block's image, then
  the point's 3 columns) and loss weight w_o = rho'(|r_o|^2) (every supported loss has rho'' <= 0, so ceres' corrector
  is sqrt(rho'), see query_reference):
    Hcc = sum w Jc^T Jc,  gc = sum w Jc^T r,  Hpp_p = sum w Jp^T Jp,  gp_p = sum w Jp^T r,  W_o = w Jc_o^T Jp_o.
  Tangent columns are mapped as query_reference.normal_equations maps them (QuaternionManifold plus-Jacobian, the free
  tvec components, the free intrinsics in parameter order, oracle_lib.ba_layout's column order).
  LM diagonal (pxr_lm.cuh jacobi_scale / lm_damping, ba_d2_kernel): s = 1 / (1 + sqrt(diag H)) (1 without Jacobi
  scaling), D2 = clamp(diag H s^2, min_lm_diagonal, max_lm_diagonal) / (radius s^2), in unscaled variables.
  Reduced system (ba_init_reduced_kernel, ba_point_inverse_kernel and the pair walk; orc_ba.h SolveDamped), unscaled:
    V_p = Hpp_p + diag(D2_p),   S = Hcc + diag(D2_c) - sum_p sum_{o,o' in p} W_o V_p^-1 W_o'^T,
    rhs = -gc + sum_p sum_{o in p} W_o V_p^-1 gp_p,   S dc = rhs,   dp = -V_p^-1 (gp_p + sum_{o in p} W_o^T dc),
    model cost change = -g^T d - d^T H d / 2  (H undamped; orc_ba.h ModelCostChange).
  Everything is accumulated in np.longdouble and block-sparse: Hcc and S are dense nc x nc, points are 3 x 3 blocks, and
  the pair terms are formed point by point in chunks of points and summed per image pair; the nl x nl matrix is never
  formed.  The camera system is solved by LAPACK in float64 and two steps of iterative refinement with long-double
  residuals (the scheme test_gpu_reduced_solve relies on); the points are back-substituted in long double.

Error scales (first order; |X| is the entrywise absolute value, X_a the matching sum of absolute terms)
  Inputs.  Every sum of terms a linearisation forms is trusted to KAPPA times the same sum of absolute terms, KAPPA =
  query_reference.KAPPA = 1e-9 (derived there from the record-level agreement of the kernels with the oracle):
    |dHcc| <= k Acc,  |dgc| <= k ac,  |dHpp| <= k Hpp_a,  |dgp| <= k gp_a,  |dW| <= k W_a,
  with Acc = sum |w| |Jc|^T |Jc|, ac = sum |w| |Jc|^T |r|_a and so on.  A residual is a difference r = f - ref of the
  interpolated descriptor and the reference, whose errors are relative to |f| and |ref|, not to |r|: the observation a
  point's reference was taken from has r = 0 up to rounding (exactly 0 in one implementation, 1e-13 in another), so
  |r|_a = |f| + |ref| (= |r| for problems without references).  The factored Jacobians J = G^T P of
  BAHandle.evaluate_jacobians (G = d r / d(u, v) [2, C], P [2, cols]) use the upper bound
  |J|^T |J| <= |P|^T (|G| |G|^T) |P| for the sum of absolute terms.
  D2 follows diag H: its relative change is at most that of diag H, so D2 carries the scale D2_a = D2 A_ii / H_ii.
  Inverse.  d(V^-1) = -V^-1 dV V^-1, so |d(V^-1)| <= k |V^-1| V_a |V^-1| with V_a = Hpp_a + diag(D2_a) (this is the
  componentwise form of the cond(V_p) weighting: |V^-1| V_a |V^-1| <= cond(V_p) |V^-1| in the Skeel sense).
  S and rhs.  d(W V^-1 W'^T) = dW V^-1 W'^T + W V^-1 dW'^T + W d(V^-1) W'^T, and |W| <= W_a, so
    E_S   = k (Acc + diag(D2_a,c) + sum_p sum_{o,o'} W_a,o M_p W_a,o'^T),   M_p = 2 |V_p^-1| + |V_p^-1| V_a,p |V_p^-1|
    E_rhs = k (ac + sum_p sum_o W_a,o M_p gp_a,p)                                 (|gp| <= gp_a the same way)
  Camera step.  (S + dS)(x + dx) = rhs + drhs gives |dx| <= |S^-1| (E_S |x| + E_rhs) to first order (Higham, Accuracy
  and Stability of Numerical Algorithms, 2nd ed., ch. 7), with |S^-1| formed explicitly.  The fp64 Cholesky that
  solves S adds its backward error |dS| <= gamma_{3n} |L| |L^T| <= 3 n u sqrt(S_ii S_jj) (Higham Thm 10.4 and the two
  triangular solves, u = 2^-53, Cauchy-Schwarz on the rows of L), which is added to E_S for the step only.
  Points.  dp = -V^-1 v, v = gp + sum W^T dc:  |d dp| <= |V^-1| E_v + k |V^-1| V_a |V^-1| |v|,
    E_v = k (gp_a + sum_o W_a,o^T |dc_o|) + sum_o W_a,o^T |d dc_o|.
  Model cost change.  (H + D) d = -g, so its first-order change is -(g + H d)^T dd - dg^T d - d^T dH d / 2 =
  (D d)^T dd - dg^T d - d^T dH d / 2:  E_mcc = |D d|^T |dd| + k (a^T |d| + |d|^T A |d| / 2).
  The camera bound is made exact rather than first order: with X = |S^-1| E_S and y = |S^-1| (E_S |x| + E_rhs),
  |dx| <= (I - X)^-1 y = sum_k X^k y.  With eta = max_i (X y)_i / y_i, X y <= eta y entrywise, so X^k y <= eta^k y and
  |dx| <= y / (1 - eta); linearize requires eta < 1/2 (IllConditioned otherwise).  The point and cost-change bounds drop
  the products of two perturbations, each at most eta of its term.  Jacobi scaling would multiply an entry's error and
  its scale by the same positive factor, so each comparator's ratio is computed on the unscaled entries directly."""
import numpy as np
import scipy.linalg

import oracle_lib as O
import query_reference as Q
from pixsfm._pixsfm import _capi

LD = np.longdouble
KAPPA = Q.KAPPA
U64 = 2.0 ** -53


# ---- layout --------------------------------------------------------------------------------------------------------
def layout(prob):
    """oracle_lib.ba_layout plus, per image, its camera columns (pose block, then its camera's free intrinsics; the
    index nc pads images with fewer than DC columns) and, per image, the ambient source of each of those columns"""
    nc, nl, pose_off, intr_off, point_off = O.ba_layout(prob)
    n_img = len(prob.img_cam)
    cols, rot, tsrc, csrc = [], np.zeros(n_img, bool), [], []
    for i in range(n_img):
        cam = int(prob.img_cam[i])
        c, ts, ks = [], [], []
        if pose_off[i] >= 0:
            rot[i] = True
            tfree = [a for a in range(3) if not (int(prob.tvec_const_mask[i]) >> a) & 1]
            c += [int(pose_off[i]) + j for j in range(3 + len(tfree))]
            ts = tfree
        if intr_off[cam] >= 0:
            ks = Q.free_params(int(prob.cam_model[cam]), int(prob.cam_const_mask[cam]))
            c += [int(intr_off[cam]) + j for j in range(len(ks))]
        cols.append(c); tsrc.append(ts); csrc.append(ks)
    DC = max(1, max(len(c) for c in cols))
    cols_img = np.full((n_img, DC), nc, np.int64)
    for i, c in enumerate(cols):
        cols_img[i, :len(c)] = c
    order = np.argsort(prob.obs_pt, kind="stable")
    pts = np.asarray(prob.obs_pt)[order]
    npts = len(prob.xyz)
    start = np.searchsorted(pts, np.arange(npts + 1))
    return dict(nc=nc, nl=nl, pose_off=pose_off, intr_off=intr_off, point_off=point_off, DC=DC, cols_img=cols_img,
                rot=rot, tsrc=tsrc, csrc=csrc, order=order, start=start, n_img=n_img, npts=npts)


def _local(lay, img, t_cols, X_cols, cam_cols, src, rot_fn):
    """[n, m, DC + 3] local Jacobian from ambient rows src [n, m, *]: the camera columns of each observation's image,
    then X"""
    n, m = src.shape[0], src.shape[1]
    DC = lay["DC"]
    out = np.zeros((n, m, DC + 3), LD)
    for i in np.unique(img):
        sel = np.nonzero(img == i)[0]
        c = 0
        if lay["rot"][i]:
            out[sel, :, 0:3] = rot_fn(sel, i)
            c = 3
            for a in lay["tsrc"][i]:
                out[sel, :, c] = src[sel, :, t_cols[a]]; c += 1
        for k in lay["csrc"][i]:
            out[sel, :, c] = src[sel, :, cam_cols + k]; c += 1
    out[:, :, DC:] = src[:, :, X_cols:X_cols + 3]
    return out


def _residual_scale(prob, obs, r):
    """error scale |r|_a of residuals r = f - ref: |f| + |ref| (|r| without references), see the module docstring"""
    if prob.refs is None:
        return np.abs(r)
    ref = np.asarray(prob.refs, LD)[np.asarray(prob.obs_pt)[obs]]
    return np.abs(r + ref) + np.abs(ref)


def _weights(s, loss_type, loss_scale):
    rho = np.array([Q.loss(loss_type, loss_scale, x) for x in np.asarray(s, np.float64)]).reshape(-1, 3)
    return rho[:, 0], rho[:, 1]


# ---- per-observation blocks ------------------------------------------------------------------------------------
def oracle_blocks(prob, interp, loss_type, loss_scale):
    """blocks(obs) -> (M, M_a, v, v_a, rho) from the oracle's forward-mode Jets (oracle_lib.ba_block_jacobians):
    M = w J^T J, v = w J^T r over [camera columns | X] and their sums of absolute terms"""
    r, J = O.ba_block_jacobians(prob, interp)
    qv = np.asarray(prob.qvec)

    def blocks(lay, obs):
        img = np.asarray(prob.obs_img)[obs]
        Jo = J[obs]
        rot = lambda sel, i: np.asarray(Jo[sel, :, 0:4], LD) @ np.asarray(Q.plus_jacobian(qv[i]), LD)
        Jl = _local(lay, img, (4, 5, 6), 7, 10, Jo, rot)
        rl = np.asarray(r[obs], LD)
        rho0, w = _weights((rl * rl).sum(1), loss_type, loss_scale)
        w = np.asarray(w, LD)
        Jt = Jl.transpose(0, 2, 1)
        M = np.matmul(Jt, Jl) * w[:, None, None]
        Ma = np.matmul(np.abs(Jt), np.abs(Jl)) * np.abs(w)[:, None, None]
        v = np.matmul(Jt, rl[:, :, None])[:, :, 0] * w[:, None]
        va = np.matmul(np.abs(Jt), _residual_scale(prob, obs, rl)[:, :, None])[:, :, 0] * np.abs(w)[:, None]
        return M, Ma, v, va, rho0
    return blocks


def factored_blocks(prob, jac, loss_type, loss_scale):
    """blocks(obs) from BAHandle.evaluate_jacobians' factored Jacobians J = grad^T P (grad [2, C] = d r / d(u, v),
    P = juv [2, rot3 | t3 | X3 | K] with tangent rotation columns); the sums of absolute terms use the upper bound
    |J|^T |J| <= |P|^T (|G| |G|^T) |P| (and |J|^T |r|_a <= |P|^T |G| |r|_a)"""
    res, grad, juv = jac["residuals"], jac["grad"], jac["juv"]

    def blocks(lay, obs):
        img = np.asarray(prob.obs_img)[obs]
        P = juv[obs]
        Pl = _local(lay, img, (3, 4, 5), 6, 9, P, lambda sel, i: P[sel, :, 0:3])
        g = np.asarray(grad[obs], LD)
        rl = np.asarray(res[obs], LD)
        rho0, w = _weights((rl * rl).sum(1), loss_type, loss_scale)
        w = np.asarray(w, LD)
        G = np.matmul(g, g.transpose(0, 2, 1))
        Ga = np.matmul(np.abs(g), np.abs(g).transpose(0, 2, 1))
        Gr = np.matmul(g, rl[:, :, None])
        Gra = np.matmul(np.abs(g), _residual_scale(prob, obs, rl)[:, :, None])
        Pt = Pl.transpose(0, 2, 1)
        M = np.matmul(Pt, np.matmul(G, Pl)) * w[:, None, None]
        Ma = np.matmul(np.abs(Pt), np.matmul(Ga, np.abs(Pl))) * np.abs(w)[:, None, None]
        v = np.matmul(Pt, Gr)[:, :, 0] * w[:, None]
        va = np.matmul(np.abs(Pt), Gra)[:, :, 0] * np.abs(w)[:, None]
        return M, Ma, v, va, rho0
    return blocks


class IllConditioned(ValueError):
    """the damped S is too ill-conditioned for its error scale to bound the step (eta >= 1/2, see the docstring)"""


RADII = (1e4, 1e3, 1e2, 1e1)


def linearize_at_largest_radius(prob, blocks, so, radii=RADII, **kw):
    """linearize at the first radius of `radii` at which the step's bound holds (a smaller radius damps more and
    conditions S better; the reference's "radius" says which)"""
    for radius in radii:
        try:
            return linearize(prob, blocks, so, radius, **kw)
        except IllConditioned:
            continue
    raise IllConditioned("no radius of %s bounds the step" % (radii,))


# ---- the reference -------------------------------------------------------------------------------------------------
def _damping(diag, so, radius):
    diag = np.asarray(diag, LD)
    s = LD(1) / (LD(1) + np.sqrt(diag)) if so.jacobi_scaling else np.ones_like(diag)
    s2 = s * s
    return np.minimum(np.maximum(diag * s2, LD(so.min_lm_diagonal)), LD(so.max_lm_diagonal)) / (LD(radius) * s2)


def _inv3(V):
    """inverses of symmetric positive definite 3 x 3 blocks [n, 3, 3] in long double (adjugate / determinant)"""
    a, b, c, d, e, f = V[:, 0, 0], V[:, 0, 1], V[:, 0, 2], V[:, 1, 1], V[:, 1, 2], V[:, 2, 2]
    A, B, Cc = d * f - e * e, c * e - b * f, b * e - c * d
    det = a * A + b * B + Cc * c
    assert np.all(a > 0) and np.all(a * d - b * b > 0) and np.all(det > 0), "V_p is not positive definite"
    out = np.stack([A, B, Cc, B, a * f - c * c, b * c - a * e, Cc, b * c - a * e, a * d - b * b], 1).reshape(-1, 3, 3)
    return out / det[:, None, None]


def _scatter_by_key(dst, keys, blocks, rows, cols):
    """dst[rows[k], cols[k]] += sum of blocks with key k (rows / cols [n_keys, *] column lists of each key)"""
    if len(keys) == 0:
        return
    o = np.argsort(keys, kind="stable")
    uk, st = np.unique(keys[o], return_index=True)
    R = np.add.reduceat(blocks[o], st, axis=0)
    if dst.ndim == 2:
        np.add.at(dst, (rows(uk)[:, :, None], cols(uk)[:, None, :]), R)
    else:
        np.add.at(dst, rows(uk), R)


def linearize(prob, blocks, so, radius, chunk_points=2000):
    """the reference of one debug_linearize call -> dict of long-double outputs and float64 error scales (see the
    module docstring).  blocks: oracle_blocks(...) or factored_blocks(...)"""
    lay = layout(prob)
    nc, nl, DC, n_img = lay["nc"], lay["nl"], lay["DC"], lay["n_img"]
    ci = lay["cols_img"]
    point_off = lay["point_off"]
    obs_img = np.asarray(prob.obs_img)
    n_obs, npts = len(obs_img), lay["npts"]
    N = nc + 1
    Hcc = np.zeros((N, N), LD); Acc = np.zeros((N, N), LD); gc = np.zeros(N, LD); ac = np.zeros(N, LD)
    Sp = np.zeros((N, N), LD); ESp = np.zeros((N, N), LD); rp = np.zeros(N, LD); Erp = np.zeros(N, LD)
    Hpp = np.zeros((npts, 3, 3), LD); Hppa = np.zeros((npts, 3, 3), LD); gp = np.zeros((npts, 3), LD)
    gpa = np.zeros((npts, 3), LD)
    Vinv = np.zeros((npts, 3, 3), LD); Q3 = np.zeros((npts, 3, 3), LD); D2p = np.zeros((npts, 3), LD)
    W = np.zeros((n_obs, DC, 3), LD); Wa = np.zeros((n_obs, DC, 3), LD)      # in layout order (sorted by point)
    cost = LD(0)
    order, start = lay["order"], lay["start"]
    img_rows = lambda k: ci[k]
    pair_rows = lambda k: ci[k // n_img]
    pair_cols = lambda k: ci[k % n_img]
    for p0 in range(0, npts, chunk_points):
        p1 = min(npts, p0 + chunk_points)
        o0, o1 = start[p0], start[p1]
        if o1 == o0:
            continue
        obs = order[o0:o1]
        img = obs_img[obs]
        M, Ma, v, va, rho0 = blocks(lay, obs)
        cost += (np.asarray(rho0, LD) * LD(0.5)).sum()
        for dst, src in ((Hcc, M), (Acc, Ma)):
            _scatter_by_key(dst, img, src[:, :DC, :DC], img_rows, img_rows)
        for dst, src in ((gc, v), (ac, va)):
            _scatter_by_key(dst, img, src[:, :DC], img_rows, None)
        W[o0:o1] = M[:, :DC, DC:]; Wa[o0:o1] = Ma[:, :DC, DC:]
        pl = np.repeat(np.arange(p0, p1), np.diff(start[p0:p1 + 1]))      # point of each observation
        seg = start[p0:p1] - o0
        nonempty = np.diff(start[p0:p1 + 1]) > 0
        idx = seg[nonempty]
        pts = np.arange(p0, p1)[nonempty]
        Hpp[pts] = np.add.reduceat(M[:, DC:, DC:], idx, axis=0)
        Hppa[pts] = np.add.reduceat(Ma[:, DC:, DC:], idx, axis=0)
        gp[pts] = np.add.reduceat(v[:, DC:], idx, axis=0); gpa[pts] = np.add.reduceat(va[:, DC:], idx, axis=0)
        var = pts[point_off[pts] >= 0]
        if len(var) == 0:
            continue
        dg = np.diagonal(Hpp[var], axis1=1, axis2=2)
        dga = np.diagonal(Hppa[var], axis1=1, axis2=2)
        D2 = _damping(dg, so, radius)
        D2a = D2 * np.where(dg > 0, dga / np.where(dg > 0, dg, 1), 1)
        D2p[var] = D2
        Vi = _inv3(Hpp[var] + D2[:, :, None] * np.eye(3, dtype=LD))
        Va = Hppa[var] + D2a[:, :, None] * np.eye(3, dtype=LD)
        Vi_a = np.abs(Vi)
        Qv = np.matmul(Vi_a, np.matmul(Va, Vi_a))
        Vinv[var] = Vi; Q3[var] = Qv
        Mvar = 2 * Vi_a + Qv
        # observations of variable points, their T = W V^-1 and T_a = W_a M_p
        isvar = point_off[pl] >= 0
        ol = np.nonzero(isvar)[0]
        slot = np.full(npts, -1, np.int64); slot[var] = np.arange(len(var))
        sp = slot[pl[ol]]
        Wl, Wal = W[o0:o1][ol], Wa[o0:o1][ol]
        T = np.matmul(Wl, Vi[sp]); Ta = np.matmul(Wal, Mvar[sp])
        _scatter_by_key(rp, img[ol], np.matmul(T, gp[var][sp][:, :, None])[:, :, 0], img_rows, None)
        _scatter_by_key(Erp, img[ol], np.matmul(Ta, gpa[var][sp][:, :, None])[:, :, 0], img_rows, None)
        # observation pairs (a, b), b <= a, of every variable point
        L = np.bincount(sp, minlength=len(var))
        s0 = np.concatenate([[0], np.cumsum(L)[:-1]])
        npair = L * (L + 1) // 2
        pp = np.repeat(np.arange(len(var)), npair)
        k = np.arange(len(pp)) - np.repeat(np.concatenate([[0], np.cumsum(npair)[:-1]]), npair)
        a = ((np.sqrt(8.0 * k + 1) - 1) // 2).astype(np.int64)
        a += (a + 1) * (a + 2) // 2 <= k; a -= a * (a + 1) // 2 > k
        b = k - a * (a + 1) // 2
        ia, ib = s0[pp] + a, s0[pp] + b
        off = ia != ib
        for dst, X, Y in ((Sp, T, Wl), (ESp, Ta, Wal)):
            P = np.matmul(X[ia], Y[ib].transpose(0, 2, 1))
            key = img[ol][ia] * n_img + img[ol][ib]
            keyT = img[ol][ib[off]] * n_img + img[ol][ia[off]]
            _scatter_by_key(dst, np.concatenate([key, keyT]), np.concatenate([P, P[off].transpose(0, 2, 1)]),
                            pair_rows, pair_cols)
            del P
    Hcc, Acc, gc, ac = Hcc[:nc, :nc], Acc[:nc, :nc], gc[:nc], ac[:nc]
    Sp, ESp, rp, Erp = Sp[:nc, :nc], ESp[:nc, :nc], rp[:nc], Erp[:nc]
    dgc = np.diagonal(Hcc).copy()
    D2c = _damping(dgc, so, radius)
    D2ca = D2c * np.where(dgc > 0, np.diagonal(Acc) / np.where(dgc > 0, dgc, 1), 1)
    S = Hcc - Sp
    S[np.diag_indices(nc)] += D2c
    rhs = -gc + rp
    del Sp
    Acc = np.asarray(Acc, np.float64)          # scales need no long double; free the long-double pair scale early
    ES = KAPPA * (Acc + np.asarray(ESp, np.float64))
    del ESp
    ES[np.diag_indices(nc)] += KAPPA * np.asarray(D2ca, np.float64)
    Erhs = np.asarray(KAPPA * (ac + Erp), np.float64)
    # camera step: fp64 LAPACK + two refinement steps with long-double residuals; |S^-1| explicitly
    if nc:
        F = scipy.linalg.cho_factor(np.asarray(S, np.float64), lower=True)
        x = np.asarray(scipy.linalg.cho_solve(F, np.asarray(rhs, np.float64)), LD)
        for _ in range(2):
            x += np.asarray(scipy.linalg.cho_solve(F, np.asarray(rhs - S @ x, np.float64)), LD)
        Sinv = np.abs(scipy.linalg.cho_solve(F, np.eye(nc)))
        ax = np.abs(np.asarray(x, np.float64))
        sd = np.sqrt(np.asarray(np.diagonal(S), np.float64))
        ESc = lambda z: ES @ z + 3 * nc * U64 * sd * (sd @ z)
        y = Sinv @ (ESc(ax) + Erhs)
        Xy = Sinv @ ESc(y)
        eta = float(np.max(np.where(y > 0, Xy / np.where(y > 0, y, 1.0), np.where(Xy > 0, np.inf, 0.0))))
        if not eta < 0.5:
            raise IllConditioned("max (|S^-1| E_S y) / y = %g at radius %g" % (eta, radius))
        Ec = y / (1 - eta)
        del Sinv
    else:
        x = np.zeros(0, LD); Ec = np.zeros(0); eta = 0.0
    # points: back-substitution in long double, in layout order
    xe = np.concatenate([x, [LD(0)]]); Ece = np.concatenate([Ec, [0.0]]); axe = np.abs(np.asarray(xe, np.float64))
    oi = obs_img[order]
    pl_all = np.repeat(np.arange(npts), np.diff(start))
    vsum = np.zeros((npts, 3), LD)
    np.add.at(vsum, pl_all, np.matmul(W.transpose(0, 2, 1), xe[ci[oi]][:, :, None])[:, :, 0])
    Waf = np.asarray(Wa, np.float64)
    e1 = np.zeros((npts, 3)); e2 = np.zeros((npts, 3))
    np.add.at(e1, pl_all, np.matmul(Waf.transpose(0, 2, 1), axe[ci[oi]][:, :, None])[:, :, 0])
    np.add.at(e2, pl_all, np.matmul(Waf.transpose(0, 2, 1), Ece[ci[oi]][:, :, None])[:, :, 0])
    vv = gp + vsum
    dp = -np.matmul(Vinv, vv[:, :, None])[:, :, 0]
    Ev = KAPPA * (np.asarray(gpa, np.float64) + e1) + e2
    Ep = np.matmul(np.abs(np.asarray(Vinv, np.float64)), Ev[:, :, None])[:, :, 0] + \
        KAPPA * np.matmul(np.asarray(Q3, np.float64), np.abs(np.asarray(vv, np.float64))[:, :, None])[:, :, 0]
    var = np.nonzero(point_off >= 0)[0]
    delta = np.zeros(nl, LD); Ed = np.zeros(nl)
    delta[:nc] = x; Ed[:nc] = Ec
    pcols = point_off[var][:, None] + np.arange(3)
    delta[pcols] = dp[var]; Ed[pcols] = Ep[var]
    # model cost change: -g^T d - d^T H d / 2 over the blocks
    dpv = np.zeros((npts, 3), LD); dpv[var] = dp[var]
    dpo = dpv[pl_all]
    cross = (xe[ci[oi]][:, :, None] * W * dpo[:, None, :]).sum()
    dHd = x @ (Hcc @ x) + np.einsum("pi,pij,pj->", dpv, Hpp, dpv) + 2 * cross
    gd = gc @ x + (gp * dpv).sum()
    mcc = -gd - dHd / 2
    ad = np.abs(np.asarray(delta, np.float64))
    adp = np.abs(np.asarray(dpv, np.float64))
    crossa = (axe[ci[oi]][:, :, None] * Waf * adp[pl_all][:, None, :]).sum()
    dAd = ad[:nc] @ (Acc @ ad[:nc]) + \
        np.einsum("pi,pij,pj->", adp, np.asarray(Hppa, np.float64), adp) + 2 * crossa
    aabs = float(np.asarray(ac, np.float64) @ ad[:nc] + (np.asarray(gpa, np.float64) * adp).sum())
    Dd = np.zeros(nl)
    Dd[:nc] = np.asarray(D2c * x, np.float64)
    Dd[pcols] = np.asarray(D2p[var] * dp[var], np.float64)
    Emcc = float(np.abs(Dd) @ Ed + KAPPA * (aabs + dAd / 2))
    return dict(radius=radius, nc=nc, nl=nl, cost=cost, Hcc=Hcc, gc=gc, Hpp=Hpp, gp=gp, S=S, rhs=rhs, delta=delta,
                model_cost_change=mcc, eta=eta, Acc=Acc, ac=ac, Hppa=Hppa, gpa=gpa, ES=ES, Erhs=Erhs, Edelta=Ed,
                Emcc=Emcc,
                W=W, Wa=Wa, Vinv=Vinv, layout=lay, obs_img=obs_img)


# ---- comparators: worst ratio of error to error scale --------------------------------------------------------------
def _ratio(diff, scale):
    diff = np.abs(np.asarray(diff, np.float64)); scale = np.asarray(scale, np.float64)
    if np.any(diff[scale == 0] != 0):
        return np.inf
    return float(np.max(np.where(scale > 0, diff / np.where(scale > 0, scale, 1.0), 0.0), initial=0.0))


def _lower(M):
    """lower triangle in float64: rounding the reference to float64 moves an entry by at most 2^-53 |entry|, and
    |S| <= E_S / KAPPA, |Hcc| <= Acc, so by at most 1.2e-7 of its error scale"""
    return np.tril(np.asarray(M, np.float64))


def hcc_error(got, ref):
    """lower triangle of Hcc against KAPPA * Acc"""
    return _ratio(_lower(got) - _lower(ref["Hcc"]), np.tril(KAPPA * ref["Acc"]))


def gc_error(got, ref):
    return _ratio(np.asarray(got, LD) - ref["gc"], KAPPA * np.asarray(ref["ac"], np.float64))


def hpp_error(got, ref):
    var = ref["layout"]["point_off"] >= 0
    return _ratio((np.asarray(got, LD) - ref["Hpp"])[var], KAPPA * np.asarray(ref["Hppa"], np.float64)[var])


def gp_error(got, ref):
    var = ref["layout"]["point_off"] >= 0
    return _ratio((np.asarray(got, LD) - ref["gp"])[var], KAPPA * np.asarray(ref["gpa"], np.float64)[var])


def s_error(got, ref):
    """lower triangle of the damped Schur complement against E_S"""
    return _ratio(_lower(got) - _lower(ref["S"]), np.tril(ref["ES"]))


def rhs_error(got, ref):
    return _ratio(np.asarray(got, LD) - ref["rhs"], ref["Erhs"])


def delta_error(got, ref):
    """cameras and points of the step against the first-order bound"""
    return _ratio(np.asarray(got, LD) - ref["delta"], ref["Edelta"])


def mcc_error(got, ref):
    return _ratio(LD(got) - ref["model_cost_change"], ref["Emcc"])


def all_errors(got, ref, dense=True):
    out = dict(delta=delta_error(got["delta"], ref), model_cost_change=mcc_error(got["model_cost_change"], ref),
               gc=gc_error(got["gc"], ref), Hpp=hpp_error(got["Hpp"], ref), gp=gp_error(got["gp"], ref))
    if dense:
        out.update(Hcc=hcc_error(got["Hcc"], ref), S=s_error(got["S"], ref), rhs=rhs_error(got["rhs"], ref))
    return out


# ---- one point's Schur terms (for mutation checks) -----------------------------------------------------------------
def point_terms(ref, p, W=None):
    """point p's contribution sum_{o,o'} W_o V^-1 W_o'^T to the dense [nc, nc] matrix it is subtracted from, and its
    [nc] rhs term sum_o W_o V^-1 gp (W: optional replacement [L, DC, 3] of the point's W blocks)"""
    lay = ref["layout"]
    nc, ci = lay["nc"], lay["cols_img"]
    o0, o1 = lay["start"][p], lay["start"][p + 1]
    Wp = ref["W"][o0:o1] if W is None else np.asarray(W, LD)
    cols = ci[ref["obs_img"][lay["order"][o0:o1]]]
    T = np.matmul(Wp, ref["Vinv"][p])
    S = np.zeros((nc + 1, nc + 1), LD); r = np.zeros(nc + 1, LD)
    for a in range(len(Wp)):
        np.add.at(r, cols[a], T[a] @ ref["gp"][p])
        for b in range(len(Wp)):
            np.add.at(S, (cols[a][:, None], cols[b][None, :]), T[a] @ Wp[b].T)
    return S[:nc, :nc], r[:nc], cols


def default_options(**kw):
    return _capi.default_ba_options(use_inner_iterations=0, **kw)
