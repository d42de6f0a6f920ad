"""numpy restatement of point triangulation from known poses (include/pxr.h, csrc/pxr_tri.cu): hloc's epipolar errors,
the midpoint N-view point, the exhaustive / sampled observation pairs, MSAC selection with the refit, triangulation
angles and reprojection errors.  It takes normalised image points (the device moves pixels there with its own
ImageToWorld, which tests/test_gpu_pnp.py checks), so it is independent of the camera models.  Also: synthetic scenes
for the tests and the benchmark."""
import numpy as np

from pnp_reference import M64, quat_to_rot, splitmix64

TRI_OK, TRI_TOO_FEW_INLIERS, TRI_ANGLE_TOO_SMALL = range(3)


# ---- verification
def epipolar_errors(x0, x1, q0, t0, q1, t1):
    """hloc's compute_epipolar_errors for normalised points x0, x1 [n, 2] of two posed images -> (d0, d1) [n]"""
    R0, R1 = quat_to_rot(q0), quat_to_rot(q1)
    R = R1 @ R0.T
    t = np.asarray(t1, np.float64) - R @ np.asarray(t0, np.float64)
    E = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]]) @ R
    h0 = np.column_stack([x0, np.ones(len(x0))])
    h1 = np.column_stack([x1, np.ones(len(x1))])
    l1 = h0 @ E.T                       # E x0: the line in image 1
    l0 = h1 @ E                         # E^T x1: the line in image 0
    dist = np.abs(np.sum(h0 * l0, axis=1))
    return dist / np.linalg.norm(l0[:, :2], axis=1), dist / np.linalg.norm(l1[:, :2], axis=1)


def mean_focal(model, params):
    return params[0] if model in (0, 2, 3) else 0.5 * (params[0] + params[1])


# ---- rays, points, angles
def rays(xn, q, t):
    """world unit rays d and camera centres c [n, 3] of normalised points xn [n, 2] seen from (q, t)"""
    R = quat_to_rot(q)
    d = np.column_stack([xn, np.ones(len(xn))]) @ R                # rows R^T (u, v, 1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    c = np.broadcast_to(-R.T @ np.asarray(t, np.float64), d.shape).copy()
    return d, c


def angle_between(a, b):
    return np.arctan2(np.linalg.norm(np.cross(a, b), axis=-1), np.sum(a * b, axis=-1))


def folded(a):
    return np.minimum(a, np.pi - a)


def midpoint(d, c):
    """X = (sum (I - d d^T))^-1 sum (I - d d^T) c, or None when the system is numerically singular"""
    P = np.eye(3)[None] - d[:, :, None] * d[:, None, :]
    A, b = P.sum(0), np.einsum("kij,kj->i", P, c)
    tr = np.trace(A) / 3.0
    if not np.linalg.det(A) > 1e-14 * tr ** 3:
        return None
    return np.linalg.solve(A, b)


def errors(d, c, X):
    """angular errors [n] (radians) and whether X is in front of each ray"""
    v = X[None, :] - c
    return angle_between(d, v), np.sum(d * v, axis=1) > 0


def max_tri_angle(c, X, mask=None):
    idx = np.flatnonzero(np.ones(len(c), bool) if mask is None else mask)
    if len(idx) < 2:
        return 0.0
    i, j = np.triu_indices(len(idx), 1)
    a, b = X - c[idx[i]], X - c[idx[j]]
    return float(folded(angle_between(a, b)).max())


# ---- hypotheses
def pair_sample(seed, key, h, n):
    """the observation pair hypothesis h of a sampled track draws, or None"""
    s0 = splitmix64((seed ^ splitmix64(key & M64)) & M64)
    idx = []
    for d in range(64):
        w = splitmix64(s0 ^ ((h << 8) & M64) ^ d)
        i = ((w >> 32) * n) >> 32
        if i not in idx:
            idx.append(i)
            if len(idx) == 2:
                return tuple(idx)
    return None


def hypothesis_pairs(n, max_pairs, seed, key):
    """[(i, j) or None] in hypothesis order"""
    if n * (n - 1) // 2 <= max_pairs:
        return [(i, j) for i in range(n) for j in range(i + 1, n)]
    return [pair_sample(seed, key, h, n) for h in range(max_pairs)]


def triangulate_track(d, c, min_angle=1.5, create_max_angle_error=2.0, max_pairs=1024, seed=0, key=0):
    """one track's RANSAC + refit -> dict(xyz, status, inliers (bool [n]), n_inliers, angle (degrees), best)"""
    n = len(d)
    min_a, tau = np.radians(min_angle), np.radians(create_max_angle_error)
    best, best_h, best_X = np.inf, -1, None
    for h, pr in enumerate(hypothesis_pairs(n, max_pairs, seed, key)):
        if pr is None:
            continue
        i, j = pr
        if not folded(angle_between(d[i], d[j])) >= min_a:
            continue
        X = midpoint(d[[i, j]], c[[i, j]])
        if X is None:
            continue
        e, front = errors(d, c, X)
        score = float(np.where(front & (e < tau), e * e, tau * tau).sum())
        if score < best:
            best, best_h, best_X = score, h, X
    out = dict(xyz=np.zeros(3), status=TRI_ANGLE_TOO_SMALL, inliers=np.zeros(n, bool), n_inliers=0, angle=0.0, best=best_h)
    if best_h < 0:
        return out

    def inl(X):
        e, front = errors(d, c, X)
        return front & (e <= tau)

    X, S = best_X, inl(best_X)
    status = TRI_OK
    if S.sum() < 2:
        status = TRI_TOO_FEW_INLIERS
    else:
        X1 = midpoint(d[S], c[S])
        if X1 is None:
            status = TRI_ANGLE_TOO_SMALL
        else:
            X, S1 = X1, inl(X1)
            if not np.array_equal(S1, S):
                S = S1
                if S.sum() < 2:
                    status = TRI_TOO_FEW_INLIERS
                else:
                    X2 = midpoint(d[S], c[S])
                    if X2 is None:
                        status = TRI_ANGLE_TOO_SMALL
                    else:
                        X = X2
    ang = max_tri_angle(c, X, S) if S.sum() >= 2 else 0.0
    if status == TRI_OK and not ang >= min_a:
        status = TRI_ANGLE_TOO_SMALL
    out.update(xyz=X, status=status, inliers=S, n_inliers=int(S.sum()), angle=np.degrees(ang))
    return out


def reprojection_errors(model, params, q, t, X, xy):
    """pixel errors [n] of points X [n, 3] against xy [n, 2] in one image; +inf behind the camera"""
    from pixsfm.util.cameras import normalized_to_image
    pc = X @ quat_to_rot(q).T + np.asarray(t, np.float64)
    err = np.full(len(X), np.inf)
    front = pc[:, 2] > 2.220446049250313e-16
    if front.any():
        px = normalized_to_image(model, params, pc[front, :2] / pc[front, 2:3])
        err[front] = np.linalg.norm(px - xy[front], axis=1)
    return err


# ---- scenes
CAMERAS = {0: [500.0, 320, 240], 1: [510.0, 490.0, 320, 240], 2: [500.0, 320, 240, 0.05], 3: [500.0, 320, 240, 0.05, -0.02],
           4: [510.0, 490.0, 320, 240, 0.05, -0.02, 0.001, -0.002], 5: [500.0, 505.0, 320, 240, 0.02, -0.01, 0.003, -0.001],
           6: [510.0, 490.0, 320, 240, 0.05, -0.02, 0.001, -0.002, 0.003, 0.01, -0.005, 0.002]}


def padded(params):
    p = np.zeros(12)
    p[:len(params)] = params
    return p


def ring_poses(n_images, radius=6.0, seed=0, jitter=0.05, arc=np.radians(120)):
    """cameras on an arc of a ring around the origin, looking at it, all at distance `radius` -> qvec [n, 4], tvec [n, 3]"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    qv, tv = [], []
    for k in range(n_images):
        a = arc * (k / max(n_images - 1, 1) - 0.5)
        C = np.array([radius * np.sin(a), 0.4 * np.sin(3 * a), -radius * np.cos(a)])
        z = -C / np.linalg.norm(C)
        x = np.cross([0.0, 1.0, 0.0], z); x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        R = Rotation.from_rotvec(rng.normal(0, jitter, 3)).as_matrix() @ R
        q = Rotation.from_matrix(R).as_quat()
        qv.append([q[3], q[0], q[1], q[2]])
        tv.append(-R @ C)
    return np.array(qv), np.array(tv)


def project_normalised(q, t, X):
    pc = X @ quat_to_rot(q).T + t
    return pc[:, :2] / pc[:, 2:3]
