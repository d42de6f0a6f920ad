"""Host restatement of absolute pose estimation (csrc/pxr_pnp.cu, include/pxr.h "batched absolute pose estimation"):
the sample stream, Lambda Twist P3P, the support measure, local optimisation and the dynamic trial count, with the
device code's operation order (the device file is compiled without fused multiply-add), so P3P and every residual
come out the same to the last bit; only sums over correspondences run in another order."""
import math

import numpy as np

M64 = (1 << 64) - 1
ROUND_TRIALS = 128
LO_STEPS = 3
DBL_EPS = 2.220446049250313e-16


def splitmix64(x):
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def sample(seed, trial, n):
    """the three correspondence indices trial `trial` draws, or None"""
    s0 = splitmix64(seed & M64)
    idx = []
    for d in range(64):
        w = splitmix64(s0 ^ ((trial << 8) & M64) ^ d)
        i = ((w >> 32) * n) >> 32
        if i not in idx:
            idx.append(i)
            if len(idx) == 3:
                return idx
    return None


# ---- Lambda Twist P3P (Persson & Nordberg, ECCV 2018)
def _root2real(b, c):
    v = b * b - 4.0 * c
    if v < 0.0:
        return False, 0.5 * b, 0.5 * b
    y = math.sqrt(v)
    r1 = 0.5 * (-b + y) if b < 0.0 else 0.5 * (-b - y)
    r2 = c / r1 if r1 != 0.0 else math.inf
    return True, r1, r2


def _cubick(b, c, d):
    """a real root of x^3 + b x^2 + c x + d"""
    if b * b >= 3.0 * c:
        v = math.sqrt(b * b - 3.0 * c)
        t1 = (-b - v) / 3.0
        k = ((t1 + b) * t1 + c) * t1 + d
        if k > 0.0:
            r0 = t1 - _sqrt(_div(-k, 3.0 * t1 + b))
        else:
            t2 = (-b + v) / 3.0
            k = ((t2 + b) * t2 + c) * t2 + d
            r0 = t2 + _sqrt(_div(-k, 3.0 * t2 + b))
    else:
        r0 = -b / 3.0
        if abs((3.0 * r0 + 2.0 * b) * r0 + c) < 1e-4:
            r0 += 1.0
    for i in range(50):
        fx = ((r0 + b) * r0 + c) * r0 + d
        if i >= 7 and abs(fx) <= DBL_EPS:
            break
        fpx = (3.0 * r0 + 2.0 * b) * r0 + c
        r0 = r0 - _div(fx, fpx)
    return r0


def _sqrt(x):
    return math.sqrt(x) if x >= 0.0 else math.nan


def _div(a, b):
    if b == 0.0:
        return math.nan if a == 0.0 or a != a else math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def _eig_known0(x):
    """eigenvectors (columns) and eigenvalues of the symmetric 3x3 x (row-major list) with one eigenvalue 0"""
    v3 = [x[3] * x[7] - x[6] * x[4], x[6] * x[1] - x[7] * x[0], x[4] * x[0] - x[3] * x[1]]
    n3 = _sqrt(v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2])
    v3 = [_div(v3[0], n3), _div(v3[1], n3), _div(v3[2], n3)]
    x01_squared = x[1] * x[1]
    b = -x[0] - x[4] - x[8]
    c = -x01_squared - x[2] * x[2] - x[5] * x[5] + x[0] * (x[4] + x[8]) + x[4] * x[8]
    _, e1, e2 = _root2real(b, c)
    if abs(e1) < abs(e2):
        e1, e2 = e2, e1
    mx0011 = -x[0] * x[4]
    prec_0 = x[1] * x[5] - x[2] * x[4]
    prec_1 = x[1] * x[2] - x[0] * x[5]
    vs = []
    for e in (e1, e2):
        tmp = _div(1.0, e * (x[0] + x[4]) + mx0011 - e * e + x01_squared)
        a1 = -(e * x[2] + prec_0) * tmp
        a2 = -(e * x[5] + prec_1) * tmp
        rnorm = _div(1.0, _sqrt(a1 * a1 + a2 * a2 + 1.0))
        vs.append([a1 * rnorm, a2 * rnorm, rnorm])
    V = [vs[0][0], vs[1][0], v3[0], vs[0][1], vs[1][1], v3[1], vs[0][2], vs[1][2], v3[2]]   # row-major, columns = vectors
    return V, (e1, e2, 0.0)


def _refine_L(L, a12, a13, a23, b12, b13, b23):
    l1, l2, l3 = L
    for _ in range(5):
        r1 = l1 * l1 + l2 * l2 + b12 * l1 * l2 - a12
        r2 = l1 * l1 + l3 * l3 + b13 * l1 * l3 - a13
        r3 = l2 * l2 + l3 * l3 + b23 * l2 * l3 - a23
        e0 = abs(r1) + abs(r2) + abs(r3)
        if not (e0 > 0.0):
            break
        a = 2.0 * l1 + b12 * l2; b = 2.0 * l2 + b12 * l1
        c = 2.0 * l1 + b13 * l3; e = 2.0 * l3 + b13 * l1
        f = 2.0 * l2 + b23 * l3; g = 2.0 * l3 + b23 * l2
        idet = _div(1.0, -a * e * f - b * c * g)
        d1 = (-e * f * r1 - b * g * r2 + b * e * r3) * idet
        d2 = (-c * g * r1 + a * g * r2 - a * e * r3) * idet
        d3 = (c * f * r1 - a * f * r2 - b * c * r3) * idet
        m1, m2, m3 = l1 - d1, l2 - d2, l3 - d3
        s1 = m1 * m1 + m2 * m2 + b12 * m1 * m2 - a12
        s2 = m1 * m1 + m3 * m3 + b13 * m1 * m3 - a13
        s3 = m2 * m2 + m3 * m3 + b23 * m2 * m3 - a23
        if not (abs(s1) + abs(s2) + abs(s3) < e0):
            break
        l1, l2, l3 = m1, m2, m3
    return l1, l2, l3


def p3p(x, X):
    """x [3,2] normalised image points, X [3,3] world points -> list of (R [3,3], t [3]) world->camera"""
    y = []
    for k in range(3):
        u, v = float(x[k][0]), float(x[k][1])
        nrm = math.sqrt(u * u + v * v + 1.0)
        y.append((u / nrm, v / nrm, 1.0 / nrm))
    Xw = [[float(X[k][j]) for j in range(3)] for k in range(3)]
    dot = lambda p, q: p[0] * q[0] + p[1] * q[1] + p[2] * q[2]
    sub = lambda p, q: [p[0] - q[0], p[1] - q[1], p[2] - q[2]]
    cross = lambda p, q: [p[1] * q[2] - p[2] * q[1], p[2] * q[0] - p[0] * q[2], p[0] * q[1] - p[1] * q[0]]
    b12, b13, b23 = -2.0 * dot(y[0], y[1]), -2.0 * dot(y[0], y[2]), -2.0 * dot(y[1], y[2])
    d12, d13, d23 = sub(Xw[0], Xw[1]), sub(Xw[0], Xw[2]), sub(Xw[1], Xw[2])
    d12xd13 = cross(d12, d13)
    a12, a13, a23 = dot(d12, d12), dot(d13, d13), dot(d23, d23)
    c31, c23, c12 = -0.5 * b13, -0.5 * b23, -0.5 * b12
    blob = c12 * c23 * c31 - 1.0
    s31_squared, s23_squared, s12_squared = 1.0 - c31 * c31, 1.0 - c23 * c23, 1.0 - c12 * c12
    p3 = a13 * (a23 * s31_squared - a13 * s23_squared)
    p2 = 2.0 * blob * a23 * a13 + a13 * (2.0 * a12 + a13) * s23_squared + a23 * (a23 - a12) * s31_squared
    p1 = a23 * (a13 - a23) * s12_squared - a12 * a12 * s23_squared - 2.0 * a12 * (blob * a23 + a13 * s23_squared)
    p0 = a12 * (a12 * s23_squared - a23 * s12_squared)
    if not (p3 != 0.0):
        return []
    ip3 = 1.0 / p3
    g = _cubick(p2 * ip3, p1 * ip3, p0 * ip3)
    A = [a23 * (1.0 - g), (a23 * b12) * 0.5, (a23 * b13 * g) * (-0.5),
         0.0, a23 - a12 + a13 * g, b23 * (a13 * g - a12) * 0.5,
         0.0, 0.0, g * (a13 - a23) - a12]
    A[3], A[6], A[7] = A[1], A[2], A[5]
    V, L = _eig_known0(A)
    v = _sqrt(max(0.0, _div(-L[1], L[0])))
    Ls = []
    for s in (v, -v):
        w2 = _div(1.0, s * V[1] - V[0])
        w0 = (V[3] - s * V[4]) * w2
        w1 = (V[6] - s * V[7]) * w2
        a = _div(1.0, (a13 - a12) * w1 * w1 - a12 * b13 * w1 - a12)
        b = (a13 * b12 * w1 - a12 * b13 * w0 - 2.0 * w0 * w1 * (a12 - a13)) * a
        c = ((a13 - a12) * w0 * w0 + a13 * b12 * w0 + a13) * a
        if b * b - 4.0 * c >= 0.0:
            _, tau1, tau2 = _root2real(b, c)
            for tau in (tau1, tau2):
                if tau > 0.0:
                    d = _div(a23, tau * (b23 + tau) + 1.0)
                    if d > 0.0:
                        l2 = math.sqrt(d)
                        l3 = tau * l2
                        l1 = w0 * l2 + w1 * l3
                        if l1 >= 0.0:
                            Ls.append((l1, l2, l3))
    # inverse of the matrix with columns d12, d13, d12 x d13 (adjugate / determinant)
    Mx = [[d12[0], d13[0], d12xd13[0]], [d12[1], d13[1], d12xd13[1]], [d12[2], d13[2], d12xd13[2]]]
    det = (Mx[0][0] * (Mx[1][1] * Mx[2][2] - Mx[1][2] * Mx[2][1]) - Mx[0][1] * (Mx[1][0] * Mx[2][2] - Mx[1][2] * Mx[2][0]) +
           Mx[0][2] * (Mx[1][0] * Mx[2][1] - Mx[1][1] * Mx[2][0]))
    if not (det != 0.0) or not math.isfinite(det):
        return []
    idet = 1.0 / det
    Xi = [[(Mx[1][1] * Mx[2][2] - Mx[1][2] * Mx[2][1]) * idet, (Mx[0][2] * Mx[2][1] - Mx[0][1] * Mx[2][2]) * idet,
           (Mx[0][1] * Mx[1][2] - Mx[0][2] * Mx[1][1]) * idet],
          [(Mx[1][2] * Mx[2][0] - Mx[1][0] * Mx[2][2]) * idet, (Mx[0][0] * Mx[2][2] - Mx[0][2] * Mx[2][0]) * idet,
           (Mx[0][2] * Mx[1][0] - Mx[0][0] * Mx[1][2]) * idet],
          [(Mx[1][0] * Mx[2][1] - Mx[1][1] * Mx[2][0]) * idet, (Mx[0][1] * Mx[2][0] - Mx[0][0] * Mx[2][1]) * idet,
           (Mx[0][0] * Mx[1][1] - Mx[0][1] * Mx[1][0]) * idet]]
    out = []
    for L3 in Ls:
        l1, l2, l3 = _refine_L(L3, a12, a13, a23, b12, b13, b23)
        ry1 = [y[0][j] * l1 for j in range(3)]
        ry2 = [y[1][j] * l2 for j in range(3)]
        ry3 = [y[2][j] * l3 for j in range(3)]
        e1, e2 = sub(ry1, ry2), sub(ry1, ry3)
        e3 = cross(e1, e2)
        Y = [[e1[0], e2[0], e3[0]], [e1[1], e2[1], e3[1]], [e1[2], e2[2], e3[2]]]
        R = [[Y[i][0] * Xi[0][j] + Y[i][1] * Xi[1][j] + Y[i][2] * Xi[2][j] for j in range(3)] for i in range(3)]
        t = [ry1[i] - (R[i][0] * Xw[0][0] + R[i][1] * Xw[0][1] + R[i][2] * Xw[0][2]) for i in range(3)]
        R, t = np.array(R), np.array(t)
        if np.all(np.isfinite(R)) and np.all(np.isfinite(t)):
            out.append((R, t))
    return out


def rot_to_quat(R):
    """rotation matrix -> unit quaternion (w, x, y, z), w >= 0 (the device's formula)"""
    R = [[float(R[i][j]) for j in range(3)] for i in range(3)]
    tr = R[0][0] + R[1][1] + R[2][2]
    if tr > 0.0:
        s = math.sqrt(tr + 1.0) * 2.0
        q = [0.25 * s, (R[2][1] - R[1][2]) / s, (R[0][2] - R[2][0]) / s, (R[1][0] - R[0][1]) / s]
    elif R[0][0] > R[1][1] and R[0][0] > R[2][2]:
        s = math.sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]) * 2.0
        q = [(R[2][1] - R[1][2]) / s, 0.25 * s, (R[0][1] + R[1][0]) / s, (R[0][2] + R[2][0]) / s]
    elif R[1][1] > R[2][2]:
        s = math.sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]) * 2.0
        q = [(R[0][2] - R[2][0]) / s, (R[0][1] + R[1][0]) / s, 0.25 * s, (R[1][2] + R[2][1]) / s]
    else:
        s = math.sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]) * 2.0
        q = [(R[1][0] - R[0][1]) / s, (R[0][2] + R[2][0]) / s, (R[1][2] + R[2][1]) / s, 0.25 * s]
    n = math.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    q = [c / n for c in q]
    if q[0] < 0.0:
        q = [-c for c in q]
    return np.array(q)


def quat_to_rot(q):
    q = np.asarray(q, np.float64) / np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


# ---- RANSAC
def residuals(R, t, uv, X):
    """squared normalised-plane reprojection errors and the in-front test, elementwise in the device's order"""
    x = R[0, 0] * X[:, 0] + R[0, 1] * X[:, 1] + R[0, 2] * X[:, 2] + t[0]
    y = R[1, 0] * X[:, 0] + R[1, 1] * X[:, 1] + R[1, 2] * X[:, 2] + t[1]
    z = R[2, 0] * X[:, 0] + R[2, 1] * X[:, 1] + R[2, 2] * X[:, 2] + t[2]
    with np.errstate(divide="ignore", invalid="ignore"):
        iz = 1.0 / z
        du = x * iz - uv[:, 0]
        dv = y * iz - uv[:, 1]
        r = du * du + dv * dv
    return r, z > DBL_EPS


def support(R, t, uv, X, thr2):
    r, front = residuals(R, t, uv, X)
    inl = front & (r <= thr2)
    return int(inl.sum()), float(r[inl].sum()), inl


def _better(a, b):
    """support a = (count, sum) strictly better than b"""
    return a[0] > b[0] or (a[0] == b[0] and a[1] < b[1])


def required_trials(n_inliers, n, confidence, multiplier, min_trials, max_trials):
    if n_inliers <= 0:
        return max_trials
    ratio = n_inliers / float(n)
    nom = 1.0 - confidence
    if nom <= 0.0:
        req = float(max_trials)
    else:
        denom = 1.0 - ratio * ratio * ratio
        if denom <= 0.0:
            req = 1.0
        elif denom == 1.0:
            req = float(max_trials)
        else:
            req = math.ceil(math.log(nom) / math.log(denom) * multiplier)
    return int(min(max(req, float(min_trials)), float(max_trials)))


def _exp_so3(w):
    th = math.sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2])
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th < 1e-12:
        return np.eye(3) + K
    K = K / th
    return np.eye(3) + math.sin(th) * K + (1.0 - math.cos(th)) * (K @ K)


def local_optimize(R, t, uv, X, thr2):
    """LO_STEPS Gauss-Newton steps on (left rotation increment, translation) over the inliers of (R, t)"""
    _, _, inl = support(R, t, uv, X, thr2)
    P, Q = X[inl], uv[inl]
    for _ in range(LO_STEPS):
        p = P @ R.T
        Xc = p + t
        iz = 1.0 / Xc[:, 2]
        r = np.stack([Xc[:, 0] * iz - Q[:, 0], Xc[:, 1] * iz - Q[:, 1]], 1)
        J = np.zeros((len(P), 2, 6))
        a0 = np.stack([iz, np.zeros_like(iz), -Xc[:, 0] * iz * iz], 1)
        a1 = np.stack([np.zeros_like(iz), iz, -Xc[:, 1] * iz * iz], 1)
        for row, a in ((0, a0), (1, a1)):
            J[:, row, 0] = -a[:, 1] * p[:, 2] + a[:, 2] * p[:, 1]
            J[:, row, 1] = a[:, 0] * p[:, 2] - a[:, 2] * p[:, 0]
            J[:, row, 2] = -a[:, 0] * p[:, 1] + a[:, 1] * p[:, 0]
            J[:, row, 3:] = a
        H = np.einsum("nki,nkj->ij", J, J)
        g = np.einsum("nki,nk->i", J, r)
        try:
            L = np.linalg.cholesky(H)
        except np.linalg.LinAlgError:
            break
        d = -np.linalg.solve(L.T, np.linalg.solve(L, g))
        R = _exp_so3(d[:3]) @ R
        t = t + d[3:]
    return R, t


def ransac(uv, X, thr, seed, min_trials=1000, max_trials=100000, confidence=0.9999, multiplier=3.0):
    """-> dict(R, t, count, sum, trial, solution, lo, num_trials, inliers) or None when nothing was found"""
    n = len(uv)
    if n < 3:
        return None
    thr2 = thr * thr
    best, best_sup, best_idx, lo = None, (-1, math.inf), -1, False
    rnd = 0
    while True:
        hyps = []
        for k in range(ROUND_TRIALS):
            trial = rnd * ROUND_TRIALS + k
            if trial >= max_trials:
                break
            idx = sample(seed, trial, n)
            if idx is None:
                continue
            for s, (R, t) in enumerate(p3p(uv[idx], X[idx])):
                hyps.append((4 * trial + s, R, t))
        rb, rb_sup = None, (-1, math.inf)
        for h, R, t in hyps:
            c, sm, _ = support(R, t, uv, X, thr2)
            if _better((c, sm), rb_sup):
                rb, rb_sup = (h, R, t), (c, sm)
        if rb is not None and _better(rb_sup, best_sup):
            best_idx, best, best_sup, lo = rb[0], (rb[1], rb[2]), rb_sup, False
            R2, t2 = local_optimize(best[0], best[1], uv, X, thr2)
            if best_sup[0] > 3 and np.all(np.isfinite(R2)) and np.all(np.isfinite(t2)):
                c, sm, _ = support(R2, t2, uv, X, thr2)
                if _better((c, sm), best_sup):
                    best, best_sup, lo = (R2, t2), (c, sm), True
        rnd += 1
        n_run = min(rnd * ROUND_TRIALS, max_trials)
        if n_run >= required_trials(best_sup[0], n, confidence, multiplier, min_trials, max_trials):
            break
    if best is None:
        return dict(count=0, num_trials=n_run, trial=-1, solution=-1)
    _, _, inl = support(best[0], best[1], uv, X, thr2)
    return dict(R=best[0], t=best[1], count=best_sup[0], sum=best_sup[1], trial=best_idx >> 2, solution=best_idx & 3,
                lo=lo, num_trials=n_run, inliers=inl)
