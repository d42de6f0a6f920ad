"""Geometric (reprojection-error) BA scenes and an independent scipy solve of them (test infrastructure).

The scenes follow the recipe of the reference's bundle_optimizer_test.cc (colmap::GenerateReconstruction): 100 points
drawn from U(-1, 1)^3, per image a SIMPLE_RADIAL camera with f = 1200 on a 1000 x 1000 image, identity rotation,
tvec = (U(-1, 1), U(-1, 1), 10), and keypoints = exact projections + U(-2, 2) px noise.  `CASES` are its nine setups.
`scipy_solve` minimises the same gauge-fixed problem (the constancy masks the problem builder resolved) with
scipy.optimize.least_squares, using pixsfm.util.cameras.world_to_image and a rotation tangent per variable pose."""
import numpy as np

from pixsfm._pixsfm import _bundle_adjustment as ba
from pixsfm._pixsfm._capi import CAMERA_NUM_PARAMS
from pixsfm.util import colmap_types as ct
from pixsfm.util.cameras import world_to_image


def make_reconstruction(n_images, n_points=100, seed=0, model=2, noise=2.0):
    rng = np.random.default_rng(seed)
    rec = ct.Reconstruction()
    xyz = rng.uniform(-1.0, 1.0, (n_points, 3))
    for p in range(n_points):
        rec.add_point3D(p + 1, xyz[p])
    for i in range(n_images):
        params = {0: [1200.0, 500.0, 500.0], 1: [1200.0, 1210.0, 500.0, 500.0], 2: [1200.0, 500.0, 500.0, 0.0],
                  3: [1200.0, 500.0, 500.0, 0.0, 0.0], 4: [1200.0, 1210.0, 500.0, 500.0, 0.01, -0.01, 1e-3, -1e-3],
                  5: [1200.0, 1210.0, 500.0, 500.0, 0.01, -0.01, 1e-3, -1e-3],
                  6: [1200.0, 1210.0, 500.0, 500.0, 0.01, -0.01, 1e-3, -1e-3, 1e-3, 0.0, 0.0, 0.0]}[model]
        rec.add_camera(ct.Camera(i + 1, model, 1000, 1000, params))
        q = np.array([1.0, 0.0, 0.0, 0.0])
        t = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), 10.0])
        xy = world_to_image(model, params, q, t, xyz) + rng.uniform(-noise, noise, (n_points, 2))
        rec.add_image(ct.Image(i + 1, str(i), i + 1, q, t, [ct.Point2D(v) for v in xy]))
        for p in range(n_points):
            rec.add_observation(p + 1, i + 1, p)
    return rec


def _setup(images, const_poses=(), const_tvec=None, const_cameras=(), var_points=(), const_points=()):
    s = ba.BundleAdjustmentSetup()
    s.add_images(images)
    for i in const_poses:
        s.set_constant_pose(i)
    if const_tvec:
        s.set_constant_tvec(*const_tvec)
    for c in const_cameras:
        s.set_constant_camera(c)
    for p in var_points:
        s.add_variable_point(p)
    for p in const_points:
        s.add_constant_point(p)
    return s


# name -> (n_images, setup factory, BundleOptimizerOptions overrides): the cases of bundle_optimizer_test.cc
CASES = {
    "two_view": (2, lambda: _setup([1, 2], [1], (2, [0])), {}),
    "two_view_constant_camera": (2, lambda: _setup([1, 2], [1, 2], None, [1]), {}),
    "partially_contained_tracks": (3, lambda: _setup([1, 2], [1, 2]), {}),
    "partially_contained_tracks_force_point": (3, lambda: _setup([1, 2], [1, 2], None, (), [2], [3]), {}),
    "constant_points": (2, lambda: _setup([1, 2], [1, 2], None, (), (), [2, 3]), {}),
    "variable_image": (3, lambda: _setup([1, 2, 3], [1], (2, [0])), {}),
    "constant_focal_length": (2, lambda: _setup([1, 2], [1], (2, [0])), {"refine_focal_length": False}),
    "variable_principal_point": (2, lambda: _setup([1, 2], [1], (2, [0])), {"refine_principal_point": True}),
    "constant_extra_param": (2, lambda: _setup([1, 2], [1], (2, [0])), {"refine_extra_params": False}),
}


def case(name, seed=0):
    """-> (reconstruction, setup, BundleOptimizerOptions with the trivial loss of the reference's TestBA)"""
    n_images, make_setup, over = CASES[name]
    opts = ba.BundleOptimizerOptions(dict(over, loss={"name": "trivial", "params": []}, print_summary=False))
    return make_reconstruction(n_images, seed=seed), make_setup(), opts


def _qplus(q, d):
    n = np.linalg.norm(d)
    if n == 0.0:
        return q.copy()
    z = np.concatenate([[np.cos(n)], np.sin(n) / n * d])
    return np.array([z[0] * q[0] - z[1] * q[1] - z[2] * q[2] - z[3] * q[3],
                     z[0] * q[1] + z[1] * q[0] + z[2] * q[3] - z[3] * q[2],
                     z[0] * q[2] - z[1] * q[3] + z[2] * q[0] + z[3] * q[1],
                     z[0] * q[3] + z[1] * q[2] - z[2] * q[1] + z[3] * q[0]])


def scipy_solve(prob, start=None):
    """a least-squares optimum (trivial loss) of the problem by scipy, from the problem's parameters or from `start`
    = (cam_params, qvec, tvec, xyz) -> the same tuple"""
    from scipy.optimize import least_squares
    cam0, q0, t0, X0 = (np.array(a, np.float64) for a in (start or (prob.cam_params, prob.qvec, prob.tvec, prob.xyz)))
    blocks = []     # (kind, index, entries)
    for i in range(len(q0)):
        if not prob.pose_const[i]:
            blocks.append(("rot", i, 3))
            free_t = [k for k in range(3) if not (int(prob.tvec_const_mask[i]) >> k) & 1]
            if free_t:
                blocks.append(("t", i, free_t))
    for c in range(len(cam0)):
        k = CAMERA_NUM_PARAMS[int(prob.cam_model[c])]
        free = [j for j in range(k) if not (int(prob.cam_const_mask[c]) >> j) & 1]
        if free:
            blocks.append(("cam", c, free))
    for p in range(len(X0)):
        if not prob.point_const[p]:
            blocks.append(("X", p, 3))

    def unpack(v):
        cam, q, t, X = cam0.copy(), q0.copy(), t0.copy(), X0.copy()
        o = 0
        for kind, i, e in blocks:
            n = 3 if kind in ("rot", "X") else len(e)
            seg = v[o:o + n]; o += n
            if kind == "rot":
                q[i] = _qplus(q0[i], seg)
            elif kind == "t":
                t[i, e] = t0[i, e] + seg
            elif kind == "cam":
                cam[i, e] = cam0[i, e] + seg
            else:
                X[i] = X0[i] + seg
        return cam, q, t, X

    def residuals(v):
        cam, q, t, X = unpack(v)
        r = np.empty((prob.n_obs, 2))
        for i in range(len(q)):
            sel = np.flatnonzero(prob.obs_img == i)
            c = int(prob.img_cam[i]); model = int(prob.cam_model[c])
            r[sel] = world_to_image(model, cam[c, :CAMERA_NUM_PARAMS[model]], q[i], t[i], X[prob.obs_pt[sel]]) - prob.obs_xy[sel]
        return r.reshape(-1)

    n = sum(3 if kind in ("rot", "X") else len(e) for kind, _, e in blocks)
    sol = least_squares(residuals, np.zeros(n), method="lm", xtol=1e-14, ftol=1e-14, gtol=1e-14, max_nfev=100 * (n + 1))
    cam, q, t, X = unpack(sol.x)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return cam, q, t, X


def geometric_problem(rec, setup, options):
    """the BAProblem GeometricBundleOptimizer builds (host only: pxr_problem_build)"""
    prob, ir = ba.build_problem(rec, None, setup, options)
    return prob, ir


def assert_close_to(prob_params, ref, tol=1e-4):
    cam, q, t, X = prob_params
    rc, rq, rt, rX = ref
    qs = q * np.sign(np.sum(q * rq, axis=1, keepdims=True))
    np.testing.assert_allclose(cam[:, 0], rc[:, 0], rtol=tol, atol=0)        # focal lengths: relative, as the GPU tests
    np.testing.assert_allclose(cam[:, 1:], rc[:, 1:], atol=tol, rtol=0)
    np.testing.assert_allclose(qs, rq, atol=tol, rtol=0)
    np.testing.assert_allclose(t, rt, atol=tol, rtol=0)
    np.testing.assert_allclose(X, rX, atol=tol, rtol=0)
