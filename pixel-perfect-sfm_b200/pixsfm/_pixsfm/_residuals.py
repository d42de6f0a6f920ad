"""Mirror of `pixsfm._pixsfm._residuals` (pixsfm/residuals/bindings.cc:14-30): the cost-functor factories.

The reference hands pyceres users a `ceres::CostFunction*`; here a factory returns an evaluate-only object with the
same construction arguments and the same parameter-block order as the functor's `operator()`
(residuals/src/feature_reference.h:98-137: `(qvec[4], tvec[3], xyz[3], cam[k])`; constant pose, :157-207:
`(xyz[3], cam[k])`; geometric, residuals/src/geometric.h:16-41 = colmap::BundleAdjustmentCostFunction).
`evaluate(*parameter_blocks)` = `ceres::CostFunction::Evaluate`: residuals [num_residuals] and one row-major Jacobian
[num_residuals, block_size] per parameter block, AMBIENT coordinates (4 quaternion columns, as Jets give them).

All arithmetic runs in libpxr.so on the GPU (pxr_ba_evaluate_jacobians over a one-observation problem): the bicubic
kernel K1 writes r and G = [dr/du, dr/dv], the projection kernel K0 writes P = d(u,v)/d(rotation tangent, t, X, cam);
this layer only multiplies the two factors and maps the 3 tangent columns to the 4 quaternion columns.

Registered dimensions: the reference registers (CHANNELS, N_NODES) = (128,1) and (1,1) and throws
"Unsupported dimensions (CHANNELS,N_NODES)." for the rest (feature_reference.h:273-283); the device kernels exist for
every channel count of the BA path, so 1, 3, 4, 8, 16, 32, 64, 128, 256 with one node are accepted.
`FeatureMetricCostFunctor` (patch-warp / NCC, N_NODES=16, featuremetric.h:342-377) is outside SURVEY section 8 and
raises the same exception the reference raises for an unregistered combination."""
import numpy as np

from . import _capi, _engine
from ._base import InterpolationConfig

_CHANNELS = (1, 3, 4, 8, 16, 32, 64, 128, 256)


def _interp(cfg):
    cfg = cfg if isinstance(cfg, InterpolationConfig) else InterpolationConfig(cfg)
    cfg.validate_for_device()
    return cfg


def _tangent_to_ambient(q):
    """3x4 matrix E/|q| with d(tangent) = E dq / |q|: the left-multiplicative QuaternionManifold tangent delta of
    q' = exp(delta) (x) q as a function of an ambient change dq of the (normalised-inside-the-functor) quaternion:
    delta = vec(dq^ (x) q^*), q^ = q/|q|;  E q^ = 0, so the radial component drops out as it does under the Jets."""
    n = np.linalg.norm(q)
    w, v = q[0] / n, np.asarray(q[1:]) / n
    vx = np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])
    E = np.concatenate([-v.reshape(3, 1), w * np.eye(3) + vx], axis=1)
    return E / n


class _FunctorBase:
    def parameter_block_sizes(self):
        return list(self._blocks)

    def num_residuals(self):
        return self._nres

    def __call__(self, *blocks):
        return self.evaluate(*blocks)[0]


class _FeatureReferenceFunctor(_FunctorBase):
    def __init__(self, camera_model_id, patch, reference_descriptor, interpolation_config, qvec=None, tvec=None,
                 use_reference=True):
        self.interp = _interp(interpolation_config)
        self.model = int(camera_model_id)
        if self.model not in _capi.CAMERA_NUM_PARAMS:
            raise ValueError("unknown camera model id %d" % self.model)
        self.k = _capi.CAMERA_NUM_PARAMS[self.model]
        data = np.ascontiguousarray(patch.data)
        if data.ndim != 3:
            raise ValueError("patch must be [H,W,C]")
        channels, n_nodes = data.shape[2], len(self.interp.nodes)
        ref = np.asarray(reference_descriptor, np.float64)
        ref = ref.reshape(1, -1) if ref.ndim == 1 else ref
        if ref.shape[0] != n_nodes or ref.shape[1] != channels:      # THROW_CHECK_EQ(rows, n_nodes) / (cols, channels)
            raise ValueError("reference_descriptor must be [n_nodes, channels]")
        if n_nodes != 1 or channels not in _CHANNELS:
            raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")
        self.patch, self._data = patch, data
        self.ref = ref[0].copy() if use_reference else None
        self.const_pose = qvec is not None
        self.qvec = None if qvec is None else np.array(qvec, np.float64).reshape(4)
        self.tvec = None if tvec is None else np.array(tvec, np.float64).reshape(3)
        self._nres = channels
        self._blocks = [3, self.k] if self.const_pose else [4, 3, 3, self.k]

    def _problem(self, q, t, X, cam):
        return _capi.BAProblem(cam_model=[self.model], cam_params=[np.asarray(cam, np.float64)], cam_const_mask=[0],
                               qvec=[q], tvec=[t], img_cam=[0], pose_const=[0], tvec_const_mask=[0], xyz=[X],
                               point_const=[0], obs_img=[0], obs_pt=[0], patches=self._data[None],
                               corner=[np.asarray(self.patch.corner, np.int32)], scale=[np.asarray(self.patch.scale, np.float64)],
                               refs=None if self.ref is None else self.ref[None],
                               upsampling_factor=getattr(self.patch, "upsampling_factor", 1.0))

    def evaluate(self, *blocks):
        if len(blocks) != len(self._blocks):
            raise ValueError("expected %d parameter blocks %s" % (len(self._blocks), self._blocks))
        if self.const_pose:
            q, t = self.qvec, self.tvec
            X, cam = (np.asarray(b, np.float64).reshape(-1) for b in blocks)
        else:
            q, t, X, cam = (np.asarray(b, np.float64).reshape(-1) for b in blocks)
        if len(q) != 4 or len(t) != 3 or len(X) != 3 or len(cam) != self.k:
            raise ValueError("parameter block sizes must be %s" % self._blocks)
        ic = _capi.default_interp(self.interp.l2_normalize, self.interp.use_float_simd)
        h = _engine.BAHandle(self._problem(q, t, X, cam), ic, _capi.default_ba_options(use_inner_iterations=0))
        try:
            out = h.evaluate_jacobians()
        finally:
            h.close()
        r, G, P = out["residuals"][0], out["grad"][0], out["juv"][0]       # [C], [2,C], [2,9+K]
        J = G.T @ P                                                          # [C, 9+K]: rot3 | t3 | X3 | cam
        J_X, J_cam = J[:, 6:9].copy(), J[:, 9:9 + self.k].copy()
        if self.const_pose:
            return r, [J_X, J_cam]
        return r, [J[:, 0:3] @ _tangent_to_ambient(q), J[:, 3:6].copy(), J_X, J_cam]


def FeatureReferenceCostFunctor(camera_model_id, patch, reference_descriptor, interpolation_config):
    """residuals/bindings.cc:15-16 -> CreateFeatureReferenceCostFunctor<dtype> (feature_reference.h:256-287).
    As in the reference, the descriptor is only shape-checked: the factory passes `nullptr` for it (:269-270), so the
    functor returns the interpolated (L2-normalised) features themselves, not `f - reference`."""
    return _FeatureReferenceFunctor(camera_model_id, patch, reference_descriptor, interpolation_config, use_reference=False)


def FeatureReferenceConstantPoseCostFunctor(camera_model_id, qvec, tvec, patch, reference_descriptor, interpolation_config):
    """residuals/bindings.cc:17-18 -> CreateFeatureReferenceConstantPoseCostFunctor<dtype> (feature_reference.h:289-321):
    parameter blocks (xyz[3], cam[k]); residual = f - reference."""
    return _FeatureReferenceFunctor(camera_model_id, patch, reference_descriptor, interpolation_config, qvec=qvec, tvec=tvec)


def FeatureMetricCostFunctor(camera, patch, src_camera, src_patch, interpolation_config):
    """residuals/bindings.cc:19 -> CreateFeatureMetricCostFunctor<dtype> (featuremetric.h:342-377): the patch-warp
    functor, registered for (3,16) and (1,16) only.  Not on the hot path (SURVEY section 8: unranked)."""
    raise ValueError("Unsupported dimensions (CHANNELS,N_NODES).")


class _GeometricFunctor(_FunctorBase):
    """colmap::BundleAdjustmentCostFunction / ...ConstantPoseCostFunction: residual = WorldToImage(...) - point2D"""

    def __init__(self, camera_model_id, point2D, qvec=None, tvec=None):
        self.model = int(camera_model_id)
        if self.model not in _capi.CAMERA_NUM_PARAMS:
            raise ValueError("unknown camera model id %d" % self.model)
        self.k = _capi.CAMERA_NUM_PARAMS[self.model]
        self.point2D = np.array(point2D, np.float64).reshape(2)
        self.const_pose = qvec is not None
        self.qvec = None if qvec is None else np.array(qvec, np.float64).reshape(4)
        self.tvec = None if tvec is None else np.array(tvec, np.float64).reshape(3)
        self._nres = 2
        self._blocks = [3, self.k] if self.const_pose else [4, 3, 3, self.k]

    def evaluate(self, *blocks):
        if len(blocks) != len(self._blocks):
            raise ValueError("expected %d parameter blocks %s" % (len(self._blocks), self._blocks))
        if self.const_pose:
            q, t = self.qvec, self.tvec
            X, cam = (np.asarray(b, np.float64).reshape(-1) for b in blocks)
        else:
            q, t, X, cam = (np.asarray(b, np.float64).reshape(-1) for b in blocks)
        # a one-observation geometric problem: the residual comes from the geometric evaluation kernel, P = d(xy)/d(theta)
        # from K0 (G is the identity)
        prob = _capi.BAProblem(cam_model=[self.model], cam_params=[cam], cam_const_mask=[0], qvec=[q], tvec=[t], img_cam=[0],
                               pose_const=[0], tvec_const_mask=[0], xyz=[X], point_const=[0], obs_img=[0], obs_pt=[0],
                               patches=None, corner=None, scale=None, obs_xy=self.point2D[None])
        h = _engine.BAHandle(prob, options=_capi.default_ba_options(use_inner_iterations=0))
        try:
            out = h.evaluate_jacobians()
        finally:
            h.close()
        P = out["juv"][0]
        r = out["residuals"][0]
        J_X, J_cam = P[:, 6:9].copy(), P[:, 9:9 + self.k].copy()
        if self.const_pose:
            return r, [J_X, J_cam]
        return r, [P[:, 0:3] @ _tangent_to_ambient(q), P[:, 3:6].copy(), J_X, J_cam]


def GeometricCostFunctor(camera_model_id, point2D):
    """residuals/bindings.cc:26 (geometric.h:16-27)"""
    return _GeometricFunctor(camera_model_id, point2D)


def GeometricConstantPoseCostFunctor(camera_model_id, qvec, tvec, point2D):
    """residuals/bindings.cc:27-28 (geometric.h:29-41)"""
    return _GeometricFunctor(camera_model_id, point2D, qvec=qvec, tvec=tvec)
