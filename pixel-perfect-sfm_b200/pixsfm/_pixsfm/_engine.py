"""Thin object wrappers over the C-ABI handles (plumbing only; no arithmetic)."""
import ctypes as C

import numpy as np

from . import _capi


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class BAHandle:
    """pxr_ba: a BA problem resident on the device (== FeatureReferenceBundleOptimizer.set_up; a problem with obs_xy
    is a geometric one, == GeometricBundleOptimizer.set_up)."""

    def __init__(self, problem, interp=None, options=None, ctx=None):
        self.ctx = ctx or _capi.default_context()
        self.lib = self.ctx.lib
        self.problem = problem
        self.interp = interp or _capi.default_interp()
        self.options = options or _capi.default_ba_options()
        self._desc = problem.desc()
        self.handle = C.c_void_p()
        if problem.obs_xy is not None:      # geometric problem: pxr_ba_create_geometric (the interpolation is not used)
            _capi.check(self.lib.pxr_ba_create_geometric(self.ctx.handle, C.byref(self._desc), _p(problem.obs_xy),
                                                         C.byref(self.options), C.byref(self.handle)))
        else:
            _capi.check(self.lib.pxr_ba_create(self.ctx.handle, C.byref(self._desc), C.byref(self.interp),
                                               C.byref(self.options), C.byref(self.handle)))

    def close(self):
        if self.handle:
            self.lib.pxr_ba_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def evaluate(self, residuals=False):
        n = self.problem.n_obs
        out = dict(sq_norm=np.zeros(n), gtr=np.zeros((n, 2)), gtg=np.zeros((n, 3)), xy=np.zeros((n, 2)))
        res = np.zeros((n, self.problem.residuals_per_obs)) if residuals else None
        cost = C.c_double()
        _capi.check(self.lib.pxr_ba_evaluate(self.handle, _p(out["sq_norm"]), _p(out["gtr"]), _p(out["gtg"]),
                                             _p(out["xy"]), _p(res), C.byref(cost)))
        out["cost"] = cost.value
        if residuals:
            out["residuals"] = res
        return out

    def evaluate_jacobians(self):
        """residuals [n,C], grad [n,2,C] (d r/d u, d r/d v), juv [n,2,9+K] (d(u,v)/d(rot3|t3|X3|cam K)), xy [n,2]:
        pxr_ba_evaluate_jacobians, the factored form of every block's ceres-style Jacobian (J = grad^T-rows x juv)"""
        n, Cc = self.problem.n_obs, self.problem.residuals_per_obs
        kmax = int(np.asarray(self.problem.cam_params).shape[1])
        res, grad, xy = np.zeros((n, Cc)), np.zeros((n, 2, Cc)), np.zeros((n, 2))
        juv = np.zeros((n, 2, 9 + kmax)); w = C.c_int32()
        _capi.check(self.lib.pxr_ba_evaluate_jacobians(self.handle, _p(res), _p(grad), _p(juv), C.byref(w), _p(xy)))
        juv = juv.reshape(-1)[: n * 2 * w.value].reshape(n, 2, w.value)
        return dict(residuals=res, grad=grad, juv=juv, xy=xy)

    def debug_linearize(self, nc, nl, radius=1e4, dense=True):
        """dense=False leaves Hcc / S out (the block-sparse and block-mode paths never form them)"""
        npts = len(self.problem.xyz)
        out = dict(gc=np.zeros(nc), Hpp=np.zeros((npts, 3, 3)), gp=np.zeros((npts, 3)), rhs=np.zeros(nc), delta=np.zeros(nl))
        if dense:
            out.update(Hcc=np.zeros((nc, nc)), S=np.zeros((nc, nc)))
        cost = C.c_double(); mcc = C.c_double()
        _capi.check(self.lib.pxr_ba_debug_linearize(self.handle, C.c_double(radius), C.byref(cost), _p(out.get("Hcc")),
                                                    _p(out["gc"]), _p(out["Hpp"]), _p(out["gp"]), _p(out.get("S")),
                                                    _p(out["rhs"]) if dense else None, _p(out["delta"]), C.byref(mcc)))
        out["cost"] = cost.value; out["model_cost_change"] = mcc.value
        return out

    def debug_reduced_solve(self, S, rhs, factor=False):
        """pxr_ba_debug_reduced_solve: the handle's reduced-system solver on S x = rhs (S [nc, nc], lower triangle read)
        -> dict(x, status (_capi.REDUCED_SOLVE_*), linear_iterations, factor [nc+1, nc] on the Cholesky paths when asked)"""
        S = np.ascontiguousarray(S, np.float64); rhs = np.ascontiguousarray(rhs, np.float64)
        nc = len(rhs)
        if S.shape != (nc, nc):
            raise ValueError("S must be [nc, nc] for rhs of length nc")
        x = np.zeros(nc); fac = np.full((nc + 1, nc), np.nan) if factor else None
        status = C.c_int(); iters = C.c_int()
        _capi.check(self.lib.pxr_ba_debug_reduced_solve(self.handle, _p(S), _p(rhs), _p(x), _p(fac), C.byref(status),
                                                        C.byref(iters)))
        out = dict(x=x, status=status.value, linear_iterations=iters.value)
        if factor:
            out["factor"] = fac
        return out

    def debug_inner_iterations(self):
        _capi.check(self.lib.pxr_ba_debug_inner_iterations(self.handle))

    def debug_eval_list(self, items, count_on_device=False):
        """[n_obs, 8] per-observation K1 record after K0 + K1 over the observation list `items` (NaN rows elsewhere)"""
        items = np.ascontiguousarray(items, np.int64)
        out = np.empty((self.problem.n_obs, 8))
        _capi.check(self.lib.pxr_ba_debug_eval_list(self.handle, _p(items), C.c_int64(len(items)),
                                                    int(bool(count_on_device)), _p(out)))
        return out

    def debug_project_point(self, items, count_on_device=False):
        """the rounds' point-only projection over the observation list `items` next to the full one: uv [n_obs, 2] and
        jpt [n_obs, 2, 3] (d(uv)/dX, NaN rows outside the list) and uv_full [n_obs, 2] of the full projection"""
        items = np.ascontiguousarray(items, np.int64)
        n = self.problem.n_obs
        uv, jpt, uv_full = np.empty((n, 2)), np.empty((n, 2, 3)), np.empty((n, 2))
        _capi.check(self.lib.pxr_ba_debug_project_point(self.handle, _p(items), C.c_int64(len(items)),
                                                        int(bool(count_on_device)), _p(uv), _p(jpt), _p(uv_full)))
        return dict(uv=uv, jpt=jpt, uv_full=uv_full)

    def debug_project(self, jac):
        """K0 over all observations, cost-only (jac False) or with Jacobians: uv [n_obs, 2] and xy [n_obs, 2]"""
        n = self.problem.n_obs
        uv, xy = np.empty((n, 2)), np.empty((n, 2))
        _capi.check(self.lib.pxr_ba_debug_project(self.handle, int(bool(jac)), _p(uv), _p(xy)))
        return dict(uv=uv, xy=xy)

    def debug_inner_capture(self, enable=True):
        """keep every round's lists in the batched inner iterations that follow (the host waits for every round)"""
        _capi.check(self.lib.pxr_ba_debug_inner_capture(self.handle, int(bool(enable))))

    def debug_inner_round_lists(self):
        """the captured rounds of the most recent batched inner iterations: per round a dict of its point list, its
        observation list and, per listed point, whether the round's step kernel kept it active"""
        out = []
        for r in range(10 ** 6):
            npt, nob = C.c_int64(), C.c_int64()
            if self.lib.pxr_ba_debug_inner_round_lists(self.handle, r, None, None, None, C.byref(npt), C.byref(nob)) != 0:
                break
            pl, ol, act = np.empty(npt.value, np.int64), np.empty(nob.value, np.int64), np.empty(npt.value, np.uint8)
            _capi.check(self.lib.pxr_ba_debug_inner_round_lists(self.handle, r, _p(pl), _p(ol), _p(act), None, None))
            out.append(dict(points=pl, obs=ol, active=act.astype(bool)))
        return out

    def debug_eval_records(self, mode=1):
        """[n_obs, 8] per-observation K1 record after K0 + K1 over all observations, mode 0 (cost only: column 0, NaN
        elsewhere) or 1 (Jacobian)"""
        out = np.empty((self.problem.n_obs, 8))
        _capi.check(self.lib.pxr_ba_debug_eval_records(self.handle, int(mode), _p(out)))
        return out

    def debug_inner_rounds(self, enable_timing=-1, capacity=64):
        """rounds of the most recent batched inner iterations: [n, 2] (active observations, active points) per round and
        the per-round device ms (-1 where round timing was off); enable_timing >= 0 switches round timing for later calls"""
        counts = np.zeros((capacity, 2), np.uint64); ms = np.zeros(capacity); n = C.c_int()
        _capi.check(self.lib.pxr_ba_debug_inner_rounds(self.handle, int(enable_timing), int(capacity), _p(counts), _p(ms),
                                                       C.byref(n)))
        k = min(n.value, capacity)
        return counts[:k], ms[:k]

    def debug_inner_round_split(self, capacity=64):
        """[n, 3] stream ms of each round of the most recent batched inner iterations, split at the ends of K0, K1 and the
        step kernel (-1 where round timing was off during that call)"""
        ms = np.zeros((capacity, 3)); n = C.c_int()
        _capi.check(self.lib.pxr_ba_debug_inner_round_split(self.handle, int(capacity), _p(ms), C.byref(n)))
        return ms[:min(n.value, capacity)]

    def solve(self, capacity=512):
        s = _capi.make_summary(capacity)
        _capi.check(self.lib.pxr_ba_solve(self.handle, C.byref(s)))
        return _capi.summary_to_dict(s)

    def iterate(self, n, capacity=512):
        s = _capi.make_summary(capacity)
        _capi.check(self.lib.pxr_ba_iterate(self.handle, int(n), C.byref(s)))
        return _capi.summary_to_dict(s)

    def kernel_timing(self, enable=-1, which=1, read=True):
        ms = C.c_double(); cnt = C.c_int()
        _capi.check(self.lib.pxr_ba_kernel_timing(self.handle, int(enable), int(which),
                                                  C.byref(ms) if read else None, C.byref(cnt) if read else None))
        return ms.value, cnt.value

    def read_params(self):
        """Copies the current device parameters back into the BAProblem arrays."""
        p = self.problem
        _capi.check(self.lib.pxr_ba_read_params(self.handle, _p(p.cam_params), _p(p.qvec), _p(p.tvec), _p(p.xyz)))

    def reset(self, cam_params, qvec, tvec, xyz):
        """pxr_ba_reset: back to the given parameters, LM trajectory forgotten (patches / work space stay resident)"""
        arrs = [np.ascontiguousarray(a, np.float64) for a in (cam_params, qvec, tvec, xyz)]
        _capi.check(self.lib.pxr_ba_reset(self.handle, *[_p(a) for a in arrs]))

    def time_stage(self, stage, iters):
        ms = C.c_double()
        _capi.check(self.lib.pxr_ba_time_stage(self.handle, int(stage), int(iters), C.byref(ms)))
        return ms.value


def k1_half_warps(dtype, channels, n_items, ctx=None):
    """pxr_fm_k1_half_warps: half-warps of the K1 launch over n_items items of a (dtype, channels) patch slab"""
    ctx = ctx or _capi.default_context()
    hw = C.c_int64()
    _capi.check(ctx.lib.pxr_fm_k1_half_warps(ctx.handle, _capi.DTYPE_IDS[np.dtype(dtype)], int(channels),
                                              C.c_int64(int(n_items)), C.byref(hw)))
    return hw.value


def ba_run(problem, interp=None, options=None, ctx=None, capacity=512):
    """pxr_ba_run (pxr_ba_run_geometric for a problem with obs_xy): upload, solve, write the refined parameters back
    into `problem` (in place)."""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    options = options or _capi.default_ba_options()
    d = problem.desc()
    s = _capi.make_summary(capacity)
    if problem.obs_xy is not None:          # geometric problem: pxr_ba_run_geometric
        _capi.check(ctx.lib.pxr_ba_run_geometric(ctx.handle, C.byref(d), _p(problem.obs_xy), C.byref(options), C.byref(s)))
    else:
        _capi.check(ctx.lib.pxr_ba_run(ctx.handle, C.byref(d), C.byref(interp), C.byref(options), C.byref(s)))
    return _capi.summary_to_dict(s)


def qba_run(batch, interp=None, options=None, ctx=None, capacity=0):
    """pxr_qba_run: solves every query of a _capi.QBABatch and writes the refined qvec / tvec / cam_params back into
    it (in place).  -> (list of per-query dicts with the pxr_qba_result fields and, with capacity > 0, `iterations`,
    dict(n_waves, h2d_bytes, solve_time_s, total_time_s, kernel_launches, message))"""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    options = options or _capi.default_ba_options(use_inner_iterations=0)
    d = batch.desc()
    nq = batch.n_queries
    res = (_capi.QBAResult * max(nq, 1))()
    its = (_capi.IterationSummary * max(nq * capacity, 1))()
    nw = C.c_int32()
    tot = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_qba_run(ctx.handle, C.byref(d), C.byref(interp), C.byref(options), res,
                                    its if capacity else None, int(capacity), C.byref(nw), C.byref(tot)))
    out = []
    for q in range(nq):
        r = {f[0]: getattr(res[q], f[0]) for f in _capi.QBAResult._fields_}
        if capacity:
            k = min(r["num_iterations"], capacity)
            r["iterations"] = [{f[0]: getattr(its[q * capacity + i], f[0]) for f in _capi.IterationSummary._fields_}
                               for i in range(k)]
        out.append(r)
    t = _capi.summary_to_dict(tot)
    return out, dict(n_waves=nw.value, h2d_bytes=t["h2d_bytes"], solve_time_s=t["solve_time_s"],
                     total_time_s=t["total_time_s"], kernel_launches=t["kernel_launches"], message=t["message"])


def qba_plan_waves(batch):
    """pxr_qba_plan_waves: (first query of every wave + the end, uploaded bytes per wave) — host computation"""
    lib = _capi.load_lib()
    d = batch.desc()
    nq = batch.n_queries
    begin = np.zeros(nq + 1, np.int32); nbytes = np.zeros(max(nq, 1)); nw = C.c_int32()
    _capi.check(lib.pxr_qba_plan_waves(C.byref(d), _p(begin), C.byref(nw), _p(nbytes)))
    return begin[:nw.value + 1].copy(), nbytes[:nw.value].copy()


def qba_debug_linearize(batch, interp=None, options=None, ctx=None):
    """pxr_qba_debug_linearize: every query's cost, J^T J (lower, [nq, 18, 18]) and J^T r ([nq, 18]) at the batch's
    parameters, and every block's projection xy [n_obs, 2] and K1 record [n_obs, 8]"""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    options = options or _capi.default_ba_options(use_inner_iterations=0)
    d = batch.desc()
    nq, m = batch.n_queries, int(batch.obs_begin[-1])
    out = dict(cost=np.zeros(nq), H=np.zeros((nq, 18, 18)), g=np.zeros((nq, 18)), xy=np.zeros((m, 2)),
               rec=np.zeros((m, 8)))
    _capi.check(ctx.lib.pxr_qba_debug_linearize(ctx.handle, C.byref(d), C.byref(interp), C.byref(options),
                                                _p(out["cost"]), _p(out["H"]), _p(out["g"]), _p(out["xy"]),
                                                _p(out["rec"])))
    return out


def pnp_run(batch, options=None, ctx=None):
    """pxr_pnp_run: absolute pose estimation for every query of a _capi.PnPBatch, one launch for the batch; writes qvec /
    tvec (successful queries), cam_params (when refinement refines intrinsics) and inlier_mask into it.  -> (list of
    per-query dicts with the pxr_pnp_result fields, dict(solve_time_s, total_time_s, kernel_launches, h2d_bytes))"""
    ctx = ctx or _capi.default_context()
    options = options or _capi.default_pnp_options()
    d = batch.desc()
    nq = batch.n_queries
    res = (_capi.PnPResult * max(nq, 1))()
    tot = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_pnp_run(ctx.handle, C.byref(d), C.byref(options), res, C.byref(tot)))
    out = [{f[0]: getattr(res[q], f[0]) for f in _capi.PnPResult._fields_} for q in range(nq)]
    t = _capi.summary_to_dict(tot)
    return out, dict(solve_time_s=t["solve_time_s"], total_time_s=t["total_time_s"], kernel_launches=t["kernel_launches"],
                     h2d_bytes=t["h2d_bytes"])


def pnp_debug_image_to_world(model, params, xy, ctx=None):
    """pxr_pnp_debug_image_to_world: the device's ImageToWorld of pixels xy [n, 2] -> [n, 2]"""
    ctx = ctx or _capi.default_context()
    p = np.zeros(_capi.PXR_MAX_CAM_PARAMS)
    p[:len(params)] = params
    xy = np.ascontiguousarray(xy, np.float64).reshape(-1, 2)
    out = np.zeros_like(xy)
    _capi.check(ctx.lib.pxr_pnp_debug_image_to_world(ctx.handle, C.c_int32(int(model)), _p(p), C.c_int64(len(xy)), _p(xy),
                                                     _p(out)))
    return out


def pnp_debug_p3p(x, X, ctx=None):
    """pxr_pnp_debug_p3p: the device's P3P of triplets x [n, 3, 2] (normalised) and X [n, 3, 3] -> (poses [n, 4, 7]
    (qvec with w >= 0 | tvec), n_sol [n])"""
    ctx = ctx or _capi.default_context()
    x = np.ascontiguousarray(x, np.float64).reshape(-1, 3, 2)
    X = np.ascontiguousarray(X, np.float64).reshape(-1, 3, 3)
    poses = np.zeros((len(x), 4, 7))
    n_sol = np.zeros(len(x), np.int32)
    _capi.check(ctx.lib.pxr_pnp_debug_p3p(ctx.handle, C.c_int64(len(x)), _p(x), _p(X), _p(poses), _p(n_sol)))
    return poses, n_sol


def _timing(tot):
    t = _capi.summary_to_dict(tot)
    return dict(solve_time_s=t["solve_time_s"], total_time_s=t["total_time_s"], kernel_launches=t["kernel_launches"],
                h2d_bytes=t["h2d_bytes"])


def tri_verify(scene, match_img, match_xy, match_noise, max_error=4.0, ctx=None):
    """pxr_tri_verify: geometric verification of matches against the known poses of a _capi.TriScene.  match_img [n, 2]
    image indices, match_xy [n, 4] pixels (x0, y0, x1, y1), match_noise [n, 2] -> (keep bool [n], err [n, 2] epipolar
    distances in the normalised plane, timing dict)"""
    ctx = ctx or _capi.default_context()
    mi = np.ascontiguousarray(match_img, np.int32).reshape(-1, 2)
    mx = np.ascontiguousarray(match_xy, np.float64).reshape(-1, 4)
    mn = np.ascontiguousarray(match_noise, np.float64).reshape(-1, 2)
    if not (len(mi) == len(mx) == len(mn)):
        raise ValueError("match_img, match_xy and match_noise differ in length")
    keep = np.zeros(len(mi), np.uint8)
    err = np.zeros((len(mi), 2))
    d = scene.desc()
    tot = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_tri_verify(ctx.handle, C.byref(d), C.c_int64(len(mi)), _p(mi), _p(mx), _p(mn),
                                       C.c_double(max_error), _p(keep), _p(err), C.byref(tot)))
    return keep.astype(bool), err, _timing(tot)


def tri_run(scene, options=None, ctx=None):
    """pxr_tri_run: robust triangulation of every track of a _capi.TriScene -> dict(xyz [nt, 3], status [nt] (TRI_*),
    n_inliers [nt], tri_angle [nt] degrees, obs_inlier bool [n_obs], obs_error [n_obs] pixels, timing)"""
    ctx = ctx or _capi.default_context()
    options = options or _capi.default_tri_options()
    nt, no = scene.n_tracks, int(scene.track_begin[-1])
    out = dict(xyz=np.zeros((nt, 3)), status=np.zeros(nt, np.int32), n_inliers=np.zeros(nt, np.int32),
               tri_angle=np.zeros(nt), obs_inlier=np.zeros(no, np.uint8), obs_error=np.zeros(no))
    d = scene.desc()
    tot = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_tri_run(ctx.handle, C.byref(d), C.byref(options), _p(out["xyz"]), _p(out["status"]),
                                    _p(out["n_inliers"]), _p(out["tri_angle"]), _p(out["obs_inlier"]), _p(out["obs_error"]),
                                    C.byref(tot)))
    out["obs_inlier"] = out["obs_inlier"].astype(bool)
    out["timing"] = _timing(tot)
    return out


def tri_evaluate(scene, xyz, ctx=None):
    """pxr_tri_evaluate: pixel reprojection errors [n_obs] (+inf behind the camera) and triangulation angles [nt]
    (degrees, every observation) of the points xyz [nt, 3] -> (obs_error, tri_angle, timing)"""
    ctx = ctx or _capi.default_context()
    xyz = np.ascontiguousarray(xyz, np.float64).reshape(-1, 3)
    if len(xyz) != scene.n_tracks:
        raise ValueError("xyz must hold one point per track")
    err, ang = np.zeros(int(scene.track_begin[-1])), np.zeros(scene.n_tracks)
    d = scene.desc()
    tot = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_tri_evaluate(ctx.handle, C.byref(d), _p(xyz), _p(err), _p(ang), C.byref(tot)))
    return err, ang, _timing(tot)


class PinnedArray:
    """A numpy array in pinned (page-locked, device-mapped) host memory from pxr_host_alloc_pinned: the patch source
    pxr_ba_run reads tap windows from directly (window residency, csrc/pxr_resident.cuh) and full-rate DMA otherwise.
    `array` is the numpy view; the memory is released by close() / when the object dies."""

    def __init__(self, shape, dtype, ctx=None):
        self.ctx = ctx or _capi.default_context()
        self.array = None
        dtype = np.dtype(dtype)
        nbytes = int(np.prod(shape)) * dtype.itemsize
        self._ptr = C.c_void_p()
        _capi.check(self.ctx.lib.pxr_host_alloc_pinned(C.byref(self._ptr), C.c_size_t(max(nbytes, 1))))
        buf = (C.c_uint8 * max(nbytes, 1)).from_address(self._ptr.value)
        self.array = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def close(self):
        if self._ptr:
            self.array = None
            self.ctx.lib.pxr_host_free_pinned(self._ptr)
            self._ptr = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def refs_compute(problem, interp=None, loss_type=1, loss_scale=0.25, iters=100, ctx=None):
    """pxr_refs_compute == ReferenceExtractor.run: -> (refs [n_points,C] f64, src_obs [n_points])"""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    d = problem.desc()
    refs = np.zeros((len(problem.xyz), problem.channels))
    src = np.zeros(len(problem.xyz), np.int64)
    s = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_refs_compute(ctx.handle, C.byref(d), C.byref(interp), int(loss_type), C.c_double(loss_scale),
                                         int(iters), _p(refs), _p(src), C.byref(s)))
    return refs, src


def obs_descriptors(problem, interp=None, ctx=None):
    """pxr_obs_descriptors: [n_obs, C] descriptors at the current projections (Reference.observations)"""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    d = problem.desc()
    out = np.zeros((problem.n_obs, problem.channels))
    _capi.check(ctx.lib.pxr_obs_descriptors(ctx.handle, C.byref(d), C.byref(interp), _p(out)))
    return out


def costmaps_compute(problem, interp=None, cfg=None, refs=None, to_host=True, to_device=False, ctx=None):
    """pxr_costmaps_compute == CostMapExtractor.run: reference extraction (unless cfg.compute_refs == 0) and one
    cost patch per observation patch.  -> dict(costmaps [n_patches,ph,pw,OC] in the patch dtype or None,
    device_ptr or None, refs [n_points,C], src_obs [n_points])"""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    cfg = cfg or _capi.default_costmap_config()
    d = problem.desc()
    n_points = len(problem.xyz)
    if refs is None:
        refs = np.zeros((n_points, problem.channels))
    else:
        refs = np.ascontiguousarray(refs, np.float64)
    src = np.full(n_points, -1, np.int64)
    oc = 3 if cfg.as_gradientfield else 1
    n_patches = d.n_patches if d.n_patches else d.n_obs
    out = np.zeros((n_patches, problem.ph, problem.pw, oc), problem.patch_np_dtype) if to_host else None
    dptr = C.c_void_p()
    s = _capi.make_summary(0)
    _capi.check(ctx.lib.pxr_costmaps_compute(ctx.handle, C.byref(d), C.byref(interp), C.byref(cfg), _p(refs), _p(src),
                                             _p(out) if to_host else None, C.byref(dptr) if to_device else None,
                                             C.byref(s)))
    return {"costmaps": out, "device_ptr": dptr.value if to_device else None, "refs": refs, "src_obs": src,
            "summary": _capi.summary_to_dict(s)}


def synth_patches_device(n_patches, ps, channels, uv0, field_id, seed=0, noise=0.01, ctx=None):
    """Device-side synthetic patch slab (fp16). Returns the device pointer (int)."""
    ctx = ctx or _capi.default_context()
    uv0 = np.ascontiguousarray(uv0, np.float64); field_id = np.ascontiguousarray(field_id, np.int64)
    out = C.c_void_p()
    _capi.check(ctx.lib.pxr_synth_patches_device(ctx.handle, C.byref(out), C.c_int64(n_patches), int(ps), int(channels),
                                                 _p(uv0), _p(field_id), C.c_uint64(seed), C.c_double(noise)))
    return out.value


def device_free(ptr, ctx=None):
    ctx = ctx or _capi.default_context()
    _capi.check(ctx.lib.pxr_device_free(ctx.handle, C.c_void_p(ptr)))


def memcpy_d2h(host_array, dev_ptr, nbytes, ctx=None):
    ctx = ctx or _capi.default_context()
    _capi.check(ctx.lib.pxr_memcpy_d2h(ctx.handle, _p(host_array), C.c_void_p(dev_ptr), C.c_size_t(nbytes)))


def ka_run(problem, interp=None, options=None, ctx=None):
    """pxr_ka_run == FeatureMetricKeypointOptimizer.run: refines problem.keypoints IN PLACE.  A _capi.QKABatch (one
    query-mode problem per query) is solved by pxr_qka_run, which also fills problem.results per query and adds
    `n_waves` to the summary."""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    options = options or _capi.default_ka_options()
    s = _capi.make_summary(0)
    if isinstance(problem, _capi.QKABatch):
        d = problem.qka_desc()
        res = (_capi.QKAResult * max(problem.n_queries, 1))()
        nw = C.c_int32()
        _capi.check(ctx.lib.pxr_qka_run(ctx.handle, C.byref(d), C.byref(interp), C.byref(options), res, C.byref(nw),
                                        C.byref(s)))
        problem.results = [{f[0]: getattr(res[q], f[0]) for f in _capi.QKAResult._fields_} for q in range(problem.n_queries)]
        out = _capi.summary_to_dict(s)
        out["n_waves"] = nw.value
        return out
    d = problem.desc()
    _capi.check(ctx.lib.pxr_ka_run(ctx.handle, C.byref(d), C.byref(interp), C.byref(options), C.byref(s)))
    return _capi.summary_to_dict(s)


def graph_labels(node_image, edge_src, edge_dst, edge_sim):
    """compute_track_labels / compute_score_labels / compute_root_labels on flat arrays (host, bit-exact)."""
    lib = _capi.load_lib()
    node_image = np.ascontiguousarray(node_image, np.int32)
    es = np.ascontiguousarray(edge_src, np.int64); ed = np.ascontiguousarray(edge_dst, np.int64)
    sim = np.ascontiguousarray(edge_sim, np.float64)
    n = len(node_image)
    tl = np.zeros(n, np.int64); sc = np.zeros(n); rt = np.zeros(n, np.uint8)
    _capi.check(lib.pxr_graph_track_labels(C.c_int64(n), _p(node_image), C.c_int64(len(es)), _p(es), _p(ed), _p(sim), _p(tl)))
    _capi.check(lib.pxr_graph_score_labels(C.c_int64(n), C.c_int64(len(es)), _p(es), _p(ed), _p(sim), _p(tl), _p(sc)))
    _capi.check(lib.pxr_graph_root_labels(C.c_int64(n), _p(tl), _p(sc), _p(rt)))
    return tl, sc, rt


def ka_problem_labels(track_labels, max_per_problem=50):
    lib = _capi.load_lib()
    tl = np.ascontiguousarray(track_labels, np.int64)
    out = np.zeros(len(tl), np.int32); nb = C.c_int32()
    _capi.check(lib.pxr_ka_problem_labels(C.c_int64(len(tl)), _p(tl), int(max_per_problem), _p(out), C.byref(nb)))
    return out, nb.value


def ka_shard_plan(problem_weight, world):
    """pxr_shard_ka_problems: rank of every packed KA problem (whole problems per rank, no collective needed)"""
    lib = _capi.load_lib()
    w = np.ascontiguousarray(problem_weight, np.int64)
    out = np.zeros(len(w), np.int32)
    _capi.check(lib.pxr_shard_ka_problems(C.c_int32(len(w)), _p(w), int(world), _p(out)))
    return out


def ba_estimate_device_bytes(problem, options=None):
    """pxr_ba_estimate_device_bytes: what the solve will take on the device (host computation) ->
    dict(patches, state, reduced_system, total) in bytes"""
    lib = _capi.load_lib()
    d = problem.desc()
    out = [C.c_double(), C.c_double(), C.c_double()]
    _capi.check(lib.pxr_ba_estimate_device_bytes(C.byref(d), C.byref(options) if options is not None else None,
                                                 C.byref(out[0]), C.byref(out[1]), C.byref(out[2])))
    p, s, r = (o.value for o in out)
    return {"patches": p, "state": s, "reduced_system": r, "total": p + s + r}


class DeviceSlab:
    """A [N,H,W,C] array in device memory owned by libpxr (returned by pxr_extract_patches); exposes the CUDA array
    interface, so FeatureMap / DevicePatches take it like a torch tensor.  Freed with the object."""

    def __init__(self, ptr, shape, dtype, ctx):
        self.ptr, self.shape, self.dtype, self._ctx = int(ptr), tuple(int(v) for v in shape), np.dtype(dtype), ctx
        self.__cuda_array_interface__ = {"shape": self.shape, "typestr": self.dtype.str, "data": (self.ptr, False),
                                         "version": 3, "strides": None}

    def __del__(self):
        try:
            if self.ptr:
                self._ctx.lib.pxr_device_free(self._ctx.handle, C.c_void_p(self.ptr))
                self.ptr = 0
        except Exception:      # interpreter shutdown
            pass


def extract_patches(dense, corners, patch_size, l2_normalize=True, out_dtype=np.float16, channels_first=True,
                    to_host=False, ctx=None):
    """pxr_extract_patches: windows of ONE dense map, gathered on the device.  `dense` is a host numpy array or anything
    with __cuda_array_interface__ (a contiguous torch.cuda tensor), [C,H,W] (or [H,W,C] with channels_first=False).
    -> DeviceSlab [n, ps, ps, C] (or a numpy array with to_host=True)"""
    ctx = ctx or _capi.default_context()
    cai = getattr(dense, "__cuda_array_interface__", None)
    if cai is not None:
        if cai.get("strides") is not None:
            raise ValueError("the dense map must be contiguous")
        shape, in_dtype, ptr, on_dev = tuple(cai["shape"]), np.dtype(cai["typestr"]), int(cai["data"][0]), 1
    else:
        dense = np.ascontiguousarray(dense)
        shape, in_dtype, ptr, on_dev = dense.shape, dense.dtype, dense.ctypes.data, 0
    if len(shape) == 4 and shape[0] == 1:
        shape = shape[1:]
    if len(shape) != 3 or in_dtype not in _capi.DTYPE_IDS or np.dtype(out_dtype) not in _capi.DTYPE_IDS:
        raise ValueError("a dense map is a [C,H,W] / [H,W,C] float16/32/64 array")
    ch, h, w = shape if channels_first else (shape[2], shape[0], shape[1])
    corners = np.ascontiguousarray(corners, np.int32).reshape(-1, 2)
    n = len(corners)
    out = np.zeros((n, patch_size, patch_size, ch), out_dtype) if to_host else None
    if n == 0:
        return out if to_host else DeviceSlab(0, (0, patch_size, patch_size, ch), out_dtype, ctx)
    dptr = C.c_void_p()
    _capi.check(ctx.lib.pxr_extract_patches(ctx.handle, C.c_void_p(ptr), on_dev, _capi.DTYPE_IDS[in_dtype], int(ch), int(h),
                                            int(w), int(bool(channels_first)), _p(corners), C.c_int64(n), int(patch_size),
                                            int(bool(l2_normalize)), _capi.DTYPE_IDS[np.dtype(out_dtype)],
                                            _p(out) if to_host else None, None if to_host else C.byref(dptr)))
    return out if to_host else DeviceSlab(dptr.value, (n, patch_size, patch_size, ch), out_dtype, ctx)


def dsift_map_size(height, width, num_spatial_bins=4, spatial_bin_size=4):
    """(H', W') of the dense SIFT map of a height x width image (stride 1, padding 1, as the reference's dsift model)"""
    extra = 2 * (spatial_bin_size // 2) - spatial_bin_size + 1 + 3 - num_spatial_bins
    return height + extra, width + extra


def dsift(image, corners=None, patch_size=16, num_ang_bins=8, num_spatial_bins=4, spatial_bin_size=4, clipval=0.2,
          rootsift=True, l2_normalize=True, out_dtype=np.float16, to_host=False, ctx=None):
    """pxr_dsift: dense SIFT of ONE [H,W] uint8 grayscale image (a host numpy array or anything with
    __cuda_array_interface__).  With `corners` [n,2] (x0, y0) in map coordinates -> the windows [n, ps, ps, C]; without
    -> the whole map [1, H', W', C].  A DeviceSlab, or a numpy array with to_host=True."""
    ctx = ctx or _capi.default_context()
    cai = getattr(image, "__cuda_array_interface__", None)
    if cai is not None:
        if cai.get("strides") is not None:
            raise ValueError("the image must be contiguous")
        shape, in_dtype, ptr, on_dev = tuple(cai["shape"]), np.dtype(cai["typestr"]), int(cai["data"][0]), 1
    else:
        image = np.ascontiguousarray(image)
        shape, in_dtype, ptr, on_dev = image.shape, image.dtype, image.ctypes.data, 0
    if len(shape) != 2 or in_dtype != np.uint8 or np.dtype(out_dtype) not in _capi.DTYPE_IDS:
        raise ValueError("an image is a [H,W] uint8 array and the output float16/32/64")
    h, w = shape
    ch = num_ang_bins * num_spatial_bins ** 2
    if corners is None:
        out_shape, c_corners, n = (1,) + dsift_map_size(h, w, num_spatial_bins, spatial_bin_size) + (ch,), None, 0
    else:
        c_corners = np.ascontiguousarray(corners, np.int32).reshape(-1, 2)
        n = len(c_corners)
        out_shape = (n, patch_size, patch_size, ch)
    out = np.zeros(out_shape, out_dtype) if to_host else None
    dptr = C.c_void_p()
    _capi.check(ctx.lib.pxr_dsift(ctx.handle, C.c_void_p(ptr), on_dev, int(h), int(w), int(num_ang_bins),
                                  int(num_spatial_bins), int(spatial_bin_size), C.c_float(clipval), int(bool(rootsift)),
                                  int(bool(l2_normalize)), _p(c_corners), C.c_int64(n), int(patch_size),
                                  _capi.DTYPE_IDS[np.dtype(out_dtype)], _p(out) if to_host else None,
                                  None if to_host else C.byref(dptr)))
    return out if to_host else DeviceSlab(dptr.value or 0, out_shape, out_dtype, ctx)



S2DNET_FLOATS = 64 * 27 + 64 + 64 * 64 * 9 + 64 + 64 * 64 + 64 + 128 * 64 * 25 + 128


class S2DNetWeights:
    """pxr_s2dnet_weights: S2DNet's four layers uploaded once in the kernel's layout; freed with the object"""

    def __init__(self, handle, ctx):
        self.handle, self._ctx = handle, ctx

    def __del__(self):
        try:
            if self.handle:
                self._ctx.lib.pxr_s2dnet_weights_destroy(C.c_void_p(self.handle))
                self.handle = 0
        except Exception:      # interpreter shutdown
            pass


def s2dnet_weights(packed, ctx=None):
    """pxr_s2dnet_weights_create: `packed` is the S2DNET_FLOATS float32 values of include/pxr.h (conv1_1, conv1_2, 1x1 and
    5x5 weight and bias in PyTorch's layouts, the BatchNorm folded into the last) -> S2DNetWeights"""
    ctx = ctx or _capi.default_context()
    packed = np.ascontiguousarray(packed, np.float32).ravel()
    handle = C.c_void_p()
    _capi.check(ctx.lib.pxr_s2dnet_weights_create(ctx.handle, _p(packed), C.c_int64(packed.size), C.byref(handle)))
    return S2DNetWeights(handle.value, ctx)


def s2dnet(image, weights, corners=None, patch_size=16, l2_normalize=True, out_dtype=np.float16, to_host=False, ctx=None):
    """pxr_s2dnet: S2DNet features of ONE [H,W,3] uint8 RGB image (a host numpy array or anything with
    __cuda_array_interface__).  With `corners` [n,2] (x0, y0) -> the windows [n, ps, ps, 128]; without -> the whole map
    [1, H, W, 128].  A DeviceSlab, or a numpy array with to_host=True."""
    ctx = ctx or _capi.default_context()
    cai = getattr(image, "__cuda_array_interface__", None)
    if cai is not None:
        if cai.get("strides") is not None:
            raise ValueError("the image must be contiguous")
        shape, in_dtype, ptr, on_dev = tuple(cai["shape"]), np.dtype(cai["typestr"]), int(cai["data"][0]), 1
    else:
        image = np.ascontiguousarray(image)
        shape, in_dtype, ptr, on_dev = image.shape, image.dtype, image.ctypes.data, 0
    if len(shape) != 3 or shape[2] != 3 or in_dtype != np.uint8 or np.dtype(out_dtype) not in _capi.DTYPE_IDS:
        raise ValueError("an image is a [H,W,3] uint8 array and the output float16/32/64")
    h, w = shape[:2]
    if corners is None:
        out_shape, c_corners, n = (1, h, w, 128), None, 0
    else:
        c_corners = np.ascontiguousarray(corners, np.int32).reshape(-1, 2)
        n = len(c_corners)
        out_shape = (n, patch_size, patch_size, 128)
    out = np.zeros(out_shape, out_dtype) if to_host else None
    dptr = C.c_void_p()
    _capi.check(ctx.lib.pxr_s2dnet(ctx.handle, C.c_void_p(weights.handle), C.c_void_p(ptr), on_dev, int(h), int(w),
                                   _p(c_corners), C.c_int64(n), int(patch_size), int(bool(l2_normalize)),
                                   _capi.DTYPE_IDS[np.dtype(out_dtype)], _p(out) if to_host else None,
                                   None if to_host else C.byref(dptr)))
    return out if to_host else DeviceSlab(dptr.value or 0, out_shape, out_dtype, ctx)

def interpolate_patches(patches, corners, scales, item_patch, xys, interp=None, upsampling_factor=1.0, ctx=None):
    """pxr_interpolate_descriptors: the (bicubic, optionally L2-normalised) descriptor of patch item_patch[i] of a host
    [N,H,W,C] patch array at IMAGE coordinates xys[i] -> [n_items, C] float64"""
    ctx = ctx or _capi.default_context()
    interp = interp or _capi.default_interp()
    patches = np.ascontiguousarray(patches)
    if patches.ndim != 4 or patches.dtype not in _capi.DTYPE_IDS:
        raise ValueError("patches must be a [N,H,W,C] float16/32/64 array")
    corners = np.ascontiguousarray(corners, np.int32).reshape(-1, 2)
    scales = np.ascontiguousarray(scales, np.float64).reshape(-1, 2)
    item_patch = np.ascontiguousarray(item_patch, np.int64).reshape(-1)
    xys = np.ascontiguousarray(xys, np.float64).reshape(-1, 2)
    if len(corners) != len(patches) or len(scales) != len(patches) or len(item_patch) != len(xys):
        raise ValueError("one corner and scale per patch, one patch index per query point")
    out = np.zeros((len(xys), patches.shape[3]))
    _capi.check(ctx.lib.pxr_interpolate_descriptors(
        ctx.handle, _p(patches), C.c_int64(len(patches)), _capi.DTYPE_IDS[patches.dtype], int(patches.shape[1]),
        int(patches.shape[2]), int(patches.shape[3]), _p(corners), _p(scales), C.c_double(upsampling_factor),
        C.c_int64(len(xys)), _p(item_patch), _p(xys), C.byref(interp), _p(out)))
    return out


def query_match_run(blocks, corners, scales, item_query, item_patch, xys, cand_begin, cand_end, cand, interp=None,
                    with_desc=False, ctx=None):
    """pxr_query_match_run: per item the descriptor of patch item_patch[i] of query item_query[i]'s block (host numpy
    or device memory) at xys[i], and the first of the candidate rows [cand_begin[i], cand_end[i]) of `cand` (a host
    [n, C] float64 array, or device memory with __cuda_array_interface__, read in place) closest to it.
    -> (best row [n_items] int64, -1 for an empty range; squared distance [n_items]; descriptors [n_items, C] or None)"""
    interp = interp or _capi.default_interp()
    ptrs, counts, (ph, pw, ch), dt = _capi._patch_blocks(blocks)
    corners = np.ascontiguousarray(corners, np.int32).reshape(-1, 2)
    scales = np.ascontiguousarray(scales, np.float64).reshape(-1, 2)
    item_query = np.ascontiguousarray(item_query, np.int32)
    item_patch = np.ascontiguousarray(item_patch, np.int64)
    xys = np.ascontiguousarray(xys, np.float64).reshape(-1, 2)
    cb = np.ascontiguousarray(cand_begin, np.int64); ce = np.ascontiguousarray(cand_end, np.int64)
    n = len(item_query)
    if not (len(item_patch) == len(xys) == len(cb) == len(ce) == n):
        raise ValueError("one query, patch, point and candidate range per item")
    cai = getattr(cand, "__cuda_array_interface__", None)
    if cai is not None:
        shape = tuple(cai["shape"])
        contiguous = cai.get("strides") is None or tuple(cai["strides"]) == (ch * 8, 8)
        if np.dtype(cai["typestr"]) != np.dtype("<f8") or len(shape) != 2 or (shape[0] and shape[1] != ch) or not contiguous:
            raise ValueError("the candidate table must be a C-contiguous [n, %d] float64 array" % ch)
        n_cand, cptr, on_dev = int(shape[0]), C.c_void_p(int(cai["data"][0])), 1
    else:
        cand = np.ascontiguousarray(cand, np.float64)
        if len(cand) and (cand.ndim != 2 or cand.shape[1] != ch):
            raise ValueError("the candidate table must be [n, %d] (one descriptor of the patches' channels per row)" % ch)
        cand = cand.reshape(-1, ch)
        n_cand, cptr, on_dev = len(cand), _p(cand), 0
    ctx = ctx or _capi.default_context()
    best, dmin = np.zeros(n, np.int64), np.zeros(n)
    desc = np.zeros((n, ch)) if with_desc else None
    _capi.check(ctx.lib.pxr_query_match_run(
        ctx.handle, C.c_int32(len(counts)), C.cast(ptrs, C.c_void_p), _p(counts), _p(corners), _p(scales), C.c_double(1.0),
        int(ph), int(pw), int(ch), int(dt), C.c_int64(n), _p(item_query), _p(item_patch), _p(xys), _p(cb), _p(ce), cptr,
        C.c_int64(n_cand), int(on_dev), C.byref(interp), _p(best), _p(dmin), _p(desc)))
    return best, dmin, desc


def device_array(a):
    """a host array copied to device memory (a torch CUDA tensor: its __cuda_array_interface__ is what the library
    reads; freed with the tensor)"""
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda")
