"""Seeded BA scenes that each land on one named cell of the host's kernel selection, and a Python restatement of
that selection.

The reduced-camera-system assembly picks its kernels from the problem's shape (camera columns per image, the largest
camera model) and from A/B environment switches.  `expected_paths(prob, env)` restates those rules; it must follow:
  - BA::launch_schur_pairs     (csrc/pxr_ba.cu)        dense-sink pair walk
  - BA::launch_sp_schur_pairs  (csrc/pxr_ba.cu)        block-sparse-sink pair walk (PXR_PCG_SPARSE, block mode)
  - BA::build / BA::build_block (csrc/pxr_ba.cu, csrc/pxr_ba_block.cu)   normal-equation build
  - BA::project                (csrc/pxr_ba.cu)        projection + Jacobian of (u, v)
  - BA::create                 (csrc/pxr_ba.cu)        column layout, sparse_schur / block_mode, per-image chunks
test_dispatch_coverage.py asserts that SCENES x DENSE_ENVS and SCENES x SPARSE_ENVS reach every kernel those functions
can launch, so a change to the dispatch shows up as a failing CPU test instead of silently lost coverage; the GPU
parity tests (test_gpu_dispatch_matrix.py) run exactly these rows against the oracle.

Scenes are returned without reference descriptors; `with_refs` adds them from the oracle."""
import numpy as np

from pixsfm._pixsfm import _capi
from pixsfm.util import synthetic

# plausible parameters for every camera model (SIMPLE_RADIAL's are the synthetic generator's own)
MODEL_PARAMS = {
    0: [1200.0, 500.0, 500.0],                                              # SIMPLE_PINHOLE
    1: [1200.0, 1190.0, 500.0, 502.0],                                      # PINHOLE
    2: [1200.0, 500.0, 500.0, 0.0],                                         # SIMPLE_RADIAL
    3: [1200.0, 500.0, 500.0, 0.02, -0.01],                                 # RADIAL
    4: [1200.0, 1195.0, 500.0, 501.0, 0.02, -0.01, 1e-3, -2e-3],            # OPENCV
    5: [1200.0, 1195.0, 500.0, 501.0, 0.01, -0.005, 0.002, -0.001],         # OPENCV_FISHEYE
    6: [1200.0, 1195.0, 500.0, 501.0, 0.02, -0.01, 1e-3, -2e-3, 0.003, 0.01, -0.004, 0.002],  # FULL_OPENCV
}

PAIR_CHUNK = 128          # BA::build_schur_pairs kChunk: observation pairs per warp
IMAGE_CHUNK = 128         # BA::create: observations per ba_build_cam_kernel chunk
STATIC_SMEM = 48 * 1024   # staged variants launch without opting in to more shared memory


def _rebuild(prob, **kw):
    f = dict(cam_model=prob.cam_model, cam_params=prob.cam_params, cam_const_mask=prob.cam_const_mask, qvec=prob.qvec,
             tvec=prob.tvec, img_cam=prob.img_cam, pose_const=prob.pose_const, tvec_const_mask=prob.tvec_const_mask,
             xyz=prob.xyz, point_const=prob.point_const, obs_img=prob.obs_img, obs_pt=prob.obs_pt,
             patches=prob.patches, corner=prob.corner, scale=prob.scale)
    f.update(kw)
    return _capi.BAProblem(**f)


def _mask(model, free):
    """cam_const_mask that keeps the parameter groups in `free` ('f' focal, 'p' principal point, 'e' extra) variable"""
    groups = dict(zip("fpe", _capi.CAMERA_PARAM_GROUPS[model]))
    const = 0
    for g, bits in groups.items():
        if g not in free:
            const |= bits
    full = (1 << _capi.CAMERA_NUM_PARAMS[model]) - 1
    return 0xFFFFFFFF if const & full == full else const


def _with_cameras(prob, models, img_cam, free):
    """replace the cameras: one entry of models / free per camera, img_cam per image"""
    models = np.asarray(models, np.int32)
    params = np.zeros((len(models), _capi.PXR_MAX_CAM_PARAMS))
    for c, m in enumerate(models):
        params[c, :len(MODEL_PARAMS[m])] = MODEL_PARAMS[m]
    masks = np.array([_mask(int(m), f) for m, f in zip(models, free)], np.uint32)
    return _rebuild(prob, cam_model=models, cam_params=params, cam_const_mask=masks, img_cam=np.asarray(img_cam, np.int32))


def _base(n_cams=5, n_points=40, track_len=4, seed=0):
    prob, _ = synthetic.make_ba_scene(n_cams=n_cams, n_points=n_points, track_len=track_len, channels=16, seed=seed,
                                      dtype=np.float32)
    return prob


def _one_model(model, free, seed):
    prob = _base(seed=seed)
    n = len(prob.img_cam)
    return _with_cameras(prob, [model] * n, np.arange(n), [free] * n)


def _mixed(opencv_free, seed=21):
    # SIMPLE_RADIAL shared by images 0-2, one OPENCV shared by images 3 and 5, SIMPLE_PINHOLE on image 4
    prob = _base(n_cams=6, n_points=50, track_len=4, seed=seed)
    return _with_cameras(prob, [2, 4, 0], [0, 0, 0, 1, 2, 1], ["fe", opencv_free, "f"])


def _pose_and_intrinsics_only(seed=22):
    prob = _base(n_cams=6, n_points=50, track_len=4, seed=seed)
    prob = _with_cameras(prob, [2] * 6, np.arange(6), ["", "fe", "", "fe", "fe", "f"])
    prob.pose_const[:] = [1, 0, 0, 1, 0, 0]         # image 0: nothing variable; image 3: intrinsics only
    prob.tvec_const_mask[:] = [0, 1, 0, 0, 0b101, 0b010]
    return prob                                       # image 2: pose only (its camera is constant)


def _duplicate_observations(seed=23, every=3):
    """every `every`-th point is observed twice in one image (two detections a pixel apart): observation pairs of one
    point inside one image, i.e. non-self pairs on a diagonal image block"""
    prob = _base(seed=seed)
    order, shift = [], []
    for p in range(len(prob.xyz)):
        idx = np.flatnonzero(prob.obs_pt == p)
        order.extend(idx); shift.extend([0] * len(idx))
        if p % every == 0:
            order.append(idx[len(idx) // 2]); shift.append(1)
    order = np.array(order)
    corner = prob.corner[order].copy()
    corner[:, 0] += np.array(shift, np.int32)
    return _rebuild(prob, obs_img=prob.obs_img[order], obs_pt=prob.obs_pt[order],
                    patches=np.ascontiguousarray(prob.patches[order]), corner=corner, scale=prob.scale[order])


def _multi_chunk(seed=24):
    # every point in all three images: each image pair key holds 150 > 128 pairs, each image 150 > 128 observations
    return _base(n_cams=3, n_points=150, track_len=3, seed=seed)


# name -> builder.  The comment is the cell the scene lands on (checked by test_dispatch_coverage.py).
SCENES = {
    "k3_dc7": lambda: _one_model(0, "f", 30),          # SIMPLE_PINHOLE, dcmax 9 (odd), staged build
    "k4_dc8": lambda: _one_model(2, "fe", 31),         # SIMPLE_RADIAL, dcmax 10, staged build
    "k5_dc7": lambda: _one_model(3, "f", 32),          # RADIAL, dcmax 11 (odd), staged build
    "k8_dc8": lambda: _one_model(4, "f", 33),          # OPENCV, dcmax 14, staged build over 48 KiB -> unstaged
    "k12_dc8": lambda: _one_model(6, "f", 34),         # FULL_OPENCV, dcmax 18, unstaged build
    "k8_dc14": lambda: _one_model(4, "fpe", 35),       # OPENCV all free: more than 8 columns, generic walk
    "mixed_dc8": lambda: _mixed("f"),                  # three models, shared + per-image cameras, dc 5..8
    "mixed_dc14": lambda: _mixed("fpe"),               # generic walk with both fast and generic chunks
    "pose_intr_only": _pose_and_intrinsics_only,       # dc 0, pose-only, intrinsics-only, partial tvec masks
    "dup_obs": _duplicate_observations,                # same-image non-self pairs
    "multi_chunk": _multi_chunk,                       # keys and images spanning several 128-chunks
}

SCHUR_KERNELS = ("fused", "mma", "staged", "direct")
# the dense-sink switch matrix: every PXR_SCHUR_KERNEL x PXR_SCHUR_CTAS, and the build / projection switches
DENSE_ENVS = [{}] + [{"PXR_SCHUR_KERNEL": k, "PXR_SCHUR_CTAS": c} for k in SCHUR_KERNELS for c in ("3", "4")] + \
             [{"PXR_BUILD_ATOMIC": "1"}, {"PXR_BUILD_UNSTAGED": "1"}, {"PXR_PROJECT_UNSTAGED": "1"}]
# the block-sparse sink (only for images of at most 8 columns): ITERATIVE_SCHUR on image-pair blocks, and block mode
SPARSE_ENVS = [dict(base, PXR_SCHUR_KERNEL=k) for base in ({"PXR_PCG_SPARSE": "1"}, {"PXR_BLOCK_ASSEMBLY": "1"})
               for k in SCHUR_KERNELS]
SPARSE_SCENES = [n for n in SCENES if "dc14" not in n]


def env_id(env):
    return "-".join("%s=%s" % (k.replace("PXR_", "").lower(), v) for k, v in sorted(env.items())) or "default"


def with_refs(prob, ic=None):
    """reference descriptors from the oracle, slightly off the observed ones so no residual vanishes"""
    import oracle_lib as O
    refs, _ = O.refs_compute(prob, ic or _capi.default_interp())
    prob.refs = refs * 0.95 + 0.002
    return prob


# ---------------------------------------------------------------------------------------------- the selection rules
def shape(prob):
    """what the host derives from a problem before it picks kernels (BA::create)"""
    models = [int(m) for m in prob.cam_model]
    K = max(_capi.CAMERA_NUM_PARAMS[m] for m in models)
    cam_cols = []
    for m, mask in zip(models, prob.cam_const_mask):
        k = _capi.CAMERA_NUM_PARAMS[m]
        full = (1 << k) - 1
        cm = int(mask) & full
        cam_cols.append(0 if cm == full else k - bin(cm).count("1"))
    img_dc = []
    for i in range(len(prob.img_cam)):
        pose = 0 if prob.pose_const[i] else 6 - bin(int(prob.tvec_const_mask[i]) & 7).count("1")
        img_dc.append(pose + cam_cols[int(prob.img_cam[i])])
    return dict(K=K, dcmax=6 + K, juv_stride=2 * (9 + K), img_dc=np.array(img_dc), img_dc_max=max(img_dc))


def _pairs(prob):
    """(image x, image y, self) of every observation pair of a variable point, as BA::build_schur_pairs forms them"""
    out = []
    for p in range(len(prob.xyz)):
        if prob.point_const[p]:
            continue
        idx = np.flatnonzero(prob.obs_pt == p)
        for a in range(len(idx)):
            for b in range(a + 1):
                ia, ib = int(prob.obs_img[idx[a]]), int(prob.obs_img[idx[b]])
                out.append((max(ia, ib), min(ia, ib), a == b))
    return out


def cells(prob):
    """structural cells of a scene beyond the kernel choice"""
    sh = shape(prob)
    pairs = _pairs(prob)
    keys = {}
    for k in pairs:
        keys[k] = keys.get(k, 0) + 1
    out = set()
    if any(x == y and not s for x, y, s in pairs):
        out.add("same_image_non_self_pairs")
    if max(keys.values()) > PAIR_CHUNK:
        out.add("key_over_one_chunk")
    dc = sh["img_dc"]
    per_img = np.bincount(prob.obs_img[dc[prob.obs_img] > 0], minlength=len(dc))
    if sh["img_dc_max"] <= 8 and per_img.max() > IMAGE_CHUNK:
        out.add("image_over_one_chunk")
    if (dc == 0).any():
        out.add("image_without_columns")
    if any(prob.pose_const[i] and dc[i] > 0 for i in range(len(dc))):
        out.add("intrinsics_only_image")
    if any(not prob.pose_const[i] and dc[i] == 6 - bin(int(prob.tvec_const_mask[i]) & 7).count("1") for i in range(len(dc))):
        out.add("pose_only_image")
    if any((int(m) & 7) not in (0, 1, 7) for i, m in enumerate(prob.tvec_const_mask) if not prob.pose_const[i]):
        out.add("partial_tvec_masks")       # beyond the gauge's single constant x of image 1
    if len(set(int(m) for m in prob.cam_model)) > 1:
        out.add("mixed_models")
    if len(set(int(c) for c in prob.img_cam)) < len(prob.img_cam) and len(prob.cam_model) > 1:
        out.add("shared_and_per_image_cameras")
    if sh["img_dc_max"] > 8:
        fast = any(dc[x] <= 8 and dc[y] <= 8 for x, y, _ in pairs)
        generic = any(dc[x] > 8 or dc[y] > 8 for x, y, _ in pairs)
        if fast and generic:
            out.add("generic_walk_fast_and_generic_chunks")
    return out


def expected_paths(prob, env, linear_solver=0):
    """the kernels the host launches for one linearisation + step of `prob` under the switches `env`
    (environment variable -> value), with kernel template arguments written as in the CUDA source"""
    sh = shape(prob)
    K, dcmax, juv_stride, dc_max = sh["K"], sh["dcmax"], sh["juv_stride"], sh["img_dc_max"]
    n_obs = len(prob.obs_pt)
    on = lambda k: k in env
    e = env.get("PXR_SCHUR_KERNEL", "")
    kernel = {"m": "mma", "s": "staged", "d": "direct"}.get(e[:1], "fused")
    ctas = int(env.get("PXR_SCHUR_CTAS", "0"))
    small8 = dc_max <= 8
    # BA::create
    sparse_schur = linear_solver == 3 and small8 and n_obs > 0 and on("PXR_PCG_SPARSE")
    block_mode = small8 and on("PXR_BLOCK_ASSEMBLY")
    io_chunks = small8 and n_obs > 0 and bool((sh["img_dc"][prob.obs_img] > 0).any())
    paths = set()
    # BA::project (the Jacobian pass)
    if not on("PXR_PROJECT_UNSTAGED") and 128 * (juv_stride | 1) * 8 <= STATIC_SMEM:
        paths.add("ba_project_staged_kernel")
    else:
        paths.add("ba_project_kernel<true>")
    # BA::build / BA::build_block
    build_smem = 128 * ((max(juv_stride, 3 * dcmax) | 1) + 9) * 8
    staged_ok = not on("PXR_BUILD_UNSTAGED") and build_smem <= STATIC_SMEM
    if block_mode:
        paths.add("ba_build_staged_kernel" if io_chunks and staged_ok else "ba_build_kernel<true>/chunked")
        if io_chunks:
            paths.add("ba_build_cam_kernel")
    else:
        chunked = io_chunks and (sparse_schur or not on("PXR_BUILD_ATOMIC"))
        if small8 and chunked and staged_ok:
            paths.add("ba_build_staged_kernel")
        elif small8:
            paths.add("ba_build_kernel<true>/" + ("chunked" if chunked else "atomic"))
        else:
            paths.add("ba_build_kernel<false>/atomic")
        if chunked:
            paths.add("ba_build_cam_kernel")
    # BA::launch_sp_schur_pairs (block-sparse sink) or BA::launch_schur_pairs (dense sink)
    small = dc_max <= 8 and dcmax >= 9
    if sparse_schur or block_mode:
        if dcmax >= 9 and kernel == "fused":
            paths.add("sp_schur_pairs_kernel<4>")
        else:
            paths.add("ba_schur_prep_kernel")
            if dcmax >= 9 and kernel == "mma":
                paths.add("sp_schur_pairs_kernel<3>")
            elif dcmax >= 9 and kernel == "staged":
                paths.add("sp_schur_pairs_kernel<1>" if dcmax % 2 == 0 else "sp_schur_pairs_kernel<2>")
            else:
                paths.add("sp_schur_pairs_kernel<0>")
        return paths
    if small and kernel == "fused":
        paths.add("ba_schur_pairs_mma_kernel<3, true>" if ctas == 3 else "ba_schur_pairs_mma_kernel<4, true>")
        return paths
    paths.add("ba_schur_prep_kernel")
    if small and kernel == "mma":
        paths.add("ba_schur_pairs_mma_kernel<4, false>" if ctas == 4 else "ba_schur_pairs_mma_kernel<3, false>")
    elif small and kernel == "staged":
        vec = dcmax % 2 == 0
        paths.add("ba_schur_pairs_staged_kernel<%s, %d>" % ("true" if vec else "false", 3 if ctas == 3 else 4))
    elif dc_max <= 8:
        paths.add("ba_schur_pairs_kernel<true>")
    else:
        paths.add("ba_schur_pairs_kernel<false>")
    return paths


# Every kernel the four selecting functions can launch for a linearisation.  Keep in step with the CUDA source.
ALL_PATHS = {
    # BA::project
    "ba_project_staged_kernel", "ba_project_kernel<true>",
    # BA::build / BA::build_block
    "ba_build_staged_kernel", "ba_build_kernel<true>/chunked", "ba_build_kernel<true>/atomic",
    "ba_build_kernel<false>/atomic", "ba_build_cam_kernel",
    # BA::launch_schur_pairs
    "ba_schur_prep_kernel",
    "ba_schur_pairs_mma_kernel<3, true>", "ba_schur_pairs_mma_kernel<4, true>",
    "ba_schur_pairs_mma_kernel<3, false>", "ba_schur_pairs_mma_kernel<4, false>",
    "ba_schur_pairs_staged_kernel<true, 3>", "ba_schur_pairs_staged_kernel<true, 4>",
    "ba_schur_pairs_staged_kernel<false, 3>", "ba_schur_pairs_staged_kernel<false, 4>",
    "ba_schur_pairs_kernel<true>", "ba_schur_pairs_kernel<false>",
    # BA::launch_sp_schur_pairs
    "sp_schur_pairs_kernel<0>", "sp_schur_pairs_kernel<1>", "sp_schur_pairs_kernel<2>",
    "sp_schur_pairs_kernel<3>", "sp_schur_pairs_kernel<4>",
}

ALL_CELLS = {"same_image_non_self_pairs", "key_over_one_chunk", "image_over_one_chunk", "image_without_columns",
             "intrinsics_only_image", "pose_only_image", "partial_tvec_masks", "mixed_models",
             "shared_and_per_image_cameras", "generic_walk_fast_and_generic_chunks"}
