"""S2DNet (num_layers 1) per image on one GPU: the fused kernel at the keypoints' windows, the same kernel over the whole
map, and the reference's path — torch's cuDNN forward in fp32 (TF32 at torch's default), F.normalize, then
pxr_extract_patches, which cuts the windows and casts them to half.

Workloads: 1600 x 1200 and 2000 x 1500 RGB images (the extractor's default max_edge and the dsift preset's), 2 000 and
8 000 keypoints, 16 x 16 windows, plus 8 x 8 windows (the low_memory shape); fp16 output, seeded weights.  Times are
CUDA-event medians of three runs after warm-up.  TFLOP/s counts 494 976 FLOP per output pixel (two per multiply-add
of the four convolutions), not the halo each tile recomputes; the share of the data sheet's 989 TFLOP/s dense FP16
bounds compute only, not bandwidth.  Peak device memory is taken per arm from torch's allocator statistics plus the
kernel's own output.  Prints one JSON line per workload; with --out also writes them to that file."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "pixel-perfect-sfm_b200"), os.path.join(ROOT, "tests")]

FLOP_PER_PIXEL = 2 * (27 * 64 + 576 * 64 + 64 * 64 + 1600 * 128)     # 494 976
PEAK_FP16 = 989e12


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _time(fn, runs=3, reps=5):
    import torch
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / reps * 1e-3)
    return float(np.median(times))


def _peak(fn, extra_bytes=0):
    """peak device memory of one call above what was allocated before it, in bytes"""
    import torch
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del out
    return int(peak + extra_bytes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="JSON file for the results (optional)")
    args = ap.parse_args()
    import torch
    import torch.nn.functional as Fn
    from scipy.ndimage import gaussian_filter
    import s2dnet_reference as R
    from pixsfm._pixsfm import _engine
    from pixsfm.features.extractor import patch_corners
    from pixsfm.features.models.s2dnet import pack_state_dict
    if not torch.cuda.is_available():
        raise SystemExit("s2dnet_bench needs a CUDA device")
    card = _card()
    sd = R.seeded_state_dict(0)
    weights = _engine.s2dnet_weights(pack_state_dict(sd))
    rows = []
    for (w, h) in ((1600, 1200), (2000, 1500)):
        rng = np.random.default_rng(w)
        img = np.stack([gaussian_filter(rng.random((h, w)), 1.5) for _ in range(3)], -1)
        img = np.clip((img - img.min()) / (img.max() - img.min()) * 255, 0, 255).astype(np.uint8)
        dev_img = torch.from_numpy(img).cuda()
        for n, ps in ((2000, 16), (8000, 16), (2000, 8), (8000, 8)):
            C = 128
            kps = rng.uniform(0, (w, h), (n, 2))
            corners = patch_corners(kps, np.array([1.0, 1.0]), ps, (w, h))

            def sparse():
                return _engine.s2dnet(dev_img, weights, corners, ps)

            def dense():
                return _engine.s2dnet(dev_img, weights, None, ps)

            def cudnn():
                with torch.no_grad():
                    m = R.forward(dev_img, sd, l2_normalize=False, dtype=torch.float32, device="cuda")
                    m = Fn.normalize(m, dim=-1).contiguous()
                return _engine.extract_patches(m, corners, ps, False, np.float16, channels_first=False)   # half cast here

            t_sparse, t_dense, t_cudnn = _time(sparse), _time(dense), _time(cudnn)
            a = torch.as_tensor(sparse(), device="cuda").float().cpu().numpy()
            full = torch.as_tensor(dense(), device="cuda").float().cpu().numpy()[0]
            c = torch.as_tensor(cudnn(), device="cuda").float().cpu().numpy()
            windows = np.stack([full[y:y + ps, x:x + ps] for x, y in corners])
            px_sparse, px_dense = n * ps * ps, h * w
            row = dict(image=[w, h], keypoints=n, patch_size=ps, channels=C, dtype="float16", card=card,
                       sparse_s=t_sparse, dense_s=t_dense, cudnn_s=t_cudnn,
                       sparse_TFLOPs=px_sparse * FLOP_PER_PIXEL / t_sparse / 1e12,
                       dense_TFLOPs=px_dense * FLOP_PER_PIXEL / t_dense / 1e12,
                       cudnn_TFLOPs=px_dense * FLOP_PER_PIXEL / t_cudnn / 1e12,
                       sparse_share_of_fp16_peak=px_sparse * FLOP_PER_PIXEL / t_sparse / PEAK_FP16,
                       dense_share_of_fp16_peak=px_dense * FLOP_PER_PIXEL / t_dense / PEAK_FP16,
                       peak_bytes_sparse=_peak(sparse, px_sparse * C * 2),
                       peak_bytes_dense=_peak(dense, px_dense * C * 2),
                       peak_bytes_cudnn=_peak(cudnn, px_sparse * C * 2),
                       sparse_vs_dense_max_abs=float(np.abs(a - windows).max()),
                       sparse_vs_cudnn_max_abs=float(np.abs(a - c).max()))
            assert row["sparse_vs_dense_max_abs"] == 0.0, row
            print(json.dumps(row), flush=True)
            rows.append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
