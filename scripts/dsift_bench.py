"""Dense SIFT per image on one GPU: the fused sparse kernel, the same kernel over the whole map, and the convolution form
in torch (tests/dsift_oracle.py (a) in float32 on the GPU, then normalise, cast to fp16 and cut the windows with
pxr_extract_patches) — a stand-in for the reference's kornia path without its device -> host copy.

Workloads: 1600 x 1200 and 2000 x 1500 grayscale images (the extractor's default max_edge and the dsift preset's),
2 000 and 8 000 keypoints, 16 x 16 windows, fp16, default descriptor (A 8, S 4, b 4: C 128).  Times are CUDA-event
medians of three runs after warm-up; bytes/s counts the image bytes plus the output bytes.  The arms' outputs are
compared at every timed size.  Prints one JSON line per workload; with --out also writes them to that file."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "pixel-perfect-sfm_b200"), os.path.join(ROOT, "tests")]


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _time(fn, runs=3, reps=10):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="JSON file for the results (optional)")
    args = ap.parse_args()
    import torch
    from scipy.ndimage import gaussian_filter
    import dsift_oracle as D
    from pixsfm._pixsfm import _engine
    from pixsfm.features.extractor import patch_corners
    if not torch.cuda.is_available():
        raise SystemExit("dsift_bench needs a CUDA device")
    card = _card()
    rows = []
    for (w, h) in ((1600, 1200), (2000, 1500)):
        rng = np.random.default_rng(w)
        img = np.clip(gaussian_filter(rng.random((h, w)), 1.5) * 255 * 4 - 382, 0, 255).astype(np.uint8)
        dev_img = torch.from_numpy(img).cuda()
        for n in (2000, 8000):
            ps, C = 16, 128
            kps = rng.uniform(0, (w, h), (n, 2))
            corners = patch_corners(kps, np.array([1.0, 1.0]), ps, (w, h))

            def sparse():
                return _engine.dsift(dev_img, corners, ps)

            def dense():
                return _engine.dsift(dev_img, None, ps)

            def conv():
                m = D.dsift_conv(dev_img, dtype=torch.float32, device="cuda", l2_normalize=False, as_tensor=True)
                return _engine.extract_patches(m, corners, ps, True, np.float16, channels_first=False)

            t_sparse, t_dense, t_conv = _time(sparse), _time(dense), _time(conv)
            a = torch.as_tensor(sparse(), device="cuda").float().cpu().numpy()
            full = torch.as_tensor(dense(), device="cuda").float().cpu().numpy()[0]
            c = torch.as_tensor(conv(), device="cuda").float().cpu().numpy()
            windows = np.stack([full[y:y + ps, x:x + ps] for x, y in corners])
            in_bytes = img.nbytes
            row = dict(image=[w, h], keypoints=n, patch_size=ps, channels=C, dtype="float16", card=card,
                       sparse_s=t_sparse, dense_s=t_dense, conv_torch_s=t_conv,
                       sparse_GBps=(in_bytes + n * ps * ps * C * 2) / t_sparse / 1e9,
                       dense_GBps=(in_bytes + h * w * C * 2) / t_dense / 1e9,
                       conv_torch_GBps=(in_bytes + n * ps * ps * C * 2) / t_conv / 1e9,
                       sparse_vs_dense_max_abs=float(np.abs(a - windows).max()),
                       sparse_vs_conv_max_abs=float(np.abs(a - c).max()))
            assert row["sparse_vs_dense_max_abs"] == 0.0, row
            assert row["sparse_vs_conv_max_abs"] < 1e-2, row
            print(json.dumps(row), flush=True)
            rows.append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
