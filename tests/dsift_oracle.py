"""Two independent float64 restatements of the dense SIFT descriptor csrc/pxr_dsift.cu computes (the reference's `dsift`
model: kornia's DenseSIFTDescriptor with stride 1 and padding 1; parity with kornia itself is unverified), and the
bound on how far the kernel's fp32 arithmetic may lie from them.

  (a) `dsift_conv`: the convolution form, in torch — gradients, orientation binning, the triangular pooling kernel as
      one grouped conv2d, the spatial gather as a one-hot grouped conv2d with padding 1, then the normalisations.
      Runs on the CPU or on CUDA (the benchmark's stand-in for the reference's path).
  (b) `dsift_loops`: plain per-pixel loops in Python / numpy.

Both return the map [H', W', C], C = A * S * S, channel a * S^2 + i * S + j."""
import math

import numpy as np


def map_size(h, w, S=4, b=4):
    extra = 2 * (b // 2) - b + 1 + 3 - S
    return h + extra, w + extra


def _normalize(x, p, dim):
    import torch
    return x / torch.clamp(torch.linalg.vector_norm(x, ord=p, dim=dim, keepdim=True), min=1e-12)


def dsift_conv(image, A=8, S=4, b=4, clipval=0.2, rootsift=True, l2_normalize=True, dtype=None, device="cpu",
               intermediates=False, as_tensor=False):
    """(a).  `image` is a uint8 numpy array or torch tensor.  With intermediates=True also returns a dict of per-pixel
    quantities the fp32 bound needs; with as_tensor=True the map stays a torch tensor on `device`."""
    import torch
    import torch.nn.functional as F
    dtype = dtype or torch.float64
    if not isinstance(image, torch.Tensor):
        image = torch.as_tensor(np.array(image))
    I = image.to(device=device, dtype=dtype)[None, None] / 255.0
    Ip = F.pad(I, (1, 1, 1, 1), mode="replicate")
    gx = 0.5 * (Ip[..., 1:-1, 2:] - Ip[..., 1:-1, :-2])
    gy = 0.5 * (Ip[..., 2:, 1:-1] - Ip[..., :-2, 1:-1])
    mag = torch.sqrt(gx * gx + gy * gy + 1e-10)
    o = A * (torch.atan2(gy, gx + 1e-10) + 2 * math.pi) / (2 * math.pi)
    k = torch.floor(o)
    w = o - k
    b0 = torch.remainder(k, A).long()
    b1 = torch.remainder(b0 + 1, A)
    E = torch.zeros((1, A) + I.shape[2:], dtype=dtype, device=device)
    E.scatter_add_(1, b0, (1 - w) * mag)
    E.scatter_add_(1, b1, w * mag)
    t = b / 2.0 - torch.abs(torch.arange(b, dtype=dtype, device=device) + 0.5 - b / 2.0)
    K = (t[:, None] * t[None, :]) / (b / 2.0) ** 2
    P = F.conv2d(E, K.expand(A, 1, b, b), padding=b // 2, groups=A)
    onehot = torch.zeros((A * S * S, 1, S, S), dtype=dtype)
    for c in range(A * S * S):
        onehot[c, 0, (c // S) % S, c % S] = 1.0
    onehot = onehot.to(device)
    D = F.conv2d(P, onehot, padding=1, groups=A)
    v1 = _normalize(D, 2, 1)
    clamped = torch.clamp(v1, 0.0, clipval)
    v2 = _normalize(clamped, 2, 1)
    v = v2
    if rootsift:
        x = _normalize(v2, 1, 1)
        v = torch.sqrt(x + 1e-10)
    if l2_normalize:
        v = _normalize(v, 2, 1)
    out = v[0].permute(1, 2, 0).contiguous()
    if as_tensor:
        return out
    if not intermediates:
        return out.cpu().numpy()
    extra = {"clamped_norm": torch.linalg.vector_norm(clamped, dim=1)[0].cpu().numpy(),
             "l1": torch.linalg.vector_norm(v2, ord=1, dim=1)[0].cpu().numpy(),
             "x": (_normalize(v2, 1, 1) if rootsift else v2)[0].permute(1, 2, 0).cpu().numpy()}
    return out.cpu().numpy(), extra


def dsift_loops(image, A=8, S=4, b=4, clipval=0.2, rootsift=True, l2_normalize=True):
    """(b)"""
    G = np.asarray(image)
    H, W = G.shape
    I = G.astype(np.float64) / 255.0

    def at(y, x):
        return I[min(max(y, 0), H - 1), min(max(x, 0), W - 1)]

    E = np.zeros((A, H, W))
    for y in range(H):
        for x in range(W):
            gx = 0.5 * (at(y, x + 1) - at(y, x - 1))
            gy = 0.5 * (at(y + 1, x) - at(y - 1, x))
            mag = math.sqrt(gx * gx + gy * gy + 1e-10)
            o = A * (math.atan2(gy, gx + 1e-10) + 2 * math.pi) / (2 * math.pi)
            k = math.floor(o)
            wt = o - k
            E[k % A, y, x] += (1 - wt) * mag
            E[(k % A + 1) % A, y, x] += wt * mag
    hb = b // 2
    Hp, Wp = H + 2 * hb - b + 1, W + 2 * hb - b + 1
    t = [b / 2.0 - abs(u + 0.5 - b / 2.0) for u in range(b)]
    P = np.zeros((A, Hp, Wp))
    for a in range(A):
        for py in range(Hp):
            for px in range(Wp):
                s = 0.0
                for u in range(b):
                    for v in range(b):
                        ey, ex = py - hb + u, px - hb + v
                        if 0 <= ey < H and 0 <= ex < W:
                            s += t[u] * t[v] / (b / 2.0) ** 2 * E[a, ey, ex]
                P[a, py, px] = s
    Hm, Wm = map_size(H, W, S, b)
    C = A * S * S
    out = np.zeros((Hm, Wm, C))
    for y in range(Hm):
        for x in range(Wm):
            d = np.zeros(C)
            for a in range(A):
                for i in range(S):
                    for j in range(S):
                        py, px = y - 1 + i, x - 1 + j
                        if 0 <= py < Hp and 0 <= px < Wp:
                            d[a * S * S + i * S + j] = P[a, py, px]
            v = np.clip(d / max(math.sqrt(float(np.sum(d * d))), 1e-12), 0.0, clipval)
            v = v / max(math.sqrt(float(np.sum(v * v))), 1e-12)
            if rootsift:
                v = np.sqrt(v / max(float(np.sum(np.abs(v))), 1e-12) + 1e-10)
            if l2_normalize:
                v = v / max(math.sqrt(float(np.sum(v * v))), 1e-12)
            out[y, x] = v
    return out


U32 = 2.0 ** -24


def fp32_bound(ref, extra, A=8, S=4, b=4, rootsift=True, l2_normalize=True, out_dtype=np.float32):
    """Per-element bound on |kernel - ref| for the kernel's fp32 arithmetic (ref, extra = dsift_conv(..., intermediates=True)).

    u = 2^-24.  The orientation o = A (atan2 + 2 pi) / (2 pi) lies below 2A; atan2f (CUDA: <= 2 ulp), the add, the product
    and the quotient leave it within eps_w = 8 ulp of 2A, and so is the fraction w = o - floor(o) (floor is exact, and E
    is continuous across the jumps of floor).  A pixel's error in E_a is at most eps_w * mag in each of its two bins, so
    the pooled map (sums of non-negative terms, relative rounding (4b + 8) u) has ||dD|| <= (A eps_w + (4b + 8) u) ||D||.
    Then, with torch's normalize semantics:
      x / ||x||          moves by at most 2 ||dx|| / ||x||           -> e1 = 2 e_D,  e2 = 2 e1 / ||clamp(v1)|| (+ 2u each)
      clamp              is 1-Lipschitz
      rootsift           x = v / |v|_1 moves by (e2 + x sqrt(C) e2) / |v|_1 element-wise, and
                         |sqrt(x + 1e-10) - sqrt(y + 1e-10)| = |x - y| / (sqrt(x + 1e-10) + sqrt(y + 1e-10))
      l2_normalize       r / ||r|| with ||r|| = 1 moves element c by at most dr_c + |r_c| ||dr||  (rootsift), 2 dr else
    plus the final rounding: u |ref| for fp32 output, one fp16 rounding (2^-11 |ref|, 2^-25 below 2^-14) for fp16."""
    C = ref.shape[-1]
    eps_w = 8.0 * 2.0 ** (math.ceil(math.log2(2 * A)) - 24)
    e_D = A * eps_w + (4 * b + 8) * U32
    e1 = 2 * e_D + 2 * U32
    e2 = (2 * e1 / np.maximum(extra["clamped_norm"], 1e-12) + 2 * U32)[..., None]
    if rootsift:
        x = extra["x"]
        s1 = np.maximum(extra["l1"], 1.0)[..., None]
        dx = (e2 + x * math.sqrt(C) * e2) / s1 + 2 * U32 * x
        dr = dx / (np.sqrt(x + 1e-10) + np.sqrt(np.maximum(x - dx, 0.0) + 1e-10)) + U32
        if l2_normalize:
            r = np.sqrt(x + 1e-10)
            dr = dr + r * np.linalg.norm(dr, axis=-1, keepdims=True) + 2 * U32
    else:
        dr = np.broadcast_to(e2, ref.shape)
        if l2_normalize:
            dr = 2 * dr + 2 * U32
    bound = dr + U32 * np.abs(ref)
    if np.dtype(out_dtype) == np.float16:
        bound = bound + np.maximum(2.0 ** -11 * np.abs(ref), 2.0 ** -25)
    return bound
