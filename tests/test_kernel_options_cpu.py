"""CPU side of the kernel-option matrix (test_gpu_kernel_options.py).

1. The instance lists of the CUDA sources, read with a regex, against the parameter rows of the GPU file: adding or
   dropping a kernel instance fails here instead of silently leaving it untested.
2. The oracle's reference extraction (RobustMeanIRLS + closest observation, irls_optim.h:23-71 and
   reference_extractor.h:239-272 of the reference) against a plain numpy restatement in extended precision, at the
   track lengths, losses and options the GPU file compares the device kernel at.  The GPU file trusts the oracle for
   these cases; this pins the oracle first."""
import itertools
import os
import re

import numpy as np

import oracle_lib as O
import test_gpu_kernel_options as G
from pixsfm._pixsfm import _capi

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pixel-perfect-sfm_b200", "csrc")
CTYPES = {"__half": "float16", "float": "float32", "double": "float64"}
DTYPES = {"PXR_F16": "float16", "PXR_F32": "float32", "PXR_F64": "float64"}


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _body(text, head):
    """the brace-balanced body of the first function whose signature contains `head`"""
    i = text.index(head)
    i = text.index("{", i)
    depth = 0
    for j in range(i, len(text)):
        depth += {"{": 1, "}": -1}.get(text[j], 0)
        if depth == 0:
            return text[i:j + 1]
    raise AssertionError("unbalanced braces after " + head)


def _rows(fn):
    """every parameter row of a test function: the product of its parametrize marks, as dicts"""
    axes = []
    for m in getattr(fn, "pytestmark", []):
        if m.name != "parametrize":
            continue
        names = [n.strip() for n in m.args[0].split(",")]
        vals = [v if len(names) > 1 else (v,) for v in m.args[1]]
        axes.append([dict(zip(names, v)) for v in vals])
    for combo in itertools.product(*axes):
        row = {}
        for d in combo:
            row.update(d)
        yield row


def _dt(v):
    return np.dtype(v).name


def fm_instances():
    """(dtype, C) pairs fm_supported (pxr_ba.cu) accepts"""
    body = _body(_src("pxr_ba.cu"), "int fm_supported(int dtype, int C)")
    out = set()
    m = re.search(r"if \(\(((?:C == \d+(?: \|\| )?)+)\) && \(((?:dtype == PXR_F\d+(?: \|\| )?)+)\)\) return 1;", body)
    assert m, "the C < 8 line of fm_supported"
    for c in re.findall(r"\d+", m.group(1)):
        for d in re.findall(r"PXR_F\d+", m.group(2)):
            out.add((DTYPES[d], int(c)))
    lines = re.findall(r"if \(dtype == (PXR_F\d+)\) return ((?:C == \d+(?: \|\| )?)+);", body)
    assert len(lines) == 3
    for d, cs in lines:
        for c in re.findall(r"\d+", cs):
            out.add((DTYPES[d], int(c)))
    return out


def ka_instances():
    """(dtype, C, FS, REF) of every ka_solve_kernel launch_ka can start"""
    src = _src("pxr_ka.cu")
    pairs = {(CTYPES[t], int(c)) for t, c in re.findall(r"PXR_KA_CASE\((__half|float|double), (\d+)\)", src)}
    launch = _body(src, "static int launch_ka(")
    modes = {(fs == "true", ref == "true") for fs, ref in
             re.findall(r"PXR_LAUNCH\(ctx, \(ka_solve_kernel<T, C, (true|false), (true|false)>\)", launch)}
    # float-SIMD in query mode is refused before the launch
    assert re.search(r"if \(ref\) \{\s*if \(fs\) return fail\(PXR_ERR_UNSUPPORTED", launch)
    return {(d, c, fs, ref) for d, c in pairs for fs, ref in modes}


def qba_instances():
    """(dtype, C, FS) of every qba_solve_kernel launch_qba can start"""
    body = _body(_src("pxr_qba.cu"), "static int launch_qba(")
    pairs = {(CTYPES[t], int(c)) for t, c in re.findall(r"PXR_QBA_CASE\((__half|float|double), (\d+)\)", body)}
    fs = {v == "true" for v in re.findall(r"launch_qba_t<T, CC, (true|false)>", body)}
    return {(d, c, f) for d, c in pairs for f in fs}


def irls_channels():
    body = _body(_src("pxr_refs.cu"), "static int refs_on_device(")
    return {int(c) for c in re.findall(r"case (\d+): PXR_TRY\(launch_irls<\1>", body)}


def test_instance_lists_are_read_from_the_sources():
    assert len(fm_instances()) == 20                        # 11 feature instances + 9 for the 1/3/4-channel maps
    assert len(ka_instances()) == 27 and len(qba_instances()) == 22
    assert irls_channels() == {8, 16, 32, 64, 128, 256}


def test_k1_rows_cover_every_instance_with_both_interpolations():
    want = {(d, c) for d, c in fm_instances() if c >= 8}
    got = {(_dt(r["dtype"]), r["channels"], r["fs"], r["l2"], (r["ph"], r["pw"])) for r in _rows(G.test_k1_and_inner_options)}
    assert {(d, c) for d, c, *_ in got} == want
    for d, c in want:
        assert {(fs, l2, s) for dd, cc, fs, l2, s in got if (dd, cc) == (d, c)} == \
            set(itertools.product((0, 1), (1, 0), ((16, 16), (8, 8))))
    small = {(_dt(r["dtype"]), r["channels"]) for r in _rows(G.test_k1_and_inner_small_channels_float_simd)}
    assert small == {(d, c) for d, c in fm_instances() if c < 8}


def test_ka_rows_cover_every_instance():
    rows = {(_dt(r["dtype"]), r["channels"], bool(r["fs"]), False) for r in _rows(G.test_ka_instance_options)}
    rows |= {(_dt(r["dtype"]), r["channels"], False, True) for r in _rows(G.test_query_ka_instance)}
    assert rows == ka_instances()
    for d, c, fs, _ in ka_instances():
        if fs:   # the float-SIMD query instance is not built: its refusal is a row of its own
            assert (d, c) in {(_dt(r["dtype"]), r["channels"]) for r in _rows(G.test_query_ka_refuses_float_simd)}
    l2 = {(_dt(r["dtype"]), r["channels"], r["fs"], r["l2"]) for r in _rows(G.test_ka_instance_options)}
    assert len(l2) == 9 * 2 * 2


def test_qba_rows_cover_every_instance():
    fs_rows = {(_dt(r["dtype"]), r["channels"], True) for r in _rows(G.test_qba_float_simd_instance)}
    assert fs_rows == {i for i in qba_instances() if i[2]}
    # the plain instances are the rows of test_gpu_qba_batch.py (every pair with the default interpolation)
    import test_gpu_qba_batch as Q
    plain = {(_dt(r["dtype"]), r["channels"], False) for r in _rows(Q.test_other_instances_match_single_query_path)}
    plain.add(("float16", 128, False))      # the default scene of every other test there
    assert plain == {i for i in qba_instances() if not i[2]}


def test_irls_rows_cover_every_channel_count():
    got = {r["channels"] for r in _rows(G.test_irls_every_channel_count)}
    assert got == irls_channels()
    assert set(G.IRLS_LENGTHS) == {1, 2, 31, 32, 33, 64, 65, 128, 129, 255, 256}
    assert {r["loss"] for r in _rows(G.test_irls_lengths_and_losses)} == set(_capi.LOSS_IDS.values())


# ---- 2. a plain restatement of reference extraction, in extended precision

def _rho(loss_type, a, s):
    """ceres' rho(s) of the five losses (the reference's loss factory) in long double"""
    a = np.longdouble(a)
    b = a * a
    if loss_type == 0:
        return s
    if loss_type == 1:
        return b * np.log1p(s / b)
    if loss_type == 2:
        return 2 * a * np.sqrt(s) - b if s > b else s
    if loss_type == 3:
        return 2 * b * (np.sqrt(1 + s / b) - 1)
    if loss_type == 4:
        return a * np.arctan2(s, a)
    raise ValueError(loss_type)


def irls_reference(D, loss_type, loss_scale, iters, l2):
    """RobustMeanIRLS (weights 1/rho(|d_i - mu|^2), normalised each round; an observation with rho == 0 is the mean)
    then the first observation closest to the mean.  D: [n, C] descriptors -> (index into D, round of the early exit
    or None)"""
    D = np.asarray(D, np.longdouble)
    w = np.ones(len(D), np.longdouble)
    mean, exit_round = None, None
    for k in range(iters):
        w = w / w.sum()
        mean = (D * w[:, None]).sum(0)
        if l2:
            nn = np.sqrt((mean * mean).sum())
            if nn > 0:
                mean = mean / nn
        early = None
        for i in range(len(D)):
            r = _rho(loss_type, loss_scale, ((D[i] - mean) ** 2).sum())
            if not r > 0:
                early = i
                break
            w[i] = 1 / r
        if early is not None:
            mean, exit_round = D[early], k
            break
    return int(np.argmin(((D - mean) ** 2).sum(1))), exit_round


LOSS_SCALES = {0: 1.0, 1: 0.25, 2: 0.1, 3: 0.1, 4: 0.2}


def test_irls_reference_restatement_agrees_with_the_oracle():
    prob, dup_points = G.irls_scene(channels=16, lengths=G.IRLS_LENGTHS)
    tl = np.bincount(prob.obs_pt, minlength=len(prob.xyz))
    first = np.concatenate([[0], np.cumsum(tl)])
    for l2 in (1, 0):
        ic = _capi.default_interp(l2_normalize=l2)
        D = G.oracle_descriptors(prob, ic)
        for loss_type in sorted(set(_capi.LOSS_IDS.values())):
            scale = LOSS_SCALES[loss_type]
            refs, src = O.refs_compute(prob, ic, loss_type, scale, 100)
            for p in range(len(prob.xyz)):
                Dp = D[first[p]:first[p + 1]]
                k, _ = irls_reference(Dp, loss_type, scale, 100, l2)
                if tl[p] == 2 and p not in dup_points:      # an exact tie: either observation is right
                    assert min(np.abs(refs[p] - d).max() for d in Dp) <= 1e-12
                    continue
                assert src[p] == first[p] + k, (l2, loss_type, p, tl[p])
                assert np.abs(refs[p] - Dp[k]).max() <= 1e-12, (l2, loss_type, p, tl[p])
    # the identical-descriptor tracks really hold two equal descriptors; the pair alone exits early in the first round
    # and keeps its first observation
    ic = _capi.default_interp(l2_normalize=0)
    D = G.oracle_descriptors(prob, ic)
    for p in dup_points:
        assert np.array_equal(D[first[p]], D[first[p] + 1])
    p = dup_points[0]
    assert tl[p] == 2 and irls_reference(D[first[p]:first[p + 1]], 1, 0.25, 100, 0) == (0, 0)
    assert O.refs_compute(prob, ic, 1, 0.25, 100)[1][p] == first[p]


def test_irls_early_exit_is_taken_on_identical_descriptors():
    """with two identical descriptors and no normalisation the mean equals them exactly in the first round: rho(0) == 0
    ends the iteration there, whatever the loss"""
    rng = np.random.default_rng(0)
    d = rng.normal(size=16)
    D = np.stack([d, d])
    for loss_type in sorted(set(_capi.LOSS_IDS.values())):
        assert irls_reference(D, loss_type, LOSS_SCALES[loss_type], 100, 0) == (0, 0)
