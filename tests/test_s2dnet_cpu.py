"""S2DNet without a GPU: the float64 restatement against torchvision's modules, the BatchNorm fold, the model's option and
weight rules, FeatureExtractor's image loading (the kernel replaced by the restatement), the C-ABI's argument checks,
and the drivers' rule for building the extractor."""
import ctypes as C

import numpy as np
import pytest

import s2dnet_reference as R
from pixsfm._pixsfm import _capi, _engine
from pixsfm.features.extractor import FeatureExtractor, patch_corners
from pixsfm.features.models import s2dnet as S
from pixsfm.features.models.s2dnet import S2DNet, fold_batchnorm, pack_state_dict


def _rgb(h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3)).astype(np.uint8)


def test_restatement_matches_torchvision_modules():
    torch = pytest.importorskip("torch")
    tv = pytest.importorskip("torchvision")
    sd = R.seeded_state_dict(3)

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.encoder = torch.nn.ModuleList(list(tv.models.vgg16().features.children())[:4])
            layer = torch.nn.Sequential(torch.nn.Conv2d(64, 64, 1), torch.nn.ReLU(), torch.nn.Conv2d(64, 128, 5, padding=2),
                                        torch.nn.BatchNorm2d(128))
            self.adaptation_layers = torch.nn.Module()
            self.adaptation_layers.add_module("adap_layer_0", layer)

        def forward(self, x):
            for m in self.encoder:
                x = m(x)
            return self.adaptation_layers.adap_layer_0(x)

    net = Net().double().eval()
    params = net.state_dict()
    net.load_state_dict({k: v for k, v in sd.items() if k in params})
    assert set(params) <= set(sd)
    for h, w in ((7, 9), (13, 5)):
        img = _rgb(h, w, h + w)
        x = torch.from_numpy(img).permute(2, 0, 1)[None].double() / 255
        x = (x - torch.tensor(R.MEAN, dtype=torch.float64)[:, None, None]) / torch.tensor(R.STD, dtype=torch.float64)[:, None, None]
        with torch.no_grad():
            want = net(x)[0].permute(1, 2, 0)
        got = R.forward(img, sd, l2_normalize=False)
        assert float((got - want).abs().max()) < 1e-12


def test_batchnorm_fold_equals_the_unfolded_layer():
    torch = pytest.importorskip("torch")
    import torch.nn.functional as Fn
    sd = {k: v.double() for k, v in R.seeded_state_dict(1).items() if v.is_floating_point()}
    a = R.ADAP
    x = torch.randn(1, 64, 9, 11, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
    want = Fn.batch_norm(Fn.conv2d(x, sd[a + "2.weight"], sd[a + "2.bias"], padding=2), sd[a + "3.running_mean"],
                         sd[a + "3.running_var"], sd[a + "3.weight"], sd[a + "3.bias"], training=False, eps=1e-5)
    w, b = fold_batchnorm(sd[a + "2.weight"], sd[a + "2.bias"], sd[a + "3.weight"], sd[a + "3.bias"],
                          sd[a + "3.running_mean"], sd[a + "3.running_var"])
    got = Fn.conv2d(x, torch.from_numpy(w), torch.from_numpy(b), padding=2)
    assert float((got - want).abs().max()) < 1e-12


def test_packed_weights_follow_the_header_order():
    sd = R.seeded_state_dict(2)
    packed = pack_state_dict(sd)
    assert packed.dtype == np.float32 and packed.size == _engine.S2DNET_FLOATS == 247808
    assert np.array_equal(packed[:1728], sd["encoder.0.weight"].numpy().ravel())
    a = R.ADAP
    w, b = fold_batchnorm(sd[a + "2.weight"], sd[a + "2.bias"], sd[a + "3.weight"], sd[a + "3.bias"],
                          sd[a + "3.running_mean"], sd[a + "3.running_var"])
    assert np.array_equal(packed[-128:], b.astype(np.float32))
    assert np.array_equal(packed[-128 - 204800:-128], w.astype(np.float32).ravel())


def test_model_options_and_weight_rules(tmp_path, monkeypatch):
    made = []
    monkeypatch.setattr(_engine, "s2dnet_weights", lambda packed, ctx=None: made.append(packed) or "w")
    ckpt = R.write_checkpoint(tmp_path / "w.pth", seed=0)
    m = S2DNet({"name": "s2dnet", "checkpoint_path": str(ckpt), "checkpointing": 2, "remove_pooling_layers": True,
                "combine": True})
    assert m.output_dims == [128] and m.scales == [1] and m.map_size(5, 7) == (5, 7) and m.image_mode == "RGB"
    assert made and np.array_equal(made[-1], pack_state_dict(R.seeded_state_dict(0)))
    for bad in ({"num_layers": 2}, {"num_layers": 3}, {"output_dim": 64}, {"pretrained": "imagenet"},
                {"pretrained": None}, {"layers": 1}):
        with pytest.raises(ValueError):
            S2DNet(dict(bad, checkpoint_path=str(ckpt)))
    sd = R.seeded_state_dict(0)
    del sd["encoder.2.bias"]
    with pytest.raises(ValueError, match="encoder.2.bias"):
        S2DNet({"checkpoint_path": str(R.write_checkpoint(tmp_path / "missing.pth", state_dict=sd))})
    sd = R.seeded_state_dict(0)
    sd[R.ADAP + "2.weight"] = sd[R.ADAP + "2.weight"][:64]
    with pytest.raises(ValueError, match="shape"):
        S2DNet({"checkpoint_path": str(R.write_checkpoint(tmp_path / "shape.pth", state_dict=sd))})


def test_a_missing_weights_file_raises_without_a_download(tmp_path, monkeypatch):
    import socket
    import subprocess

    def no_network(*a, **k):
        raise AssertionError("no network call may be made")
    monkeypatch.setattr(socket, "create_connection", no_network)
    monkeypatch.setattr(subprocess, "call", no_network)
    monkeypatch.setattr(subprocess, "run", no_network)
    where = tmp_path / "nowhere" / "s2dnet_weights.pth"
    with pytest.raises(ValueError, match="not part of this package") as e:
        S2DNet({"checkpoint_path": str(where)})
    assert str(where) in str(e.value) and "checkpoint_path" in str(e.value)
    assert not where.parent.exists()
    if not S.DEFAULT_CHECKPOINT.exists():
        with pytest.raises(ValueError, match="not part of this package") as e:
            S2DNet({})
        assert str(S.DEFAULT_CHECKPOINT) in str(e.value)


def _fake_s2dnet(calls):
    """_engine.s2dnet with the float64 restatement in place of the kernel (host output only)"""
    def run(image, weights, corners=None, patch_size=16, l2_normalize=True, out_dtype=np.float16, to_host=False, ctx=None):
        calls.append((image.shape, corners is None, to_host))
        full = np.ascontiguousarray(R.forward(image, R.seeded_state_dict(0), l2_normalize).numpy(), out_dtype)
        if corners is None:
            return full[None]
        return np.stack([full[y:y + patch_size, x:x + patch_size] for x, y in np.asarray(corners)])
    return run


@pytest.mark.parametrize("mode", ["RGB", "L", "RGBA"])
def test_extractor_loads_rgb_resizes_and_extracts(tmp_path, monkeypatch, mode):
    from PIL import Image
    calls = []
    monkeypatch.setattr(_engine, "s2dnet_weights", lambda packed, ctx=None: "w")
    monkeypatch.setattr(_engine, "s2dnet", _fake_s2dnet(calls))
    ckpt = R.write_checkpoint(tmp_path / "w.pth", seed=0)
    rng = np.random.default_rng(0)
    src = Image.fromarray((rng.random((61, 97, 3)) * 255).astype(np.uint8), "RGB").convert(mode)
    src.save(str(tmp_path / "a.png"))
    conf = {"model": {"checkpoint_path": str(ckpt)}, "max_edge": 50, "pyr_scales": [1.0, 0.6], "dtype": "float",
            "patch_size": 6}
    ex = FeatureExtractor(conf)
    assert ex.conf["model"]["name"] == "s2dnet" and ex.channels_per_level == [128, 128]
    levels, size = ex.load_image(tmp_path / "a.png")
    assert size == (97, 61) and [lv.shape for lv in levels] == [(31, 50, 3), (19, 30, 3)]
    want = np.asarray(Image.open(tmp_path / "a.png").resize((50, 31), Image.LANCZOS).convert("RGB"))
    assert levels[0].dtype == np.uint8 and np.array_equal(levels[0], want)
    kps = np.array([[5.0, 3.0], [48.5, 30.2], [90.0, 59.0], [40.0, 20.0]])
    fm = ex.features_from_image_list(tmp_path, ["a.png"], {"a.png": kps})
    assert fm.num_levels == 2 and fm.fset(0).channels == 128
    for level, img in enumerate(levels):
        fmap = fm.fset(level).fmap("a.png")
        h, w = img.shape[:2]
        assert np.allclose(fmap.scale, (w / 97, h / 61)) and fmap.is_sparse
        corners = patch_corners(kps, fmap.scale, 6, (w, h))
        assert np.array_equal(fmap.corners, corners)
        full = R.forward(img, R.seeded_state_dict(0)).numpy().astype(np.float32)
        for k, (x, y) in enumerate(corners):
            assert np.array_equal(fmap.patches[k], full[y:y + 6, x:x + 6])
    assert all(not dense and host for _, dense, host in calls)


def test_c_abi_rejects_malformed_arguments_without_a_device():
    lib = _capi.load_lib()
    packed = np.zeros(_engine.S2DNET_FLOATS, np.float32)
    out = C.c_void_p()
    assert lib.pxr_s2dnet_weights_create(None, _capi.ptr(packed), C.c_int64(packed.size - 1), C.byref(out)) == \
        _capi.PXR_ERR_INVALID_ARGUMENT and b"247808" in lib.pxr_last_error()
    bad = packed.copy()
    bad[5] = np.nan
    assert lib.pxr_s2dnet_weights_create(None, _capi.ptr(bad), C.c_int64(bad.size), C.byref(out)) == \
        _capi.PXR_ERR_INVALID_ARGUMENT and b"finite" in lib.pxr_last_error()
    bad = packed.copy()
    bad[1728 + 64 + 7] = 1e5                                      # conv1_2 weight outside fp16
    assert lib.pxr_s2dnet_weights_create(None, _capi.ptr(bad), C.c_int64(bad.size), C.byref(out)) == \
        _capi.PXR_ERR_INVALID_ARGUMENT and b"fp16" in lib.pxr_last_error()
    assert lib.pxr_s2dnet_weights_create(None, _capi.ptr(packed), C.c_int64(packed.size), C.byref(out)) == \
        _capi.PXR_ERR_INVALID_ARGUMENT and b"NULL" in lib.pxr_last_error()
    lib.pxr_s2dnet_weights_destroy(None)

    img = _rgb(40, 50, 0)
    res = np.zeros((4, 16, 16, 128), np.float16)

    def run(corners, n, ps, dtype=0, h=40, w=50):
        c = None if corners is None else _capi.ptr(np.ascontiguousarray(corners, np.int32))
        return lib.pxr_s2dnet(None, None, _capi.ptr(img), 0, h, w, c, C.c_int64(n), ps, 1, dtype, _capi.ptr(res), None)
    for corners, msg in (([[-1, 0]], b"leaves the"), ([[0, -1]], b"leaves the"), ([[35, 0]], b"leaves the"),
                         ([[0, 25]], b"leaves the")):
        assert run(corners, 1, 16) == _capi.PXR_ERR_INVALID_ARGUMENT and msg in lib.pxr_last_error()
    assert run([[0, 0]], 1, 41) == _capi.PXR_ERR_INVALID_ARGUMENT and b"window size" in lib.pxr_last_error()
    assert run([[0, 0]], 1, 16, dtype=3) == _capi.PXR_ERR_INVALID_ARGUMENT and b"dtype" in lib.pxr_last_error()
    assert run(None, 0, 16, h=0) == _capi.PXR_ERR_INVALID_ARGUMENT and b"empty" in lib.pxr_last_error()
    assert run(None, 0, 16) == _capi.PXR_ERR_INVALID_ARGUMENT and b"NULL" in lib.pxr_last_error()


def test_drivers_build_the_s2dnet_extractor_only_with_weights(tmp_path, monkeypatch):
    from pixsfm.localization.main import QueryLocalizer
    from pixsfm.refine_colmap import PixSfM
    from recon_util import make_reconstruction
    monkeypatch.setattr(_engine, "s2dnet_weights", lambda packed, ctx=None: "w")
    ckpt = R.write_checkpoint(tmp_path / "w.pth", seed=0)
    with_weights = {"dense_features": {"model": {"name": "s2dnet", "checkpoint_path": str(ckpt)}}}
    s = PixSfM(with_weights)
    assert isinstance(s.extractor, FeatureExtractor) and isinstance(s.extractor.model, S2DNet)
    s_default = PixSfM({"dense_features": {"model": {"checkpoint_path": str(ckpt)}}})
    assert isinstance(s_default.extractor.model, S2DNet)
    rec = make_reconstruction(n_cams=3, n_points=10, track_len=3, channels=8, seed=1)[0]
    loc = QueryLocalizer(rec, {"localization": with_weights}, image_dir=tmp_path, references=[{}])
    assert isinstance(loc.extractor, FeatureExtractor) and isinstance(loc.extractor.model, S2DNet)
    if not S.DEFAULT_CHECKPOINT.exists():
        assert PixSfM().extractor is None
        assert PixSfM({"dense_features": {"model": {"name": "s2dnet"}}}).extractor is None
        assert QueryLocalizer(rec, {}, references=[{}]).extractor is None
        with pytest.raises(ValueError, match="no feature_manager given") as e:
            PixSfM()._features("features_from_graph", None, None, None)
        assert str(S.DEFAULT_CHECKPOINT) in str(e.value)
    assert PixSfM({"dense_features": {"model": {"name": "vgg16"}}}).extractor is None
