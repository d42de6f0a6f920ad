"""Dense SIFT without a GPU: the two oracle restatements against each other, the map size, the `dsift` preset against
the reference's configs/dsift.yaml, FeatureExtractor's options and image loading (the kernel replaced by oracle (a)),
and the drivers building the extractor from the preset."""
import os

import numpy as np
import pytest
import yaml

import dsift_oracle as D
from pixsfm._pixsfm import _engine
from pixsfm.features.extractor import FeatureExtractor, patch_corners
from pixsfm.features.models import DSIFT

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "configs", "dsift.yaml")
AS = [(4, 2), (4, 4), (8, 2), (8, 4)]


def _image(h, w, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (h, w)).astype(np.uint8)
    img[: h // 3, : w // 3] = 77                         # flat region: zero gradients
    img[h // 2, :] = 200                                 # horizontal edge: gy only
    return img


@pytest.mark.parametrize("A,S", AS)
@pytest.mark.parametrize("b", [3, 4, 5])
def test_conv_and_loop_oracles_agree(A, S, b):
    for k, (h, w) in enumerate([(11, 14), (9, 7)]):
        img = _image(h, w, 10 * A + S + b + k)
        rootsift, l2 = bool(k % 2 == 0), bool((b + k) % 2)
        a = D.dsift_conv(img, A, S, b, 0.2, rootsift, l2)
        c = D.dsift_loops(img, A, S, b, 0.2, rootsift, l2)
        assert a.shape == c.shape == D.map_size(h, w, S, b) + (A * S * S,)
        assert np.abs(a - c).max() < 1e-12


@pytest.mark.parametrize("S,b", [(4, 4), (4, 3), (4, 5), (2, 4), (2, 1), (4, 8)])
def test_map_size_formula(S, b):
    h, w = 23, 31
    extra = 2 * (b // 2) - b + 1 + 2 - S + 1
    assert _engine.dsift_map_size(h, w, S, b) == (h + extra, w + extra) == D.map_size(h, w, S, b)
    assert DSIFT({"num_spatial_bins": S, "spatial_bin_size": b}).map_size(h, w) == (h + extra, w + extra)
    assert D.dsift_conv(_image(h, w, 0), 4, S, b).shape[:2] == (h + extra, w + extra)
    if S == 4 and b == 4:
        assert extra == 0


def _resolve(top):
    from pixsfm.refine_colmap import _resolve_references
    return {k: _resolve_references(v, top) if isinstance(v, dict) else v for k, v in top.items()}


def test_dsift_preset_is_the_reference_file():
    from pixsfm.configs import default_configs, parse_config_path
    with open(GOLDEN) as f:
        golden = _resolve(yaml.safe_load(f))
    assert parse_config_path("dsift") == golden == default_configs["dsift"]()


def test_dsift_model_and_extractor_options():
    m = DSIFT()
    assert m.output_dims == [128] and m.scales == [1]
    assert DSIFT({"name": "dsift", "num_ang_bins": 4, "num_spatial_bins": 2}).output_dims == [16]
    for bad in ({"num_ang_bins": 6}, {"num_spatial_bins": 3}, {"spatial_bin_size": 0}, {"spatial_bin_size": 9},
                {"clipval": 0.0}, {"bins": 4}):
        with pytest.raises(ValueError):
            DSIFT(bad)
    ex = FeatureExtractor({"model": {"name": "dsift"}})
    assert ex.conf["max_edge"] == 1600 and ex.conf["resize"] == "LANCZOS" and ex.conf["pyr_scales"] == [1.0]
    assert ex.channels_per_level == [128]
    with pytest.raises(ValueError, match="not part of this package"):
        FeatureExtractor({})                                        # the reference's default model is s2dnet
    with pytest.raises(ValueError, match="not part of this package"):
        FeatureExtractor({"model": {"name": "vgg16"}})
    with pytest.raises(ValueError, match="GPU only"):
        FeatureExtractor({"model": {"name": "dsift"}, "device": "cpu"})
    with pytest.raises(ValueError, match="unknown extractor options"):
        FeatureExtractor({"model": {"name": "dsift"}, "maxedge": 100})
    with pytest.raises(ValueError):
        FeatureExtractor({"model": {"name": "dsift", "num_ang_bins": 5}})
    with pytest.raises(ValueError):
        FeatureExtractor({"model": {"name": "dsift"}, "resize": "NEAREST"})


def _fake_dsift(calls):
    """_engine.dsift with oracle (a) in place of the kernel (host output only)"""
    def run(image, corners=None, patch_size=16, num_ang_bins=8, num_spatial_bins=4, spatial_bin_size=4, clipval=0.2,
            rootsift=True, l2_normalize=True, out_dtype=np.float16, to_host=False, ctx=None):
        calls.append((image.shape, corners is None, to_host))
        full = D.dsift_conv(image, num_ang_bins, num_spatial_bins, spatial_bin_size, clipval, rootsift, l2_normalize)
        full = full.astype(out_dtype)
        if corners is None:
            return full[None]
        return np.stack([full[y:y + patch_size, x:x + patch_size] for x, y in np.asarray(corners)])
    return run


def _write_png(path, h, w, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    rgb = (rng.random((h, w, 3)) * 255).astype(np.uint8)
    Image.fromarray(rgb, "RGB").save(str(path))
    return rgb


def test_extractor_loads_resizes_and_extracts(tmp_path, monkeypatch):
    from PIL import Image
    calls = []
    monkeypatch.setattr(_engine, "dsift", _fake_dsift(calls))
    (tmp_path / "imgs").mkdir()
    _write_png(tmp_path / "imgs" / "a.png", 61, 97, 0)
    conf = {"model": {"name": "dsift", "num_ang_bins": 4, "num_spatial_bins": 2}, "max_edge": 50,
            "pyr_scales": [1.0, 0.6], "dtype": "float", "patch_size": 6}
    ex = FeatureExtractor(conf)
    levels, size = ex.load_image(tmp_path / "imgs" / "a.png")
    assert size == (97, 61) and [lv.shape for lv in levels] == [(31, 50), (19, 30)]
    want = np.asarray(Image.open(tmp_path / "imgs" / "a.png").resize((50, 31), Image.LANCZOS).convert("L"))
    assert levels[0].dtype == np.uint8 and np.array_equal(levels[0], want)

    kps = np.array([[5.0, 3.0], [48.5, 30.2], [90.0, 59.0], [40.0, 20.0]])
    fm = ex.features_from_image_list(tmp_path / "imgs", ["a.png"], {"a.png": kps})
    assert fm.num_levels == 2 and fm.fset(0).channels == 16
    for level, img in enumerate(levels):
        fmap = fm.fset(level).fmap("a.png")
        h, w = D.map_size(*img.shape, 2, 4)
        assert np.allclose(fmap.scale, (w / 97, h / 61)) and fmap.is_sparse
        corners = patch_corners(kps, fmap.scale, 6, (w, h))
        assert np.array_equal(fmap.corners, corners)
        full = D.dsift_conv(img, 4, 2, 4).astype(np.float32)
        for k, (x, y) in enumerate(corners):
            assert np.array_equal(fmap.patches[k], full[y:y + 6, x:x + 6])
    assert all(not dense and host for _, dense, host in calls)

    # a path instead of image_dir / name (QueryLocalizer._query_features), and more patches than the map: dense
    many = np.tile(kps, (20, 1))
    fm2 = ex.features_from_image_list(None, [str(tmp_path / "imgs" / "a.png")], {str(tmp_path / "imgs" / "a.png"): many})
    dense = fm2.fset(0).fmap(str(tmp_path / "imgs" / "a.png"))
    assert not dense.is_sparse and dense.patches.shape == (1,) + D.map_size(31, 50, 2, 4) + (16,)
    assert np.array_equal(dense.patches[0], D.dsift_conv(levels[0], 4, 2, 4).astype(np.float32))

    # the cache round trip: written once, then read back instead of extracted
    cached = FeatureExtractor(dict(conf, use_cache=True, load_cache_on_init=True))
    n = len(calls)
    fm3 = cached.features_from_image_list(tmp_path / "imgs", ["a.png"], {"a.png": kps}, cache_path=tmp_path / "c.h5")
    assert (tmp_path / "c.h5").exists() and len(calls) == n + 2
    fm4 = cached.features_from_image_list(tmp_path / "imgs", ["a.png"], {"a.png": kps}, cache_path=tmp_path / "c.h5")
    assert len(calls) == n + 2
    for level in range(2):
        a, b = fm.fset(level).fmap("a.png"), fm4.fset(level).fmap("a.png")
        assert np.array_equal(np.asarray(a.patches), np.asarray(fm3.fset(level).fmap("a.png").patches))
        assert np.array_equal(a.corners, b.corners) and np.array_equal(np.asarray(a.patches), np.asarray(b.patches))


def test_drivers_build_the_extractor_from_the_preset(tmp_path):
    from pathlib import Path
    from pixsfm.localization.main import QueryLocalizer
    from pixsfm.refine_colmap import PixSfM
    from recon_util import make_reconstruction
    s = PixSfM("dsift")
    assert isinstance(s.extractor, FeatureExtractor) and s.extractor.conf["max_edge"] == 2000
    assert s.extractor.conf["model"]["spatial_bin_size"] == 4 and s.extractor.conf["dtype"] == "half"
    assert s.resolve_cache_path(None, tmp_path) == Path(tmp_path) / "dsift_featuremaps_sparse.h5"
    s2 = PixSfM(GOLDEN)
    assert isinstance(s2.extractor, FeatureExtractor) and s2.extractor.conf == s.extractor.conf
    assert PixSfM().extractor is None
    rec = make_reconstruction(n_cams=3, n_points=10, track_len=3, channels=8, seed=1)[0]
    loc = QueryLocalizer(rec, "dsift", image_dir=tmp_path, references=[{}])
    assert isinstance(loc.extractor, FeatureExtractor) and loc.extractor.conf["max_edge"] == 2000
    loc2 = QueryLocalizer(rec, GOLDEN, image_dir=tmp_path, references=[{}])
    assert isinstance(loc2.extractor, FeatureExtractor)
    assert QueryLocalizer(rec, {}, references=[{}]).extractor is None
