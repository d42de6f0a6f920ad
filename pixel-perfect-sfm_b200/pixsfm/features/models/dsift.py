"""Dense SIFT (reference features/models/dsift.py: kornia's DenseSIFTDescriptor with stride 1 and padding 1), computed
by libpxr's fused kernel (csrc/pxr_dsift.cu) — only at the keypoints' windows when the features are sparse.  The
descriptor follows the structure of kornia's; bit parity with kornia is unverified."""
from ..extractor import _DTYPES as DTYPES
from ..._pixsfm import _engine


class DSIFT:
    default_conf = {"num_ang_bins": 8, "num_spatial_bins": 4, "spatial_bin_size": 4, "rootsift": True, "clipval": 0.2}
    image_mode = "L"

    def __init__(self, conf=None):
        conf = dict(conf or {})
        conf.pop("name", None)
        unknown = set(conf) - set(self.default_conf)
        if unknown:
            raise ValueError("unknown dsift options: %s" % sorted(unknown))
        self.conf = dict(self.default_conf, **conf)
        c = self.conf
        if c["num_ang_bins"] not in (4, 8) or c["num_spatial_bins"] not in (2, 4):
            raise ValueError("dsift supports num_ang_bins 4 or 8 and num_spatial_bins 2 or 4 (got %r, %r)"
                             % (c["num_ang_bins"], c["num_spatial_bins"]))
        if not isinstance(c["spatial_bin_size"], int) or not 1 <= c["spatial_bin_size"] <= 8:
            raise ValueError("dsift supports spatial_bin_size 1..8 (got %r)" % (c["spatial_bin_size"],))
        if not float(c["clipval"]) > 0:
            raise ValueError("clipval must be positive (got %r)" % (c["clipval"],))
        self.output_dims = [c["num_ang_bins"] * c["num_spatial_bins"] ** 2]
        self.scales = [1]

    def map_size(self, height, width):
        """(H', W') of the descriptor map of a height x width image"""
        return _engine.dsift_map_size(height, width, self.conf["num_spatial_bins"], self.conf["spatial_bin_size"])

    def __call__(self, image, corners=None, patch_size=16, l2_normalize=True, dtype="half", to_host=True):
        """[H,W] uint8 image -> the windows at `corners` [n, ps, ps, C], or the whole map [1, H', W', C]"""
        c = self.conf
        return _engine.dsift(image, corners, patch_size, c["num_ang_bins"], c["num_spatial_bins"], c["spatial_bin_size"],
                             float(c["clipval"]), bool(c["rootsift"]), l2_normalize, DTYPES[dtype], to_host)
