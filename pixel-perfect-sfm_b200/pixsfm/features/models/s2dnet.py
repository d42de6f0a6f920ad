"""S2DNet with one hypercolumn layer (reference features/models/s2dnet.py at `num_layers: 1`, the default of every shipped
configuration but pixsfm_eth3d_d2net.yaml): VGG16's conv1_1 / ReLU / conv1_2 / ReLU and one adaptation layer
(1x1 conv / ReLU / 5x5 conv / BatchNorm), computed by libpxr's fused kernel (csrc/pxr_s2dnet.cu) — only at the keypoints'
windows when the features are sparse.  Nothing is pooled at this depth, so the map is the size of the image.

The weights are one local file the user supplies (the reference downloads it to the same package-relative place); it is
never downloaded here.  Unlike the reference, which silently keeps random initial values for a missing or mis-shaped
key, every required key must be present with its shape."""
from pathlib import Path

import numpy as np

from ..extractor import _DTYPES as DTYPES
from ..._pixsfm import _engine

DEFAULT_CHECKPOINT = Path(__file__).parent / "checkpoints" / "s2dnet_weights.pth"
BN_EPS = 1e-5
_ADAP = "adaptation_layers.adap_layer_0."
# key -> shape of every tensor the reference's module takes from the checkpoint at num_layers 1
REQUIRED_KEYS = {"encoder.0.weight": (64, 3, 3, 3), "encoder.0.bias": (64,),
                 "encoder.2.weight": (64, 64, 3, 3), "encoder.2.bias": (64,),
                 _ADAP + "0.weight": (64, 64, 1, 1), _ADAP + "0.bias": (64,),
                 _ADAP + "2.weight": (128, 64, 5, 5), _ADAP + "2.bias": (128,),
                 _ADAP + "3.weight": (128,), _ADAP + "3.bias": (128,),
                 _ADAP + "3.running_mean": (128,), _ADAP + "3.running_var": (128,)}


def fold_batchnorm(weight, bias, gamma, beta, mean, var, eps=BN_EPS):
    """the eval-mode BatchNorm after a convolution folded into it, in float64 -> (weight, bias)"""
    weight, bias, gamma, beta, mean, var = (np.asarray(v, np.float64) for v in (weight, bias, gamma, beta, mean, var))
    s = gamma / np.sqrt(var + eps)
    return weight * s[:, None, None, None], (bias - mean) * s + beta


def pack_state_dict(state_dict):
    """the float32 array pxr_s2dnet_weights_create takes (include/pxr.h) from the reference's state dict (tensors or
    arrays); extra keys are ignored, a missing or mis-shaped required key raises ValueError"""
    arrays = {}
    for key, shape in REQUIRED_KEYS.items():
        if key not in state_dict:
            raise ValueError("the S2DNet checkpoint has no %r" % key)
        v = state_dict[key]
        v = np.asarray(v.detach().cpu().double().numpy() if hasattr(v, "detach") else v, np.float64)
        if v.shape != shape:
            raise ValueError("S2DNet checkpoint key %r has shape %s, not %s" % (key, v.shape, shape))
        arrays[key] = v
    w4, b4 = fold_batchnorm(arrays[_ADAP + "2.weight"], arrays[_ADAP + "2.bias"], arrays[_ADAP + "3.weight"],
                            arrays[_ADAP + "3.bias"], arrays[_ADAP + "3.running_mean"], arrays[_ADAP + "3.running_var"])
    parts = [arrays["encoder.0.weight"], arrays["encoder.0.bias"], arrays["encoder.2.weight"], arrays["encoder.2.bias"],
             arrays[_ADAP + "0.weight"], arrays[_ADAP + "0.bias"], w4, b4]
    return np.concatenate([p.ravel() for p in parts]).astype(np.float32)


def load_state_dict(path):
    """the checkpoint's state dict, read with torch (imported here, as _engine does)"""
    path = Path(path)
    if not path.is_file():
        raise ValueError("the S2DNet weights are not part of this package and are never downloaded: no file at %s. Put "
                         "s2dnet_weights.pth there or set the model's checkpoint_path" % path)
    import torch
    return torch.load(str(path), map_location="cpu", weights_only=True)["state_dict"]


class S2DNet:
    default_conf = {"num_layers": 1, "checkpointing": None, "output_dim": 128, "pretrained": "s2dnet",
                    "remove_pooling_layers": False, "combine": False, "checkpoint_path": None}
    image_mode = "RGB"

    def __init__(self, conf=None):
        conf = dict(conf or {})
        conf.pop("name", None)
        unknown = set(conf) - set(self.default_conf)
        if unknown:
            raise ValueError("unknown s2dnet options: %s" % sorted(unknown))
        self.conf = c = dict(self.default_conf, **conf)
        if c["num_layers"] != 1:
            raise ValueError("s2dnet is computed here at num_layers 1 only (got %r)" % (c["num_layers"],))
        if c["output_dim"] != 128:
            raise ValueError("s2dnet's checkpoint has output_dim 128 (got %r)" % (c["output_dim"],))
        if c["pretrained"] != "s2dnet":
            raise ValueError("s2dnet runs with its trained weights only (pretrained %r would leave it untrained)"
                             % (c["pretrained"],))
        # checkpointing only saves training memory; remove_pooling_layers and combine change nothing at one layer
        self.checkpoint_path = Path(c["checkpoint_path"]) if c["checkpoint_path"] is not None else DEFAULT_CHECKPOINT
        self.output_dims = [128]
        self.scales = [1]
        self.weights = _engine.s2dnet_weights(pack_state_dict(load_state_dict(self.checkpoint_path)))

    def map_size(self, height, width):
        """(H', W') of the feature map of a height x width image: the image's"""
        return height, width

    def __call__(self, image, corners=None, patch_size=16, l2_normalize=True, dtype="half", to_host=True):
        """[H,W,3] uint8 RGB image -> the windows at `corners` [n, ps, ps, 128], or the whole map [1, H, W, 128]"""
        return _engine.s2dnet(image, self.weights, corners, patch_size, l2_normalize, DTYPES[dtype], to_host)
