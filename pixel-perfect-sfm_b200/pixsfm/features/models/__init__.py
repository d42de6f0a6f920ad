"""The dense feature models this package computes itself (reference pixsfm/features/models/): `dsift`, and `s2dnet` at
num_layers 1 from a local weights file.  VGG and the deeper S2DNet levels are not here."""
from .dsift import DSIFT  # noqa: F401
from .s2dnet import S2DNet  # noqa: F401
