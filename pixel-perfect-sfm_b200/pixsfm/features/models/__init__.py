"""The dense feature models this package computes itself (reference pixsfm/features/models/).  Only `dsift` is here:
S2DNet and VGG need downloaded weights and their convolutions are cuDNN's work."""
from .dsift import DSIFT  # noqa: F401
