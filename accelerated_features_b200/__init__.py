"""accelerated_features_b200: XFeat inference hot path as hand-written sm_90a CUDA kernels (drop-in `XFeat` class)."""
from .xfeat import XFeat  # noqa: F401

__all__ = ["XFeat"]
__version__ = "0.1.0"
