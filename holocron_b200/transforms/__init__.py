"""Image transforms of holocron.transforms on a batched CUDA resampling kernel."""
from .interpolation import RandomZoomOut, Resize

__all__ = ["RandomZoomOut", "Resize"]
