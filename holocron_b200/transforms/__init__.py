"""Image transforms of holocron.transforms, and the random transforms of the reference's classification recipe, on
batched CUDA kernels."""
from .augmentation import RandomErasing, RandomHorizontalFlip, RandomResizedCrop, TrivialAugmentWide
from .interpolation import RandomZoomOut, Resize

__all__ = ["RandomErasing", "RandomHorizontalFlip", "RandomResizedCrop", "RandomZoomOut", "Resize", "TrivialAugmentWide"]
