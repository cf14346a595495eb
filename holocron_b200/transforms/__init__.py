"""Image transforms of holocron.transforms, and the random transforms of the reference's classification, segmentation
and detection recipes, on batched CUDA kernels."""
from .augmentation import ColorJitter, RandomErasing, RandomHorizontalFlip, RandomResizedCrop, TrivialAugmentWide
from .classification import Normalize
from .interpolation import RandomZoomOut, Resize

__all__ = ["ColorJitter", "Normalize", "RandomErasing", "RandomHorizontalFlip", "RandomResizedCrop", "RandomZoomOut",
           "Resize", "TrivialAugmentWide"]
