"""Image transforms of holocron.transforms, and the random transforms of the reference's classification, segmentation
and detection recipes, on batched CUDA kernels."""
from .augmentation import ColorJitter, RandomErasing, RandomHorizontalFlip, RandomResizedCrop, TrivialAugmentWide
from .interpolation import RandomZoomOut, Resize

__all__ = ["ColorJitter", "RandomErasing", "RandomHorizontalFlip", "RandomResizedCrop", "RandomZoomOut", "Resize",
           "TrivialAugmentWide"]
