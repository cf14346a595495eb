"""holocron_b200: H100-native (sm_90a) implementation of the data-parallel training hot path of frgfm/Holocron.

Public surface mirrors ``holocron.nn`` / ``holocron.nn.functional`` / ``holocron.ops`` / ``holocron.optim`` /
``holocron.models`` for the hot-path components (see DESIGN.md). All compute goes through the C-ABI CUDA library
``holocron_b200/csrc/libholocron_b200.so`` declared in ``include/holocron_b200.h``.
"""
from . import nn, ops, optim, models, trainer, transforms, utils  # noqa: F401
from ._lib import HolocronB200Error, lib, lib_path  # noqa: F401

__version__ = "0.1.0"
