"""Model-building and checkpoint-format helpers mirroring holocron/models/utils.py (conv_sequence :28-86,
load_pretrained_params :89-113, fuse_conv_bn :116-143, model_from_hf_hub :146-175, _configure_model :178-188,
_checkpoint_from_hub_config :191-206) plus the writers the reference keeps in its scripts (HF-hub folder layout,
references/clean_checkpoint.py)."""
import hashlib
import json
import logging
from pathlib import Path
from typing import Any, Callable, Dict, List, Optional, Sequence, Tuple, TypeVar, Union

import torch
from torch import nn

from .checkpoints import Checkpoint, Dataset, Evaluation, LoadingMeta, PreProcessing, TrainingRecipe

__all__ = ["clean_checkpoint", "conv_sequence", "fuse_conv_bn", "load_pretrained_params", "model_from_hf_hub",
           "save_hf_hub_folder"]

logger = logging.getLogger(__name__)

M = TypeVar("M", bound=nn.Module)


def conv_sequence(
    in_channels: int,
    out_channels: int,
    act_layer: Optional[nn.Module] = None,
    norm_layer: Optional[Callable[[int], nn.Module]] = None,
    drop_layer: Optional[Callable[..., nn.Module]] = None,
    conv_layer: Optional[Callable[..., nn.Module]] = None,
    bn_channels: Optional[int] = None,
    attention_layer: Optional[Callable[[int], nn.Module]] = None,
    blurpool: bool = False,
    **kwargs: Any,
) -> List[nn.Module]:
    """Builds ``[conv(bias = norm is None), norm, act, attention, drop(inplace=True)]`` with the reference's ordering
    and bias rule. ``blurpool`` is outside the hot path and not supported here."""
    if blurpool:
        raise NotImplementedError("conv_sequence(blurpool=True) is not supported: no model here builds a blur-pooled "
                                  "block; use holocron_b200.nn.BlurPool2d directly")
    if conv_layer is None:
        conv_layer = nn.Conv2d
    if bn_channels is None:
        bn_channels = out_channels
    # a convolution followed by a normalisation layer does not need a bias
    kwargs["bias"] = kwargs.get("bias", norm_layer is None)
    layers: List[nn.Module] = [conv_layer(in_channels, out_channels, **kwargs)]
    if callable(norm_layer):
        layers.append(norm_layer(bn_channels))
    if callable(act_layer):
        layers.append(act_layer)
    if callable(attention_layer):
        layers.append(attention_layer(bn_channels))
    if callable(drop_layer):
        layers.append(drop_layer(inplace=True))
    return layers


def fuse_conv_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d) -> Tuple[torch.Tensor, torch.Tensor]:
    """Folds an (eval-mode) BatchNorm into the preceding convolution: returns the fused kernel and bias.

    k' = gamma / sqrt(running_var + eps) * k ;  b' = beta - gamma * running_mean / sqrt(running_var + eps) (+ scaled conv bias).
    Weight-sized host-side arithmetic in fp32 (one-off at re-parametrisation time), same operation order as the
    reference so the re-parametrised logits keep their argmax (BASELINE.json config 1).
    """
    if bn.bias.data.shape[0] != conv.weight.data.shape[0]:
        raise AssertionError("expected same number of output channels for both `conv` and `bn`")
    scale = bn.weight.data / torch.sqrt(bn.running_var + bn.eps)
    fused_bias = bn.bias.data - scale * bn.running_mean
    if conv.bias is not None:
        logger.warning("convolution layers placed before batch normalization should not have a bias.")
        fused_bias += scale * conv.bias.data
    fused_kernel = scale.view(-1, 1, 1, 1) * conv.weight.data
    return fused_kernel, fused_bias


# ------------------------------------------------------------------------------------------------ checkpoint formats
def load_pretrained_params(model: nn.Module, url: Optional[str] = None, progress: bool = True,
                           key_replacement: Optional[Tuple[str, str]] = None, key_filter: Optional[str] = None) -> None:
    """Loads a ``state_dict`` from ``url`` into ``model`` (reference models/utils.py:89-113): keys optionally filtered by
    prefix, then renamed. ``file://`` URLs are served from the local disk by ``torch.hub``; the module trees of this
    package carry the reference's parameter names, so its released checkpoints load unchanged."""
    if url is None:
        logger.warning("Invalid model URL, using default initialization.")
        return
    state_dict = torch.hub.load_state_dict_from_url(url, progress=progress, map_location="cpu")
    if isinstance(key_filter, str):
        state_dict = {k: v for k, v in state_dict.items() if k.startswith(key_filter)}
    if isinstance(key_replacement, tuple):
        state_dict = {k.replace(*key_replacement): v for k, v in state_dict.items()}
    model.load_state_dict(state_dict)


def _configure_model(model: M, checkpoint: Union[Checkpoint, None], **kwargs: Any) -> M:
    """reference models/utils.py:178-188: remembers the checkpoint description and loads its parameters."""
    model.default_cfg = checkpoint  # type: ignore[assignment]
    if isinstance(checkpoint, Checkpoint):
        load_pretrained_params(model, checkpoint.meta.url, **kwargs)
    return model


def _requested_checkpoint(pretrained: bool, checkpoint: Union[Checkpoint, None]) -> Union[Checkpoint, None]:
    """The factories' ``pretrained`` / ``checkpoint`` arguments. The reference falls back to a table of released checkpoints
    (GitHub URLs) when ``pretrained`` is set without a checkpoint; there is no network here and the table is not shipped."""
    if checkpoint is not None and not isinstance(checkpoint, Checkpoint):
        raise TypeError(f"`checkpoint` is expected to be a holocron_b200.models.checkpoints.Checkpoint, got {type(checkpoint)}")
    if pretrained and checkpoint is None:
        raise NotImplementedError("the released checkpoints need network access: pass checkpoint=Checkpoint(...) (its "
                                  "meta.url may be a file:// URL) or load a reference state_dict - the module tree and "
                                  "parameter names are identical")
    return checkpoint


def _checkpoint_from_hub_config(hub_config: Dict[str, Any]) -> Checkpoint:
    """reference models/utils.py:191-206."""
    return Checkpoint(
        evaluation=Evaluation(dataset=Dataset.IMAGENETTE, results={}),
        meta=LoadingMeta(url="N/A", sha256="N/A", size=0, num_params=0, arch=hub_config["arch"],
                         categories=hub_config["classes"]),
        pre_processing=PreProcessing(input_shape=hub_config["input_shape"], mean=hub_config["mean"], std=hub_config["std"]),
        recipe=TrainingRecipe(commit=None, script="references/classification/train.py", args=None),
    )


def model_from_hf_hub(repo_id: str, **kwargs: Any) -> nn.Module:
    """Instantiates a model from a HuggingFace-hub repository laid out like the reference's (``config.json`` with ``arch``,
    ``classes``, ``input_shape``, ``mean``, ``std`` + ``pytorch_model.bin``) - reference models/utils.py:146-175. ``kwargs`` go
    to ``hf_hub_download`` (``local_files_only=True`` / ``cache_dir=`` work offline; :func:`save_hf_hub_folder` writes the
    same two files)."""
    from huggingface_hub import hf_hub_download

    from .. import models
    with Path(hf_hub_download(repo_id, filename="config.json", **kwargs)).open("rb") as f:
        cfg = json.load(f)
    model = models.__dict__[cfg["arch"]](num_classes=len(cfg["classes"]), pretrained=False)
    if getattr(model, "default_cfg", None) is None:
        model.default_cfg = cfg
    elif isinstance(model.default_cfg, Checkpoint):
        model.default_cfg = _checkpoint_from_hub_config(cfg)
    else:
        model.default_cfg.update(cfg)
    state_dict = torch.load(hf_hub_download(repo_id, filename="pytorch_model.bin", **kwargs), map_location="cpu")
    model.load_state_dict(state_dict)
    return model


def save_hf_hub_folder(model: nn.Module, folder: Union[str, Path], arch: str, classes: Sequence[str],
                       input_shape: Sequence[int] = (3, 224, 224), mean: Sequence[float] = (0.485, 0.456, 0.406),
                       std: Sequence[float] = (0.229, 0.224, 0.225), **extra: Any) -> Path:
    """Writes the two files :func:`model_from_hf_hub` (here and in the reference) reads: ``config.json`` and
    ``pytorch_model.bin`` (CPU tensors, the reference's parameter names). Returns the folder."""
    folder = Path(folder)
    folder.mkdir(parents=True, exist_ok=True)
    cfg = {"arch": arch, "classes": list(classes), "input_shape": list(input_shape), "mean": list(mean), "std": list(std),
           **extra}
    (folder / "config.json").write_text(json.dumps(cfg, indent=2))
    torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, folder / "pytorch_model.bin")
    return folder


def clean_checkpoint(checkpoint: Union[str, Path], outfile: Union[str, Path]) -> str:
    """Training checkpoint (``Trainer.save``: epoch / step / losses / model / optimizer / scheduler state) -> the bare model
    ``state_dict`` in the legacy (non-zip) serialisation the reference releases, and its SHA-256 (the first 8 hex digits
    go into the released file name) - reference references/clean_checkpoint.py:12-18."""
    state = torch.load(checkpoint, map_location="cpu")["model"]
    torch.save(state, outfile, _use_new_zipfile_serialization=False)
    with Path(outfile).open("rb") as f:
        return hashlib.sha256(f.read()).hexdigest()
