"""Small model pieces for the SyncBatchNorm tests: each one exercises a different fused BatchNorm consumer."""
import torch
from torch import nn

from holocron_b200.models._blocks import FusedSequential
from holocron_b200.models.classification.mobileone import MobileOneBlock
from holocron_b200.models.classification.repvgg import RepBlock
from holocron_b200.models.classification.resnet import Bottleneck
from holocron_b200.models.classification.rexnet import ReXBlock
from holocron_b200.models.detection.yolov4 import _units


def repvgg_stage() -> nn.Module:
    """RepVGG-A0 stage 2 entry: a stride-2 two-branch block and a three-branch block (identity BatchNorm)."""
    return nn.Sequential(RepBlock(48, 96, 2, identity=False), RepBlock(96, 96, 1, identity=True))


def rexnet_se_block() -> nn.Module:
    return ReXBlock(in_channels=32, channels=40, t=6, stride=1, use_se=True)


def yolov4_neck_unit() -> nn.Module:
    """Two conv-BN-Mish units of a YOLOv4 PAN, DropBlock off."""
    return FusedSequential(*_units([(64, 32, 1), (32, 64, 3)], nn.Mish(inplace=True), nn.BatchNorm2d, None, None))


def resnet_bottleneck() -> nn.Module:
    return Bottleneck(64, 16, act_layer=nn.ReLU(inplace=True), norm_layer=nn.BatchNorm2d)


def mobileone_block() -> nn.Module:
    return MobileOneBlock(32, 64, overparam_factor=2)


# name -> (builder, input channels, spatial size)
CASES = {
    "repvgg_stage": (repvgg_stage, 48, 32),
    "rexnet_se": (rexnet_se_block, 32, 16),
    "yolov4_neck_unit": (yolov4_neck_unit, 64, 32),
    "resnet_bottleneck": (resnet_bottleneck, 64, 16),
    "mobileone": (mobileone_block, 32, 16),
}


def build(name: str, seed: int = 0, sync: bool = False) -> nn.Module:
    builder = CASES[name][0]
    torch.manual_seed(seed)
    model = builder()
    with torch.no_grad():     # non-trivial affine parameters and running statistics
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.3, 0.3)
                m.running_mean.uniform_(-0.5, 0.5)
                m.running_var.uniform_(0.5, 1.5)
    return nn.SyncBatchNorm.convert_sync_batchnorm(model) if sync else model


def inputs(name: str, n: int, seed: int = 1):
    """Seeded (x, output-gradient weights generator seed): x [n, C, S, S] fp32."""
    _, c, s = CASES[name]
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, c, s, s, generator=g)
