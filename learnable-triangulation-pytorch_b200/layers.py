"""The `conv` and `norm` hooks of the backbone (pose_resnet.py) and the V2V net (v2v.py), with their torch defaults.

Every block's forward takes a `conv` hook, a function (module, x) -> y that applies a convolution module, and a `norm` hook, a
function (module, x, relu=False, residual=None) -> act(module(x) + residual) that applies a BatchNorm together with the ReLU right
after it and, at the end of a residual unit, the shortcut add.  None stands for the torch formulas below; the training backends
pass the native ones (autograd_ops.backbone_conv / v2v_conv and autograd_ops.batch_norm).
"""
import torch.nn.functional as F
from torch import nn

# The concrete classes, not _ConvNd / _BatchNorm: a SyncBatchNorm-converted model keeps calling its SyncBatchNorm and ReLU modules.
CONVS = (nn.Conv2d, nn.ConvTranspose2d, nn.Conv3d, nn.ConvTranspose3d)
NORMS = (nn.BatchNorm2d, nn.BatchNorm3d)


def torch_conv(m, x):
    return m(x)


def torch_norm(m, x, relu=False, residual=None):
    """relu(m(x) + residual), ReLU and residual optional.  The ReLU runs in place on the fresh BatchNorm output or sum, as the
    models' nn.ReLU(inplace=True) modules do."""
    y = m(x)
    if residual is not None:
        y = y + residual
    return F.relu(y, inplace=True) if relu else y


def defaults(conv, norm):
    """(conv, norm) with None replaced by the torch formulas."""
    return conv or torch_conv, norm or torch_norm


def run(seq, x, conv=None, norm=None):
    """nn.Sequential.forward with every convolution through `conv` and every BatchNorm, fused with an nn.ReLU directly after it,
    through `norm`; other modules are called as they are."""
    conv, norm = defaults(conv, norm)
    mods = list(seq)
    i = 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, NORMS):
            relu = i + 1 < len(mods) and isinstance(mods[i + 1], nn.ReLU)
            x = norm(m, x, relu=relu)
            i += 2 if relu else 1
        else:
            x = conv(m, x) if isinstance(m, CONVS) else m(x)
            i += 1
    return x
