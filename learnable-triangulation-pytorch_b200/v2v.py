"""V2V 3D encoder-decoder (volumetric hourglass).

Host-side mirror of `/root/reference/mvn/models/v2v.py:141-180` (V2VModel) with the
reference's module names, so `state_dict()` keys match:
front_layers.{0..3}, encoder_decoder.{encoder_res*,decoder_res*,decoder_upsample*,skip_res*,mid_res},
back_layers.{0..2}, output_layer.

Parameters live here; inference runs through the native planner in engine.py.
The torch forward below is the autograd / CPU plumbing path (backend="torch").  Every forward takes the `conv` and `norm` hooks of
layers.py: `conv` applies each Conv3d / ConvTranspose3d (v2v_backend="native": autograd_ops.v2v_conv), `norm` each BatchNorm3d
together with the ReLU right after it and, in a Res3DBlock, the residual add (norm_backend="native": autograd_ops.batch_norm).
None, the default, stands for the torch formulas in layers.py.  Pooling and the decoder's `upsample + skip` adds are always torch, but
for the max-pool backward under torch.use_deterministic_algorithms (autograd_ops.MaxPool3dFn).
A ReLU module right after a BatchNorm is applied by `norm`, not called as a module, so a forward hook registered on it does not fire.
"""
import torch
import torch.nn.functional as F
from torch import nn

from .layers import defaults, run


class Basic3DBlock(nn.Module):
    """conv(k) + BN + ReLU (reference v2v.py:7-17)."""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.block = nn.Sequential(nn.Conv3d(cin, cout, k, 1, (k - 1) // 2), nn.BatchNorm3d(cout), nn.ReLU(True))

    def forward(self, x, conv=None, norm=None):
        return run(self.block, x, conv, norm)


class Res3DBlock(nn.Module):
    """relu(BN(conv3(relu(BN(conv3 x)))) + skip(x)); skip = 1x1x1 conv + BN when cin != cout (ref :20-42)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.res_branch = nn.Sequential(
            nn.Conv3d(cin, cout, 3, 1, 1), nn.BatchNorm3d(cout), nn.ReLU(True),
            nn.Conv3d(cout, cout, 3, 1, 1), nn.BatchNorm3d(cout))
        self.skip_con = nn.Sequential() if cin == cout else nn.Sequential(
            nn.Conv3d(cin, cout, 1, 1, 0), nn.BatchNorm3d(cout))

    def forward(self, x, conv=None, norm=None):
        conv, norm = defaults(conv, norm)
        rb = self.res_branch
        y = norm(rb[1], conv(rb[0], x), relu=True)
        z = conv(rb[3], y)
        return norm(rb[4], z, relu=True, residual=run(self.skip_con, x, conv, norm))


class Pool3DBlock(nn.Module):
    def __init__(self, pool_size):
        super().__init__()
        self.pool_size = pool_size

    def forward(self, x):
        if torch.are_deterministic_algorithms_enabled() and x.is_cuda and torch.is_grad_enabled():
            from .autograd_ops import MaxPool3dFn       # torch's CUDA max_pool3d backward is not deterministic
            return MaxPool3dFn.apply(x, self.pool_size)
        return F.max_pool3d(x, self.pool_size, self.pool_size)


class Upsample3DBlock(nn.Module):
    """ConvTranspose3d(k=2, s=2) + BN + ReLU (reference :54-66)."""

    def __init__(self, cin, cout, kernel_size, stride):
        super().__init__()
        assert kernel_size == 2 and stride == 2
        self.block = nn.Sequential(nn.ConvTranspose3d(cin, cout, 2, 2, 0, 0), nn.BatchNorm3d(cout), nn.ReLU(True))

    def forward(self, x, conv=None, norm=None):
        return run(self.block, x, conv, norm)


# (level, encoder channels in->out); decoder mirrors it. reference v2v.py:73-101
_ENC = ((1, 32, 64), (2, 64, 128), (3, 128, 128), (4, 128, 128), (5, 128, 128))
_DEC = ((5, 128, 128), (4, 128, 128), (3, 128, 128), (2, 128, 64), (1, 64, 32))


class EncoderDecorder(nn.Module):  # (sic) the reference's class name
    def __init__(self):
        super().__init__()
        for lvl, cin, cout in _ENC:
            setattr(self, "encoder_pool%d" % lvl, Pool3DBlock(2))
            setattr(self, "encoder_res%d" % lvl, Res3DBlock(cin, cout))
        self.mid_res = Res3DBlock(128, 128)
        for lvl, cin, cout in _DEC:
            setattr(self, "decoder_res%d" % lvl, Res3DBlock(cin, cin))
            setattr(self, "decoder_upsample%d" % lvl, Upsample3DBlock(cin, cout, 2, 2))
        for lvl, cin, _ in _ENC:
            setattr(self, "skip_res%d" % lvl, Res3DBlock(cin, cin))

    def forward(self, x, conv=None, norm=None):
        skips = {}
        for lvl, _, _ in _ENC:
            skips[lvl] = getattr(self, "skip_res%d" % lvl)(x, conv, norm)
            x = getattr(self, "encoder_res%d" % lvl)(getattr(self, "encoder_pool%d" % lvl)(x), conv, norm)
        x = self.mid_res(x, conv, norm)
        for lvl, _, _ in _DEC:
            x = getattr(self, "decoder_upsample%d" % lvl)(getattr(self, "decoder_res%d" % lvl)(x, conv, norm), conv, norm) + skips[lvl]
        return x


class V2VModel(nn.Module):
    def __init__(self, input_channels, output_channels):
        super().__init__()
        self.front_layers = nn.Sequential(
            Basic3DBlock(input_channels, 16, 7), Res3DBlock(16, 32), Res3DBlock(32, 32), Res3DBlock(32, 32))
        self.encoder_decoder = EncoderDecorder()
        self.back_layers = nn.Sequential(Res3DBlock(32, 32), Basic3DBlock(32, 32, 1), Basic3DBlock(32, 32, 1))
        self.output_layer = nn.Conv3d(32, output_channels, 1, 1, 0)
        # Xavier-normal weights, zero bias on every (transposed) conv, reference :171-180
        for m in self.modules():
            if isinstance(m, (nn.Conv3d, nn.ConvTranspose3d)):
                nn.init.xavier_normal_(m.weight)
                nn.init.constant_(m.bias, 0)

    def forward(self, x, conv=None, norm=None):
        conv, norm = defaults(conv, norm)
        for blk in self.front_layers:
            x = blk(x, conv, norm)
        x = self.encoder_decoder(x, conv, norm)
        for blk in self.back_layers:
            x = blk(x, conv, norm)
        return conv(self.output_layer, x)
