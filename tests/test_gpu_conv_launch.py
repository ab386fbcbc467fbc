"""The training convolutions launch packed filters exactly as the inference engine does (engine.launch_conv): on the same split-fp16
input, ConvNdFn's forward equals NativeEngine._conv bit for bit -- same kernel, filter, scale and split-K scratch."""
import pytest
import torch

from lt_b200 import autograd_ops as A
from lt_b200 import capi, engine as eng_mod
from test_gpu_ops import _engine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.mark.parametrize("cin,cout,k,stride,dims", [
    (32, 32, (3, 3, 3), (1, 1, 1), (6, 9, 16)),       # full-resolution V2V width: LT_CONV_TC_FOLD with the lines kernel's scale
    (32, 16, (7, 7, 7), (1, 1, 1), (5, 6, 16)),       # V2V front layer: 16-wide float32 output, conv_tc_kernel
    (64, 128, (3, 3), (2, 2), (17, 15)),              # backbone 3x3 stride 2
    (256, 512, (1, 1), (2, 2), (12, 10)),             # backbone downsample 1x1 stride 2
], ids=["3^3 32->32 W16", "7^3 32->16", "3x3 s2", "1x1 s2"])
def test_training_forward_equals_engine_conv(cin, cout, k, stride, dims):
    torch.manual_seed(cin + cout + len(k))
    nd = len(k)
    conv = (torch.nn.Conv3d if nd == 3 else torch.nn.Conv2d)(cin, cout, k, stride, tuple(kk // 2 for kk in k)).to(DEV)
    x = torch.randn(2, cin, *dims, device=DEV)
    with torch.no_grad():
        y_train = A.ConvNdFn.apply(x, conv.weight, conv.bias, conv.stride, conv.padding)
        e = _engine("tc")
        pk = e._pack_conv(conv, None, out_fmt=capi.FMT_F32)
        x_s = A._to_s32(A._cl(x), eng_mod._round_up(cin, 32))
        y_eng = e._conv(eng_mod.Act.view(x_s), pk, relu=False, out_fmt=capi.FMT_F32, out_c=eng_mod._round_up(cout, 4))
    assert y_eng.C == eng_mod._round_up(cout, 4)
    assert torch.equal(y_train, A._from_cl(y_eng.data, cout, nd))
