"""GPU tests of the full-resolution V2V convolution kernel (conv_fold_kernel) at the edges of its tiling: one halo box feeds every
kw tap (A fragments loaded with ldmatrix from the swizzled box), the 3^3 filter stays resident while each consumer warpgroup
owns whole 8 x 8 x 2 tiles, and the 7^3 filter streams through its own ring over 8 x 16 x 2 tiles."""
import copy

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lt_b200 import capi
from test_gpu_ops import _engine, _bn_for, act_from_nchw, act_to_nchw, DEV
from test_gpu_tc import TOL

pytestmark = pytest.mark.gpu

RS_CASES = [
    # (cout, k, (D, H, W), batch)
    (32, 3, (5, 13, 20), 2),     # D odd with BD = 2, H not a multiple of 8, 16 < W < 64 and not a multiple of 8
    (16, 3, (3, 9, 17), 1),      # Cout 16 (N tile 16), a one-column last w tile
    (32, 3, (4, 8, 16), 1),      # the narrowest volume: both w edges of one tile read the zero fill
    (16, 7, (5, 19, 27), 1),     # 7^3: H not a multiple of 16, W not a multiple of 8
    (32, 7, (3, 11, 16), 2),     # 7^3 with a 32-wide N tile: the kw shift reads zero fill on both sides of every tile
    (32, 3, (32, 40, 48), 2),    # 960 tiles: at least 3 tiles per consumer warpgroup on any H100
    (16, 7, (24, 48, 64), 2),    # 576 tiles: at least 4 tiles per CTA
]


def _run(e, pk, xa, ra, out=None):
    launched = []
    orig = capi.conv_nd
    capi.conv_nd = lambda d, *a: (launched.append(a[-1]), orig(d, *a))[1]
    try:
        ya = e._conv(xa, pk, relu=True, residual=ra, res_mode=capi.RES_BEFORE_RELU, out=out)
    finally:
        capi.conv_nd = orig
    torch.cuda.synchronize()
    return ya, launched


@pytest.mark.parametrize("case", RS_CASES)
def test_conv_fold_rs(case):
    cout, k, spatial, N = case
    torch.manual_seed(1000 + cout + k + spatial[2])
    conv = torch.nn.Conv3d(32, cout, k, 1, k // 2, bias=True).eval()
    bn = _bn_for(conv, 5)
    x = torch.randn(N, 32, *spatial)
    res = torch.randn(N, cout, *spatial)
    with torch.no_grad():   # float64 reference on the device: no TF32
        ref_conv, ref_bn = copy.deepcopy(conv).to(DEV).double(), copy.deepcopy(bn).to(DEV).double()
        want = F.relu(ref_bn(ref_conv(x.to(DEV).double())) + res.to(DEV).double()).cpu()
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV), cin_pad=32)
    assert pk.w_fold is not None
    xa = act_from_nchw(x, capi.FMT_S32, pad_c=32)
    ra = act_from_nchw(res, capi.FMT_S32, pad_c=32)

    ya, launched = _run(e, pk, xa, ra)
    assert launched == [capi.CONV_TC_FOLD]
    got = act_to_nchw(ya).cpu()
    err = rel_err(got[:, :cout].double().numpy(), want.numpy())
    print("conv_fold rs %s rel err vs torch %.2e" % (case, err))
    assert err < TOL["tc"]
    if cout < 32:
        assert float(got[:, cout:].abs().max()) == 0.0

    yb, _ = _run(e, pk, xa, ra)
    assert torch.equal(ya.data, yb.data), "run-to-run results differ"

    rin = act_from_nchw(res, capi.FMT_S32, pad_c=32)
    yi, _ = _run(e, pk, xa, rin, out=rin)
    assert yi is rin and torch.equal(yi.data, ya.data), "in-place residual differs from out of place"

    pk.w_fold = None   # the generic implicit-GEMM kernel on the same packed layer
    yg, launched = _run(e, pk, xa, ra)
    assert launched == [capi.CONV_TC]
    gen = act_to_nchw(yg).cpu()[:, :cout]
    err_g = rel_err(got[:, :cout].numpy(), gen.numpy())
    print("conv_fold rs %s rel err vs conv_tc %.2e" % (case, err_g))
    assert err_g < TOL["tc"]
