"""GPU tests of the kw-wide 3^3 kernel behind LT_CONV_TC_FOLD (conv_lines_kernel): whole W lines as the m64 rows (one line at
W = 64, floor(64 / W) stacked lines below, spare rows masked), (kw, Cout) as the N of each product, the kw sum formed in the
epilogue across lanes and warps, and the (n, h block, d) planes cut into one contiguous range per CTA.  Each case runs the
float64, run-to-run, in-place and against-conv_tc checks of test_gpu_fold_rs; 3^3 layers wider than 64 run on conv_tc_kernel."""
import copy

import pytest
import torch
import torch.nn.functional as F

import test_gpu_fold_rs as fold_rs
from conftest import rel_err
from lt_b200 import capi
from test_gpu_ops import _engine, _bn_for, act_from_nchw, act_to_nchw, DEV
from test_gpu_tc import TOL

pytestmark = pytest.mark.gpu

LINES_CASES = [
    # (cout, k, (D, H, W), batch)
    (32, 3, (6, 8, 64), 1),       # W = 64: one line per m64 block, two per CTA
    (32, 3, (5, 12, 32), 2),      # W = 32: two stacked lines per m64 block
    (32, 3, (4, 16, 16), 1),      # W = 16: four stacked lines, every warp's rows 0 and 15 at line ends
    (32, 3, (3, 14, 20), 2),      # W = 20: three lines and four masked rows per block
    (32, 3, (4, 10, 48), 1),      # W = 48: one line and sixteen masked rows per block
    (32, 3, (7, 9, 64), 1),       # D and H odd: a half-empty last h block
    (16, 3, (5, 11, 64), 2),      # Cout 16 (N = 48), H odd
    (16, 3, (3, 7, 24), 1),       # Cout 16 with two stacked lines
    (32, 3, (64, 64, 64), 2),     # the benchmark's grid, batch 2: several d pieces per (n, h block) column
]


@pytest.mark.parametrize("case", LINES_CASES)
def test_conv_lines(case):
    fold_rs.test_conv_fold_rs(case)


def test_conv_lines_wide_routes_to_conv_tc():
    """A 3^3 layer wider than 64 has no kw-wide tile: it runs on conv_tc_kernel, with the same results."""
    cout, k, spatial, N = 32, 3, (3, 5, 80), 1
    torch.manual_seed(77)
    conv = torch.nn.Conv3d(32, cout, k, 1, k // 2, bias=True).eval()
    bn = _bn_for(conv, 5)
    x = torch.randn(N, 32, *spatial)
    res = torch.randn(N, cout, *spatial)
    with torch.no_grad():
        ref_conv, ref_bn = copy.deepcopy(conv).to(DEV).double(), copy.deepcopy(bn).to(DEV).double()
        want = F.relu(ref_bn(ref_conv(x.to(DEV).double())) + res.to(DEV).double()).cpu()
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV), cin_pad=32)
    assert pk.w_fold is not None
    ya, launched = fold_rs._run(e, pk, act_from_nchw(x, capi.FMT_S32, pad_c=32), act_from_nchw(res, capi.FMT_S32, pad_c=32))
    assert launched == [capi.CONV_TC]
    err = rel_err(act_to_nchw(ya).cpu()[:, :cout].double().numpy(), want.numpy())
    print("3^3 W = 80 rel err vs torch %.2e" % err)
    assert err < TOL["tc"]
