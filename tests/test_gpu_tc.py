"""GPU parity tests of the wgmma/TMA convolution path (through the C ABI): GEMM core self-test, conv vs the
fp32 torch reference of the same op, transposed-conv phases, and tensor-core vs FFMA kernels at larger sizes."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lt_b200 import capi
from test_gpu_ops import _engine, _bn_for, act_from_nchw, act_to_nchw, DEV

pytestmark = pytest.mark.gpu

# fp32-grade: 3-term split-fp16 products;  fp16-grade: high parts only
TOL = {"tc": 2e-5, "tc1": 3e-3}


@pytest.mark.parametrize("mnk", [(128, 16, 64), (128, 32, 128), (256, 64, 64), (384, 128, 256), (200, 256, 512), (128, 48, 64)])
def test_tc_gemm_selftest(mnk):
    M, N, K = mnk
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(DEV).half().contiguous()
    b = torch.randn(N, K, generator=g).to(DEV).half().contiguous()
    d = torch.zeros(M * N + 2 * N, dtype=torch.float32, device=DEV)
    capi.tc_gemm_selftest(a, b, d, M, N, K)
    torch.cuda.synchronize()
    got = d[:M * N].view(M, N).cpu().double()
    want = a.cpu().double() @ b.cpu().double().t()
    assert rel_err(got.numpy(), want.numpy()) < 1e-5     # fp16 products are exact in fp32; only summation order differs


TC_CASES = [
    # (dims, cin, cout, k, pad, spatial, batch)
    (2, 64, 64, 1, 0, (16, 8), 1),
    (2, 64, 64, 1, 0, (12, 12), 3),
    (2, 256, 64, 1, 0, (24, 24), 2),
    (2, 64, 256, 1, 0, (12, 12), 2),
    (2, 64, 64, 3, 1, (12, 12), 2),
    (2, 128, 128, 3, 1, (9, 7), 3),
    (3, 32, 32, 3, 1, (8, 8, 8), 2),
    (3, 32, 16, 7, 3, (8, 8, 8), 1),
    (3, 16, 32, 3, 1, (8, 8, 8), 1),
    (3, 32, 17, 1, 0, (8, 8, 8), 2),
    (3, 128, 128, 3, 1, (2, 2, 2), 2),
    (3, 64, 128, 3, 1, (4, 4, 4), 1),
]


@pytest.mark.parametrize("case", TC_CASES)
@pytest.mark.parametrize("mode", ["tc", "tc1"])
def test_conv_tc_vs_torch(case, mode):
    dims, cin, cout, k, pad, spatial, N = case
    torch.manual_seed(cin * 13 + cout + k)
    conv = (torch.nn.Conv2d if dims == 2 else torch.nn.Conv3d)(cin, cout, k, 1, pad, bias=(dims == 3)).eval()
    bn = _bn_for(conv, 7)
    x = torch.randn(N, cin, *spatial)
    with torch.no_grad():
        y0 = bn(conv(x))
        res = torch.randn_like(y0)
        want = F.relu(y0 + res)
    e = _engine(mode)
    cin_p = (cin + 31) // 32 * 32
    cout_p = (cout + 31) // 32 * 32
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV), cin_pad=cin_p)
    assert pk.impl in (capi.CONV_TC, capi.CONV_TC1)
    xa = act_from_nchw(x, capi.FMT_S32, pad_c=cin_p)
    ra = act_from_nchw(res, capi.FMT_S32, pad_c=cout_p)
    ya = e._conv(xa, pk, relu=True, residual=ra, res_mode=capi.RES_BEFORE_RELU)
    torch.cuda.synchronize()
    full = act_to_nchw(ya).cpu()
    got = full[:, :cout]
    if dims == 2:
        got = got.squeeze(2)
    err = rel_err(got.numpy(), want.numpy())
    print("conv_tc[%s] %s rel err %.2e" % (mode, case, err))
    assert err < TOL[mode]
    if cout_p > cout:
        assert float(full[:, cout:].abs().max()) == 0.0, "padding channels must be written as zeros"


@pytest.mark.parametrize("case", [(128, 128, 3, (2, 2, 2), 8), (128, 128, 3, (4, 4, 4), 8), (128, 128, 3, (8, 8, 8), 8), (64, 128, 3, (5, 3, 4), 2),
                                  (256, 96, 1, (4, 4, 4), 2)])
@pytest.mark.parametrize("res_mode", ["none", "before", "after"])
def test_conv_tc_splitk_matches_single_pass(case, res_mode):
    """Deep V2V levels (v2v.py:75-101: 2^3..8^3 volumes) have fewer M tiles than SMs: the K loop is split over blockIdx.z
    and summed by splitk_reduce_kernel.  Same result as the single-pass kernel up to fp32 summation order."""
    cin, cout, k, spatial, N = case
    torch.manual_seed(cin + cout + spatial[0])
    conv = torch.nn.Conv3d(cin, cout, k, 1, k // 2, bias=True).eval()
    bn = _bn_for(conv, 3)
    x = torch.randn(N, cin, *spatial)
    mode = {"none": capi.RES_NONE, "before": capi.RES_BEFORE_RELU, "after": capi.RES_AFTER_RELU}[res_mode]
    with torch.no_grad():
        y0 = bn(conv(x))
        res = torch.randn_like(y0)
        want = {"none": F.relu(y0), "before": F.relu(y0 + res), "after": F.relu(y0) + res}[res_mode]
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    xa = act_from_nchw(x, capi.FMT_S32)
    ra = act_from_nchw(res, capi.FMT_S32) if res_mode != "none" else None
    y_split = act_to_nchw(e._conv(xa, pk, relu=True, residual=ra, res_mode=mode), cout).cpu()
    e._splitk_ws = torch.empty(0, dtype=torch.uint8, device=DEV)      # no workspace -> single pass
    y_single = act_to_nchw(e._conv(xa, pk, relu=True, residual=ra, res_mode=mode), cout).cpu()
    torch.cuda.synchronize()
    err = rel_err(y_split.numpy(), want.numpy())
    diff = rel_err(y_split.numpy(), y_single.numpy())
    print("splitk %s res=%s rel err %.2e, vs single pass %.2e" % (case, res_mode, err, diff))
    assert err < TOL["tc"] and diff < 5e-6


@pytest.mark.parametrize("case", [(64, 256, 1, (48, 48), 8), (128, 512, 1, (24, 24), 20), (256, 1024, 1, (24, 24), 9),
                                  (256, 512, 2, (48, 48), 6), (192, 384, 1, (40, 24), 5)])
@pytest.mark.parametrize("res_mode", ["none", "before"])
def test_conv_tc_b_resident_vs_torch(case, res_mode):
    """1x1 layers with <= 8 K chunks and >= 256 outputs take the B-resident persistent variant (weights of the CTA's 64-wide
    N sub-tile stay in shared memory; CTA = (N tile, M stream)): uneven tile counts per stream, residual prefetch, stride 2."""
    cin, cout, stride, spatial, N = case
    torch.manual_seed(cin + cout + N)
    conv = torch.nn.Conv2d(cin, cout, 1, stride, 0, bias=False).eval()
    bn = _bn_for(conv, 5)
    x = torch.randn(N, cin, *spatial)
    with torch.no_grad():
        y0 = bn(conv(x))
        res = torch.randn_like(y0)
        want = F.relu(y0 + res) if res_mode == "before" else F.relu(y0)
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    ra = act_from_nchw(res, capi.FMT_S32) if res_mode == "before" else None
    ya = e._conv(act_from_nchw(x, capi.FMT_S32), pk, relu=True, residual=ra,
                 res_mode=capi.RES_BEFORE_RELU if res_mode == "before" else capi.RES_NONE)
    torch.cuda.synchronize()
    err = rel_err(act_to_nchw(ya, cout).squeeze(2).cpu().numpy(), want.numpy())
    print("conv_tc b-resident %s %s rel err %.2e" % (case, res_mode, err))
    assert err < TOL["tc"]


@pytest.mark.parametrize("case", [(64, 64, 3, 2, 1, (12, 12), 2), (64, 128, 1, 2, 0, (12, 12), 2), (128, 128, 3, 2, 1, (48, 48), 4),
                                  (256, 512, 1, 2, 0, (48, 48), 4)])
def test_conv_tc_stride2_vs_torch(case):
    """Stride-2 convs of the trunk (pose_resnet.py:62-69,236-243) through TMA traversal strides."""
    cin, cout, k, stride, pad, spatial, N = case
    torch.manual_seed(cin + cout + k)
    conv = torch.nn.Conv2d(cin, cout, k, stride, pad, bias=False).eval()
    bn = _bn_for(conv, 11)
    x = torch.randn(N, cin, *spatial)
    with torch.no_grad():
        want = F.relu(bn(conv(x)))
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    assert pk.impl == capi.CONV_TC
    ya = e._conv(act_from_nchw(x, capi.FMT_S32), pk, relu=True)
    torch.cuda.synchronize()
    err = rel_err(act_to_nchw(ya, cout).squeeze(2).cpu().numpy(), want.numpy())
    print("conv_tc stride2 %s rel err %.2e" % (case, err))
    assert err < TOL["tc"]


def test_stem_space_to_depth_vs_torch():
    """7x7 stride-2 stem (pose_resnet.py:205-208) as a 4x4 conv over the space-to-depth image, on the tensor cores."""
    torch.manual_seed(5)
    conv = torch.nn.Conv2d(3, 64, 7, 2, 3, bias=False).eval()
    bn = _bn_for(conv, 4)
    x = torch.randn(3, 3, 64, 96)
    with torch.no_grad():
        want = F.relu(bn(conv(x)))
    e = _engine("tc")
    pk = e._pack_stem_s2d(conv.to(DEV), bn.to(DEV))
    from lt_b200.engine import Act
    xa = Act(3, 1, 32, 48, 32, capi.FMT_S32, DEV)
    capi.stem_s2d(x.to(DEV).contiguous(), xa.data, 3, 3, 64, 96)
    ya = e._conv(xa, pk, relu=True, out_dims=(1, 32, 48))
    torch.cuda.synchronize()
    err = rel_err(act_to_nchw(ya, 64).squeeze(2).cpu().numpy(), want.numpy())
    print("stem s2d rel err %.2e" % err)
    assert err < TOL["tc"]


FOLD_CASES = [
    # (cin, cout, k, (D, H, W), batch)   -- Cin = 32 cubic stride-1 layers of the V2V net (v2v.py:146, :24-28)
    (32, 32, 3, (8, 8, 16), 1),
    (32, 32, 3, (9, 11, 18), 2),      # partial tiles in x (18 = 14 + 4) and y (11 = 8 + 3)
    (16, 32, 3, (6, 16, 32), 1),      # 16 input channels stored 32 wide
    (32, 16, 7, (8, 8, 16), 1),       # 7^3, weights streamed
    (32, 16, 7, (7, 13, 25), 2),
    (32, 32, 3, (32, 32, 32), 2),     # many tiles per persistent CTA
    (32, 16, 7, (5, 10, 64), 1),      # 7^3 on a 64-wide volume: full-width tiles (2 lines of 64), 3-row edge exchange
    (32, 16, 7, (4, 7, 71), 2),       # 32-row window with a partial last window (71 = 2*26 + 19)
    (32, 32, 3, (3, 5, 64), 2),       # full-width tiles, 64-wide lines: the kw shift crosses warps (edge-row exchange), partial y block
    (16, 32, 3, (4, 64, 64), 1),      # full-width 64^2 planes, 16 input channels stored 32 wide
    (32, 16, 7, (9, 9, 32), 1),       # full-width, one line per warp
    (32, 32, 3, (3, 5, 64), 1),       # odd tile count (9): the last pair's second CTA runs an out-of-range tile
]


@pytest.mark.parametrize("case", FOLD_CASES)
@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("variant", ["pair", "one_cta", "staged", "windowed", "default"])
def test_conv_fold_vs_torch(case, with_res, variant):
    # the variants set the kw-fold options of lt_options, which the sm_90a kernel accepts and ignores: every variant must agree
    if variant != "default":
        capi.set_options(fold_pair=2 * int(variant in ("pair", "staged")), fold_fullw=int(variant != "windowed"), fold_direct=int(variant != "staged"))
    try:
        _fold_case(case, with_res)
    finally:
        capi.set_options(fold_pair=1, fold_fullw=1, fold_direct=0)


def _fold_case(case, with_res):
    cin, cout, k, spatial, N = case
    torch.manual_seed(cin + cout + k + spatial[2])
    conv = torch.nn.Conv3d(cin, cout, k, 1, k // 2, bias=True).eval()
    bn = _bn_for(conv, 13)
    x = torch.randn(N, cin, *spatial)
    with torch.no_grad():
        y0 = bn(conv(x))
        res = torch.randn_like(y0)
        want = F.relu(y0 + res) if with_res else F.relu(y0)
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV), cin_pad=32)
    assert pk.w_fold is not None
    xa = act_from_nchw(x, capi.FMT_S32, pad_c=32)
    ra = act_from_nchw(res, capi.FMT_S32, pad_c=32) if with_res else None
    launched = []
    orig = capi.conv_nd
    capi.conv_nd = lambda d, *a: (launched.append(a[-1]), orig(d, *a))[1]
    try:
        ya = e._conv(xa, pk, relu=True, residual=ra, res_mode=capi.RES_BEFORE_RELU if with_res else capi.RES_NONE)
    finally:
        capi.conv_nd = orig
    torch.cuda.synchronize()
    assert launched == [capi.CONV_TC_FOLD], "the kw-folded kernel must have been selected"
    full = act_to_nchw(ya).cpu()
    err = rel_err(full[:, :cout].numpy(), want.numpy())
    print("conv_fold %s res=%s rel err %.2e" % (case, with_res, err))
    assert err < TOL["tc"]
    if cout < 32:
        assert float(full[:, cout:].abs().max()) == 0.0


WIDE_CASES = [
    # (dims, cin, cout, k, stride, pad, spatial, batch, res_mode)  -- layers with Cout % 128 == 0 (Nt = 128)
    (2, 256, 1024, 1, 1, 0, (24, 24), 9, "before"),     # 1x1 expand of a bottleneck: 8 N tiles, odd M-tile count (41)
    (2, 1024, 256, 1, 1, 0, (24, 24), 8, "none"),       # 1x1 reduce: 32 K chunks
    (2, 256, 256, 3, 1, 1, (24, 24), 32, "none"),       # 3x3: padding through TMA zero fill
    (2, 128, 128, 3, 1, 1, (48, 48), 3, "none"),        # Nt = 128
    (2, 128, 512, 1, 1, 0, (48, 48), 3, "before"),
    (2, 64, 256, 1, 1, 0, (96, 96), 2, "before"),       # 2 K chunks per tile: epilogue-bound
    (2, 256, 512, 1, 2, 0, (48, 48), 4, "none"),        # stride-2 downsample through TMA traversal strides
    (2, 128, 128, 3, 2, 1, (48, 48), 16, "none"),
    (2, 512, 2048, 1, 1, 0, (12, 12), 6, "before"),
    (3, 128, 128, 3, 1, 1, (16, 16, 16), 8, "before"),  # V2V 16^3 level
    (3, 64, 128, 3, 1, 1, (16, 16, 16), 4, "after"),
    (2, 96, 384, 1, 1, 0, (40, 24), 5, "before"),       # CoutP = 384 = 3 x 128
]


@pytest.mark.parametrize("acc", ["single", "two"])
@pytest.mark.parametrize("case", WIDE_CASES)
def test_conv_tc_wide_vs_torch(case, acc):
    """LT_CONV_TC on the wide layers (Cout % 128 == 0) against the fp32 torch op, under both settings of lt_options.pair_two_acc (which
    has no effect)."""
    capi.set_options(pair_two_acc=int(acc == "two"))
    try:
        _wide_case(case)
    finally:
        capi.set_options(pair_two_acc=1)


def _wide_case(case):
    dims, cin, cout, k, stride, pad, spatial, N, res_mode = case
    torch.manual_seed(cin + cout + k + N)
    conv = (torch.nn.Conv2d if dims == 2 else torch.nn.Conv3d)(cin, cout, k, stride, pad, bias=(dims == 3)).eval()
    bn = _bn_for(conv, 17)
    x = torch.randn(N, cin, *spatial)
    mode = {"none": capi.RES_NONE, "before": capi.RES_BEFORE_RELU, "after": capi.RES_AFTER_RELU}[res_mode]
    with torch.no_grad():
        y0 = bn(conv(x))
        res = torch.randn_like(y0)
        want = {"none": F.relu(y0), "before": F.relu(y0 + res), "after": F.relu(y0) + res}[res_mode]
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    assert pk.impl == capi.CONV_TC
    ra = act_from_nchw(res, capi.FMT_S32) if res_mode != "none" else None
    launched = []
    orig = capi.conv_nd
    capi.conv_nd = lambda d, *a: (launched.append(a[-1]), orig(d, *a))[1]
    try:
        ya = e._conv(act_from_nchw(x, capi.FMT_S32), pk, relu=True, residual=ra, res_mode=mode)
    finally:
        capi.conv_nd = orig
    torch.cuda.synchronize()
    assert launched == [capi.CONV_TC], "the generic tensor-core kernel must have been selected"
    got = act_to_nchw(ya, cout).cpu()
    if dims == 2:
        got = got.squeeze(2)
    err = rel_err(got.numpy(), want.numpy())
    print("conv_tc wide %s rel err %.2e" % (case, err))
    assert err < TOL["tc"]


def test_conv_tc_wide_deconv_phases_vs_torch():
    """k4 s2 p1 transposed conv 256 -> 256 (pose_resnet.py:266-291) as four stride-phase 2x2 convs on the tensor-core kernel."""
    torch.manual_seed(14)
    e = _engine("tc")
    dc = torch.nn.ConvTranspose2d(256, 256, 4, 2, 1, 0, bias=False).eval()
    bn = _bn_for(dc, 2)
    x = torch.randn(6, 256, 24, 24)
    with torch.no_grad():
        want = F.relu(bn(dc(x)))
    launched = []
    orig = capi.conv_nd
    capi.conv_nd = lambda d, *a: (launched.append(a[-1]), orig(d, *a))[1]
    try:
        got = act_to_nchw(e._deconv2d(act_from_nchw(x, capi.FMT_S32), e._pack_deconv2d_k4s2(dc.to(DEV), bn.to(DEV)))).squeeze(2).cpu()
    finally:
        capi.conv_nd = orig
    assert launched == [capi.CONV_TC] * 4
    assert rel_err(got.numpy(), want.numpy()) < TOL["tc"]


@pytest.mark.parametrize("cin,cout,spatial,N", [(64, 32, (32, 32, 32), 2), (128, 64, (16, 16, 16), 4), (128, 128, (8, 8, 8), 2), (128, 128, (2, 2, 2), 8)])
def test_deconv3d_merged_single_gemm_vs_torch(cin, cout, spatial, N):
    """ConvTranspose3d(k=2, s=2) + BN + ReLU + skip (v2v.py:54-66, :118-137) as ONE GEMM with N = 8 x Cout and grouped output
    (lt_conv_desc.ogd/ogh/ogw) on the tensor-core kernel, from a 32^3 input level down to 2^3."""
    torch.manual_seed(cin + cout + spatial[0])
    e = _engine("tc")
    dc = torch.nn.ConvTranspose3d(cin, cout, 2, 2).eval()
    bn = _bn_for(dc, 3)
    x = torch.randn(N, cin, *spatial)
    skip = torch.randn(N, cout, *[2 * v for v in spatial])
    with torch.no_grad():
        want = F.relu(bn(dc(x))) + skip
    pk = e._pack_deconv3d_k2s2(dc.to(DEV), bn.to(DEV))
    assert not isinstance(pk, dict) and pk.groups == 8
    launched = []
    orig = capi.conv_nd
    capi.conv_nd = lambda d, *a: (launched.append(a[-1]), orig(d, *a))[1]
    try:
        got = act_to_nchw(e._deconv3d(act_from_nchw(x, capi.FMT_S32), pk, act_from_nchw(skip, capi.FMT_S32))).cpu()
    finally:
        capi.conv_nd = orig
    torch.cuda.synchronize()
    assert len(launched) == 1
    err = rel_err(got.numpy(), want.numpy())
    print("deconv3d merged %d->%d %s N=%d impl=%d rel err %.2e" % (cin, cout, spatial, N, launched[0], err))
    assert err < TOL["tc"]


def test_conv_tc_fp32_output_and_no_residual():
    torch.manual_seed(3)
    conv = torch.nn.Conv2d(256, 32, 1).eval()
    x = torch.randn(2, 256, 24, 24)
    with torch.no_grad():
        want = conv(x)
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), None, out_fmt=capi.FMT_F32)
    ya = e._conv(act_from_nchw(x, capi.FMT_S32), pk, relu=False, out_fmt=capi.FMT_F32)
    assert ya.fmt == capi.FMT_F32
    assert rel_err(act_to_nchw(ya, 32).squeeze(2).cpu().numpy(), want.numpy()) < TOL["tc"]


def test_deconv_phases_tc_vs_torch():
    torch.manual_seed(4)
    e = _engine("tc")
    dc = torch.nn.ConvTranspose2d(64, 64, 4, 2, 1, 0, bias=False).eval()
    bn = _bn_for(dc, 2)
    x = torch.randn(2, 64, 6, 12)
    with torch.no_grad():
        want = F.relu(bn(dc(x)))
    got = act_to_nchw(e._deconv2d(act_from_nchw(x, capi.FMT_S32), e._pack_deconv2d_k4s2(dc.to(DEV), bn.to(DEV)))).squeeze(2).cpu()
    assert rel_err(got.numpy(), want.numpy()) < TOL["tc"]
    dc3 = torch.nn.ConvTranspose3d(64, 32, 2, 2).eval()
    bn3 = _bn_for(dc3, 3)
    x3 = torch.randn(2, 64, 4, 4, 4)
    skip = torch.randn(2, 32, 8, 8, 8)
    with torch.no_grad():
        want3 = F.relu(bn3(dc3(x3))) + skip
    got3 = act_to_nchw(e._deconv3d(act_from_nchw(x3, capi.FMT_S32), e._pack_deconv3d_k2s2(dc3.to(DEV), bn3.to(DEV)),
                                   act_from_nchw(skip, capi.FMT_S32))).cpu()
    assert rel_err(got3.numpy(), want3.numpy()) < TOL["tc"]


@pytest.mark.parametrize("case", [(2, 256, 1024, 1, 0, (24, 24), 32), (2, 256, 256, 3, 1, (24, 24), 32), (3, 32, 32, 3, 1, (64, 64, 64), 1)])
def test_conv_tc_vs_ffma_at_config2_sizes(case):
    """Sizes of BASELINE config #2 the CPU oracle cannot reach quickly: tensor-core kernel vs the exact-fp32 FFMA kernel."""
    dims, cin, cout, k, pad, spatial, N = case
    torch.manual_seed(9)
    conv = (torch.nn.Conv2d if dims == 2 else torch.nn.Conv3d)(cin, cout, k, 1, pad, bias=False).eval().to(DEV)
    bn = _bn_for(conv, 1).to(DEV)
    x = torch.randn(N, cin, *spatial, device=DEV)
    e_tc, e_ff = _engine("tc"), _engine("simt")
    y_tc = act_to_nchw(e_tc._conv(act_from_nchw(x, capi.FMT_S32), e_tc._pack_conv(conv, bn), relu=True))
    y_ff = act_to_nchw(e_ff._conv(act_from_nchw(x, capi.FMT_F32), e_ff._pack_conv(conv, bn), relu=True))
    torch.cuda.synchronize()
    err = rel_err(y_tc.cpu().numpy(), y_ff.cpu().numpy())
    print("conv_tc vs ffma %s rel err %.2e" % (case, err))
    assert err < TOL["tc"]


@pytest.mark.parametrize("J,FC", [(17, 20), (15, 16)])
@pytest.mark.parametrize("spatial,N", [((16, 16, 16), 2), ((5, 6, 7), 3), ((64, 64, 16), 1)])
def test_v2v_tail_fused_vs_torch(spatial, N, J, FC):
    """back_layers[1], back_layers[2], output_layer (v2v.py:154-160,168-169) as one kernel (csrc/conv_tail.cu) vs the three torch ops;
    row counts that are not a multiple of the 128-voxel tile included.  J = 15 packs the output filter as 16 rows, which the kernel's
    32-row weight load extends with zeros."""
    torch.manual_seed(21)
    c1, c2, c3 = torch.nn.Conv3d(32, 32, 1).eval(), torch.nn.Conv3d(32, 32, 1).eval(), torch.nn.Conv3d(32, J, 1).eval()
    bn1, bn2 = _bn_for(c1, 5), _bn_for(c2, 6)
    x = torch.randn(N, 32, *spatial)
    with torch.no_grad():
        want = c3(F.relu(bn2(c2(F.relu(bn1(c1(x)))))))
    e = _engine("tc")
    b1 = e._pack_conv(c1.to(DEV), bn1.to(DEV))
    b2 = e._pack_conv(c2.to(DEV), bn2.to(DEV))
    b3 = e._pack_conv(c3.to(DEV), None, out_fmt=capi.FMT_F32)
    xa = act_from_nchw(x, capi.FMT_S32)
    rows = xa.pixels
    logits = torch.full((rows, FC), 7.0, dtype=torch.float32, device=DEV)
    capi.v2v_tail(xa.data, b1.w, b2.w, b3.w, b1.scale, b1.shift, b2.scale, b2.shift, b3.scale, b3.shift, logits, rows, FC)
    torch.cuda.synchronize()
    got = logits.view(N, *spatial, FC).permute(0, 4, 1, 2, 3).cpu()
    err = rel_err(got[:, :J].numpy(), want.numpy())
    print("v2v tail %s N=%d J=%d rel err %.2e" % (spatial, N, J, err))
    assert err < TOL["tc"] * 2          # three chained layers
    assert float(got[:, J:].abs().max()) == 0.0


@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("spatial,N", [((32, 32, 16), 3), ((64, 64, 16), 2), ((64, 64, 64), 1)])
def test_v2v_tail_with_softargmax_statistics(spatial, N, softmax):
    """lt_v2v_tail_stats_fwd + lt_softargmax3d_finish_fwd (statistics pass of op.py:84-96 fused into the kernel that produces the logits)
    vs the unfused pair lt_v2v_tail_fwd + lt_softargmax3d_fwd on the same inputs: identical logits, key points / volumes to fp32
    summation-order accuracy, equal arg-max.  Shapes: one tile per CTA with CTAs that own no tile of some samples (identity partials),
    several tiles per CTA across a sample boundary (flush), and a full 64^3 volume."""
    torch.manual_seed(5)
    c1, c2, c3 = torch.nn.Conv3d(32, 32, 1).eval(), torch.nn.Conv3d(32, 32, 1).eval(), torch.nn.Conv3d(32, 17, 1).eval()
    with torch.no_grad():
        c3.weight.mul_(6.0)      # logit spread of a few units: peaked softmax
    bn1, bn2 = _bn_for(c1, 5), _bn_for(c2, 6)
    x = torch.randn(N, 32, *spatial)
    e = _engine("tc")
    b1 = e._pack_conv(c1.to(DEV), bn1.to(DEV))
    b2 = e._pack_conv(c2.to(DEV), bn2.to(DEV))
    b3 = e._pack_conv(c3.to(DEV), None, out_fmt=capi.FMT_F32)
    xa = act_from_nchw(x, capi.FMT_S32)
    nvox, J, FC, mult = spatial[0] * spatial[1] * spatial[2], 17, 20, 1.7
    coord = (torch.randn(N, nvox, 3) * 600).to(DEV)
    args = (xa.data, b1.w, b2.w, b3.w, b1.scale, b1.shift, b2.scale, b2.shift, b3.scale, b3.shift)
    ws_bytes = capi.softargmax3d_workspace_bytes(N, J, nvox)
    # unfused
    lg0 = torch.empty((N * nvox, FC), dtype=torch.float32, device=DEV)
    capi.v2v_tail(*args, lg0, N * nvox, FC)
    v0 = torch.empty((N, J, nvox), dtype=torch.float32, device=DEV)
    kp0 = torch.empty((N, J, 3), dtype=torch.float32, device=DEV)
    ws0 = torch.empty(ws_bytes // 4 + 1, dtype=torch.float32, device=DEV)
    capi.softargmax3d(lg0, nvox * FC, FC, 1, coord, v0, kp0, ws0, N, J, nvox, mult, softmax)
    # fused (twice: the partials of every (sample, CTA) must be rewritten by each call)
    for _ in range(2):
        lg1 = torch.full((N * nvox, FC), 3.0, dtype=torch.float32, device=DEV)
        ws1 = torch.full((ws_bytes // 4 + 1,), float("nan"), dtype=torch.float32, device=DEV)
        G = capi.v2v_tail_stats(*args, lg1, N, nvox, FC, coord, J, mult, int(softmax), ws1)
        v1 = torch.full((N, J, nvox), -1.0, dtype=torch.float32, device=DEV)
        kp1 = torch.empty((N, J, 3), dtype=torch.float32, device=DEV)
        capi.softargmax3d_finish(lg1, nvox * FC, FC, coord, v1, kp1, ws1, N, J, nvox, G, mult, int(softmax))
        torch.cuda.synchronize()
        assert G >= 1 and torch.equal(lg0, lg1), "the statistics variant must not change the logits"
        err_kp = rel_err(kp1.cpu().numpy(), kp0.cpu().numpy())
        err_v = rel_err(v1.cpu().numpy(), v0.cpu().numpy())
        print("tail + statistics %s N=%d softmax=%s G=%d: keypoints %.2e volumes %.2e" % (spatial, N, softmax, G, err_kp, err_v))
        assert err_kp < 3e-5 and err_v < 3e-5
        assert torch.equal(v1.argmax(-1), v0.argmax(-1))
