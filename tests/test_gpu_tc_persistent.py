"""Persistent conv_tc_kernel: CTAs that run several work units in a row (one operand ring across tile boundaries), the N-tile-
fastest unit order, and the modelled K split, against torch and the FFMA path."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lt_b200 import capi
from test_gpu_ops import _engine, _bn_for, act_from_nchw, act_to_nchw, DEV

pytestmark = pytest.mark.gpu

TOL = {"tc": 2e-5, "tc1": 3e-3}
RES = {"none": capi.RES_NONE, "before": capi.RES_BEFORE_RELU, "after": capi.RES_AFTER_RELU}

# (cin, cout, k, stride, spatial, batch): M tiles of 128 positions odd / even and well above 132 (several units per CTA);
# Cout 16 / 32 / 64 / 128 / 256 / 1024 gives N tiles of 16 / 32 / 64 / 128 and 1, 2, 8 of them
CASES = [
    (64, 16, 1, 1, (24, 24), 33),      # 594 M tiles x 1 N tile of 16
    (64, 32, 3, 1, (16, 24), 35),      # 105 M tiles (odd, < SMs), Nt 32
    (128, 64, 1, 1, (32, 32), 34),     # 272 M tiles, Nt 64
    (256, 256, 3, 1, (24, 24), 8),     # 36 M tiles x 2 N tiles, 72 chunks
    (256, 1024, 1, 1, (24, 24), 9),    # 41 M tiles (odd) x 8 N tiles of 128
    (512, 512, 3, 1, (12, 12), 32),    # layer-4 shape: 144 x 4 tiles, split by the launch model
    (128, 256, 1, 2, (48, 48), 7),     # stride 2, 126 M tiles x 2 N tiles
    (128, 128, 3, 2, (48, 48), 8),     # stride 2, 3x3
]


def _c32(c):
    return (c + 31) // 32 * 32


def _run(e, pk, x, res, mode, out_fmt=None):
    return e._conv(x, pk, relu=True, residual=res, res_mode=mode, out_fmt=out_fmt)


def _case(case, res_mode, seed):
    cin, cout, k, stride, spatial, N = case
    torch.manual_seed(seed)
    conv = torch.nn.Conv2d(cin, cout, k, stride, k // 2, bias=False).eval()
    bn = _bn_for(conv, 3)
    x = torch.randn(N, cin, *spatial)
    with torch.no_grad():
        y0 = bn(conv(x))
        res = torch.randn_like(y0)
        want = {"none": F.relu(y0), "before": F.relu(y0 + res), "after": F.relu(y0) + res}[res_mode]
    return conv, bn, x, res, want


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("res_mode", ["none", "before", "after"])
def test_persistent_vs_torch_and_ffma(case, res_mode):
    conv, bn, x, res, want = _case(case, res_mode, sum(case[:4]))
    cout = case[1]
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    ra = act_from_nchw(res, capi.FMT_S32, pad_c=_c32(cout)) if res_mode != "none" else None
    y1 = act_to_nchw(_run(e, pk, act_from_nchw(x, capi.FMT_S32), ra, RES[res_mode]), cout).squeeze(2).cpu()
    y2 = act_to_nchw(_run(e, pk, act_from_nchw(x, capi.FMT_S32), ra, RES[res_mode]), cout).squeeze(2).cpu()
    es = _engine("simt")
    pks = es._pack_conv(conv.to(DEV), bn.to(DEV))
    rs = act_from_nchw(res, capi.FMT_F32, pad_c=pks.cout_p) if res_mode != "none" else None
    ys = act_to_nchw(_run(es, pks, act_from_nchw(x, capi.FMT_F32), rs, RES[res_mode]), cout).squeeze(2).cpu()
    torch.cuda.synchronize()
    err, err_s = rel_err(y1.numpy(), want.numpy()), rel_err(y1.numpy(), ys.numpy())
    print("persistent %s res=%s rel err %.2e vs torch, %.2e vs ffma" % (case, res_mode, err, err_s))
    assert torch.equal(y1, y2), "two runs must be bit-identical"
    assert err < TOL["tc"] and err_s < TOL["tc"]


@pytest.mark.parametrize("case", CASES)
def test_persistent_tc1_and_fp32_output(case):
    conv, bn, x, res, want = _case(case, "before", 7 + case[1])
    cout = case[1]
    e = _engine("tc1")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    y = act_to_nchw(_run(e, pk, act_from_nchw(x, capi.FMT_S32), act_from_nchw(res, capi.FMT_S32, pad_c=_c32(cout)),
                    capi.RES_BEFORE_RELU), cout).squeeze(2).cpu()
    e3 = _engine("tc")
    pk3 = e3._pack_conv(conv.to(DEV), bn.to(DEV))
    yf = _run(e3, pk3, act_from_nchw(x, capi.FMT_S32), act_from_nchw(res, capi.FMT_F32, pad_c=pk3.cout_p), capi.RES_BEFORE_RELU,
              out_fmt=capi.FMT_F32)
    assert yf.fmt == capi.FMT_F32
    yf = act_to_nchw(yf, cout).squeeze(2).cpu()
    torch.cuda.synchronize()
    assert rel_err(y.numpy(), want.numpy()) < TOL["tc1"]
    assert rel_err(yf.numpy(), want.numpy()) < TOL["tc"]


@pytest.mark.parametrize("case", [c for c in CASES if c[1] >= 256 or c[2] == 3])
def test_modelled_split_matches_no_split(case):
    """The K split chosen by lt_conv_tc_plan sums its partial tiles in a fixed order: within 5e-6 of tc_splitk = 0 and
    bit-identical run to run."""
    conv, bn, x, res, want = _case(case, "before", 11 + case[0])
    cout = case[1]
    e = _engine("tc")
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    xa, ra = act_from_nchw(x, capi.FMT_S32), act_from_nchw(res, capi.FMT_S32, pad_c=_c32(cout))
    ys = [act_to_nchw(_run(e, pk, xa, ra, capi.RES_BEFORE_RELU), cout).cpu() for _ in range(2)]
    old = capi.get_options()["tc_splitk"]
    try:
        capi.set_options(tc_splitk=0)
        y0 = act_to_nchw(_run(e, pk, xa, ra, capi.RES_BEFORE_RELU), cout).cpu()
    finally:
        capi.set_options(tc_splitk=old)
    torch.cuda.synchronize()
    assert torch.equal(ys[0], ys[1])
    assert rel_err(ys[0].numpy(), y0.numpy()) < 5e-6
    assert rel_err(y0.squeeze(2).numpy(), want.numpy()) < TOL["tc"]


def test_grouped_deconv3d_persistent():
    """k2 s2 transposed conv + skip as one grouped GEMM (8 N tiles of 128 routed to the 8 output phases), 256 M tiles."""
    torch.manual_seed(5)
    cin, cout, spatial, N = 128, 128, (16, 16, 16), 8
    e = _engine("tc")
    dc = torch.nn.ConvTranspose3d(cin, cout, 2, 2).eval()
    bn = _bn_for(dc, 3)
    x = torch.randn(N, cin, *spatial)
    skip = torch.randn(N, cout, *[2 * v for v in spatial])
    with torch.no_grad():
        want = F.relu(bn(dc(x))) + skip
    pk = e._pack_deconv3d_k2s2(dc.to(DEV), bn.to(DEV))
    assert pk.groups == 8
    xa, sa = act_from_nchw(x, capi.FMT_S32), act_from_nchw(skip, capi.FMT_S32)
    got = [act_to_nchw(e._deconv3d(xa, pk, sa)).cpu() for _ in range(2)]
    torch.cuda.synchronize()
    assert torch.equal(got[0], got[1])
    assert rel_err(got[0].numpy(), want.numpy()) < TOL["tc"]


@pytest.mark.parametrize("mnk", [(128 * 301, 64, 128), (128 * 133 + 5, 128, 64), (256, 256, 512)])
def test_selftest_gemm_many_units(mnk):
    """The plain-fp16 self-test GEMM through the same persistent kernel, with more M tiles than SMs."""
    M, N, K = mnk
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(DEV).half().contiguous()
    b = torch.randn(N, K, generator=g).to(DEV).half().contiguous()
    d = torch.zeros(M * N + 2 * N, dtype=torch.float32, device=DEV)
    capi.tc_gemm_selftest(a, b, d, M, N, K)
    torch.cuda.synchronize()
    got = d[:M * N].view(M, N).cpu().double()
    want = a.cpu().double() @ b.cpu().double().t()
    assert rel_err(got.numpy(), want.numpy()) < 1e-5
