"""conv_tc_kernel's shared-memory staged epilogue (residual tile in and output tile out by TMA): partial M tiles, several units
per CTA handing the buffer over, in-place residual, float32 outputs narrower than the N tile, stride-phase and grouped outputs.

Every launch here runs without a split-K workspace, so it ends in conv_tc_kernel's own epilogue rather than in
splitk_reduce_kernel; the `plans` fixture records lt_conv_tc_plan for each launch, and the tests assert the path they cover."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lt_b200 import capi
from test_gpu_ops import _engine, _bn_for, act_from_nchw, act_to_nchw, DEV

pytestmark = pytest.mark.gpu

TOL = 2e-5
RES = {"none": capi.RES_NONE, "before": capi.RES_BEFORE_RELU, "after": capi.RES_AFTER_RELU}

# (cin, cout, k, stride, spatial, batch)
CASES = [
    (64, 256, 1, 1, (13, 11), 5),      # partial M tiles in W and H, several images per tile
    (128, 96, 3, 1, (7, 9), 3),        # N tile of 32 x 3, partial tiles
    (64, 256, 1, 1, (24, 24), 45),     # 2 N tiles of 128, more units than SMs: several units per CTA
    (256, 1024, 1, 1, (24, 24), 3),    # N tile 128, 8 N tiles
    (128, 128, 3, 2, (17, 15), 4),     # stride 2, partial tiles
]


def _single_pass_engine():
    e = _engine("tc")
    e._splitk_ws = torch.empty(0, dtype=torch.uint8, device=DEV)      # no workspace -> never split
    return e


@pytest.fixture
def plans(monkeypatch):
    """lt_conv_tc_plan of every LT_CONV_TC launch the test makes, in launch order."""
    got = []
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    conv_nd = capi.conv_nd

    def hook(desc, *args):
        if args[-1] == capi.CONV_TC:
            got.append(capi.conv_tc_plan(desc, sms, capi.get_options()["tc_splitk"]))
        return conv_nd(desc, *args)

    monkeypatch.setattr(capi, "conv_nd", hook)
    return got


def _assert_staged(plans, launches):
    """`launches` launches, each one pass (no K split) with whole 32-channel slabs: the staged epilogue."""
    assert len(plans) == launches, plans
    for p in plans:
        assert p["splits"] == 1 and p["nt"] >= 32, p


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
def test_staged_vs_torch_and_repeat(case, res_mode, plans):
    conv, bn, x, res, want = _case(case, res_mode, sum(case[:3]))
    cout = case[1]
    e = _single_pass_engine()
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    xa = act_from_nchw(x, capi.FMT_S32)
    ra = act_from_nchw(res, capi.FMT_S32, pad_c=(cout + 31) // 32 * 32) if res_mode != "none" else None
    ys = [e._conv(xa, pk, relu=True, residual=ra, res_mode=RES[res_mode]) for _ in range(2)]
    y = [act_to_nchw(a, cout).squeeze(2).cpu() for a in ys]
    torch.cuda.synchronize()
    _assert_staged(plans, 2)
    if case == CASES[2]:
        assert plans[0]["m_tiles"] * plans[0]["n_tiles"] > 2 * plans[0]["grid"], plans[0]   # 3 or more units on some CTAs
    assert torch.equal(y[0], y[1]), "two runs must be bit-identical"
    assert rel_err(y[0].numpy(), want.numpy()) < TOL


@pytest.mark.parametrize("case", [CASES[0], CASES[2], CASES[3]])
@pytest.mark.parametrize("res_mode", ["before", "after"])
def test_staged_in_place_residual(case, res_mode, plans):
    """out is the residual tensor: bit-identical to the out-of-place result."""
    conv, bn, x, res, want = _case(case, res_mode, 17 + case[1])
    cout = case[1]
    e = _single_pass_engine()
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV))
    xa = act_from_nchw(x, capi.FMT_S32)
    ra = act_from_nchw(res, capi.FMT_S32, pad_c=(cout + 31) // 32 * 32)
    ref = act_to_nchw(e._conv(xa, pk, relu=True, residual=ra, res_mode=RES[res_mode]), cout).cpu()
    got = e._conv(xa, pk, relu=True, residual=ra, res_mode=RES[res_mode], out=ra)
    assert got is ra
    got = act_to_nchw(got, cout).cpu()
    torch.cuda.synchronize()
    _assert_staged(plans, 2)
    assert torch.equal(got, ref)
    assert rel_err(got.squeeze(2).numpy(), want.numpy()) < TOL


@pytest.mark.parametrize("cout,out_c", [(20, 20), (17, 20), (40, 44), (16, 16)])
def test_staged_fp32_output_narrower_than_tile(cout, out_c, plans):
    """float32 output with a channel stride FC below the padded N tile: the TMA store clips at FC.  Padded Cout 48 and 16 give
    16-channel N tiles, which keep the register epilogue."""
    torch.manual_seed(cout + out_c)
    conv = torch.nn.Conv2d(64, cout, 3, 1, 1, bias=True).eval()
    x = torch.randn(3, 64, 13, 10)
    res = torch.randn(3, cout, 13, 10)
    with torch.no_grad():
        want = F.relu(conv(x) + res)
    e = _single_pass_engine()
    pk = e._pack_conv(conv.to(DEV), None, out_fmt=capi.FMT_F32)
    xa = act_from_nchw(x, capi.FMT_S32)
    ra = act_from_nchw(res, capi.FMT_F32, pad_c=out_c)
    ys = [e._conv(xa, pk, relu=True, residual=ra, res_mode=capi.RES_BEFORE_RELU, out_fmt=capi.FMT_F32, out_c=out_c)
          for _ in range(2)]
    assert ys[0].fmt == capi.FMT_F32 and ys[0].C == out_c
    y = [a.data.cpu() for a in ys]
    torch.cuda.synchronize()
    if pk.cout_p % 32 == 0:
        _assert_staged(plans, 2)
    else:
        assert len(plans) == 2 and all(p["splits"] == 1 and p["nt"] == 16 for p in plans), plans
    assert torch.equal(y[0], y[1])
    assert rel_err(act_to_nchw(ys[0], cout).squeeze(2).cpu().numpy(), want.numpy()) < TOL


@pytest.mark.parametrize("spatial,batch", [((12, 12), 4), ((7, 9), 3)])
def test_staged_deconv2d_phases(spatial, batch, plans):
    """ConvTranspose2d(k4, s2, p1) as four stride-phase convs writing one output: each phase is a sub-lattice tensor map."""
    torch.manual_seed(batch)
    dc = torch.nn.ConvTranspose2d(64, 64, 4, 2, 1).eval()
    bn = _bn_for(dc, 2)
    x = torch.randn(batch, 64, *spatial)
    with torch.no_grad():
        want = F.relu(bn(dc(x)))
    e = _single_pass_engine()
    phases = e._pack_deconv2d_k4s2(dc.to(DEV), bn.to(DEV))
    xa = act_from_nchw(x, capi.FMT_S32)
    got = [act_to_nchw(e._deconv2d(xa, phases), 64).squeeze(2).cpu() for _ in range(2)]
    torch.cuda.synchronize()
    _assert_staged(plans, 8)
    assert torch.equal(got[0], got[1])
    assert rel_err(got[0].numpy(), want.numpy()) < TOL


@pytest.mark.parametrize("cin,cout,spatial,N", [(64, 32, (5, 6, 7), 3), (128, 64, (4, 4, 4), 2)])
def test_staged_grouped_deconv3d_skip(cin, cout, spatial, N, plans):
    """k2 s2 transposed conv + skip as one grouped GEMM with partial M tiles: one output and one skip map per output phase."""
    torch.manual_seed(cin + cout)
    e = _single_pass_engine()
    dc = torch.nn.ConvTranspose3d(cin, cout, 2, 2).eval()
    bn = _bn_for(dc, 4)
    x = torch.randn(N, cin, *spatial)
    skip = torch.randn(N, cout, *[2 * v for v in spatial])
    with torch.no_grad():
        want = F.relu(bn(dc(x))) + skip
    pk = e._pack_deconv3d_k2s2(dc.to(DEV), bn.to(DEV))
    assert pk.groups == 8
    xa, sa = act_from_nchw(x, capi.FMT_S32), act_from_nchw(skip, capi.FMT_S32)
    got = [act_to_nchw(e._deconv3d(xa, pk, sa)).cpu() for _ in range(2)]
    torch.cuda.synchronize()
    _assert_staged(plans, 2)
    assert torch.equal(got[0], got[1])
    assert rel_err(got[0].numpy(), want.numpy()) < TOL
