"""GPU parity tests of the bandwidth-bound kernels and the FFMA conv path, through the C ABI, against the CPU
oracle (oracle/vol_oracle.py) and the committed golden vectors.  Tolerances: fp32 kernels, 1e-5..1e-4 relative
to the tensor's max/spread (far inside the 1e-3 contract of BASELINE.json)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_err
from oracle import vol_oracle as O
from lt_b200 import capi, op, testing
from lt_b200.engine import Act, NativeEngine

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def cu(a):
    return torch.as_tensor(np.ascontiguousarray(a)).to(DEV)


# ------------------------------------------------------------------------------------------ unprojection
@pytest.mark.parametrize("tag", ["a", "b", "c"])
@pytest.mark.parametrize("agg", ["sum", "max", "softmax", "conf"])
def test_unproject_golden(tag, agg):
    g = np.load(os.path.join(GOLDEN, "unproject.npz"))
    out = op.unproject_heatmaps(cu(g[tag + "_heat"]), cu(g[tag + "_proj"]), cu(g[tag + "_coord"]), agg, cu(g[tag + "_conf"]))
    assert rel_err(out.cpu().numpy(), g["%s_out_%s" % (tag, agg)]) < 2e-5


def _scene(B, V, C, h, w, n, seed):
    rng = np.random.RandomState(seed)
    heat = rng.randn(B, V, C, h, w).astype(np.float32)
    cams = testing.make_cameras(V, image_size=48, radius=3000.0)
    proj = np.stack([np.stack([O.projection_after_resize(c.K, c.R, c.t, (48, 48), (h, w)) for c in cams])] * B)
    coord = np.stack([O.coord_volume(rng.randn(3) * 100 + [0, 0, 900], 2800.0, n) for _ in range(B)])
    conf = rng.rand(B, V, C).astype(np.float32)
    return heat, proj, coord, conf


@pytest.mark.parametrize("shape", [(1, 1, 32, 12, 12, 8), (2, 4, 32, 9, 13, 8), (1, 8, 32, 16, 16, 6),
                                   (1, 9, 32, 8, 8, 6), (2, 3, 5, 7, 11, 5), (1, 10, 6, 8, 8, 4), (1, 2, 64, 6, 6, 4)])
@pytest.mark.parametrize("agg", ["sum", "max", "softmax", "conf"])
def test_unproject_vs_oracle(shape, agg):
    heat, proj, coord, conf = _scene(*shape, seed=sum(shape))
    want = O.unproject_heatmaps(heat, proj, coord, agg, conf)
    got = op.unproject_heatmaps(cu(heat), cu(proj), cu(coord), agg, cu(conf)).cpu().numpy()
    assert got.shape == want.shape
    assert rel_err(got, want) < 3e-5


def test_unproject_split_output_and_partial_sum():
    B, V, C, h, w, n = 2, 4, 32, 12, 12, 8
    heat, proj, coord, conf = _scene(B, V, C, h, w, n, seed=11)
    want = O.unproject_heatmaps(heat, proj, coord, "softmax")
    feats = cu(heat).permute(0, 1, 3, 4, 2).contiguous()
    nvox = n ** 3
    out_s = torch.empty((B, nvox, 2 * C), dtype=torch.float16, device=DEV)
    capi.unproject_aggregate(feats, cu(proj), cu(coord).view(B, nvox, 3), None, out_s, capi.FMT_S32, capi.AGG["softmax"])
    out_f = torch.empty((B, nvox, C), dtype=torch.float32, device=DEV)
    capi.s32_to_f32(out_s, out_f, B * nvox, C)
    got = out_f.view(B, n, n, n, C).permute(0, 4, 1, 2, 3).cpu().numpy()
    assert rel_err(got, want) < 3e-5          # split-fp16 keeps ~22 significand bits
    # view-sharded: two "ranks" with two views each, summed partials == single pass
    parts = []
    for r in range(2):
        p = torch.empty((B, 2, nvox, C), dtype=torch.float32, device=DEV)
        capi.unproject_partial(feats[:, r::2].contiguous(), cu(proj[:, r::2]), cu(coord).view(B, nvox, 3), None, p, capi.AGG["softmax"])
        parts.append(p)
    total = parts[0] + parts[1]
    fin = torch.empty((B, nvox, C), dtype=torch.float32, device=DEV)
    capi.unproject_finalize(total, fin, capi.FMT_F32, B, C, nvox, capi.AGG["softmax"])
    assert rel_err(fin.view(B, n, n, n, C).permute(0, 4, 1, 2, 3).cpu().numpy(), want) < 3e-5


# ------------------------------------------------------------------------------------------ soft-argmax
@pytest.mark.parametrize("softmax", [True, False])
def test_softargmax_golden(softmax):
    g = np.load(os.path.join(GOLDEN, "softargmax.npz"))
    kp, v = op.integrate_tensor_3d_with_coordinates(cu(g["vols"]), cu(g["coord"]), softmax)
    assert rel_err(kp.cpu().numpy(), g["kp_%d" % softmax]) < 2e-5
    assert rel_err(v.cpu().numpy(), g["v_%d" % softmax]) < 2e-5


@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("layout", ["channels_first", "channels_last"])
def test_softargmax_vs_oracle(softmax, layout):
    rng = np.random.RandomState(3)
    B, J, n, Cp = 2, 17, 20, 32
    vols = (rng.randn(B, J, n, n, n) * 4).astype(np.float32)
    coord = (rng.randn(B, n, n, n, 3) * 700).astype(np.float32)
    mult = 1.7
    kp_w, v_w = O.integrate_tensor_3d_with_coordinates(vols * np.float32(mult), coord, softmax)
    nvox = n ** 3
    if layout == "channels_first":
        kp, v = op.integrate_tensor_3d_with_coordinates(cu(vols) * mult, cu(coord), softmax)
    else:
        cl = torch.zeros((B, nvox, Cp), dtype=torch.float32, device=DEV)
        cl[:, :, :J] = cu(vols).view(B, J, nvox).permute(0, 2, 1)
        v = torch.empty((B, J, n, n, n), dtype=torch.float32, device=DEV)
        kp = torch.empty((B, J, 3), dtype=torch.float32, device=DEV)
        ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, nvox) // 4 + 1, dtype=torch.float32, device=DEV)
        capi.softargmax3d(cl, nvox * Cp, Cp, 1, cu(coord).view(B, nvox, 3), v, kp, ws, B, J, nvox, mult, softmax)
    assert rel_err(kp.cpu().numpy(), kp_w) < 3e-5
    assert rel_err(v.cpu().numpy(), v_w) < 3e-5
    assert np.array_equal(v.view(B, J, -1).argmax(-1).cpu().numpy(), v_w.reshape(B, J, -1).argmax(-1))


@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("Cp,J,n,B", [(20, 17, 32, 3), (32, 17, 28, 2), (24, 21, 26, 1), (20, 17, 64, 2)])
def test_softargmax_fused_stream(softmax, Cp, J, n, B):
    """Fused streaming path (nvox >= 16384, voxel stride 20..32): partial tail tiles, more tiles than CTAs (64^3),
    fewer tiles than CTAs, NaN in the padding channels (must never leak), keypoints-only call."""
    rng = np.random.RandomState(Cp + n)
    vols = (rng.randn(B, J, n, n, n) * 3).astype(np.float32)
    vols[:, :, n // 3, n // 2, n // 5] += 9.0          # a clear peak per joint
    coord = (rng.randn(B, n, n, n, 3) * 700).astype(np.float32)
    mult = 1.3
    kp_w, v_w = O.integrate_tensor_3d_with_coordinates(vols * np.float32(mult), coord, softmax)
    nvox = n ** 3
    cl = torch.full((B, nvox, Cp), float("nan"), dtype=torch.float32, device=DEV)
    cl[:, :, :J] = cu(vols).view(B, J, nvox).permute(0, 2, 1)
    v = torch.empty((B, J, n, n, n), dtype=torch.float32, device=DEV)
    kp = torch.empty((B, J, 3), dtype=torch.float32, device=DEV)
    ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, nvox) // 4 + 1, dtype=torch.float32, device=DEV)
    for _ in range(2):   # twice: the per-sample counters/flags in the workspace must be re-armed by every call
        v.fill_(-1.0)
        capi.softargmax3d(cl, nvox * Cp, Cp, 1, cu(coord).view(B, nvox, 3), v, kp, ws, B, J, nvox, mult, softmax)
        assert rel_err(kp.cpu().numpy(), kp_w) < 3e-5
        assert rel_err(v.cpu().numpy(), v_w) < 3e-5
        assert np.array_equal(v.view(B, J, -1).argmax(-1).cpu().numpy(), v_w.reshape(B, J, -1).argmax(-1))
    kp2 = torch.empty_like(kp)
    capi.softargmax3d(cl, nvox * Cp, Cp, 1, cu(coord).view(B, nvox, 3), None, kp2, ws, B, J, nvox, mult, softmax)
    assert torch.equal(kp2, kp)


# ------------------------------------------------------------------------------------------ coordinate volume
@pytest.mark.parametrize("theta,transfer", [(0.0, False), (0.0, True), (1.1, False)])
def test_coord_volume(theta, transfer):
    n, B = 16, 3
    rng = np.random.RandomState(1)
    base = rng.randn(B, 3) * 300 + [0, 0, 900]
    side = 2500.0
    want = np.stack([O.coord_volume(base[b], side, n, theta, (0, 0, 1), transfer) for b in range(B)])
    out = torch.empty((B, n, n, n, 3), dtype=torch.float32, device=DEV)
    rot = np.stack([O.rotation_matrix((0, 0, 1), theta)] * B).reshape(B, 9)
    capi.coord_volume(cu(np.float32(base - side / 2)), cu(np.float32(base)), cu(np.float32([side / (n - 1)] * 3)),
                      cu(np.float32(rot)), out, transfer)
    if theta == 0.0:
        assert np.array_equal(out.cpu().numpy(), want)       # bit-exact in eval mode
    else:
        assert np.abs(out.cpu().numpy() - want).max() < 1e-3  # mm


# ------------------------------------------------------------------------------------------ FFMA conv path
class _Holder(torch.nn.Module):
    """Minimal object with the attributes NativeEngine reads (only used to reach its packing helpers)."""
    volume_size = 32


def _engine(mode):
    e = NativeEngine.__new__(NativeEngine)
    e.model, e.mode, e.use_graph = _Holder(), mode, False
    e.act_fmt = capi.FMT_F32 if mode == "simt" else capi.FMT_S32
    e.tc_impl = {"simt": capi.CONV_SIMT, "tc": capi.CONV_TC, "tc1": capi.CONV_TC1}[mode]
    e._packs, e._graphs, e.launches, e.timeline, e._epoch = {}, {}, 0, None, 0
    return e


def act_from_nchw(x, fmt, pad_c=None):
    """torch (N,C,[D,]H,W) cpu/cuda -> Act channels-last in fmt."""
    x = x.to(DEV).float()
    if x.dim() == 4:
        x = x.unsqueeze(2)
    N, C, D, H, W = x.shape
    Cp = pad_c or C
    a = Act(N, D, H, W, Cp, capi.FMT_F32, DEV, zero=True)
    a.data[..., :C] = x.permute(0, 2, 3, 4, 1)
    if fmt == capi.FMT_S32:
        s = Act(N, D, H, W, Cp, capi.FMT_S32, DEV)
        capi.f32_to_s32(a.data, s.data, a.pixels, Cp)
        return s
    return a


def act_to_nchw(a, C=None):
    if a.fmt == capi.FMT_S32:
        f = Act(a.N, a.D, a.H, a.W, a.C, capi.FMT_F32, DEV)
        capi.s32_to_f32(a.data, f.data, a.pixels, a.C)
        a = f
    out = a.data.permute(0, 4, 1, 2, 3)
    return out[:, :C] if C else out


def _bn_for(conv, seed=0):
    g = torch.Generator().manual_seed(seed)
    c = conv.out_channels
    bn = torch.nn.BatchNorm3d(c) if isinstance(conv, (torch.nn.Conv3d, torch.nn.ConvTranspose3d)) else torch.nn.BatchNorm2d(c)
    bn.weight.data = torch.rand(c, generator=g) + 0.5
    bn.bias.data = torch.randn(c, generator=g) * 0.3
    bn.running_mean = torch.randn(c, generator=g) * 0.2
    bn.running_var = torch.rand(c, generator=g) + 0.5
    return bn.eval()


CONV_CASES = [
    # (dims, cin, cout, k, stride, pad, spatial, batch)
    (2, 64, 64, 1, 1, 0, (12, 12), 2),
    (2, 32, 48, 3, 1, 1, (9, 11), 2),
    (2, 64, 128, 3, 2, 1, (12, 12), 2),
    (2, 64, 256, 1, 2, 0, (12, 12), 1),
    (2, 3, 64, 7, 2, 3, (32, 32), 2),
    (3, 32, 16, 7, 1, 3, (8, 8, 8), 1),
    (3, 16, 32, 3, 1, 1, (8, 8, 8), 2),
    (3, 32, 17, 1, 1, 0, (8, 8, 8), 1),
    (3, 128, 128, 3, 1, 1, (4, 4, 4), 2),
]


@pytest.mark.parametrize("case", CONV_CASES)
@pytest.mark.parametrize("out_fmt", [capi.FMT_F32, capi.FMT_S32])
def test_conv_simt_vs_torch(case, out_fmt):
    dims, cin, cout, k, stride, pad, spatial, N = case
    if out_fmt == capi.FMT_S32 and cout % 32:
        pytest.skip("split-fp16 output needs 32-channel blocks")
    torch.manual_seed(cin * 7 + cout)
    conv = (torch.nn.Conv2d if dims == 2 else torch.nn.Conv3d)(cin, cout, k, stride, pad, bias=(dims == 3)).eval()
    bn = _bn_for(conv, 5)
    x = torch.randn(N, cin, *spatial)
    res = torch.randn_like(bn(conv(x)))
    with torch.no_grad():
        want = F.relu(bn(conv(x)) + res)
    e = _engine("simt")
    e.act_fmt = out_fmt
    pk = e._pack_conv(conv.to(DEV), bn.to(DEV), cin_pad=4 if cin == 3 else None, force_simt=True)
    xa = act_from_nchw(x, capi.FMT_F32, pad_c=4 if cin == 3 else None)
    ra = act_from_nchw(res, out_fmt, pad_c=(cout + 3) // 4 * 4)
    ya = e._conv(xa, pk, relu=True, residual=ra, res_mode=capi.RES_BEFORE_RELU, out_fmt=out_fmt)
    got = act_to_nchw(ya, cout).cpu()
    if dims == 2:
        got = got.squeeze(2)
    assert rel_err(got.numpy(), want.numpy()) < 3e-5


def test_deconv_phases_simt_vs_torch():
    torch.manual_seed(1)
    e = _engine("simt")
    # 2-D k4 s2 p1 (pose_resnet.py:266-291)
    dc = torch.nn.ConvTranspose2d(32, 48, 4, 2, 1, 0, bias=False).eval()
    bn = _bn_for(dc, 2)
    x = torch.randn(2, 32, 6, 7)
    with torch.no_grad():
        want = F.relu(bn(dc(x)))
    got = act_to_nchw(e._deconv2d(act_from_nchw(x, capi.FMT_F32), e._pack_deconv2d_k4s2(dc.to(DEV), bn.to(DEV)))).squeeze(2).cpu()
    assert rel_err(got.numpy(), want.numpy()) < 3e-5
    # 3-D k2 s2 + skip add after ReLU (v2v.py:54-66,124-136)
    dc3 = torch.nn.ConvTranspose3d(32, 16, 2, 2).eval()
    bn3 = _bn_for(dc3, 3)
    x3 = torch.randn(2, 32, 3, 4, 5)
    skip = torch.randn(2, 16, 6, 8, 10)
    with torch.no_grad():
        want3 = F.relu(bn3(dc3(x3))) + skip
    got3 = act_to_nchw(e._deconv3d(act_from_nchw(x3, capi.FMT_F32), e._pack_deconv3d_k2s2(dc3.to(DEV), bn3.to(DEV)),
                                   act_from_nchw(skip, capi.FMT_F32))).cpu()
    assert rel_err(got3.numpy(), want3.numpy()) < 3e-5


@pytest.mark.parametrize("fmt", [capi.FMT_F32, capi.FMT_S32])
def test_maxpool(fmt):
    e = _engine("simt")
    x2 = torch.randn(2, 64, 11, 12)
    got = act_to_nchw(e._maxpool(act_from_nchw(x2, fmt), (1, 3, 3), (1, 2, 2), (0, 1, 1))).squeeze(2).cpu()
    assert rel_err(got.numpy(), F.max_pool2d(x2, 3, 2, 1).numpy()) < 2e-5
    x3 = torch.randn(2, 32, 8, 6, 4)
    got3 = act_to_nchw(e._maxpool(act_from_nchw(x3, fmt), (2, 2, 2), (2, 2, 2), (0, 0, 0))).cpu()
    assert rel_err(got3.numpy(), F.max_pool3d(x3, 2, 2).numpy()) < 2e-5


def test_split_fp16_round_trip_precision():
    x = (torch.randn(1000, 64, device=DEV) * torch.logspace(-3, 4, 64, device=DEV)).contiguous()
    s = torch.empty((1000, 128), dtype=torch.float16, device=DEV)
    capi.f32_to_s32(x, s, 1000, 64)
    y = torch.empty_like(x)
    capi.s32_to_f32(s, y, 1000, 64)
    # 22 significand bits while the (unscaled) low part is a normal fp16 number; below that an absolute floor of 2^-25
    assert bool(((x - y).abs() <= x.abs() * 2 ** -21 + 2 ** -25).all())


def test_nchw_to_nhwc_and_back():
    x = torch.randn(3, 3, 10, 14, device=DEV)
    y = torch.empty((3, 10, 14, 4), device=DEV)
    capi.nchw_to_nhwc(x, y, 3, 3, 10, 14, 4)
    assert torch.equal(y[..., :3], x.permute(0, 2, 3, 1)) and float(y[..., 3].abs().max()) == 0.0
    z = torch.empty((3, 3, 140), device=DEV)
    capi.cl_to_cf(y.view(3, 140, 4), z, 3, 140, 4, 3)
    assert torch.equal(z.view(3, 3, 10, 14), x)
