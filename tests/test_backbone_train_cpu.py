"""CPU checks of the native backbone training convolutions (autograd_ops.ConvNdFn in 2-D, ConvTranspose2dK4Fn, StemConvFn), no GPU
needed: the filter re-gathers that turn each data gradient into forward convolutions (with the grouped launch's phase scatter), the
weight-gradient kernel's index mapping (lt_test_conv_wgrad_host) on every 2-D descriptor, the device-side stem filter gather, and
the `backbone_backend` option -- all against torch autograd in float64."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from conftest import rel_err
from lt_b200 import autograd_ops as A
from lt_b200 import capi, engine


def _gather(w, base, strides, k, cin, cout):
    """torch emulation of lt_conv_gather_weights_fwd (include/lt_b200.h): element (td, th, tw, ci, co) of the canonical filter is
    w.flatten()[base + td s_td + th s_th + tw s_tw + ci s_ci + co s_co]; returned as a (cout, cin, kh, kw) Conv2d filter (kd = 1)."""
    assert k[0] == 1
    flat = w.reshape(-1)
    td, th, tw, ci, co = torch.meshgrid(*[torch.arange(n) for n in (k[0], k[1], k[2], cin, cout)], indexing="ij")
    idx = base + td * strides[0] + th * strides[1] + tw * strides[2] + ci * strides[3] + co * strides[4]
    assert int(idx.min()) >= 0 and int(idx.max()) < flat.numel()
    return flat[idx].permute(4, 3, 0, 1, 2)[:, :, 0]


# (cin, cout, (H, W), N): 3x3 stride-2 pad-1 convs at even, odd and mixed sides
S2K3_CASES = [(64, 64, (8, 10), 2), (32, 64, (13, 11), 2), (64, 32, (7, 7), 3), (96, 32, (12, 9), 2)]
S2K1_CASES = [(64, 128, (8, 10), 2), (32, 64, (13, 11), 2), (256, 32, (7, 5), 2)]
DECONV_CASES = [(64, 32, (6, 5), 2), (32, 64, (3, 4), 2), (17, 20, (4, 4), 1)]


@pytest.mark.parametrize("case", S2K3_CASES)
def test_grouped_s2_dgrad_regather_reproduces_autograd(case):
    """One 2x2 stride-1 pad-0 conv of dY (one row / column of zeros past its end, as TMA fills it) with N = 4 Cin, column block
    g = 2a + b scattered to input phase (a, b) over that phase's own extent."""
    cin, cout, (H, W), N = case
    torch.manual_seed(cin + cout + H)
    x = torch.randn(N, cin, H, W, dtype=torch.float64, requires_grad=True)
    w = torch.randn(cout, cin, 3, 3, dtype=torch.float64)
    y = F.conv2d(x, w, None, 2, 1)
    gy = torch.randn_like(y)
    y.backward(gy)
    srcs, k, pad, groups, ci, co = A.conv_s2_dgrad_filter(w.shape, (2, 2))
    assert (k, pad, groups, ci, co) == ((1, 2, 2), (0, 0, 0), (1, 2, 2), cout, cin) and len(srcs) == 4
    wp = A.pad_s2_filter(w, (2, 2))
    assert wp.shape == (cout, cin, 4, 4)
    OH, OW = y.shape[2:]
    gy_ext = F.pad(gy, (0, 1, 0, 1))
    got = torch.full_like(x, float("nan"))
    for g, (base, strides) in enumerate(srcs):
        a, b = g // 2, g % 2
        out = F.conv2d(gy_ext, _gather(wp, base, strides, k, ci, co))
        assert out.shape[2:] == (OH, OW)
        eh, ew = (H - a + 1) // 2, (W - b + 1) // 2          # the per-group extents of make_epi_maps
        assert eh <= OH and ew <= OW
        got[:, :, a::2, b::2] = out[:, :, :eh, :ew]
    assert rel_err(got.detach().numpy(), x.grad.numpy()) < 1e-12


@pytest.mark.parametrize("case", S2K1_CASES)
def test_1x1_s2_dgrad_regather_reproduces_autograd(case):
    """The transposed 1x1 filter over dY into the even phase of dX; the other three phases are zero."""
    cin, cout, (H, W), N = case
    torch.manual_seed(cin + cout + H + 1)
    x = torch.randn(N, cin, H, W, dtype=torch.float64, requires_grad=True)
    w = torch.randn(cout, cin, 1, 1, dtype=torch.float64)
    y = F.conv2d(x, w, None, 2, 0)
    gy = torch.randn_like(y)
    y.backward(gy)
    (base, strides), k, stride, pad, ci, co = A.conv3d_dgrad_filter(w.shape, (0, 0))
    assert (k, stride, pad, ci, co) == ((1, 1, 1), (1, 1, 1), (0, 0, 0), cout, cin)
    got = torch.zeros_like(x)
    got[:, :, 0::2, 0::2] = F.conv2d(gy, _gather(w, base, strides, k, ci, co))
    assert rel_err(got.detach().numpy(), x.grad.numpy()) < 1e-12


@pytest.mark.parametrize("k", [1, 3])
def test_stride1_2d_dgrad_regather_reproduces_autograd(k):
    torch.manual_seed(k)
    x = torch.randn(2, 32, 9, 7, dtype=torch.float64, requires_grad=True)
    w = torch.randn(17, 32, k, k, dtype=torch.float64)
    y = F.conv2d(x, w, None, 1, k // 2)
    gy = torch.randn_like(y)
    y.backward(gy)
    (base, strides), kk, stride, pad, ci, co = A.conv3d_dgrad_filter(w.shape, (k // 2, k // 2))
    got = F.conv2d(gy, _gather(w, base, strides, kk, ci, co), None, stride[1:], pad[1:])
    assert rel_err(got.numpy(), x.grad.numpy()) < 1e-12


@pytest.mark.parametrize("case", DECONV_CASES)
def test_deconv_k4s2_dgrad_regather_reproduces_autograd(case):
    cin, cout, (H, W), N = case
    torch.manual_seed(cin + cout + 2)
    x = torch.randn(N, cin, H, W, dtype=torch.float64, requires_grad=True)
    w = torch.randn(cin, cout, 4, 4, dtype=torch.float64)
    y = F.conv_transpose2d(x, w, None, 2, 1)
    gy = torch.randn_like(y)
    y.backward(gy)
    (base, strides), k, stride, pad, ci, co = A.conv_transpose2d_k4s2_dgrad_filter(w.shape)
    got = F.conv2d(gy, _gather(w, base, strides, k, ci, co), None, stride[1:], pad[1:])
    assert rel_err(got.numpy(), x.grad.numpy()) < 1e-12


def _cl_padded(t, cp):
    """(N, C, H, W) -> float32 channels-last (N, 1, H, W, cp), channels C .. cp-1 zero."""
    out = torch.zeros(t.shape[0], 1, *t.shape[2:], cp, dtype=torch.float32)
    out[:, 0, ..., :t.shape[1]] = t.permute(0, 2, 3, 1).float()
    return out.contiguous()


# (cin, cout, k, stride, (H, W), N)
WGRAD_CASES = [
    (64, 64, 3, 1, (9, 7), 2),
    (32, 17, 1, 1, (8, 6), 2),      # final_layer: 17 output channels padded to 32
    (256, 32, 1, 1, (5, 6), 2),     # process_features
    (64, 128, 3, 2, (13, 11), 2),
    (32, 64, 3, 2, (8, 10), 3),
    (64, 128, 1, 2, (13, 11), 2),
    (64, 256, 1, 2, (6, 6), 2),
]


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_wgrad_host_mapping_conv2d(case):
    cin, cout, k, s, (H, W), N = case
    torch.manual_seed(3 + cin + cout + k + s)
    x = torch.randn(N, cin, H, W, dtype=torch.float64)
    w = torch.randn(cout, cin, k, k, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(x.float().double(), w, None, s, k // 2)
    gy = torch.randn_like(y).float().double()
    y.backward(gy)
    d = A.conv3d_wgrad_desc(N, (1, H, W), cin, cout, (1, k, k), (0, k // 2, k // 2), (1, s, s))
    assert (d.OH, d.OW) == tuple(y.shape[2:])
    gw = torch.empty(k * k, cin, cout, dtype=torch.float32)
    capi.conv_wgrad_host(d, _cl_padded(x, d.Cin), _cl_padded(gy, d.FC), cin, cout, gw)
    got = gw.reshape(k, k, cin, cout).permute(3, 2, 0, 1)
    assert rel_err(got.numpy(), w.grad.numpy()) < 1e-6


@pytest.mark.parametrize("case", DECONV_CASES)
def test_wgrad_host_mapping_deconv_k4s2_phases(case):
    """Each 2x2 phase descriptor's weight gradient lands on its own four of the 16 taps; together they are autograd's dW."""
    cin, cout, (H, W), N = case
    torch.manual_seed(5 + cin + cout)
    x = torch.randn(N, cin, H, W, dtype=torch.float64)
    w = torch.randn(cin, cout, 4, 4, dtype=torch.float64, requires_grad=True)
    y = F.conv_transpose2d(x.float().double(), w, None, 2, 1)
    gy = torch.randn_like(y).float().double()
    y.backward(gy)
    got = torch.full((cin, cout, 4, 4), float("nan"), dtype=torch.float32)
    for py in (0, 1):
        for px in (0, 1):
            d = A.conv_transpose2d_k4s2_desc(N, (1, H, W), cin, cout, py, px)
            gw = torch.empty(4, cin, cout, dtype=torch.float32)
            capi.conv_wgrad_host(d, _cl_padded(x, d.Cin), _cl_padded(gy, d.FC), cin, cout, gw)
            got[:, :, 1 - py::2, 1 - px::2] = A.conv_transpose2d_k4s2_wgrad_scatter(gw, py, px)
    assert not torch.isnan(got).any()
    assert rel_err(got.numpy(), w.grad.numpy()) < 1e-6


def _s2d(images):
    """lt_stem_s2d_fwd's layout in float32: (N, 3, H, W) -> (N, 1, H/2, W/2, 32), channel (r 2 + s) 3 + c = img[c][2y + r][2x + s]."""
    N, C, H, W = images.shape
    out = torch.zeros(N, 1, H // 2, W // 2, 32, dtype=torch.float32)
    for r in (0, 1):
        for s in (0, 1):
            c0 = (r * 2 + s) * C
            out[:, 0, :, :, c0:c0 + C] = images[:, :, r::2, s::2].permute(0, 2, 3, 1).float()
    return out


@pytest.mark.parametrize("hw", [(16, 12), (22, 18)])
def test_wgrad_host_mapping_stem_s2d(hw):
    """The 4x4 stride-1 conv over the space-to-depth input (Cin 32, 12 real) mapped back to the (64, 3, 7, 7) stem filter."""
    H, W = hw
    N, cout = 2, 64
    torch.manual_seed(H)
    img = torch.randn(N, 3, H, W, dtype=torch.float64)
    w = torch.randn(cout, 3, 7, 7, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(img.float().double(), w, None, 2, 3)
    gy = torch.randn_like(y).float().double()
    y.backward(gy)
    d = A.stem_wgrad_desc(N, H, W, cout)
    assert (d.OH, d.OW) == tuple(y.shape[2:])
    gs = torch.empty(16, 12, cout, dtype=torch.float32)
    capi.conv_wgrad_host(d, _s2d(img), _cl_padded(gy, d.FC), 12, cout, gs)
    idx = A.stem_wgrad_index("cpu")
    assert sorted(idx.tolist()) == sorted(set(idx.tolist())) and len(idx) == 147
    got = gs.reshape(16 * 12, cout)[idx].t().reshape(cout, 3, 7, 7)
    assert rel_err(got.numpy(), w.grad.numpy()) < 1e-6


def _stem_s2d_filter_host(w):
    """The stem rearrangement as the engine did it before on the host: (64, 3, 7, 7) -> [4][4][32][64]."""
    w = w.detach().float().cpu()
    cout = w.shape[0]
    wt = torch.zeros((4, 4, 32, cout), dtype=torch.float32)
    for ai, a in enumerate(range(-2, 2)):
        for bi, b in enumerate(range(-2, 2)):
            for r in (0, 1):
                for s in (0, 1):
                    ky, kx = 2 * a + r + 3, 2 * b + s + 3
                    if 0 <= ky < 7 and 0 <= kx < 7:
                        c0 = (r * 2 + s) * 3
                        wt[ai, bi, c0:c0 + 3] = w[:, :, ky, kx].t()
    return wt


def test_device_stem_gather_matches_host_rearrangement():
    torch.manual_seed(0)
    w = torch.randn(64, 3, 7, 7)
    w[0, 0, 0, 0] = -0.0
    got = engine.stem_s2d_filter(w)
    ref = _stem_s2d_filter_host(w)
    assert got.shape == ref.shape and got.dtype == ref.dtype
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))     # bit for bit


def test_backbone_conv_rejects_unsupported_modules():
    x = torch.zeros(1, 64, 8, 8)
    for m in (nn.Conv2d(64, 64, 3, 1, 1, groups=2), nn.Conv2d(64, 64, 3, 1, 2, dilation=2), nn.Conv2d(64, 64, 3, 3, 1),
              nn.Conv2d(64, 64, 3, 1, 0), nn.Conv2d(64, 64, 2, 1, 1), nn.Conv2d(64, 64, 5, 2, 2), nn.Conv2d(64, 64, 3, (2, 1), 1),
              nn.Conv2d(64, 64, 3, 1, "same"), nn.Conv2d(64, 64, 7, 2, 3), nn.Conv2d(64, 64, 3, 1, 1, padding_mode="reflect"),
              nn.Conv2d(64, 64, 3, 2, 1, padding_mode="circular"),
              nn.ConvTranspose2d(64, 64, 2, 2, 0), nn.ConvTranspose2d(64, 64, 4, 2, 1, 1), nn.ConvTranspose2d(64, 64, 4, 1, 1),
              nn.Conv3d(64, 64, 3, 1, 1)):
        with pytest.raises(ValueError):
            A.backbone_conv(m, x)
    with pytest.raises(ValueError):     # grouped data gradient: Cin a multiple of 32
        A.backbone_conv(nn.Conv2d(48, 64, 3, 2, 1), torch.zeros(1, 48, 8, 8))
    img = torch.zeros(1, 3, 16, 16, requires_grad=True)
    with pytest.raises(ValueError, match="image gradients"):
        A.backbone_conv(nn.Conv2d(3, 64, 7, 2, 3, bias=False), img)
    with pytest.raises(ValueError):
        A.backbone_conv(nn.Conv2d(3, 64, 7, 2, 3, bias=False), torch.zeros(1, 3, 15, 16))


def test_backbone_conv_needs_cuda_tensors():
    for m, x in ((nn.Conv2d(64, 64, 3, 1, 1), torch.zeros(1, 64, 8, 8)), (nn.Conv2d(64, 64, 3, 2, 1), torch.zeros(1, 64, 8, 8)),
                 (nn.Conv2d(64, 128, 1, 2, 0), torch.zeros(1, 64, 8, 8)), (nn.ConvTranspose2d(64, 32, 4, 2, 1), torch.zeros(1, 64, 4, 4)),
                 (nn.Conv2d(3, 64, 7, 2, 3), torch.zeros(1, 3, 16, 16))):
        with pytest.raises(RuntimeError):
            A.backbone_conv(m, x)


@pytest.mark.parametrize("style,layers", [("simple", 18), ("simple", 50), ("caffe", 50)])
def test_conv_hook_reaches_every_convolution(style, layers):
    """PoseResNet.forward with a pass-through `conv` hook: the same outputs as without one, and every Conv2d / ConvTranspose2d of
    the backbone and its confidence heads goes through the hook exactly once."""
    from lt_b200 import pose_resnet, testing
    cfg = testing.make_config(num_layers=layers, style=style).model.backbone
    cfg.alg_confidences = cfg.vol_confidences = True
    torch.manual_seed(layers)
    net = pose_resnet.get_pose_net(cfg, device="cpu").eval()
    seen = []

    def hook(m, x):
        seen.append(m)
        return m(x)
    x = torch.randn(1, 3, 128, 128)
    with torch.no_grad():
        ref = net(x)
        got = net(x, hook)
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    convs = [m for m in net.modules() if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d))]
    assert len(seen) == len(convs) and {id(m) for m in seen} == {id(m) for m in convs}


def test_backbone_backend_option_is_checked():
    from lt_b200 import testing, AlgebraicTriangulationNet, VolumetricTriangulationNet
    for cls in (VolumetricTriangulationNet, AlgebraicTriangulationNet):
        def cfg():
            c = testing.make_config(num_layers=18, volume_size=32)
            c.model.use_confidences = True
            return c
        with pytest.raises(ValueError, match="backbone_backend='native' needs backend='hybrid' and conv_mode='tc'"):
            cls(cfg(), device="cpu", backend="torch", backbone_backend="native")
        with pytest.raises(ValueError, match="backbone_backend='native' needs backend='hybrid' and conv_mode='tc'"):
            cls(cfg(), device="cpu", backend="hybrid", conv_mode="simt", backbone_backend="native")
        with pytest.raises(ValueError, match="backbone_backend='native' needs"):
            cls(cfg(), device="cpu", backend="native", backbone_backend="native")
        with pytest.raises(ValueError, match="unknown backbone_backend"):
            cls(cfg(), device="cpu", backend="hybrid", backbone_backend="cudnn")
        m = cls(cfg(), device="cpu", backend="hybrid", backbone_backend="native")
        ref = cls(cfg(), device="cpu", backend="hybrid")
        assert m.backbone_backend == "native" and ref.backbone_backend == "torch"
        assert list(m.state_dict().keys()) == list(ref.state_dict().keys())
        assert [n for n, _ in m.named_modules()] == [n for n, _ in ref.named_modules()]
    m = VolumetricTriangulationNet(testing.make_config(num_layers=18, volume_size=32), device="cpu", backend="hybrid",
                                   backbone_backend="native", v2v_backend="native")
    assert (m.backbone_backend, m.v2v_backend) == ("native", "native")
