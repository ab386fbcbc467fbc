"""CPU checks of the native V2V training convolutions (autograd_ops.ConvNdFn / ConvTranspose3dFn), no GPU needed:
the filter re-gather that turns each data gradient into a forward convolution, and the weight-gradient kernel's index mapping
(lt_test_conv_wgrad_host), both against torch autograd in float64."""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lt_b200 import autograd_ops as A
from lt_b200 import capi

# (cin, cout, k, (D, H, W), N): every Conv3d shape of the V2V net (v2v.py) at small grids
CONV_CASES = [
    (32, 16, 7, (9, 8, 10), 2),     # front_layers[0]
    (16, 32, 3, (8, 9, 8), 2),      # Res3DBlock(16, 32): 16 input channels padded to 32
    (16, 32, 1, (8, 8, 9), 2),      # its 1x1x1 skip
    (32, 32, 3, (8, 8, 8), 2),
    (32, 64, 3, (5, 6, 4), 2),
    (64, 64, 3, (4, 4, 5), 2),
    (64, 128, 3, (3, 4, 4), 2),
    (128, 128, 3, (2, 3, 2), 2),
    (32, 64, 1, (4, 4, 4), 2),
    (32, 17, 1, (8, 8, 8), 2),      # output_layer: 17 output channels padded to 32
]
DECONV_CASES = [(128, 128, (2, 3, 2), 2), (128, 64, (3, 2, 4), 2), (64, 32, (4, 4, 3), 2)]


def _gather(w, base, strides, k, cin, cout):
    """torch emulation of lt_conv_gather_weights_fwd (include/lt_b200.h): element (td, th, tw, ci, co) of the canonical filter is
    w.flatten()[base + td s_td + th s_th + tw s_tw + ci s_ci + co s_co]; returned as a (cout, cin, kd, kh, kw) Conv3d filter."""
    flat = w.reshape(-1)
    td, th, tw, ci, co = torch.meshgrid(*[torch.arange(n) for n in (k[0], k[1], k[2], cin, cout)], indexing="ij")
    idx = base + td * strides[0] + th * strides[1] + tw * strides[2] + ci * strides[3] + co * strides[4]
    assert int(idx.min()) >= 0 and int(idx.max()) < flat.numel()
    return flat[idx].permute(4, 3, 0, 1, 2)


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv3d_dgrad_regather_reproduces_autograd(case):
    cin, cout, k, dims, N = case
    torch.manual_seed(cin + cout + k)
    x = torch.randn(N, cin, *dims, dtype=torch.float64, requires_grad=True)
    w = torch.randn(cout, cin, k, k, k, dtype=torch.float64)
    gy = torch.randn(N, cout, *dims, dtype=torch.float64)
    F.conv3d(x, w, None, 1, k // 2).backward(gy)
    (base, strides), kk, stride, pad, ci, co = A.conv3d_dgrad_filter(w.shape, (k // 2,) * 3)
    assert (ci, co) == (cout, cin)
    wd = _gather(w, base, strides, kk, ci, co)
    got = F.conv3d(gy, wd, None, stride, pad)
    assert rel_err(got.numpy(), x.grad.numpy()) < 1e-12


@pytest.mark.parametrize("case", DECONV_CASES)
def test_conv_transpose3d_dgrad_regather_reproduces_autograd(case):
    cin, cout, dims, N = case
    torch.manual_seed(cin + cout)
    x = torch.randn(N, cin, *dims, dtype=torch.float64, requires_grad=True)
    w = torch.randn(cin, cout, 2, 2, 2, dtype=torch.float64)
    gy = torch.randn(N, cout, *[2 * d for d in dims], dtype=torch.float64)
    F.conv_transpose3d(x, w, None, 2).backward(gy)
    (base, strides), k, stride, pad, ci, co = A.conv_transpose3d_dgrad_filter(w.shape)
    wd = _gather(w, base, strides, k, ci, co)
    got = F.conv3d(gy, wd, None, stride, pad)
    assert rel_err(got.numpy(), x.grad.numpy()) < 1e-12


def _cl_padded(t, cp):
    """(N, C, D, H, W) -> float32 channels-last (N, D, H, W, cp), channels C .. cp-1 zero."""
    out = torch.zeros(t.shape[0], *t.shape[2:], cp, dtype=torch.float32)
    out[..., :t.shape[1]] = t.permute(0, 2, 3, 4, 1).float()
    return out.contiguous()


@pytest.mark.parametrize("case", CONV_CASES)
def test_wgrad_host_mapping_conv3d(case):
    cin, cout, k, dims, N = case
    torch.manual_seed(7 + cin + cout + k)
    x = torch.randn(N, cin, *dims, dtype=torch.float64)
    w = torch.randn(cout, cin, k, k, k, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(N, cout, *dims, dtype=torch.float64)
    x32, gy32 = x.float().double(), gy.float().double()
    F.conv3d(x32, w, None, 1, k // 2).backward(gy32)
    d = A.conv3d_wgrad_desc(N, dims, cin, cout, (k, k, k), (k // 2,) * 3)
    gw = torch.empty(k ** 3, cin, cout, dtype=torch.float32)
    capi.conv_wgrad_host(d, _cl_padded(x, d.Cin), _cl_padded(gy, d.FC), cin, cout, gw)
    got = gw.reshape(k, k, k, cin, cout).permute(4, 3, 0, 1, 2)
    assert rel_err(got.numpy(), w.grad.numpy()) < 1e-6


@pytest.mark.parametrize("case", DECONV_CASES)
def test_wgrad_host_mapping_grouped_conv_transpose3d(case):
    cin, cout, dims, N = case
    torch.manual_seed(11 + cin + cout)
    x = torch.randn(N, cin, *dims, dtype=torch.float64)
    w = torch.randn(cin, cout, 2, 2, 2, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(N, cout, *[2 * s for s in dims], dtype=torch.float64)
    F.conv_transpose3d(x.float().double(), w, None, 2).backward(gy.float().double())
    d = A.conv_transpose3d_desc(N, dims, cin, cout)
    gw = torch.empty(1, cin, 8 * cout, dtype=torch.float32)
    capi.conv_wgrad_host(d, _cl_padded(x, cin), _cl_padded(gy, cout), cin, cout, gw)
    got = gw.reshape(cin, 8, cout).permute(0, 2, 1).reshape(cin, cout, 2, 2, 2)
    assert rel_err(got.numpy(), w.grad.numpy()) < 1e-6


def test_wgrad_rejects_bad_descriptors():
    d = A.conv3d_wgrad_desc(1, (4, 4, 4), 32, 32, (3, 3, 3), (1, 1, 1))
    d.in_format = capi.FMT_F32
    with pytest.raises(RuntimeError, match="split-fp16"):
        capi.conv_wgrad_host(d, torch.zeros(64, 32), torch.zeros(64, 32), 32, 32, torch.zeros(27, 32, 32))
    d = A.conv3d_wgrad_desc(1, (4, 4, 4), 32, 32, (3, 3, 3), (1, 1, 1))
    with pytest.raises(RuntimeError, match="channel counts"):
        capi.conv_wgrad_host(d, torch.zeros(64, 32), torch.zeros(64, 32), 33, 32, torch.zeros(27, 33, 32))


def test_v2v_backend_option_is_checked():
    from lt_b200 import testing, VolumetricTriangulationNet
    cfg = testing.make_config(num_layers=18, volume_size=32)
    with pytest.raises(ValueError):
        VolumetricTriangulationNet(cfg, device="cpu", backend="torch", v2v_backend="native")
    with pytest.raises(ValueError):
        VolumetricTriangulationNet(cfg, device="cpu", backend="hybrid", conv_mode="simt", v2v_backend="native")
    with pytest.raises(ValueError):
        VolumetricTriangulationNet(cfg, device="cpu", backend="hybrid", v2v_backend="cudnn")
    m = VolumetricTriangulationNet(cfg, device="cpu", backend="hybrid", v2v_backend="native")
    ref = VolumetricTriangulationNet(cfg, device="cpu", backend="hybrid")
    assert list(m.state_dict().keys()) == list(ref.state_dict().keys())
    with pytest.raises(RuntimeError):
        A.conv3d(torch.zeros(1, 32, 4, 4, 4), torch.zeros(32, 32, 3, 3, 3), None, (1, 1, 1))
