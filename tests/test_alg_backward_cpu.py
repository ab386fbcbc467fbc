"""Backward of the algebraic model's custom ops (`backend="hybrid"`) checked on the CPU.

- The DLT backward (csrc/algebraic.cu) and mode 2 of the soft-argmax backward (csrc/backward.cu) through their test hooks,
  which run the kernels' own per-item code (`__host__ __device__`) on host pointers, against torch autograd of the torch
  formulation (`torch_ops`, pinned to the reference).
- The autograd wrappers (autograd_ops.IntegrateTensor2dFn, TriangulateDltFn) with torch stand-ins for the C calls.
- Error paths that need no GPU.
The CUDA launches themselves are covered by tests/test_gpu_alg_hybrid.py."""
import ctypes

import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import autograd_ops, capi, testing, torch_ops


def _dlt_scene(B, V, J, seed):
    """Cameras on a ring, points around (0, 0, 900) mm, their projections with 2 px of noise, confidences in [0.1, 1.1)."""
    rng = np.random.RandomState(seed)
    cams = testing.make_cameras(V, image_size=384)
    P = np.repeat(np.stack([c.projection for c in cams]).astype(np.float32)[None], B, axis=0)       # (B, V, 3, 4)
    X = rng.randn(B, J, 3) * 300 + [0, 0, 900]
    Xh = np.concatenate([X, np.ones((B, J, 1))], -1)
    uvw = np.einsum("bvij,bkj->bvki", P.astype(np.float64), Xh)
    kp = (uvw[..., :2] / uvw[..., 2:3] + rng.randn(B, V, J, 2) * 2.0).astype(np.float32)
    conf = (rng.rand(B, V, J) + 0.1).astype(np.float32)
    g = rng.randn(B, J, 3).astype(np.float32)
    return [torch.from_numpy(a) for a in (P, kp, conf, g)]


@pytest.mark.parametrize("V", [2, 4, 5])
@pytest.mark.parametrize("with_conf", [True, False])
def test_dlt_backward_item_code_vs_torch_autograd(V, with_conf):
    B, J = 3, 17
    P, kp, conf, g = _dlt_scene(B, V, J, seed=10 + V)
    k = kp.clone().requires_grad_(True)
    c = conf.clone().requires_grad_(True) if with_conf else None
    out = torch_ops.triangulate_batch_of_points(P, k, c)
    (out * g).sum().backward()
    grad_kp = torch.full_like(kp, float("nan"))             # the hook writes every element
    grad_conf = torch.full_like(conf, float("nan")) if with_conf else None
    capi.triangulate_dlt_bwd_host(P, kp, conf if with_conf else None, g, grad_kp, grad_conf)
    assert float((grad_kp - k.grad).abs().max()) <= 1e-4 * float(k.grad.abs().max())
    if with_conf:
        assert float((grad_conf - c.grad).abs().max()) <= 1e-4 * float(c.grad.abs().max())


def test_dlt_backward_is_finite_on_a_tied_eigenvalue():
    """All confidences zero: A^T A = 0, every eigenvalue ties with the smallest.  The tied terms are dropped, so the gradient
    is zero rather than non-finite."""
    P, kp, conf, g = _dlt_scene(1, 3, 2, seed=3)
    grad_kp, grad_conf = torch.empty_like(kp), torch.empty_like(conf)
    capi.triangulate_dlt_bwd_host(P, kp, torch.zeros_like(conf), g, grad_kp, grad_conf)
    assert torch.isfinite(grad_kp).all() and torch.isfinite(grad_conf).all()


def _pixel_grid(B, h, w):
    ys, xs = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    return torch.stack([xs, ys, torch.zeros_like(xs)], -1).reshape(1, h * w, 3).expand(B, h * w, 3).contiguous()


@pytest.mark.parametrize("hw", [(7, 11), (12, 9)])
@pytest.mark.parametrize("softmax", [True, False])
@pytest.mark.parametrize("with_gheat", [True, False])
def test_softargmax2d_backward_item_code_vs_torch_autograd(hw, softmax, with_gheat):
    """Mode 1 (softmax) and mode 2 (ReLU, mass-normalised) of the soft-argmax backward on a pixel grid (x, y, 0)."""
    torch.manual_seed(7)
    B, J = 2, 5
    h, w = hw
    mult = 1.7
    logits = torch.randn(B, J, h, w) * 2
    g_kp, g_heat = torch.randn(B, J, 2), torch.randn(B, J, h, w)
    l = logits.clone().requires_grad_(True)
    kp, heat = torch_ops.integrate_tensor_2d(l * mult, softmax)
    loss = (kp * g_kp).sum() + ((heat * g_heat).sum() if with_gheat else 0.0)
    loss.backward()
    g3 = torch.cat([g_kp, torch.zeros(B, J, 1)], -1).contiguous()
    grad = torch.full((B, J, h * w), float("nan"))
    capi.softargmax3d_bwd_host(heat.detach().reshape(B, J, h * w).contiguous(), _pixel_grid(B, h, w), g3,
                               g_heat.reshape(B, J, h * w).contiguous() if with_gheat else None, grad, B, J, h * w, mult,
                               1 if softmax else 2)
    want = l.grad.reshape(B, J, h * w)
    assert float((grad - want).abs().max()) <= 1e-4 * float(want.abs().max())


# ---- wrapper plumbing with torch stand-ins for the C calls ------------------------------------------------------------

def _fake_softargmax(logits, bs, vs, cs, coord, out, kp, ws, B, J, nvox, mult, mode):
    assert mode in (1, 2)
    flat = logits.reshape(B, J, nvox) * mult
    p = torch.softmax(flat, -1) if mode == 1 else torch.relu(flat)
    k = p @ coord
    if mode == 2:
        k = k / p.sum(-1, keepdim=True)
    kp.copy_(k)
    out.copy_(p.view_as(out))


def _fake_softargmax_bwd(probs, coord, g_kp, g_vol, grad_logits, scratch, B, J, nvox, mult, mode):
    assert mode in (1, 2) and scratch.numel() >= mode * B * J
    p = probs.reshape(B, J, nvox)
    tk = torch.einsum("bjc,bnc->bjn", g_kp, coord)
    gv = torch.zeros_like(p) if g_vol is None else g_vol.reshape(B, J, nvox)
    if mode == 1:
        t = tk + gv
        g = mult * p * (t - (p * t).sum(-1, keepdim=True))
    else:
        M = p.sum(-1, keepdim=True)
        S = (p * tk).sum(-1, keepdim=True) / M
        g = mult * (p > 0) * (gv + (tk - S) / M)
    grad_logits.copy_(g.view_as(grad_logits))


def _fake_triangulate(proj, kp2d, conf, out):
    out.copy_(torch_ops.triangulate_batch_of_points(proj, kp2d, conf))


CALLS = []


def _fake_triangulate_bwd(proj, kp2d, conf, grad_out, grad_kp2d, grad_conf):
    CALLS.append(grad_conf is None)
    k = kp2d.clone().requires_grad_(True)
    c = None if conf is None else conf.clone().requires_grad_(grad_conf is not None)
    with torch.enable_grad():
        torch_ops.triangulate_batch_of_points(proj, k, c).backward(grad_out)
    grad_kp2d.copy_(k.grad)                      # write (not accumulate) contract of lt_triangulate_dlt_bwd
    if grad_conf is not None:
        grad_conf.copy_(c.grad)


@pytest.fixture
def fake_capi(monkeypatch):
    monkeypatch.setattr(capi, "softargmax3d", _fake_softargmax)
    monkeypatch.setattr(capi, "softargmax3d_bwd", _fake_softargmax_bwd)
    monkeypatch.setattr(capi, "softargmax3d_workspace_bytes", lambda B, J, nvox: 64)
    monkeypatch.setattr(capi, "triangulate_dlt", _fake_triangulate)
    monkeypatch.setattr(capi, "triangulate_dlt_bwd", _fake_triangulate_bwd)
    CALLS.clear()


@pytest.mark.parametrize("softmax", [True, False])
def test_integrate_2d_wrapper_gradients(fake_capi, softmax):
    torch.manual_seed(2)
    B, J, h, w = 3, 4, 6, 9
    logits = torch.randn(B, J, h, w) * 2
    g_kp, g_heat = torch.randn(B, J, 2), torch.randn(B, J, h, w)
    res = []
    for fn in (torch_ops.integrate_tensor_2d, autograd_ops.integrate_tensor_2d):
        l = logits.clone().requires_grad_(True)
        kp, heat = fn(l, softmax)
        ((kp * g_kp).sum() + (heat * g_heat).sum()).backward()
        res.append((kp.detach(), heat.detach(), l.grad))
    assert res[1][0].shape == (B, J, 2) and res[1][1].shape == (B, J, h, w)
    for a, b in zip(res[0], res[1]):
        assert torch.allclose(a, b, atol=1e-4, rtol=1e-4)
    # key-points-only loss: the heat-map gradient slot arrives as None
    grads = []
    for fn in (torch_ops.integrate_tensor_2d, autograd_ops.integrate_tensor_2d):
        l = logits.clone().requires_grad_(True)
        (fn(l, softmax)[0] * g_kp).sum().backward()
        grads.append(l.grad)
    assert torch.allclose(grads[0], grads[1], atol=1e-4, rtol=1e-4)


@pytest.mark.parametrize("with_conf", [True, False])
def test_triangulate_wrapper_gradients(fake_capi, with_conf):
    P, kp, conf, g = _dlt_scene(2, 4, 5, seed=1)
    res = []
    for fn in (torch_ops.triangulate_batch_of_points, autograd_ops.triangulate_batch_of_points):
        k = kp.clone().requires_grad_(True)
        c = conf.clone().requires_grad_(True) if with_conf else None
        out = fn(P, k, c)
        (out * g).sum().backward()
        res.append((out.detach(), k.grad, None if c is None else c.grad))
    assert res[1][0].shape == (2, 5, 3)
    assert torch.allclose(res[0][0], res[1][0], atol=1e-4)
    assert torch.allclose(res[0][1], res[1][1], atol=1e-5, rtol=1e-4)
    if with_conf:
        assert torch.allclose(res[0][2], res[1][2], atol=1e-5, rtol=1e-4)
    assert CALLS == [not with_conf]


def test_triangulate_wrapper_skips_the_confidence_gradient_when_not_needed(fake_capi):
    P, kp, conf, g = _dlt_scene(1, 3, 4, seed=2)
    k = kp.clone().requires_grad_(True)
    (autograd_ops.triangulate_batch_of_points(P, k, conf) * g).sum().backward()
    assert CALLS == [True] and k.grad is not None


# ---- errors -----------------------------------------------------------------------------------------------------------

def test_hybrid_algebraic_model_rejects_cpu_tensors():
    model = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18), device="cpu", backend="hybrid")
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    proj = torch.from_numpy(testing.image_projections(batch))
    with pytest.raises(RuntimeError, match="hybrid backend needs CUDA tensors"):
        model(images, proj, batch)


def test_softargmax_backward_rejects_an_unknown_mode():
    """The argument check runs before anything touches a device: no GPU needed."""
    B, J, n = 1, 2, 8
    buf = torch.zeros(B * J * n * 3)
    p = ctypes.c_void_p(buf.data_ptr())
    lib = capi.lib()
    assert lib.lt_softargmax3d_bwd(p, p, p, None, p, p, B, J, n, 1.0, 3, None) != 0
    assert b"mode" in lib.lt_last_error_string()
    with pytest.raises(RuntimeError, match="mode"):
        capi.softargmax3d_bwd_host(buf[:B * J * n], buf[:B * n * 3], buf[:B * J * 3], None, torch.empty(B * J * n), B, J, n, 1.0, 3)
