"""Gradient parity of the native custom-op backward kernels (`backend="hybrid"`, csrc/backward.cu) against torch autograd of
the torch formulation (`torch_ops`, itself pinned to the reference in tests/test_oracle_vs_reference.py).

Part of the default GPU suite since round 2 (first run: 14 of 15 green, the one failure was the test's own 16^3 grid
being too small for the five pooling levels of V2V)."""
import os

import numpy as np
import pytest
import torch

from lt_b200 import op, testing, torch_ops
from oracle import vol_oracle as O

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scene(B, V, C, h, w, n, seed):
    rng = np.random.RandomState(seed)
    heat = rng.randn(B, V, C, h, w).astype(np.float32)
    cams = testing.make_cameras(V, image_size=48, radius=3000.0)
    proj = np.stack([np.stack([O.projection_after_resize(c.K, c.R, c.t, (48, 48), (h, w)) for c in cams])] * B)
    coord = np.stack([O.coord_volume(rng.randn(3) * 100 + [0, 0, 900], 2800.0, n) for _ in range(B)])
    conf = rng.rand(B, V, C).astype(np.float32)
    return [torch.from_numpy(a).to(DEV) for a in (heat, proj, coord, conf)]


@pytest.mark.parametrize("shape", [(2, 4, 32, 12, 12, 8), (1, 3, 8, 9, 13, 6), (1, 9, 32, 8, 8, 5)])
@pytest.mark.parametrize("agg", ["sum", "softmax", "conf", "max"])
def test_unproject_backward_vs_torch_autograd(shape, agg):
    heat, proj, coord, conf = _scene(*shape, seed=sum(shape))
    g = torch.randn(shape[0], shape[2], shape[5], shape[5], shape[5], device=DEV)
    grads = []
    for backend in ("torch", "hybrid"):
        h_ = heat.clone().requires_grad_(True)
        c_ = conf.clone().requires_grad_(True)
        out = op.unproject_heatmaps(h_, proj, coord, agg, c_, backend=backend)
        out.backward(g)
        grads.append((out.detach(), h_.grad, c_.grad if agg == "conf" else None))
    (o0, gh0, gc0), (o1, gh1, gc1) = grads
    scale = lambda t: float(max(t.abs().max(), t.std()))
    assert float((o0 - o1).abs().max()) <= 3e-5 * scale(o0)
    assert float((gh0 - gh1).abs().max()) <= 1e-4 * scale(gh0)
    if agg == "conf":
        assert float((gc0 - gc1).abs().max()) <= 1e-4 * scale(gc0)


@pytest.mark.parametrize("softmax", [True, False])
def test_softargmax_backward_vs_torch_autograd(softmax):
    torch.manual_seed(3)
    B, J, n = 2, 17, 12
    vols = (torch.randn(B, J, n, n, n, device=DEV) * 3)
    coord = torch.randn(B, n, n, n, 3, device=DEV) * 700
    g_kp = torch.randn(B, J, 3, device=DEV)
    g_vol = torch.randn(B, J, n, n, n, device=DEV)
    grads = []
    for backend in ("torch", "hybrid"):
        v_ = vols.clone().requires_grad_(True)
        kp, p = op.integrate_tensor_3d_with_coordinates(v_, coord, softmax, backend=backend)
        ((kp * g_kp).sum() + (p * g_vol).sum()).backward()
        grads.append(v_.grad)
    scale = float(max(grads[0].abs().max(), grads[0].std()))
    assert float((grads[0] - grads[1]).abs().max()) <= 1e-4 * scale


def test_hybrid_module_training_step_matches_torch_backend():
    import lt_b200
    cfg = testing.make_config(num_layers=18, volume_size=32)   # V2V pools five times: 32 is the smallest grid
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    losses, grads = [], []
    # both backends run their convolutions through torch: in full fp32, so that TF32 rounding of cuDNN is not part of the comparison
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for backend in ("torch", "hybrid"):
            torch.manual_seed(0)
            m = lt_b200.VolumetricTriangulationNet(cfg, device=DEV, backend=backend).to(DEV).train()
            testing.randomize_weights(m, seed=0, calib_size=64, calib_views=1)
            m = m.to(DEV).eval()     # eval-mode BN / no random rotation: deterministic forward, gradients still flow
            kp = m(images.to(DEV), None, batch)[0]
            loss = (kp ** 2).mean()
            loss.backward()
            losses.append(float(loss.detach()))
            grads.append(m.process_features[0].weight.grad.clone())
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    # the native forward uses reciprocal / exp2 approximations (3e-5 on the unprojected volume); a randomly initialised V2V
    # amplifies that
    assert abs(losses[0] - losses[1]) <= 3e-3 * abs(losses[0])
    assert float((grads[0] - grads[1]).abs().max()) <= 3e-2 * float(grads[0].abs().max())
