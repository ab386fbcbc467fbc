"""Training the algebraic model on `backend="hybrid"`: gradient parity of the native 2-D soft-argmax backward (mode 2 of
lt_softargmax3d_bwd for the ReLU branch) and of the DLT backward (lt_triangulate_dlt_bwd) against torch autograd of the torch
formulation (`torch_ops`), and one training step of AlgebraicTriangulationNet against `backend="torch"`.  Bounds as in
tests/test_gpu_hybrid.py."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import multiview, op, testing

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _scale(t):
    return float(max(t.abs().max(), t.std()))


def _dlt_scene(B, V, J, seed):
    rng = np.random.RandomState(seed)
    cams = testing.make_cameras(V, image_size=384)
    P = np.repeat(np.stack([c.projection for c in cams]).astype(np.float32)[None], B, axis=0)
    X = rng.randn(B, J, 3) * 300 + [0, 0, 900]
    uvw = np.einsum("bvij,bkj->bvki", P.astype(np.float64), np.concatenate([X, np.ones((B, J, 1))], -1))
    kp = (uvw[..., :2] / uvw[..., 2:3] + rng.randn(B, V, J, 2) * 2.0).astype(np.float32)
    conf = (rng.rand(B, V, J) + 0.1).astype(np.float32)
    g = rng.randn(B, J, 3).astype(np.float32)
    return [torch.from_numpy(a).to(DEV) for a in (P, kp, conf, g)]


@pytest.mark.parametrize("V", [2, 4])
@pytest.mark.parametrize("with_conf", [True, False])
def test_triangulate_backward_vs_torch_autograd(V, with_conf):
    P, kp, conf, g = _dlt_scene(8, V, 17, seed=20 + V)
    res = []
    for backend in ("torch", "hybrid"):
        k = kp.clone().requires_grad_(True)
        c = conf.clone().requires_grad_(True) if with_conf else None
        out = multiview.triangulate_batch_of_points(P, k, c, backend=backend)
        (out * g).sum().backward()
        res.append((out.detach(), k.grad, None if c is None else c.grad))
    (o0, gk0, gc0), (o1, gk1, gc1) = res
    assert float((o0 - o1).abs().max()) <= 3e-5 * _scale(o0)
    assert float((gk0 - gk1).abs().max()) <= 1e-4 * _scale(gk0)
    if with_conf:
        assert float((gc0 - gc1).abs().max()) <= 1e-4 * _scale(gc0)


def test_hybrid_triangulation_is_part_of_the_autograd_graph():
    P, kp, conf, _ = _dlt_scene(2, 3, 5, seed=1)
    k, c = kp.clone().requires_grad_(True), conf.clone().requires_grad_(True)
    out = multiview.triangulate_batch_of_points(P, k, c, backend="hybrid")
    assert out.grad_fn is not None and out.shape == (2, 5, 3)
    out.sum().backward()
    assert k.grad is not None and c.grad is not None and bool(torch.isfinite(k.grad).all())


@pytest.mark.parametrize("softmax", [True, False])
def test_integrate_2d_backward_vs_torch_autograd(softmax):
    torch.manual_seed(4)
    B, J, h, w = 4, 17, 24, 20
    logits = torch.randn(B, J, h, w, device=DEV) * 3
    g_kp, g_heat = torch.randn(B, J, 2, device=DEV), torch.randn(B, J, h, w, device=DEV)
    res = []
    for backend in ("torch", "hybrid"):
        l = logits.clone().requires_grad_(True)
        kp, heat = op.integrate_tensor_2d(l, softmax, backend=backend)
        ((kp * g_kp).sum() + (heat * g_heat).sum()).backward()
        res.append((kp.detach(), heat.detach(), l.grad))
    (k0, h0, g0), (k1, h1, g1) = res
    assert k1.shape == (B, J, 2) and h1.shape == (B, J, h, w)
    assert float((k0 - k1).abs().max()) <= 3e-5 * _scale(k0)
    assert float((h0 - h1).abs().max()) <= 3e-5 * _scale(h0)
    assert float((g0 - g1).abs().max()) <= 1e-4 * _scale(g0)


def test_hybrid_algebraic_eval_forward_without_grad_matches_torch_backend():
    B, V, S = 1, 2, 128
    images, batch = testing.make_batch(B, V, image_size=S, seed=5)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    holder = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=6, calib_size=S)
    outs = []
    for backend in ("torch", "hybrid"):
        m = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18), device="cpu", backend=backend)
        m.load_state_dict(holder.state_dict())
        m = m.to(DEV).eval()
        with torch.no_grad():
            outs.append(m(images.to(DEV), proj, batch))
    assert len(outs[1]) == 4
    for a, b in zip(*outs):
        assert a.shape == b.shape and b.grad_fn is None
    kp3d0, kp2d0, heat0, conf0 = outs[0]
    kp3d1, kp2d1, heat1, conf1 = outs[1]
    assert float((heat0 - heat1).abs().max()) <= 3e-5 * _scale(heat0)
    assert float((kp2d0 - kp2d1).abs().max()) <= 3e-5 * _scale(kp2d0)
    assert torch.equal(conf0, conf1)                 # torch on both backends
    assert float((kp3d0 - kp3d1).abs().max()) <= 1e-3 * _scale(kp3d0)


def _masked_mae(pred, target, validity):
    """KeypointsMAELoss of the reference (mvn/models/loss.py): sum |gt - pred| * validity / (3 * max(1, sum validity))."""
    return (torch.abs(target - pred) * validity).sum() / (3 * max(1.0, float(validity.sum())))


@pytest.mark.parametrize("use_confidences", [True, False])
@pytest.mark.parametrize("heatmap_softmax", [True, False])
def test_hybrid_algebraic_training_step_matches_torch_backend(use_confidences, heatmap_softmax):
    B, V, S, J = 2, 3, 128, 17
    images, batch = testing.make_batch(B, V, image_size=S, seed=11)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    g = torch.Generator().manual_seed(12)
    target = (torch.from_numpy(np.stack([k[:, :3] for k in batch["keypoints_3d"]])).float()
              + torch.randn(B, J, 3, generator=g) * 50).to(DEV)
    validity = (torch.rand(B, J, 1, generator=g) > 0.2).float().to(DEV)

    def config():
        cfg = testing.make_alg_config(num_layers=18, use_confidences=use_confidences)
        cfg.model.heatmap_softmax = heatmap_softmax
        return cfg

    holder = lt_b200.AlgebraicTriangulationNet(config(), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
    sd = holder.state_dict()
    losses, grads = [], []
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for backend in ("torch", "hybrid"):
            m = lt_b200.AlgebraicTriangulationNet(config(), device="cpu", backend=backend)
            m.load_state_dict(sd)
            m = m.to(DEV).train()                 # batch-statistics BatchNorm; the algebraic forward has no randomness
            kp3d, kp2d, heat, conf = m(images.to(DEV), proj, batch)
            assert kp3d.shape == (B, J, 3) and kp2d.shape == (B, V, J, 2) and heat.shape[:3] == (B, V, J) and conf.shape == (B, V, J)
            loss = _masked_mae(kp3d, target, validity)
            loss.backward()
            losses.append(float(loss.detach()))
            gr = [m.backbone.final_layer.weight.grad.clone()]
            if use_confidences:
                gr.append(m.backbone.alg_confidences.head[0].weight.grad.clone())
            grads.append(gr)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    errs = [float((a - b).abs().max()) / float(a.abs().max()) for a, b in zip(*grads)]
    print("alg hybrid vs torch (conf=%s, softmax=%s): loss %.3e rel, gradients %s rel"
          % (use_confidences, heatmap_softmax, abs(losses[0] - losses[1]) / abs(losses[0]), ["%.2e" % e for e in errs]))
    # measured on an H100: loss within 7e-8, gradients within 3e-6 (relative).  Both backends run the same torch backbone, so
    # only the custom ops differ; the bounds keep a 30x margin and stay below the volumetric module test's (3e-3, 3e-2)
    assert np.isfinite(losses).all()
    assert abs(losses[0] - losses[1]) <= 1e-5 * abs(losses[0])
    for e in errs:
        assert e <= 1e-4
