"""The volumetric cross-entropy loss on the device (csrc/loss.cu through lt_b200.loss.VolumetricCELoss) against the restatement of the
reference loss (test_volumetric_ce_cpu.oracle_volumetric_ce_loss, pinned to the reference's golden there) run on CUDA, and against
the vectorised torch formulation: indices, loss, sparse gradient, composition with the hybrid soft-argmax, no host
synchronisation, determinism and one training step of the volumetric model."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import autograd_ops, loss as ce, op, testing, torch_ops
from test_volumetric_ce_cpu import oracle_volumetric_ce_loss

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _rotations(B, g):
    q = torch.randn(B, 4, generator=g, dtype=torch.float64)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(B, 3, 3)


def _problem(B, J, grid, seed):
    """Softmaxed volumes on randomly rotated cuboids (2500 mm side); two joints per sample outside the cuboid, one NaN-free point
    per voxel of the rest, validity 0 for about 10 % of the joints."""
    g = torch.Generator().manual_seed(seed)
    X, Y, Z = grid
    axes = [torch.linspace(-1250.0, 1250.0, n, dtype=torch.float64) for n in grid]
    lattice = torch.stack(torch.meshgrid(*axes, indexing="ij"), -1)                          # (X, Y, Z, 3)
    base = torch.randn(B, 3, generator=g, dtype=torch.float64) * 200 + torch.tensor([0.0, 0.0, 900.0], dtype=torch.float64)
    coord = (torch.einsum("xyzc,bdc->bxyzd", lattice, _rotations(B, g)) + base[:, None, None, None]).float()
    kp = (base[:, None] + (torch.rand(B, J, 3, generator=g, dtype=torch.float64) - 0.5) * 2200).float()
    kp[:, :min(J, 2)] += torch.tensor([4000.0, -3000.0, 2500.0])
    logits = torch.randn(B, J, X * Y * Z, generator=g) * 3
    vols = torch.softmax(logits, -1).reshape(B, J, X, Y, Z)
    valid = (torch.rand(B, J, 1, generator=g) > 0.1).float()
    return [t.to(DEV) for t in (coord, vols, kp, valid)]


def _run(fn, coord, vols, kp, valid, scale=1.0):
    v = vols.clone().requires_grad_(True)
    loss = fn(coord, v, kp, valid)
    (loss * scale).backward()
    return loss.detach(), v.grad


def _native(coord, vols, kp, valid):
    return ce.VolumetricCELoss(backend="native")(coord, vols, kp, valid)


def _index(coord, vols, kp, valid):
    B, J = vols.shape[:2]
    return autograd_ops.volumetric_ce_loss(vols.reshape(B, J, -1), coord.reshape(B, -1, 3).contiguous(), kp, valid[..., 0].contiguous())[1]


@pytest.mark.parametrize("B", [1, 5, 8])
@pytest.mark.parametrize("grid", [(64, 64, 64), (32, 32, 32), (20, 24, 28)])
@pytest.mark.parametrize("J", [1, 17, 40])
def test_op_parity_with_the_oracle_and_the_torch_formulation(B, grid, J):
    coord, vols, kp, valid = _problem(B, J, grid, seed=B * 1000 + J + grid[0])
    want_index = torch_ops.volumetric_ce_index(coord, kp)
    index = _index(coord, vols, kp, valid)
    assert torch.equal(index.long(), want_index)
    l_n, g_n = _run(_native, coord, vols, kp, valid, scale=2.5)
    for fn in (oracle_volumetric_ce_loss, torch_ops.volumetric_ce_loss):
        l_w, g_w = _run(fn, coord, vols, kp, valid, scale=2.5)
        assert abs(float(l_n) - float(l_w)) <= 1e-6 * abs(float(l_w))
        gw = g_w.reshape(B, J, -1).gather(2, want_index.unsqueeze(-1))
        gn = g_n.reshape(B, J, -1).gather(2, want_index.unsqueeze(-1))
        assert float((gn - gw).abs().max()) <= 1e-6 * float(gw.abs().max())
        assert int((g_w != 0).sum()) == int((valid[..., 0] != 0).sum())
    rest = g_n.reshape(B, J, -1).scatter(2, want_index.unsqueeze(-1), 0.0)
    assert int(torch.count_nonzero(rest)) == 0


def test_composition_with_the_hybrid_softargmax():
    """Logits -> op.integrate_tensor_3d_with_coordinates(backend="hybrid") -> CE: the logits gradient through the native CE matches
    the one through the torch formulation."""
    B, J, grid = 2, 17, (32, 32, 32)
    coord, _, kp, valid = _problem(B, J, grid, seed=5)
    logits = torch.randn(B, J, *grid, device=DEV, generator=torch.Generator(DEV).manual_seed(1)) * 3
    grads = []
    for fn in (_native, torch_ops.volumetric_ce_loss):
        l_ = logits.clone().requires_grad_(True)
        kp_pred, vols = op.integrate_tensor_3d_with_coordinates(l_, coord, True, backend="hybrid")
        (fn(coord, vols, kp, valid) + 1e-3 * kp_pred.abs().mean()).backward()
        grads.append(l_.grad)
    scale = float(grads[1].abs().max())
    assert float((grads[0] - grads[1]).abs().max()) <= 1e-5 * scale


def test_no_host_synchronisation():
    coord, vols, kp, valid = _problem(5, 17, (64, 64, 64), seed=3)
    _run(_native, coord, vols, kp, valid)                 # load the library, warm the allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _run(_native, coord, vols, kp, valid)
        with pytest.raises(RuntimeError):
            _run(oracle_volumetric_ce_loss, coord, vols, kp, valid)
    finally:
        torch.cuda.set_sync_debug_mode("default")


def test_bit_identical_from_run_to_run():
    coord, vols, kp, valid = _problem(8, 40, (64, 64, 64), seed=9)
    l0, g0 = _run(_native, coord, vols, kp, valid)
    l1, g1 = _run(_native, coord, vols, kp, valid)
    assert torch.equal(l0, l1) and torch.equal(g0, g1)


def test_hybrid_training_step_native_ce_matches_the_oracle_ce():
    """One ResNet-18 volumetric training step on backend="hybrid" with 0.1 * MAE + 0.01 * CE (the recipe's weights): the native CE
    against the oracle CE on the same forward."""
    cfg = testing.make_config(num_layers=18, volume_size=32)
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        torch.manual_seed(0)
        m = lt_b200.VolumetricTriangulationNet(cfg, device=DEV, backend="hybrid").to(DEV).train()
        testing.randomize_weights(m, seed=0, calib_size=64, calib_views=1)
        m = m.to(DEV).eval()
        kp_pred, _, vols, _, _, coord, _ = m(images.to(DEV), None, batch)
        gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
        kp_gt, valid = gt[..., :3], gt[..., 3:]
        mae = (torch.abs(kp_gt - kp_pred) * valid).sum() / (3 * valid.sum())
        params = [m.volume_net.output_layer.weight, m.process_features[0].weight]
        res = []
        for fn in (_native, oracle_volumetric_ce_loss):
            total = 0.1 * mae + 0.01 * fn(coord, vols, kp_gt, valid)
            res.append((float(total), torch.autograd.grad(total, params, retain_graph=True)))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    (l0, g0), (l1, g1) = res
    assert abs(l0 - l1) <= 1e-6 * abs(l1)
    for a, b in zip(g0, g1):
        assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max())
