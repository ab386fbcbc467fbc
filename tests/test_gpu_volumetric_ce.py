"""The volumetric cross-entropy loss on the device (csrc/loss.cu through lt_b200.loss.VolumetricCELoss) against the restatement of the
reference loss (test_volumetric_ce_cpu.oracle_volumetric_ce_loss, pinned to the reference's golden there) run on CUDA, and against
the vectorised torch formulation: indices, loss, sparse gradient, composition with the hybrid soft-argmax, no host
synchronisation, determinism and one training step of the volumetric model.

The kernels against the host hook (capi.volumetric_ce_host), which runs the same distance, key, term and gradient helpers and sums
the terms in the same order: loss, index, picked probability and the whole gradient agree bit for bit on the golden cases, on exact
ties split across CTAs, warps and a thread's voxels, on NaN coordinates and ground truth, on distances that overflow, on both
backward kernels and on the grid-stride loops of the finish and backward kernels."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import autograd_ops, capi, loss as ce, op, testing, torch_ops
from test_gpu_glue_ref import run_in_fresh_process
from test_volumetric_ce_cpu import CASES, GOLDEN, oracle_volumetric_ce_loss

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
@pytest.mark.parametrize("grid", [(64, 64, 64), (32, 32, 32), (20, 24, 28), (7, 11, 13)])
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


# ---- the kernels against the host hook, bit for bit -------------------------------------------------------------------------
CE_CHUNK = 1024                                                         # kCeChunk: voxels per CTA of ce_search_kernel


def _device_ce(probs, coord, kp, valid, grad_offset=0, grad_loss=1.0):
    """lt_volumetric_ce_fwd + lt_volumetric_ce_bwd on CPU float32 inputs (B, J, nvox), (B, nvox, 3), (B, J, 3), (B, J) -> (loss, index,
    picked, grad) on the CPU.  The gradient starts `grad_offset` floats into a NaN-filled buffer (1: not 16-byte aligned), with a
    guard of NaN after it that must survive."""
    B, J, nvox = probs.shape
    loss = torch.empty(1, device=DEV)
    index = torch.empty((B, J), dtype=torch.int32, device=DEV)
    picked = torch.empty((B, J), device=DEV)
    ws = torch.empty(capi.volumetric_ce_workspace_bytes(B, J, nvox), dtype=torch.uint8, device=DEV)
    capi.volumetric_ce(probs.to(DEV), coord.to(DEV), kp.to(DEV), valid.to(DEV), loss, index, picked, ws)
    n = B * J * nvox
    buf = torch.full((grad_offset + n + 64,), float("nan"), device=DEV)
    grad = buf[grad_offset:grad_offset + n].view(B, J, nvox)
    capi.volumetric_ce_bwd(torch.tensor([grad_loss], device=DEV), index, picked, valid.to(DEV), grad)
    torch.cuda.synchronize()
    assert bool(buf[:grad_offset].isnan().all()) and bool(buf[grad_offset + n:].isnan().all())
    return float(loss.item()), index.cpu(), picked.cpu(), grad.cpu()


def _host_ce(probs, coord, kp, valid, grad_loss=1.0):
    grad = torch.full_like(probs, float("nan"))
    loss, index, picked = capi.volumetric_ce_host(probs, coord, kp, valid, grad_loss=grad_loss, grad_probs=grad)
    return loss, index, picked, grad


def _assert_device_equals_host(probs, coord, kp, valid, grad_offset=0):
    d = _device_ce(probs, coord, kp, valid, grad_offset)
    h = _host_ce(probs, coord, kp, valid)
    assert np.float32(d[0]).view(np.int32) == np.float32(h[0]).view(np.int32), (d[0], h[0])
    assert torch.equal(d[1], h[1])
    assert torch.equal(d[2].view(torch.int32), h[2].view(torch.int32))
    assert torch.equal(d[3].view(torch.int32), h[3].view(torch.int32))
    return d


@pytest.mark.parametrize("tag", CASES)
def test_golden_cases_on_the_device(tag):
    """volumetric_ce.npz on the kernels: the golden indices (tie, NaN ground truth and validity 0 in `lattice`), the golden loss and
    gradient at the bars of test_volumetric_ce_cpu.py, and the host hook bit for bit."""
    g = np.load(GOLDEN)
    B, J = g["volumes"].shape[:2]
    probs = torch.from_numpy(g["volumes"]).reshape(B, J, -1).contiguous()
    coord = torch.from_numpy(g[tag + "_coord"]).reshape(B, -1, 3).contiguous()
    kp, valid = torch.from_numpy(g[tag + "_keypoints"]), torch.from_numpy(g["validity"])[..., 0].contiguous()
    for offset in (0, 1):
        loss, index, picked, grad = _assert_device_equals_host(probs, coord, kp, valid, offset)
        assert torch.equal(index.long(), torch.from_numpy(g[tag + "_index"]))
        assert abs(loss - float(g[tag + "_loss"][0])) <= 1e-6 * abs(float(g[tag + "_loss"][0]))
        want = torch.from_numpy(g[tag + "_grad_at_index"])
        got = grad.gather(2, index.long().unsqueeze(-1)).squeeze(-1)
        assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max())


def _far_problem(B, J, nvox, seed):
    """Voxels scattered 1e4 .. 2e4 mm away from every ground-truth point near the origin, softmaxed probabilities, mixed validity."""
    g = torch.Generator().manual_seed(seed)
    coord = (torch.rand(B, nvox, 3, generator=g) + 1.0) * 1e4 * torch.where(torch.rand(B, nvox, 3, generator=g) > 0.5, 1.0, -1.0)
    kp = torch.randn(B, J, 3, generator=g) * 100
    probs = torch.softmax(torch.randn(B, J, nvox, generator=g) * 3, -1)
    valid = (torch.rand(B, J, generator=g) > 0.2).float()
    return probs.contiguous(), coord.contiguous(), kp.contiguous(), valid.contiguous()


def _tie(coord, kp, b, j, v_low, v_high):
    """Voxels v_low < v_high exactly 1 mm from ground-truth point (b, j), one on each side along x: equal distances."""
    p = kp[b, j]
    coord[b, v_high] = p + torch.tensor([1.0, 0.0, 0.0])
    coord[b, v_low] = p - torch.tensor([1.0, 0.0, 0.0])


TIES = {"across CTAs": (100, 100 + 3 * CE_CHUNK), "across warps": (5, 37), "within a thread": (5, 5 + 256),
        "first and last CTA": (0, 4999)}


@pytest.mark.parametrize("name", list(TIES))
def test_exact_ties_go_to_the_lower_index(name):
    lo, hi = TIES[name]
    probs, coord, kp, valid = _far_problem(2, 3, 5000, seed=lo + hi)
    kp[:, 1] = kp[:, 0]                                                 # two joints share the point and so the tie
    for b in range(2):
        _tie(coord, kp, b, 0, lo, hi)
    _tie(coord, kp, 0, 2, hi - 1, hi + 1 if hi + 1 < 5000 else hi - 2)  # and one more between two other voxels
    d = _assert_device_equals_host(probs, coord, kp, valid)
    assert d[1][:, 0].tolist() == [lo, lo] and d[1][:, 1].tolist() == [lo, lo]


def test_nan_coordinates_in_a_late_cta_win_with_their_smallest_index():
    probs, coord, kp, valid = _far_problem(2, 5, 5000, seed=1)
    coord[0, 4700, 1] = float("nan")
    coord[0, 4500, 2] = float("nan")
    _tie(coord, kp, 0, 3, 10, 20)                                       # a finite tie elsewhere loses to the NaN
    d = _assert_device_equals_host(probs, coord, kp, valid)
    assert d[1][0].tolist() == [4500] * 5


def test_nan_ground_truth_and_overflowing_distances():
    probs, coord, kp, valid = _far_problem(2, 4, 3000, seed=2)
    kp[0, 1, 2] = float("nan")                                          # every distance NaN: the first voxel
    coord[1] = (torch.rand(3000, 3, generator=torch.Generator().manual_seed(3)) * 2 - 1) * 1e38
    kp[1, 0] = torch.tensor([-3e38, 0.0, 0.0])                          # every square overflows ...
    coord[1, 2500] = torch.tensor([-3e38, 1.0, 0.0])                    # ... but one: distance 1
    kp[1, 1] = torch.tensor([3.4e38, 3.4e38, 0.0])                      # every distance +inf: the first voxel
    valid[0, 1] = 1.0
    d = _assert_device_equals_host(probs, coord, kp, valid)
    assert d[1][0, 1] == 0 and d[1][1, 0] == 2500 and d[1][1, 1] == 0


SIZES = [  # (B, J, nvox, grad offset): nvox = 1 and < 1024, J < 8 and not a multiple of 8, both backward kernels, > 256 rows for the
           # finish kernel's loop, > 65535 rows for the backward's grid-stride loop
    (1, 1, 1, 0), (3, 3, 300, 0), (2, 13, 1001, 0), (2, 13, 1000, 1), (2, 8, 4096, 1), (4, 70, 600, 0), (2, 33000, 6, 0),
    (2, 33000, 8, 0), (2, 33000, 8, 1)]


@pytest.mark.parametrize("B, J, nvox, offset", SIZES)
def test_sizes_and_both_backward_kernels(B, J, nvox, offset):
    probs, coord, kp, valid = _far_problem(B, J, nvox, seed=B * J + nvox)
    coord[:, nvox // 2] = kp[:, 0] + 0.5                                 # a voxel near some joint, so not every index is the same
    _assert_device_equals_host(probs, coord, kp, valid, offset)


def profiled_ce_bwd_launches():
    """The backward of an aligned gradient with nvox % 4 == 0, then of one offset by a float, under torch.profiler -> the backward
    kernels launched."""
    from torch.profiler import ProfilerActivity, profile
    probs, coord, kp, valid = _far_problem(2, 3, 1000, seed=4)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _device_ce(probs, coord, kp, valid, 0)
        _device_ce(probs, coord, kp, valid, 1)
    evs = sorted((e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA),
                 key=lambda e: e.start_ns())
    return [e.name() for e in evs if "ce_bwd_kernel" in e.name()]


def test_both_backward_kernels_launch():
    names = run_in_fresh_process("test_gpu_volumetric_ce", "profiled_ce_bwd_launches")
    assert len(names) == 2 and "<true>" in names[0] and "<false>" in names[1], names
