"""GPU tests of the keypoint criteria kernels (lt_keypoints_loss_fwd / _bwd): the float64 restatement of the reference with the CPU
tests' bars, bitwise repeats, no host synchronisation, and a captured call equal to the eager one."""
import numpy as np
import pytest
import torch

from lt_b200 import loss as crit, testing

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KINDS = ("mse", "mse_smooth", "mae", "l2")
EPS = 2.0 ** -24


def _device(kind, pred, gt, v, threshold=400.0, grad_loss=1.0):
    p = pred.to(DEV).requires_grad_(True)
    loss = crit.keypoints_loss(kind, p, gt.to(DEV), v.to(DEV), threshold=threshold, backend="native")
    loss.backward(torch.tensor(grad_loss, device=DEV))
    torch.cuda.synchronize()
    return loss.detach().cpu(), p.grad.cpu()


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("case", testing.KEYPOINT_CASES)
@pytest.mark.parametrize("kind", KINDS)
def test_device_matches_the_float64_reference(kind, case, dim):
    pred, gt, v = testing.keypoint_case(case, dim)
    want, want_grad, mag = testing.reference_keypoints_loss64(kind, pred, gt, v)
    loss, grad = _device(kind, pred, gt, v)
    n = pred.shape[0] * pred.shape[1] * (1 if kind == "l2" else dim)
    sv = max(1.0, float(v.double().sum()))
    norm = sv if kind == "l2" else dim * sv
    if np.isnan(want):
        assert bool(torch.isnan(loss))
    else:
        assert abs(float(loss) - want) <= (n + 4) * EPS * mag / norm + EPS * abs(want)
    nan = torch.isnan(want_grad)
    assert torch.equal(torch.isnan(grad), nan)
    w = want_grad[~nan]
    assert bool(((grad[~nan].double() - w).abs() <= 4 * EPS * w.abs() + 1e-30).all())


@pytest.mark.parametrize("kind", KINDS)
def test_repeats_are_bitwise_equal(kind):
    pred, gt, v = testing.keypoint_case("plain", 3, (64, 17), seed=3)      # 1088 points: four or five per thread of the CTA
    a = _device(kind, pred, gt, v)
    for _ in range(3):
        b = _device(kind, pred, gt, v)
        assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32))      # bit patterns: L2 has NaN gradients
        assert torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def test_no_host_synchronisation():
    pred, gt, v = (t.to(DEV) for t in testing.keypoint_case("fractional"))
    p = pred.clone().requires_grad_(True)
    crit.KeypointsMSESmoothLoss(backend="native")(p, gt, v).backward()      # module loads outside the checked region
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for cls in (crit.KeypointsMSELoss, crit.KeypointsMSESmoothLoss, crit.KeypointsMAELoss, crit.KeypointsL2Loss):
            p.grad = None
            cls(backend="native")(p, gt, v).backward()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", KINDS)
def test_captured_call_equals_the_eager_call(kind):
    pred, gt, v = (t.to(DEV) for t in testing.keypoint_case("fractional", 3, (5, 17), seed=7))
    eager_p = pred.clone().requires_grad_(True)
    eager = crit.keypoints_loss(kind, eager_p, gt, v, backend="native")
    eager.backward()
    static_p = pred.clone().requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        crit.keypoints_loss(kind, static_p, gt, v, backend="native").backward()
    torch.cuda.current_stream().wait_stream(side)
    static_p.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = crit.keypoints_loss(kind, static_p, gt, v, backend="native")
        out.backward()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager.detach()) and torch.equal(static_p.grad, eager_p.grad)
