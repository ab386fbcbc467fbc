"""The keypoint criteria (lt_b200.loss.Keypoints*Loss, csrc/loss.cu) checked on the CPU.

- The kernels' term, derivative and summation code through the host hook lt_test_keypoints_loss_host, against a float64
  restatement of the reference (testing.reference_keypoints_loss, loss.py:7-49) and torch autograd through it, on graded cases:
  zero and fractional validity, MSESmooth's threshold boundary, NaN / Inf at valid and invalid points, dim 2 and 3.
- The wrapper plumbing with a torch stand-in for the C calls, the error paths and install().
The CUDA launches are covered by tests/test_gpu_keypoints_loss.py."""
import sys
import types

import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import capi, loss as crit, testing

KINDS = ("mse", "mse_smooth", "mae", "l2")
EPS = 2.0 ** -24
CASES = testing.KEYPOINT_CASES


def _host(kind, pred, gt, v, threshold=400.0, grad_loss=1.0):
    B, J, dim = pred.shape
    grad = torch.full((B * J, dim), 12345.0)
    loss, norm = capi.keypoints_loss_host(pred.reshape(-1, dim).contiguous(), gt.reshape(-1, dim).contiguous(),
                                          v.reshape(-1).contiguous(), kind, threshold, grad_loss=grad_loss, grad_pred=grad)
    return loss, norm, grad.reshape(B, J, dim)


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("kind", KINDS)
def test_host_hook_matches_the_float64_reference(kind, case, dim):
    pred, gt, v = testing.keypoint_case(case, dim)
    want, want_grad, mag = testing.reference_keypoints_loss64(kind, pred, gt, v)
    loss, norm, grad = _host(kind, pred, gt, v)
    n = pred.shape[0] * pred.shape[1] * (1 if kind == "l2" else dim)
    sv = max(1.0, float(v.double().sum()))
    assert norm == (sv if kind == "l2" else dim * sv)
    if np.isnan(want):
        assert np.isnan(loss)
    else:
        assert abs(loss - want) <= (n + 4) * EPS * mag / norm + EPS * abs(want), (loss, want)
    nan = torch.isnan(want_grad)
    assert torch.equal(torch.isnan(grad), nan), "NaN pattern of the gradient"
    w = want_grad[~nan]
    assert bool(((grad[~nan].double() - w).abs() <= 4 * EPS * w.abs() + 1e-30).all())


def test_smooth_boundary_element_takes_the_unreplaced_branch():
    pred, gt, v = testing.keypoint_case("boundary")
    _, _, grad = _host("mse_smooth", pred, gt, v)
    _, norm, grad_mse = _host("mse", pred, gt, v)
    assert grad[0, 0, 0] == grad_mse[0, 0, 0]                  # d = 400: -2 (gt - pred) v / norm
    assert grad[0, 1, 0] != grad_mse[0, 1, 0]                  # d > 400: the pow 0.1 branch
    d = 20.0009765625 ** 2
    assert abs(float(grad[0, 1, 0]) - (-0.1 * d ** -0.9 * 400 ** 0.9 * 2 * 20.0009765625 / norm)) <= 4 * EPS * abs(float(grad[0, 1, 0]))


def test_invalid_non_finite_points_give_nan_as_in_the_reference():
    pred, gt, v = testing.keypoint_case("nan_invalid")
    for kind in KINDS:
        assert np.isnan(_host(kind, pred, gt, v)[0])
        assert np.isnan(float(testing.reference_keypoints_loss(kind, pred, gt, v)))


def test_l2_gradient_is_nan_at_a_zero_length_residual():
    pred, gt, v = testing.keypoint_case("plain")
    pred[0, 0] = gt[0, 0]
    v[0, 0], v[0, 1] = 1.0, 0.0
    grad = _host("l2", pred, gt, v)[2]
    assert bool(torch.isnan(grad[0, 0]).all()) and bool(torch.isnan(grad[0, 1]).all())
    assert bool(torch.isfinite(grad[v[..., 0] > 0][1:]).all())


def test_host_hook_scales_by_grad_loss_and_repeats_bitwise():
    pred, gt, v = testing.keypoint_case("many")
    a = _host("mae", pred, gt, v, grad_loss=1.0)
    b = _host("mae", pred, gt, v, grad_loss=-3.0)
    assert a[0] == _host("mae", pred, gt, v)[0]
    assert torch.allclose(b[2], -3.0 * a[2], rtol=1e-6, atol=0)


def test_host_hook_rejects_bad_arguments():
    buf = torch.zeros(64)
    p = buf.data_ptr()
    nrm = torch.zeros(1, dtype=torch.float64).data_ptr()
    lib = capi.lib()
    assert lib.lt_test_keypoints_loss_host(p, p, p, p, nrm, None, None, 0, 400.0, 0, 3) != 0
    assert b"bad sizes" in lib.lt_last_error_string()
    assert lib.lt_test_keypoints_loss_host(p, p, p, p, nrm, None, None, 0, 400.0, 4, 0) != 0
    assert b"bad sizes" in lib.lt_last_error_string()
    assert lib.lt_test_keypoints_loss_host(p, None, p, p, nrm, None, None, 0, 400.0, 4, 3) != 0
    assert b"null pointer" in lib.lt_last_error_string()
    assert lib.lt_test_keypoints_loss_host(p, p, p, p, nrm, None, None, 4, 400.0, 4, 3) != 0
    assert b"unknown kind" in lib.lt_last_error_string()
    # the device entry points check their arguments before touching a device
    assert lib.lt_keypoints_loss_fwd(p, p, p, p, None, 0, 400.0, 4, 3, None) != 0
    assert b"null pointer" in lib.lt_last_error_string()
    assert lib.lt_keypoints_loss_bwd(p, p, p, p, nrm, p, 0, 400.0, -1, 3, None) != 0
    assert b"bad sizes" in lib.lt_last_error_string()


# ---- wrapper plumbing with a torch stand-in for the C calls ---------------------------------------------------------------

CALLS = []


def _fake_fwd(pred, gt, validity, loss, norm, kind, threshold):
    CALLS.append(("fwd", kind))
    l, n, _ = _host(kind, pred[None], gt[None], validity[None, :, None], threshold)
    loss.fill_(l)
    norm.fill_(n)


def _fake_bwd(grad_loss, pred, gt, validity, norm, grad_pred, kind, threshold):
    CALLS.append(("bwd", kind))
    grad_pred.copy_(_host(kind, pred[None], gt[None], validity[None, :, None], threshold, grad_loss=float(grad_loss))[2][0])


@pytest.fixture
def fake_capi(monkeypatch):
    monkeypatch.setattr(capi, "keypoints_loss", _fake_fwd)
    monkeypatch.setattr(capi, "keypoints_loss_bwd", _fake_bwd)
    # the module's CUDA check is the only thing that stands between CPU tensors and the (faked) kernels here
    monkeypatch.setattr(crit, "_resolve_backend", lambda backend, *t: "torch" if backend == "torch" else "native")
    CALLS.clear()


MODULES = {"mse": crit.KeypointsMSELoss, "mse_smooth": crit.KeypointsMSESmoothLoss, "mae": crit.KeypointsMAELoss,
           "l2": crit.KeypointsL2Loss}


@pytest.mark.parametrize("kind", KINDS)
def test_module_wrapper_gradients_reach_the_prediction_only(fake_capi, kind):
    pred, gt, v = testing.keypoint_case("fractional")
    res = []
    for backend in ("torch", "native"):
        p, g = pred.clone().requires_grad_(True), gt.clone().requires_grad_(True)
        out = MODULES[kind](backend=backend)(p, g, v)
        (out * 3.0).backward()
        assert out.dim() == 0 and g.grad is None
        res.append((out.detach(), p.grad))
    assert CALLS == [("fwd", kind), ("bwd", kind)]
    assert torch.allclose(res[0][0], res[1][0], rtol=1e-6, atol=0)
    assert torch.allclose(res[0][1], res[1][1], rtol=1e-5, atol=1e-9)


def test_native_path_takes_two_dimensional_validity(fake_capi):
    pred, gt, v = testing.keypoint_case("plain")
    a = crit.KeypointsMAELoss(backend="native")(pred, gt, v)
    b = crit.KeypointsMAELoss(backend="native")(pred, gt, v[..., 0])
    assert torch.equal(a, b)


def test_smooth_threshold_reaches_the_kernel(fake_capi):
    pred, gt, v = testing.keypoint_case("plain")
    a = crit.KeypointsMSESmoothLoss(threshold=50, backend="native")(pred, gt, v)
    b = crit.KeypointsMSESmoothLoss(threshold=50, backend="torch")(pred, gt, v)
    assert torch.allclose(a, b, rtol=1e-6) and not torch.allclose(a, crit.KeypointsMSESmoothLoss(backend="torch")(pred, gt, v))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("case", ["plain", "zero_validity", "fractional", "boundary"])
def test_torch_backend_matches_autograd_of_the_reference_formula(kind, case):
    pred, gt, v = testing.keypoint_case(case)
    p1, p2 = pred.clone().requires_grad_(True), pred.clone().requires_grad_(True)
    want = testing.reference_keypoints_loss(kind, p1, gt, v)
    got = MODULES[kind](backend="torch")(p2, gt, v)
    want.backward()
    got.backward()
    assert torch.allclose(got, want, rtol=1e-6, atol=0)
    assert torch.allclose(p2.grad, p1.grad, rtol=1e-5, atol=1e-12, equal_nan=True)


@pytest.mark.parametrize("backend", ["native", "hybrid", None])
def test_cpu_tensors_on_the_native_backends_raise(backend, monkeypatch):
    monkeypatch.delenv("LT_B200_BACKEND", raising=False)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        crit.KeypointsMSELoss(backend=backend)(*testing.keypoint_case("plain"))
    with pytest.raises(ValueError, match="unknown backend"):
        crit.KeypointsMSELoss(backend="cpu")(*testing.keypoint_case("plain"))


@pytest.mark.parametrize("which, shape", [
    ("pred", (3, 5)),                       # not 3-D
    ("pred", (3, 5, 0)),
    ("gt", (3, 5, 2)),                      # differs from pred
    ("gt", (3, 4, 3)),
    ("validity", (3, 5, 2)),                # not (B, J, 1) or (B, J)
    ("validity", (3, 4, 1)),
    ("validity", (15,)),
])
def test_shape_mismatches_raise_value_error(which, shape):
    args = dict(zip(("pred", "gt", "validity"), testing.keypoint_case("plain")))
    args[which] = torch.zeros(shape)
    for backend in ("torch", "native"):
        for cls in MODULES.values():
            with pytest.raises(ValueError):
                cls(backend=backend)(args["pred"], args["gt"], args["validity"])


def test_install_patches_every_reference_loss(monkeypatch):
    names = ["mvn_kp", "mvn_kp.models", "mvn_kp.models.triangulation", "mvn_kp.models.loss", "mvn_kp.utils", "mvn_kp.utils.op"]
    mods = {n: types.ModuleType(n) for n in names}
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    lt_b200.install(mods["mvn_kp"])
    ref = mods["mvn_kp.models.loss"]
    for name in ("KeypointsMSELoss", "KeypointsMSESmoothLoss", "KeypointsMAELoss", "KeypointsL2Loss", "VolumetricCELoss"):
        assert getattr(ref, name) is getattr(lt_b200.loss, name)
    assert crit.KeypointsMSESmoothLoss().threshold == 400
