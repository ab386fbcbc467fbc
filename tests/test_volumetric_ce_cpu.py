"""The volumetric cross-entropy loss (lt_b200.loss.VolumetricCELoss, csrc/loss.cu) checked on the CPU.

- A restatement of the reference loss (loss.py:52-80, below) and the vectorised torch formulation (torch_ops.volumetric_ce_loss)
  against tests/golden/volumetric_ce.npz, made from the unmodified reference.
- The kernels' distance / argmin-key / term / gradient code through the host hook lt_test_volumetric_ce_host, against the same
  fixture and on the tie, boundary and NaN cases.
- The wrapper plumbing with a torch stand-in for the C calls, the error paths and install().
The CUDA launches are covered by tests/test_gpu_volumetric_ce.py."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import autograd_ops, capi, loss as ce, torch_ops

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "volumetric_ce.npz")
CASES = ("rot", "view", "lattice")


def oracle_volumetric_ce_loss(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity):
    """Restatement of VolumetricCELoss.forward (reference loss.py:56-80): per sample (:61) the distances of every voxel to every
    ground-truth point (:62-69), torch.argmin copied to the host (:71), unravelled over the volume's grid (:72), then per joint
    the term validity[0] * -log(p + 1e-6) at that voxel added to a running sum (:74-77), divided by the number of terms (:80)."""
    loss, n_losses = 0.0, 0
    for b in range(volumes_batch_pred.shape[0]):
        kp = keypoints_gt[b]
        dists = torch.sqrt(((coord_volumes_batch[b].unsqueeze(0) - kp.reshape(kp.shape[0], 1, 1, 1, 3)) ** 2).sum(-1))
        flat = torch.argmin(dists.reshape(dists.shape[0], -1), dim=-1).detach().cpu().numpy()
        for j, (x, y, z) in enumerate(np.stack(np.unravel_index(flat, volumes_batch_pred.shape[-3:]), axis=1)):
            loss += keypoints_binary_validity[b, j][0] * (-torch.log(volumes_batch_pred[b, j, x, y, z] + 1e-6))
            n_losses += 1
    return loss / n_losses


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


def _case(g, tag):
    return (torch.from_numpy(g[tag + "_coord"]), torch.from_numpy(g["volumes"]), torch.from_numpy(g[tag + "_keypoints"]),
            torch.from_numpy(g["validity"]))


def _rel(a, b):
    return abs(float(a.detach() if torch.is_tensor(a) else a) - float(b)) / abs(float(b))


def test_golden_covers_the_edge_cases(golden):
    n = golden["volumes"].shape[-1]
    assert golden["lattice_index"][0, 3] == (4 * n + 6) * n + 2          # the tie went to the lower of two flat indices
    assert golden["lattice_index"][1, 5] == 0                           # NaN ground truth: the first NaN distance
    assert np.isnan(golden["lattice_keypoints"][1, 5]).all() and golden["validity"][0, 7, 0] == 0
    c = golden["rot_coord"].reshape(2, -1, 3)
    for b in range(2):                                                  # far-outside joints land on the boundary of the grid
        for j in (0, 1):
            i = np.unravel_index(golden["rot_index"][b, j], (n, n, n))
            assert any(k in (0, n - 1) for k in i)
    assert not np.array_equal(golden["rot_index"], golden["view_index"])


@pytest.mark.parametrize("tag", CASES)
def test_oracle_matches_the_reference_golden(golden, tag):
    coord, vols, kp, valid = _case(golden, tag)
    assert _rel(oracle_volumetric_ce_loss(coord, vols, kp, valid), golden[tag + "_loss"][0]) <= 1e-6


@pytest.mark.parametrize("tag", CASES)
def test_torch_formulation_matches_the_reference_golden(golden, tag):
    coord, vols, kp, valid = _case(golden, tag)
    B, J = vols.shape[:2]
    assert torch.equal(torch_ops.volumetric_ce_index(coord, kp), torch.from_numpy(golden[tag + "_index"]))
    v = vols.clone().requires_grad_(True)
    loss = torch_ops.volumetric_ce_loss(coord, v, kp, valid)
    loss.backward()
    assert loss.dim() == 0 and _rel(loss, golden[tag + "_loss"][0]) <= 1e-6
    grad = v.grad.reshape(B, J, -1)
    index = torch.from_numpy(golden[tag + "_index"]).unsqueeze(-1)
    want = torch.from_numpy(golden[tag + "_grad_at_index"])
    got = grad.gather(2, index).squeeze(-1)
    assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max())
    assert int((grad != 0).sum()) == int((want != 0).sum())             # nothing outside the picked voxels


@pytest.mark.parametrize("tag", CASES)
def test_host_hook_matches_the_reference_golden(golden, tag):
    coord, vols, kp, valid = _case(golden, tag)
    B, J = vols.shape[:2]
    probs = vols.reshape(B, J, -1).contiguous()
    grad = torch.full_like(probs, float("nan"))                         # the hook writes every element
    loss, index, picked = capi.volumetric_ce_host(probs, coord.reshape(B, -1, 3).contiguous(), kp, valid[..., 0].contiguous(),
                                                  grad_loss=1.0, grad_probs=grad)
    assert torch.equal(index.long(), torch.from_numpy(golden[tag + "_index"]))
    assert _rel(loss, golden[tag + "_loss"][0]) <= 1e-6
    assert torch.equal(picked, probs.gather(2, index.long().unsqueeze(-1)).squeeze(-1))
    want = torch.from_numpy(golden[tag + "_grad_at_index"])
    got = grad.gather(2, index.long().unsqueeze(-1)).squeeze(-1)
    assert float((got - want).abs().max()) <= 1e-6 * float(want.abs().max())
    mask = torch.ones_like(grad, dtype=torch.bool).scatter_(2, index.long().unsqueeze(-1), False)
    assert bool((grad[mask] == 0).all())


def _one(coord, kp):
    """host-hook argmin of explicit coordinate rows (nvox, 3) and points (J, 3)"""
    coord = torch.tensor(coord, dtype=torch.float32).reshape(1, -1, 3)
    kp = torch.tensor(kp, dtype=torch.float32).reshape(1, -1, 3)
    J = kp.shape[1]
    probs = torch.full((1, J, coord.shape[1]), 0.25)
    return capi.volumetric_ce_host(probs, coord, kp, torch.ones(1, J))[1][0].tolist()


def test_host_hook_tie_and_nan_rules():
    # equal distances: the lower index
    assert _one([[2, 0, 0], [0, 0, 0], [1, 0, 0], [1, 0, 0]], [[1, 0, 0]]) == [2]
    assert _one([[0, 0, 0], [2, 0, 0]], [[1, 0, 0]]) == [0]
    assert _one([[0, 0, 0], [1 + 2 ** -23, 0, 0]], [[0.5 + 2 ** -24, 0, 0]]) == [0]
    # NaN: a NaN ground truth makes every distance NaN (index 0); a NaN voxel wins, the first one among several
    assert _one([[5, 5, 5], [0, 0, 0]], [[float("nan"), 0, 0]]) == [0]
    assert _one([[3, 0, 0], [float("nan"), 0, 0], [1, 0, 0], [float("nan"), 0, 0]], [[1, 0, 0]]) == [1]
    # distances that overflow to inf tie with each other (index 0) and lose to any finite one
    assert _one([[1e38, 0, 0], [-1e38, 0, 0]], [[-3e38, 0, 0]]) == [0]
    assert _one([[3e38, 0, 0], [-3e38, 1, 0]], [[-3e38, 0, 0]]) == [1]


def test_torch_argmin_conventions_the_kernels_follow():
    assert int(torch.argmin(torch.tensor([3.0, float("nan"), 1.0, float("nan")]))) == 1
    assert int(torch.argmin(torch.tensor([float("inf"), float("inf")]))) == 0


def test_host_hook_compares_rounded_square_roots():
    """Two voxels whose squared distances differ but whose correctly rounded fp32 square roots are equal (what the CUDA build of
    torch.sqrt returns; the vectorised CPU one can differ by an ulp): argmin sees equal values and picks the lower index, although
    that voxel is the farther one in d^2."""
    rng = np.random.RandomState(0)
    found = 0
    for _ in range(2000):
        k = rng.uniform(-1, 1, 3).astype(np.float32)
        c0 = (k + rng.uniform(-1, 1, 3)).astype(np.float32)
        c1 = c0.copy()
        c1[0] = np.nextafter(c1[0], np.float32(np.inf) if c1[0] > k[0] else np.float32(-np.inf))
        sq = (np.stack([c1, c0]) - k) ** 2
        d2 = (sq[:, 0] + sq[:, 1]) + sq[:, 2]                            # float32, summed left to right
        d = np.sqrt(d2.astype(np.float64)).astype(np.float32)            # correctly rounded
        if d[0] == d[1] and d2[0] > d2[1]:
            found += 1
            assert _one(np.stack([c1, c0]), k[None]) == [0]
    assert found > 10


def test_host_hook_many_joints_matches_torch_formulation():
    """J larger than a joint group, non-cubic grid, random rotation-free coordinates: hook == torch formulation."""
    torch.manual_seed(4)
    B, J, X, Y, Z = 2, 21, 5, 6, 7
    coord = torch.randn(B, X, Y, Z, 3) * 300
    vols = torch.softmax(torch.randn(B, J, X * Y * Z), -1).reshape(B, J, X, Y, Z)
    kp = torch.randn(B, J, 3) * 300
    valid = (torch.rand(B, J, 2) > 0.2).float()
    want = torch_ops.volumetric_ce_loss(coord, vols, kp, valid)
    loss, index, _ = capi.volumetric_ce_host(vols.reshape(B, J, -1).contiguous(), coord.reshape(B, -1, 3).contiguous(), kp,
                                             valid[..., 0].contiguous())
    assert torch.equal(index.long(), torch_ops.volumetric_ce_index(coord, kp))
    assert _rel(loss, want) <= 1e-6


# ---- wrapper plumbing with a torch stand-in for the C calls ---------------------------------------------------------------

CALLS = []


def _fake_ce(probs, coord, kp, validity, loss, index, picked, workspace):
    CALLS.append("fwd")
    assert workspace.numel() >= 8 * probs.shape[0] * probs.shape[1]
    B, J, nvox = probs.shape
    idx = torch_ops.volumetric_ce_index(coord, kp)
    p = probs.gather(2, idx.unsqueeze(-1)).squeeze(-1)
    index.copy_(idx)
    picked.copy_(p)
    loss.copy_((validity * -torch.log(p + 1e-6)).sum().reshape(1) / (B * J))


def _fake_ce_bwd(grad_loss, index, picked, validity, grad_probs):
    CALLS.append("bwd")
    B, J, nvox = grad_probs.shape
    val = -((grad_loss / (B * J)) * validity) / (picked + 1e-6)
    grad_probs.copy_(torch.zeros_like(grad_probs).scatter_(2, index.long().unsqueeze(-1), val.unsqueeze(-1)))


@pytest.fixture
def fake_capi(monkeypatch):
    monkeypatch.setattr(capi, "volumetric_ce", _fake_ce)
    monkeypatch.setattr(capi, "volumetric_ce_bwd", _fake_ce_bwd)
    monkeypatch.setattr(capi, "volumetric_ce_workspace_bytes", lambda B, J, nvox: 8 * B * J)
    # the module's CUDA check is the only thing that stands between CPU tensors and the (faked) kernels here
    monkeypatch.setattr(ce, "_resolve_backend", lambda backend, *t: "torch" if backend == "torch" else "native")
    CALLS.clear()


@pytest.mark.parametrize("tag", CASES)
def test_module_wrapper_gradients(fake_capi, golden, tag):
    coord, vols, kp, valid = _case(golden, tag)
    res = []
    for backend in ("torch", "native"):
        v = vols.clone().requires_grad_(True)
        out = ce.VolumetricCELoss(backend=backend)(coord, v, kp, valid)
        (out * 3.0).backward()
        res.append((out.detach(), v.grad))
    assert CALLS == ["fwd", "bwd"]
    assert res[1][0].dim() == 0 and res[1][1].shape == vols.shape
    assert _rel(res[1][0], res[0][0]) <= 1e-6
    assert torch.allclose(res[0][1], res[1][1], rtol=1e-6, atol=0)


def test_module_wrapper_takes_a_non_contiguous_coordinate_view(fake_capi, golden):
    coord, vols, kp, valid = _case(golden, "rot")
    view = coord.transpose(2, 3).flip(1)                                # the same view as the golden's "view" case, not copied
    assert not view.is_contiguous()
    out = ce.VolumetricCELoss(backend="native")(view, vols, kp, valid)
    assert _rel(out, golden["view_loss"][0]) <= 1e-6


def test_function_gives_no_gradient_to_the_data(fake_capi, golden):
    coord, vols, kp, valid = _case(golden, "rot")
    B, J = vols.shape[:2]
    v, k = vols.clone().requires_grad_(True), kp.clone().requires_grad_(True)
    c = coord.clone().requires_grad_(True)
    loss, index, picked = autograd_ops.volumetric_ce_loss(v.reshape(B, J, -1), c.reshape(B, -1, 3), k, valid[..., 0])
    assert not index.requires_grad and not picked.requires_grad and index.dtype == torch.int32
    loss.backward()
    assert v.grad is not None and k.grad is None and c.grad is None


# ---- errors -----------------------------------------------------------------------------------------------------------

def _inputs(B=2, J=3, grid=(4, 5, 6)):
    return (torch.zeros(B, *grid, 3), torch.full((B, J) + grid, 0.1), torch.zeros(B, J, 3), torch.ones(B, J, 1))


@pytest.mark.parametrize("backend", ["native", "hybrid", None])
def test_cpu_tensors_on_the_native_backends_raise(backend, monkeypatch):
    monkeypatch.delenv("LT_B200_BACKEND", raising=False)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        ce.VolumetricCELoss(backend=backend)(*_inputs())


def test_environment_selects_the_backend(monkeypatch):
    monkeypatch.setenv("LT_B200_BACKEND", "torch")
    assert ce.VolumetricCELoss()(*_inputs()).dim() == 0
    monkeypatch.setenv("LT_B200_BACKEND", "native")
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        ce.VolumetricCELoss()(*_inputs())
    with pytest.raises(ValueError, match="unknown backend"):
        ce.VolumetricCELoss(backend="cpu")(*_inputs())


@pytest.mark.parametrize("which, shape", [
    ("volumes", (2, 3, 4, 5)),              # not 5-D
    ("coord", (2, 4, 5, 7, 3)),             # grid differs from the volumes'
    ("coord", (2, 4, 5, 6, 2)),             # not 3 coordinates
    ("coord", (1, 4, 5, 6, 3)),             # batch differs
    ("keypoints", (2, 4, 3)),               # joint count differs
    ("keypoints", (2, 3, 2)),
    ("validity", (2, 3)),                   # no trailing dimension
    ("validity", (2, 3, 0)),
    ("validity", (2, 4, 1)),
])
def test_shape_mismatches_raise_value_error(which, shape):
    coord, vols, kp, valid = _inputs()
    new = torch.zeros(shape)
    args = {"coord": coord, "volumes": vols, "keypoints": kp, "validity": valid}
    args[which] = new
    for backend in ("torch", "native"):
        with pytest.raises(ValueError):
            ce.VolumetricCELoss(backend=backend)(args["coord"], args["volumes"], args["keypoints"], args["validity"])


def test_host_hook_rejects_bad_sizes():
    buf = torch.zeros(64)
    p = buf.data_ptr()
    lib = capi.lib()
    assert lib.lt_test_volumetric_ce_host(p, p, p, p, p, p, p, None, None, 1, 2, 0) != 0
    assert b"bad sizes" in lib.lt_last_error_string()
    assert lib.lt_test_volumetric_ce_host(p, None, p, p, p, p, p, None, None, 1, 2, 4) != 0
    assert b"null pointer" in lib.lt_last_error_string()
    # the device entry points check their arguments before touching a device
    assert lib.lt_volumetric_ce_fwd(p, p, p, p, p, p, p, p, 8, 1, 2, 4, None) != 0
    assert b"workspace too small" in lib.lt_last_error_string()
    assert lib.lt_volumetric_ce_bwd(p, p, p, p, p, 0, 2, 4, None) != 0
    assert b"bad sizes" in lib.lt_last_error_string()


def test_install_patches_the_reference_loss(monkeypatch):
    """install() on a stand-in `mvn` package: mvn.models.loss.VolumetricCELoss becomes the native module."""
    names = ["mvn_stub", "mvn_stub.models", "mvn_stub.models.triangulation", "mvn_stub.models.loss", "mvn_stub.utils",
             "mvn_stub.utils.op"]
    mods = {n: types.ModuleType(n) for n in names}
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    sentinel = object()
    mods["mvn_stub.models.loss"].VolumetricCELoss = sentinel
    lt_b200.install(mods["mvn_stub"])
    assert mods["mvn_stub.models.loss"].VolumetricCELoss is lt_b200.loss.VolumetricCELoss
    assert mods["mvn_stub.models.triangulation"].VolumetricTriangulationNet is lt_b200.VolumetricTriangulationNet
    assert mods["mvn_stub.utils.op"].integrate_tensor_3d_with_coordinates is lt_b200.op.integrate_tensor_3d_with_coordinates
