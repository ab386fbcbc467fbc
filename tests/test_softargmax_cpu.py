"""Soft-argmax scenes and float64 references, the backward's per-item code (csrc/backward.cu) on the CPU against float64 autograd, and
the engine's choice of the fused V2V tail, all without a GPU.  The references are built on `torch_ops` (pinned to the reference by
tests/test_oracle_vs_reference.py):
- modes 0 and 1: `integrate_tensor_3d_with_coordinates` on multiplier x logits (0: ReLU without normalisation, 1: softmax);
- mode 2: sum relu * x / sum relu, the ReLU branch of `integrate_tensor_2d` (checked equal to it on a pixel grid).

Logits are float32 values on a grid of 2^-12 with |l| < 32, so l + c is exact in float32 for every offset c in OFFSETS and l x 100 is
exact too: the float64 answer of a softmax scene is the same at every offset (checked here), so the offset scenes measure how the
kernels handle a large max, not how the input was rounded.

A joint whose ReLU map has no mass (mode 2) has a NaN key point in the reference (0 / 0); the kernels give NaN as well.  Its backward
is zero in the kernels' per-item code (every p_i = 0 fails the p_i > 0 test), as in float64 autograd (the ReLU's gradient masks the
0 / 0); the other joints' gradients are unaffected.
The helpers here are shared with tests/test_gpu_softargmax.py.
"""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import capi, engine as eng_mod, testing, torch_ops
from oracle import vol_oracle as O

OFFSETS = (-1024.0, 0.0, 64.0, 1024.0)
KINDS = ("peaked", "flat", "diffuse")
Q = 2.0 ** -12                      # logit grid


def coords_for(B, nvox, seed):
    """Realistic coordinates (B, nvox, 3) float32: the first nvox voxels of a 2.5 m coordinate volume per sample (O.coord_volume)."""
    rng = np.random.RandomState(seed)
    n = max(2, int(np.ceil(round(nvox ** (1.0 / 3.0), 6))))
    while n ** 3 < nvox:
        n += 1
    return np.stack([O.coord_volume(rng.randn(3) * 100 + [0, 0, 900], 2500.0, n).reshape(-1, 3)[:nvox] for _ in range(B)]).astype(np.float32)


def pixel_grid(B, h, w):
    """(B, h * w, 3) float32 pixel grid (x, y, 0), as engine.algebraic_forward passes it."""
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    return np.ascontiguousarray(np.broadcast_to(np.stack([xs, ys, np.zeros_like(xs)], -1).reshape(1, h * w, 3), (B, h * w, 3)))


def make_logits(B, J, nvox, kind, seed, offset=0.0, zero_mass_joint=None):
    """(B, J, nvox) float32 logits on the 2^-12 grid, |l| < 32, plus `offset`.
    peaked: N(0, 2) with one +9 voxel per (sample, joint); flat: one value per (sample, joint); diffuse: N(0, 0.5).
    zero_mass_joint: that joint is <= 0 everywhere (no ReLU mass)."""
    rng = np.random.RandomState(seed)
    if kind == "peaked":
        x = rng.randn(B, J, nvox) * 2.0
        x[np.arange(B)[:, None], np.arange(J)[None, :], rng.randint(0, nvox, (B, J))] += 9.0
    elif kind == "flat":
        x = np.broadcast_to(rng.uniform(0.5, 3.0, (B, J, 1)), (B, J, nvox)).copy()
    elif kind == "diffuse":
        x = rng.randn(B, J, nvox) * 0.5
    else:
        raise ValueError(kind)
    x = np.clip(np.round(x / Q) * Q, -31.0, 31.0)
    if zero_mass_joint is not None:
        x[:, zero_mass_joint] = -np.abs(x[:, zero_mass_joint])
    out = (x + offset).astype(np.float32)
    assert np.array_equal(out.astype(np.float64) - offset, x), "logit + offset is not exact in float32"
    return out


def channels_last(x, vs):
    """(B, J, nvox) -> (B, nvox, vs) channels-last with NaN padding channels."""
    B, J, nvox = x.shape
    out = np.full((B, nvox, vs), np.nan, dtype=np.float32)
    out[:, :, :J] = x.transpose(0, 2, 1)
    return out


def reference(logits, coord, mult, mode, dtype=torch.float64, device="cpu"):
    """(key points (B, J, 3), volumes (B, J, nvox)) of op.py in `dtype`; logits (B, J, nvox), coord (B, nvox, 3) arrays or tensors."""
    l = torch.as_tensor(logits).to(device, dtype)
    c = torch.as_tensor(coord).to(device, dtype)
    z = l * mult
    if mode == 2:
        r = torch.relu(z)
        return (r @ c) / r.sum(-1, keepdim=True), r
    return torch_ops.integrate_tensor_3d_with_coordinates(z, c, bool(mode))


def scale_of(t, floor=1e-30):
    return max(float(t.abs().max()), float(t.std()) if t.numel() > 1 else 0.0, floor)


def err(a, ref, floor=1e-30):
    """max |a - ref| over the reference's scale (max |ref|, its spread, at least `floor`), both finite."""
    a, ref = a.double().cpu(), ref.double().cpu()
    return float((a - ref).abs().max()) / scale_of(ref, floor)


def grad_floor(g_kp, coord, mult):
    """Scale floor of a soft-argmax gradient, for references that are exactly zero (one voxel: the key point is that voxel's
    coordinate whatever its logit): multiplier x |d key points| x |coordinates|."""
    return mult * float(np.abs(g_kp).max()) * float(np.abs(coord).max())


def kp_err(a, ref, coord):
    """Key-point error over the coordinate scale (the spread of the coordinates the key points are averages of)."""
    return float((a.double().cpu() - ref.double().cpu()).abs().max()) / scale_of(torch.as_tensor(coord).double())


# ------------------------------------------------------------------------------------------ the scene builders' claims
@pytest.mark.parametrize("kind", KINDS)
def test_offset_scenes_have_one_float64_answer(kind):
    coord = coords_for(2, 1000, 1)
    base = reference(make_logits(2, 5, 1000, kind, 3), coord, 1.0, 1)
    for c in OFFSETS:
        kp, vol = reference(make_logits(2, 5, 1000, kind, 3, offset=c), coord, 1.0, 1)
        assert err(kp, base[0]) < 1e-12 and err(vol, base[1]) < 1e-12, c


def test_logits_times_100_are_exact_in_float32():
    x = make_logits(2, 17, 4096, "peaked", 5)
    assert np.array_equal((x * np.float32(100)).astype(np.float64), x.astype(np.float64) * 100)


def test_mode2_reference_is_the_relu_branch_of_integrate_tensor_2d():
    B, J, h, w = 2, 4, 9, 13
    x = make_logits(B, J, h * w, "peaked", 2)
    kp, vol = reference(x, pixel_grid(B, h, w), 1.7, 2)
    kp2, hm = torch_ops.integrate_tensor_2d(torch.from_numpy(x).double().reshape(B, J, h, w) * 1.7, softmax=False)
    assert torch.allclose(kp[..., :2], kp2, rtol=1e-12, atol=1e-12) and torch.equal(kp[..., 2], torch.zeros(B, J, dtype=torch.float64))
    assert torch.equal(vol, hm.reshape(B, J, -1))


def test_zero_mass_joint_has_a_nan_reference_key_point():
    x = make_logits(2, 3, 300, "diffuse", 4, zero_mass_joint=1)
    kp, _ = reference(x, coords_for(2, 300, 4), 1.0, 2)
    assert bool(torch.isnan(kp[:, 1]).all()) and bool(torch.isfinite(kp[:, [0, 2]]).all())


# ------------------------------------------------------------------------------------------ backward item code on the CPU
def reference_grad(logits, coord, mult, mode, g_kp, g_vol, dtype=torch.float64, device="cpu"):
    """d logits (B, J, nvox) of key points . g_kp (+ volumes . g_vol) by autograd in `dtype`."""
    l = torch.as_tensor(logits).to(device, dtype).requires_grad_(True)
    kp, vol = reference(l, coord, mult, mode, dtype, device)
    loss = (kp * torch.as_tensor(g_kp).to(device, dtype)).sum()
    if g_vol is not None:
        loss = loss + (vol * torch.as_tensor(g_vol).to(device, dtype)).sum()
    loss.backward()
    return l.grad, vol.detach()


def upstream(B, J, nvox, seed, coord_scale):
    """Key-point gradients (B, J, 3) and volume gradients (B, J, nvox), float32; the volume term is scaled to weigh about as much as the
    key-point term."""
    rng = np.random.RandomState(seed)
    return rng.randn(B, J, 3).astype(np.float32), (rng.randn(B, J, nvox) * coord_scale).astype(np.float32)


def host_backward(probs, coord, g_kp, g_vol, mult, mode):
    """lt_test_softargmax3d_bwd_host on CPU float32 tensors."""
    B, J, nvox = probs.shape
    grad = torch.empty(B, J, nvox)
    capi.softargmax3d_bwd_host(torch.as_tensor(probs).float().contiguous(), torch.as_tensor(coord).float().contiguous(),
                               torch.as_tensor(g_kp).float().contiguous(), None if g_vol is None else torch.as_tensor(g_vol).float().contiguous(),
                               grad, B, J, nvox, mult, mode)
    return grad


BWD_SCENES = {   # name -> (B, J, nvox, kind, coordinates)
    "B2 J5 216 peaked": (2, 5, 216, "peaked", "volume"),
    "B3 J4 1000 diffuse": (3, 4, 1000, "diffuse", "volume"),
    "B2 J3 9x13 pixels": (2, 3, 117, "peaked", "pixels"),
}


def bwd_scene(name):
    B, J, nvox, kind, cs = BWD_SCENES[name]
    coord = coords_for(B, nvox, len(name)) if cs == "volume" else pixel_grid(B, 9, 13)
    return make_logits(B, J, nvox, kind, len(name) + 1), coord


@pytest.mark.parametrize("name", list(BWD_SCENES))
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("with_gvol", [True, False])
@pytest.mark.parametrize("mult", [1.0, 1.7])
def test_backward_item_code_vs_float64(name, mode, with_gvol, mult):
    """probs = the float32 rounding of the float64 forward; yardstick rule against float32 autograd."""
    x, coord = bwd_scene(name)
    B, J, nvox = x.shape
    g_kp, g_vol = upstream(B, J, nvox, 3, 1.0 if mode == 0 else float(np.abs(coord).max()) / nvox)
    g_vol = g_vol if with_gvol else None
    want, vol = reference_grad(x, coord, mult, mode, g_kp, g_vol)
    yard, _ = reference_grad(x, coord, mult, mode, g_kp, g_vol, torch.float32)
    got = host_backward(vol.float(), coord, g_kp, g_vol, mult, mode)
    fl = 1e-6 * grad_floor(g_kp, coord, mult)
    e, y = err(got, want, fl), err(yard, want, fl)
    assert e <= max(2e-6, 2 * y), (e, y)


def test_backward_of_a_zero_mass_joint_is_zero():
    x = make_logits(2, 3, 300, "diffuse", 4, zero_mass_joint=1)
    coord = coords_for(2, 300, 4)
    g_kp, g_vol = upstream(2, 3, 300, 1, 1.0)
    want, vol = reference_grad(x, coord, 1.0, 2, g_kp, g_vol)
    got = host_backward(vol.float(), coord, g_kp, g_vol, 1.0, 2)
    assert bool((want[:, 1] == 0).all()) and bool((got[:, 1] == 0).all())
    assert err(got[:, [0, 2]], want[:, [0, 2]]) <= 2e-6


# ------------------------------------------------------------------------------------------ engine: fused tail only for a streamed layout
class _Recorder:
    def __init__(self, monkeypatch):
        self.calls = []
        monkeypatch.setattr(capi, "lib", lambda: None)
        for name in ("v2v_tail", "absmax", "conv_gather_weights", "fold_bn", "conv_fold_pack_weights", "stem_s2d", "coord_volume",
                     "unproject_aggregate", "softargmax3d", "softargmax3d_finish", "maxpool", "nchw_to_nhwc", "f32_to_s32", "s32_to_f32",
                     "cl_to_cf", "conv_tc_pack_weights", "conv_nd"):
            monkeypatch.setattr(capi, name, self.rec(name))
        monkeypatch.setattr(capi, "v2v_tail_stats", self.tail_stats)
        monkeypatch.setattr(capi, "conv_fold_weight_bytes", lambda k, co: k * k * k * ((co + 15) // 16 * 16) * 64 * 2)
        monkeypatch.setattr(capi, "conv_tc_weight_bytes", lambda t, ci, co: t * (ci // 32) * ((co + 15) // 16 * 16) * 64 * 2)
        monkeypatch.setattr(capi, "softargmax3d_workspace_bytes", lambda B, J, n: B * J * ((n + 2047) // 2048 * 5 + 2) * 4)

    def rec(self, name):
        def f(*a, **k):
            self.calls.append((name, a))
        return f

    def tail_stats(self, *a, **k):
        self.calls.append(("v2v_tail_stats", a))
        return 264

    def names(self):
        return [c[0] for c in self.calls]


@pytest.mark.parametrize("num_joints", [1, 12, 13, 16, 17, 20, 21, 32])
def test_engine_fuses_the_softargmax_statistics_only_for_a_streamed_layout(monkeypatch, num_joints):
    """The fused statistics (lt_v2v_tail_stats_fwd) are merged by lt_softargmax3d_finish_fwd, which streams compact logits of voxel
    stride 20..32: the engine fuses for J 17..20 (stride 20) and otherwise runs the tail and the full soft-argmax."""
    rec = _Recorder(monkeypatch)
    cfg = testing.make_config(num_layers=18, volume_size=32, num_joints=num_joints)
    model = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend="native", conv_mode="tc", use_cuda_graph=False).eval()
    e = eng_mod.NativeEngine(model, mode="tc", use_graph=False)
    B, V, S = 1, 2, 64
    z3 = torch.zeros(B, 3)
    kp, _, vols, _ = e.forward(torch.zeros(B, V, 3, S, S), torch.zeros(B, V, 3, 4), z3, z3, torch.zeros(3), torch.zeros(B, 9))
    assert tuple(kp.shape) == (B, num_joints, 3) and tuple(vols.shape) == (B, num_joints, 32, 32, 32)
    names = rec.names()
    fused = 17 <= num_joints <= 20
    assert names.count("v2v_tail_stats") == names.count("softargmax3d_finish") == int(fused)
    assert names.count("v2v_tail") + names.count("softargmax3d") == (0 if fused else 2)
    if not fused:
        a = [c[1] for c in rec.calls if c[0] == "softargmax3d"][0]
        assert a[2] == eng_mod._round_up(num_joints, 4) and a[3] == 1     # voxel stride = the tail's compact width, channels-last
