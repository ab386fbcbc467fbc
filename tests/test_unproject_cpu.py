"""Exact-geometry scenes for the unprojection kernels, and the backward's per-item code (csrc/backward.cu) on the CPU against
float64 autograd of `torch_ops` (itself pinned to the reference by tests/test_oracle_vs_reference.py).

An exact-geometry scene puts every bilinear tap position where float32 computes it exactly: projection rows with dyadic entries,
a depth row that gives pz = 1 for valid voxels, power-of-two maps and voxel coordinates on a dyadic lattice.  The pixel coordinate
ix = t * (w - 1), with t = x / h, then comes out exact from both kernel formulas (the division form of make_taps / bwd_taps and the
reciprocal-multiply form of unproject_v2_kernel), so the kernels can be held to a few float32 roundings of the feature arithmetic
whatever the position.  The lattice sweeps ix and iy over about [-2, size + 1]: taps exactly on 0 and size - 1, cells half outside
the map and cells fully outside it.  Some voxels sit at pz = -1 and pz = 0 (masked) and pz = 2^-60 (valid, but projected far
outside the map, so the kernels' index clamping is reached).  Projections, coordinates, features and confidences differ per sample.
The helpers here are shared with tests/test_gpu_unproject.py.
"""
from collections import namedtuple

import numpy as np
import pytest
import torch

from lt_b200 import capi, testing, torch_ops
from oracle import vol_oracle as O

AGGS = ("sum", "max", "softmax", "conf")
EDGE_Z = (-1.0, 0.0, 2.0 ** -60)
Scene = namedtuple("Scene", "feats proj coord conf")   # (B, V, h, w, C), (B, V, 3, 4), (B, nvox, 3), (B, V, C); float32 numpy


def lattice(h, w):
    """Dyadic values t (step 1/64) for which t * (size - 1) sweeps about [-2, size + 1] on the smaller side of the map that is
    longer than one pixel (a one-pixel side maps every t to 0)."""
    sides = [s for s in (h, w) if s > 1]
    size = min(sides) if sides else 2
    k = int(np.ceil(max(2.25 / (size - 1), 0.125) * 64))
    return np.arange(-k, 64 + k + 1) / 64.0


def exact_scene(B, V, C, h, w, nvox, seed, identical_views=False, feat_scale=1.0):
    """x = h * t_x and y = w * t_y with t = +-U (+ 1), U one of the voxel's X and Y: t_x / h and t_y / w are exact, and t = 0, 1 are
    on the lattice for every view.  Rows of sample b differ from those of sample 0 in every view (combination index shifted by 3b)."""
    rng = np.random.RandomState(seed)
    lat = lattice(h, w)
    L = len(lat)
    coord = np.ones((B, nvox, 3))
    i = np.arange(nvox)
    for b in range(B):
        coord[b, :, 0] = lat[rng.permutation(L)[i % L]]
        coord[b, :, 1] = lat[rng.permutation(L)[(i + i // L) % L]]
        edge = (i + 5 * b) % 13 == 0
        coord[b, edge, 2] = np.array(EDGE_Z)[(i[edge] // 13) % 3]
    proj = np.zeros((B, V, 3, 4))
    base = rng.randint(0, 8, V)
    for b in range(B):
        for v in range(V):
            k = (base[v] + 3 * b) % 8
            u, sx, sy = k & 1, (1, -1)[(k >> 1) & 1], (1, -1)[k >> 2]
            proj[b, v, 0, u], proj[b, v, 0, 3] = h * sx, h * (sx < 0)
            proj[b, v, 1, 1 - u], proj[b, v, 1, 3] = w * sy, w * (sy < 0)
            proj[b, v, 2, 2] = 1.0
    feats = (rng.randn(B, V, h, w, C) * feat_scale).astype(np.float32)
    conf = rng.uniform(0.25, 1.25, (B, V, C)).astype(np.float32)
    if identical_views:
        proj[:, 1], feats[:, 1], conf[:, 1] = proj[:, 0], feats[:, 0], conf[:, 0]
    return Scene(feats, proj.astype(np.float32), coord.astype(np.float32), conf)


def camera_scene(B, V, C, h, w, n, seed, feat_scale=1.0):
    """Ring cameras (a different ring phase per sample) and a 2.8 m cube of n^3 voxels: positions are not exact in float32."""
    rng = np.random.RandomState(seed)
    proj = np.stack([np.stack([O.projection_after_resize(c.K, c.R, c.t, (48, 48), (h, w))
                               for c in testing.make_cameras(V, image_size=48, radius=3000.0, phase=0.3 + 0.4 * b)]) for b in range(B)])
    coord = np.stack([O.coord_volume(rng.randn(3) * 100 + [0, 0, 900], 2800.0, n).reshape(-1, 3) for _ in range(B)])
    feats = (rng.randn(B, V, h, w, C) * feat_scale).astype(np.float32)
    conf = rng.uniform(0.25, 1.25, (B, V, C)).astype(np.float32)
    return Scene(feats, proj.astype(np.float32), coord.astype(np.float32), conf)


def tensors(sc, device, dtype):
    return [torch.as_tensor(a).to(device, dtype) for a in sc]


def samples(feats, proj, coord):
    """Per-view samples (B, V, C, nvox) of channels-last features (B, V, h, w, C)."""
    return torch_ops.sample_views(feats.permute(0, 1, 4, 2, 3), proj, coord)


def reference(sc, agg, device="cpu", dtype=torch.float64):
    """Aggregated volume (B, nvox, C) of torch_ops in `dtype`."""
    f, p, c, cf = tensors(sc, device, dtype)
    B, nvox = c.shape[:2]
    out = torch_ops.unproject_heatmaps(f.permute(0, 1, 4, 2, 3), p, c.reshape(B, nvox, 1, 1, 3), agg, cf)
    return out.reshape(B, -1, nvox).transpose(1, 2)


def reference_partial(sc, agg, device="cpu"):
    """View-partial aggregate (B, P, nvox, C) in float64."""
    f, p, c, cf = tensors(sc, device, torch.float64)
    return torch_ops.partial_aggregate(samples(f, p, c), agg, cf).transpose(2, 3)


def reference_grads(sc, agg, g, device="cpu", dtype=torch.float64):
    """Autograd of torch_ops: (d features (B, V, h, w, C), d conf (B, V, C) or None) for the upstream gradient g (B, nvox, C)."""
    f, p, c, cf = tensors(sc, device, dtype)
    f.requires_grad_(True)
    cf.requires_grad_(agg == "conf")
    B, nvox = c.shape[:2]
    out = torch_ops.unproject_heatmaps(f.permute(0, 1, 4, 2, 3), p, c.reshape(B, nvox, 1, 1, 3), agg, cf)
    out.backward(g.to(device, dtype).transpose(1, 2).reshape(out.shape))
    return f.grad, (cf.grad if agg == "conf" else None)


def max_near_ties(sc, device="cpu"):
    """(B, nvox, C) mask of the max aggregation's near-ties: float64 top-two gap non-zero but below 1e-5 of the output's scale.  At
    such an entry float32 may pick another view than float64 does, so the tests zero its upstream gradient in every run."""
    f, p, c, _ = tensors(sc, device, torch.float64)
    s = samples(f, p, c)
    if s.shape[1] < 2:
        return torch.zeros(s.shape[0], s.shape[3], s.shape[2], dtype=torch.bool, device=device)
    top = s.topk(2, dim=1).values
    gap = (top[:, 0] - top[:, 1]).transpose(1, 2)
    scale = max(float(top[:, 0].abs().max()), float(top[:, 0].std()))
    return (gap > 0) & (gap < 1e-5 * scale)


def scale_of(t):
    return max(float(t.abs().max()), float(t.std()), 1e-30)


def err(a, ref):
    """max |a - ref| over the reference's scale (max |ref|, its spread)."""
    return float((a.double().cpu() - ref.double().cpu()).abs().max()) / scale_of(ref.double().cpu())


# ------------------------------------------------------------------------------------------ the scene builder's claim
@pytest.mark.parametrize("hw", [(1, 1), (1, 4), (2, 1), (2, 2), (8, 32), (32, 8), (16, 16)])
def test_exact_scene_positions_are_exact_in_float32(hw):
    h, w = hw
    sc = exact_scene(2, 3, 4, h, w, 700, seed=h * 100 + w)
    X, Y, Z = (sc.coord[..., k][:, None, :].astype(np.float32) for k in range(3))
    P = sc.proj[:, :, :, :, None]
    f32 = np.float32
    px, py, pz = (X * P[:, :, r, 0] + Y * P[:, :, r, 1] + Z * P[:, :, r, 2] + P[:, :, r, 3] for r in range(3))
    X64, Y64, Z64 = (sc.coord[..., k][:, None, :].astype(np.float64) for k in range(3))
    P64 = P.astype(np.float64)
    px64, py64, pz64 = (X64 * P64[:, :, r, 0] + Y64 * P64[:, :, r, 1] + Z64 * P64[:, :, r, 2] + P64[:, :, r, 3] for r in range(3))
    assert px.dtype == np.float32 and np.array_equal(px, px64) and np.array_equal(py, py64) and np.array_equal(pz, pz64)
    zs = np.where(pz64 == 0, 1.0, pz64)
    ix64 = (px64 / zs / h) * (w - 1)
    iy64 = (py64 / zs / w) * (h - 1)
    # division form (make_taps, bwd_taps)
    z32 = np.where(pz == 0, f32(1), pz)
    ix = ((f32(2) * ((px / z32) / f32(h) - f32(0.5)) + f32(1)) / f32(2)) * f32(w - 1)
    iy = ((f32(2) * ((py / z32) / f32(w) - f32(0.5)) + f32(1)) / f32(2)) * f32(h - 1)
    assert ix.dtype == np.float32 and np.array_equal(ix, ix64) and np.array_equal(iy, iy64)
    # reciprocal-multiply form (unproject_v2_kernel) at pz = 1, where 1/pz is 1
    ok = pz == 1
    ix2 = ((f32(2) * ((px * f32(1)) * (f32(1) / f32(h)) - f32(0.5)) + f32(1)) * f32(0.5)) * f32(w - 1)
    iy2 = ((f32(2) * ((py * f32(1)) * (f32(1) / f32(w)) - f32(0.5)) + f32(1)) * f32(0.5)) * f32(h - 1)
    assert np.array_equal(ix2[ok], ix64[ok]) and np.array_equal(iy2[ok], iy64[ok])
    # every depth class, and for each side longer than one pixel every tap-edge class
    for z in (1.0,) + EDGE_Z:
        assert (pz64 == z).any(), z
    for i, size in ((ix64[ok], w), (iy64[ok], h)):
        if size == 1:
            assert (i == 0).all()
            continue
        classes = {"on 0": i == 0, "on size-1": i == size - 1, "interior": (i > 0) & (i < size - 1) & (i != np.floor(i)),
                   "half out low": (i > -1) & (i < 0), "half out high": (i > size - 1) & (i < size),
                   "out low": i <= -1, "out high": i >= size, "below -1.5": i < -1.5, "above size+0.5": i > size + 0.5}
        for name, m in classes.items():
            assert m.any(), (name, size)


def test_exact_scene_projections_differ_per_sample():
    sc = exact_scene(3, 4, 4, 8, 8, 64, seed=1)
    for b in (1, 2):
        for v in range(4):
            assert not np.array_equal(sc.proj[b, v], sc.proj[0, v])
        assert not np.array_equal(sc.coord[b], sc.coord[0]) and not np.array_equal(sc.feats[b], sc.feats[0])


# ------------------------------------------------------------------------------------------ backward item code on the CPU
def _p(t):
    assert not t.is_cuda and t.is_contiguous() and t.dtype == torch.float32
    return t.data_ptr()


def host_backward(sc, agg, g, with_gconf=True):
    """lt_test_unproject_aggregate_bwd_host: the backward kernel's per-item code on the CPU.  g (B, nvox, C) float32."""
    f, p, c, cf = (torch.from_numpy(np.ascontiguousarray(a)) for a in sc)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gf = torch.zeros_like(f)
    gc = torch.zeros(B, V, C) if (agg == "conf" and with_gconf) else None
    rc = capi.lib().lt_test_unproject_aggregate_bwd_host(_p(f), _p(p), _p(c), _p(cf) if agg == "conf" else None, _p(g.contiguous()),
                                                         _p(gf), None if gc is None else _p(gc), B, V, C, h, w, nvox, capi.AGG[agg])
    assert rc == 0, capi.lib().lt_last_error_string()
    return gf, gc


HOST_SCENES = {   # name -> (B, V, C, h, w, nvox, identical views)
    "B2 V3 C8 8x32": (2, 3, 8, 8, 32, 300, False),
    "B3 V2 C4 32x8": (3, 2, 4, 32, 8, 300, False),
    "B2 V4 C4 1x4": (2, 4, 4, 1, 4, 120, False),
    "B2 V3 C4 2x1": (2, 3, 4, 2, 1, 120, False),
    "B2 V3 C8 4x4 identical views": (2, 3, 8, 4, 4, 200, True),
}


@pytest.mark.parametrize("name", list(HOST_SCENES))
@pytest.mark.parametrize("agg", AGGS)
def test_backward_item_code_edge_scenes_vs_float64(name, agg):
    """Bar 2e-6 of scale: positions are exact, so what remains is float32 rounding of the samples, the softmax and the scatter."""
    B, V, C, h, w, nvox, ident = HOST_SCENES[name]
    sc = exact_scene(B, V, C, h, w, nvox, seed=B * 1000 + V * 100 + C + h + w, identical_views=ident)
    g = torch.from_numpy(np.random.RandomState(7).randn(B, nvox, C).astype(np.float32))
    if agg == "max":
        near = max_near_ties(sc)
        assert float(near.float().mean()) < 0.01
        g = g.masked_fill(near, 0.0)
    want_f, want_c = reference_grads(sc, agg, g)
    got_f, got_c = host_backward(sc, agg, g)
    assert err(got_f, want_f) <= 2e-6, err(got_f, want_f)
    if agg == "conf":
        assert err(got_c, want_c) <= 2e-6, err(got_c, want_c)
        got_f2, none = host_backward(sc, agg, g, with_gconf=False)
        assert none is None and torch.equal(got_f2, got_f)
