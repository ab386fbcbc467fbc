"""The fixed-order backward kernels that training under torch.use_deterministic_algorithms runs, checked on the CPU through their
lt_test_*_host hooks (the same per-item code the GPU runs): the unprojection backward without float atomics (csrc/backward.cu,
lt_unproject_aggregate_bwd_det) and V2V's max-pool backward (csrc/misc.cu, lt_maxpool3d_bwd).

Bars of the unprojection (exact-geometry scenes of tests/test_unproject_cpu.py, where every tap weight w_k is exact in float32): an
element of d features is a sum of n terms gs * w_k, one per (voxel, tap) with w_k != 0 on its pixel.  Against the float64
restatement of those terms it may differ by
- n - 1 float32 additions, summed in one order: (n - 1) u sum |terms|, u = 2^-24;
- per term, the rounding of the product gs * w_k (1) and the float32 per-view sample gradient gs: its bilinear sample, 4 taps of a
  product and an add (8), and for softmax the exp, normaliser, 1 + s - out and products (8): 17 u |term| at most,
so per element (n + 17) u sum |terms|, with the softmax magnitudes |g| p (1 + |s| + |out|) of tests/test_geometry_grad_cpu.py.
d conf of (sample, view, channel) sums nvox terms g * s (chunks in order, then the chunk partials): (nvox + 9) u sum |g| |s|.
The whole result is also held to the scale-relative bars tests/test_backward_host_cpu.py applies to the atomic kernel's hook.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lt_b200 import capi, torch_ops
from test_unproject_cpu import AGGS, exact_scene, max_near_ties, reference_grads, err, host_backward

EPS32 = 2.0 ** -24
K_TERM = 17
K_CONF = 9


def det_host(sc, agg, g, geom=False):
    """lt_test_unproject_aggregate_bwd_det_host -> (d features, d conf or None, d proj or None, d coord or None)."""
    f, p, c, cf = (torch.from_numpy(np.ascontiguousarray(a)) for a in sc)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gf = torch.zeros_like(f)
    gc = torch.zeros(B, V, C) if agg == "conf" else None
    gp = torch.full((B, V, 12), float("nan")) if geom else None
    gx = torch.full((B, nvox, 3), float("nan")) if geom else None
    capi.unproject_aggregate_bwd_det_host(f, p.reshape(B, V, 12).contiguous(), c, cf if agg == "conf" else None, g.contiguous(), gf, gc,
                                          gp, gx, capi.AGG[agg])
    return gf, gc, gp, gx


def term_reference(sc, agg, g):
    """float64 restatement of the per-tap terms: (d features, bar of d features, d conf, bar of d conf)."""
    f = torch.from_numpy(sc.feats).double()
    p = torch.from_numpy(sc.proj).double()
    c = torch.from_numpy(sc.coord).double()
    cf = torch.from_numpy(sc.conf).double()
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    c_ok = torch.nan_to_num(c, nan=0.0)
    s = torch_ops.sample_views(f.permute(0, 1, 4, 2, 3), p, c_ok).transpose(2, 3)      # (B, V, nvox, C)
    nan_vox = torch.isnan(c).any(-1)                                                     # (B, nvox): no tap (the kernels' rule)
    s = s.masked_fill(nan_vox[:, None, :, None], 0.0)
    gg = g.double().unsqueeze(1)                                                         # (B, 1, nvox, C)
    if agg == "sum":
        gs, mag = gg.expand_as(s), gg.abs().expand_as(s)
    elif agg == "conf":
        gs = gg * cf.unsqueeze(2)
        mag = gs.abs()
    elif agg == "max":
        oh = torch.zeros_like(s).scatter_(1, s.argmax(1, keepdim=True), 1.0)
        gs, mag = oh * gg, oh * gg.abs()
    else:
        pr = torch.softmax(s, 1)
        out = (s * pr).sum(1, keepdim=True)
        gs = gg * pr * (1 + s - out)
        mag = gg.abs() * pr * (1 + s.abs() + out.abs())
    X4 = torch.cat([c_ok, torch.ones_like(c_ok[..., :1])], -1)
    pj = torch.einsum("bvrk,bnk->bvnr", p, X4)
    pz = pj[..., 2]
    zs = torch.where(pz == 0, torch.ones_like(pz), pz)
    ix, iy = pj[..., 0] / zs / h * (w - 1), pj[..., 1] / zs / w * (h - 1)
    x0, y0 = ix.floor(), iy.floor()
    ref = torch.zeros(B, V, h * w, C, dtype=torch.float64)
    bar_mag = torch.zeros_like(ref)
    cnt = torch.zeros(B, V, h * w, dtype=torch.float64)
    conf_mag = torch.zeros(B, V, C, dtype=torch.float64)
    fm = f.abs().reshape(B, V, h * w, C)
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        xt, yt = x0 + dx, y0 + dy
        wt = (1 - (ix - xt).abs()) * (1 - (iy - yt).abs())
        inside = (pz > 0) & (xt >= 0) & (xt <= w - 1) & (yt >= 0) & (yt <= h - 1) & (wt != 0) & ~nan_vox[:, None, :]
        wt = torch.where(inside, wt, torch.zeros_like(wt))
        o = torch.where(inside, yt * w + xt, torch.zeros_like(xt)).long()                # (B, V, nvox)
        idx = o.unsqueeze(-1).expand(-1, -1, -1, C)
        ref.scatter_add_(2, idx, gs * wt.unsqueeze(-1))
        bar_mag.scatter_add_(2, idx, mag * wt.unsqueeze(-1))
        cnt.scatter_add_(2, o, inside.double())
        conf_mag += (g.double().abs().unsqueeze(1) * torch.gather(fm, 2, idx) * wt.unsqueeze(-1)).sum(2)
    bar = (cnt.unsqueeze(-1) + K_TERM) * EPS32 * bar_mag
    conf_ref = (gg * s).sum(2)
    conf_bar = (nvox + K_CONF) * EPS32 * conf_mag
    return ref.reshape(B, V, h, w, C), bar.reshape(B, V, h, w, C), conf_ref, conf_bar


def check_against_terms(sc, agg, g):
    want_f, bar_f, want_c, bar_c = term_reference(sc, agg, g)
    got_f, got_c, _, _ = det_host(sc, agg, g)
    over = ((got_f.double() - want_f).abs() - bar_f).max()
    assert float(over) <= 0.0, float(((got_f.double() - want_f).abs() / (bar_f + 1e-300)).max())
    if agg == "conf":
        assert float(((got_c.double() - want_c).abs() - bar_c).max()) <= 0.0
    return got_f, got_c


def upstream(sc, agg, seed=7):
    B, nvox, C = sc.coord.shape[0], sc.coord.shape[1], sc.feats.shape[-1]
    g = torch.from_numpy(np.random.RandomState(seed).randn(B, nvox, C).astype(np.float32))
    if agg == "max":
        g = g.masked_fill(max_near_ties(sc), 0.0)
    return g


SCENES = {   # name -> (B, V, C, h, w, nvox)
    "V1 C4 8x8 nvox 301": (2, 1, 4, 8, 8, 301),
    "V2 C32 8x16 nvox 257": (2, 2, 32, 8, 16, 257),
    "V4 C4 16x8 nvox 523": (1, 4, 4, 16, 8, 523),
    "V8 C4 8x8 nvox 199": (1, 8, 4, 8, 8, 199),
    "V2 C128 4x8 nvox 67": (1, 2, 128, 4, 8, 67),
}


@pytest.mark.parametrize("name", list(SCENES))
@pytest.mark.parametrize("agg", AGGS)
def test_fixed_order_backward_vs_float64_terms(name, agg):
    """Edge taps (on 0 and size - 1, half and fully outside), pz = -1, 0 and 2^-60 and a few NaN coordinates: every element of
    d features and d conf within its per-element bar, and the whole within the atomic hook's scale-relative bars."""
    B, V, C, h, w, nvox = SCENES[name]
    sc = exact_scene(B, V, C, h, w, nvox, seed=B * 1000 + V * 100 + C + h + w)
    sc.coord[:, ::37, 1] = np.nan
    g = upstream(sc, agg)
    got_f, got_c = check_against_terms(sc, agg, g)
    assert torch.isfinite(got_f).all()
    finite = sc._replace(coord=np.nan_to_num(sc.coord, nan=1e6).astype(np.float32))   # torch_ops has no NaN rule: project far away
    want_f, want_c = reference_grads(finite, agg, g)
    assert err(got_f, want_f) <= 2e-5
    if agg == "conf":
        assert err(got_c, want_c) <= 1e-4


@pytest.mark.parametrize("agg", AGGS)
def test_fixed_order_backward_every_voxel_in_one_cell(agg):
    """A far camera or a tiny cuboid: all nvox voxels share one floor cell, one sorted segment of nvox entries."""
    sc = exact_scene(2, 3, 8, 8, 8, 200, seed=11)
    sc.coord[:] = np.array([0.25, 0.5, 1.0], np.float32)
    g = upstream(sc, agg)
    got_f, _ = check_against_terms(sc, agg, g)
    assert int((got_f.abs().sum(-1) != 0).sum()) <= 2 * 3 * 4


@pytest.mark.parametrize("agg", AGGS)
def test_fixed_order_backward_geometry_outputs_match_geometry_hook(agg):
    """With the geometry outputs: d proj and d coord bit-equal to lt_unproject_aggregate_bwd_geom's hook, and d features / d conf
    bit-equal to the fixed-order hook without them."""
    from test_geometry_grad_cpu import geometry_host
    sc = exact_scene(2, 3, 8, 8, 16, 230, seed=5)
    g = upstream(sc, agg)
    gf, gc, gp, gx = det_host(sc, agg, g, geom=True)
    _, _, want_p, want_x = geometry_host(sc, agg, g)
    assert torch.equal(gp.reshape(want_p.shape), want_p) and torch.equal(gx, want_x)
    gf2, gc2, _, _ = det_host(sc, agg, g)
    assert torch.equal(gf, gf2) and (gc is None or torch.equal(gc, gc2))


def test_fixed_order_backward_sample_independent_of_batch():
    """Sample b's gradients do not depend on the other samples: a batch run equals per-sample runs bit for bit."""
    sc = exact_scene(3, 2, 8, 8, 8, 150, seed=9)
    g = upstream(sc, "conf")
    gf, gc, _, _ = det_host(sc, "conf", g)
    for b in range(3):
        one = type(sc)(*(a[b:b + 1] for a in sc))
        f1, c1, _, _ = det_host(one, "conf", g[b:b + 1])
        assert torch.equal(f1[0], gf[b]) and torch.equal(c1[0], gc[b])


def test_fixed_order_backward_close_to_atomic_hook():
    sc = exact_scene(2, 4, 8, 16, 16, 400, seed=3)
    g = upstream(sc, "softmax")
    got, _, _, _ = det_host(sc, "softmax", g)
    atomic, _ = host_backward(sc, "softmax", g)
    assert err(got, atomic) <= 1e-6


# ---- max-pool backward ------------------------------------------------------------------------------------------------------

def pool_input(N, C, D, H, W, seed, case):
    rng = np.random.RandomState(seed)
    x = rng.randint(-3, 4, (N, C, D, H, W)).astype(np.float32)          # many ties
    flat = x.reshape(-1)
    n = flat.size
    if case in ("inf", "all"):
        flat[rng.choice(n, n // 7, replace=False)] = np.inf
        flat[rng.choice(n, n // 7, replace=False)] = -np.inf
    if case in ("nan", "all"):
        flat[rng.choice(n, n // 9, replace=False)] = np.nan               # some windows get one NaN, some several
    if case == "all":
        x[0, 0, :2, :2, :2] = -np.inf                                     # a window of only -inf: its first element gets the gradient
    return torch.from_numpy(x)


def pool_cases():
    for shape in ((2, 3, 4, 4, 4), (1, 4, 5, 7, 9), (2, 8, 3, 2, 5)):
        for case in ("ties", "inf", "nan", "all"):
            for cl in (False, True):
                yield shape, case, cl


def bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("shape,case,cl", list(pool_cases()))
def test_maxpool3d_backward_host_bit_equal_torch_cpu(shape, case, cl):
    x = pool_input(*shape, seed=sum(shape), case=case)
    if cl:
        x = x.contiguous(memory_format=torch.channels_last_3d)
    gy = torch.from_numpy(np.random.RandomState(1).randn(*F.max_pool3d(x, 2, 2).shape).astype(np.float32))
    gy[0, 0, 0, 0, 0] = -0.0
    xr = x.clone().requires_grad_(True)
    F.max_pool3d(xr, 2, 2).backward(gy)
    gx = torch.full_like(x, float("nan"))
    assert gx.stride() == x.stride()
    capi.maxpool3d_bwd_host(x, gy, gx, 2)
    assert torch.equal(bits(gx), bits(xr.grad))
