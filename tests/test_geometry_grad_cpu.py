"""Gradients with respect to the geometry -- projection matrices and coordinate volumes -- through the per-item code of
csrc/backward.cu and csrc/algebraic.cu on the CPU (the lt_test_*_host hooks), against float64 autograd of `torch_ops` and, for the
DLT, against central differences of the 50-digit solve of tests/test_algebraic_ref_cpu.py.

Bars of the unprojection (exact-geometry scenes, where every tap position is exact in float32): per element, a count of float32
roundings times the sum of the magnitudes of the terms that element adds up (`geometry_magnitudes`):
- the sample derivative of a channel quad: 4 taps x (product, fma) plus the gradient product: 9; the quad's channel sum: 4; the
  sum over the C / 4 quads: C / 4; the per-view sample gradient (softmax: exp, normaliser, 1 + s - out, products): 8;
- q: the scale by (w - 1) / h, the division by pz and the x, y products: 4;
- dP sums in float64 and rounds once: 1; dX sums 3 V float32 products: 3 V.
Camera scenes (positions not exact in float32): the suite's yardstick, native error <= max(bar, 2 x float32 torch_ops error).
The helpers here are shared with tests/test_gpu_geometry_grad.py."""
import mpmath
import numpy as np
import pytest
import torch

from lt_b200 import capi, torch_ops
from test_algebraic_ref_cpu import (MP_DPS, FD_STEP, ULP32, make_scene, dlt_reference, eta, spreads, eigvec_err, mp_point, err_over_bar,
                                    item, scene_id, SCENES)
from test_unproject_cpu import AGGS, HOST_SCENES, exact_scene, camera_scene, tensors, max_near_ties, err

EPS32 = 2.0 ** -24


# ---- unprojection -----------------------------------------------------------------------------------------------------

def geometry_reference(sc, agg, g, device="cpu", dtype=torch.float64):
    """Autograd of torch_ops: (d proj (B, V, 3, 4), d coord (B, nvox, 3)) for the upstream gradient g (B, nvox, C)."""
    f, p, c, cf = tensors(sc, device, dtype)
    p.requires_grad_(True)
    c.requires_grad_(True)
    B, nvox = c.shape[:2]
    out = torch_ops.unproject_heatmaps(f.permute(0, 1, 4, 2, 3), p, c.reshape(B, nvox, 1, 1, 3), agg, cf)
    out.backward(g.to(device, dtype).transpose(1, 2).reshape(out.shape))
    return p.grad, c.grad


def geometry_magnitudes(sc, agg, g):
    """Per element of (d proj, d coord) the sum of |terms| it adds up, float64 (see the module docstring), and the rounding count."""
    f, p, c, cf = tensors(sc, "cpu", torch.float64)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    g = g.double()
    s = torch_ops.sample_views(f.permute(0, 1, 4, 2, 3), p, c)                         # (B, V, C, nvox)
    gt = g.transpose(1, 2).unsqueeze(1)                                                 # (B, 1, C, nvox)
    if agg == "sum":
        gs = gt.abs().expand_as(s)
    elif agg == "conf":
        gs = (gt * cf.unsqueeze(-1)).abs()
    elif agg == "max":
        arg = s.argmax(1, keepdim=True)
        gs = torch.zeros_like(s).scatter_(1, arg, 1.0) * gt.abs()
    else:
        pr = torch.softmax(s, 1)
        out = (s * pr).sum(1, keepdim=True)
        gs = gt.abs() * pr * (1 + s.abs() + out.abs())
    X4 = torch.cat([c, torch.ones_like(c[..., :1])], -1)                                # (B, nvox, 4)
    proj = torch.einsum("bvrk,bnk->bvnr", p, X4)
    pz = proj[..., 2]
    live_depth = pz > 0
    zs = torch.where(pz == 0, torch.ones_like(pz), pz)
    x, y = proj[..., 0] / zs, proj[..., 1] / zs
    ix, iy = x / h * (w - 1), y / w * (h - 1)
    x0, y0 = ix.floor(), iy.floor()
    fm = f.abs().reshape(B, V, h * w, C)
    Mix = torch.zeros_like(ix)
    Miy = torch.zeros_like(ix)
    live = torch.zeros_like(live_depth)
    for dxo, dyo, wx, wy in ((0, 0, lambda: y0 + 1 - iy, lambda: x0 + 1 - ix), (1, 0, lambda: y0 + 1 - iy, lambda: ix - x0),
                             (0, 1, lambda: iy - y0, lambda: x0 + 1 - ix), (1, 1, lambda: iy - y0, lambda: ix - x0)):
        xt, yt = x0 + dxo, y0 + dyo
        inside = live_depth & (xt >= 0) & (xt <= w - 1) & (yt >= 0) & (yt <= h - 1)
        live |= inside
        o = (yt.clamp(0, h - 1) * w + xt.clamp(0, w - 1)).long()                        # (B, V, nvox)
        ft = torch.gather(fm, 2, o.unsqueeze(-1).expand(-1, -1, -1, C))                # (B, V, nvox, C)
        d = (gs.transpose(2, 3) * ft).sum(-1) * inside
        Mix += wx().abs() * d
        Miy += wy().abs() * d
    Mx, My = Mix * (w - 1) / h, Miy * (h - 1) / w
    az = zs.abs()
    mq = torch.stack([Mx / az, My / az, (Mx * x.abs() + My * y.abs()) / az], -1) * live.unsqueeze(-1)   # (B, V, nvox, 3)
    m_proj = torch.einsum("bvnr,bnk->bvrk", mq, X4.abs())
    m_coord = torch.einsum("bvnr,bvrk->bnk", mq, p[..., :3].abs())
    k_q = 9 + 4 + C // 4 + 8 + 4
    return m_proj, m_coord, (k_q + 1, k_q + 3 * V)


def geometry_host(sc, agg, g):
    """lt_test_unproject_aggregate_bwd_geom_host -> (d features, d conf or None, d proj (B, V, 3, 4), d coord (B, nvox, 3))."""
    f, p, c, cf = (torch.from_numpy(np.ascontiguousarray(a)) for a in sc)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gf = torch.zeros_like(f)
    gc = torch.zeros(B, V, C) if agg == "conf" else None
    gp = torch.full((B, V, 12), float("nan"))
    gx = torch.full((B, nvox, 3), float("nan"))
    capi.unproject_aggregate_bwd_geom_host(f, p.reshape(B, V, 12).contiguous(), c, cf if agg == "conf" else None, g.contiguous(), gf, gc,
                                           gp, gx, capi.AGG[agg])
    return gf, gc, gp.reshape(B, V, 3, 4), gx


def upstream(sc, agg, seed=7):
    B, nvox, C = sc.coord.shape[0], sc.coord.shape[1], sc.feats.shape[-1]
    g = torch.from_numpy(np.random.RandomState(seed).randn(B, nvox, C).astype(np.float32))
    if agg == "max":
        g = g.masked_fill(max_near_ties(sc), 0.0)
    return g


def worst_over_bar(got, want, mag, k):
    return float(((got.double() - want.double()).abs() / (k * EPS32 * mag + 1e-30)).max())


@pytest.mark.parametrize("name", list(HOST_SCENES))
@pytest.mark.parametrize("agg", AGGS)
def test_geometry_item_code_edge_scenes_vs_float64(name, agg):
    """Taps on 0 and size - 1, half-outside cells, pz = -1, 0 and 2^-60, non-square and one-pixel maps: every element of d proj and
    d coord within its rounding bar, and the feature / confidence gradients exactly those of the plain item code."""
    B, V, C, h, w, nvox, ident = HOST_SCENES[name]
    sc = exact_scene(B, V, C, h, w, nvox, seed=B * 1000 + V * 100 + C + h + w, identical_views=ident)
    g = upstream(sc, agg)
    want_p, want_x = geometry_reference(sc, agg, g)
    m_p, m_x, (k_p, k_x) = geometry_magnitudes(sc, agg, g)
    gf, gc, gp, gx = geometry_host(sc, agg, g)
    assert torch.isfinite(gp).all() and torch.isfinite(gx).all()
    wp, wx = worst_over_bar(gp, want_p, m_p, k_p), worst_over_bar(gx, want_x, m_x, k_x)
    print("%s %s: d proj err/bar %.3g, d coord err/bar %.3g" % (name, agg, wp, wx))
    assert wp <= 1.0 and wx <= 1.0
    # voxels that fail the depth test or see no tap contribute exactly nothing: a scene of only those gives exact zeros
    from test_unproject_cpu import host_backward
    pf, pc = host_backward(sc, agg, g)
    assert torch.equal(gf, pf) and (gc is None or torch.equal(gc, pc))


def test_geometry_dead_voxels_give_exact_zeros():
    """Every voxel at pz = -1, 0 or 2^-60 (the last projected far outside the map): d proj and d coord are exactly 0, never NaN."""
    sc = exact_scene(2, 3, 8, 8, 8, 60, seed=3)
    coord = sc.coord.copy()
    coord[..., 2] = np.array([-1.0, 0.0, 2.0 ** -60], np.float32)[np.arange(60) % 3]
    sc = sc._replace(coord=coord)
    for agg in AGGS:
        _, _, gp, gx = geometry_host(sc, agg, upstream(sc, agg))
        assert not gp.any() and not gx.any(), agg


@pytest.mark.parametrize("agg", AGGS)
def test_geometry_item_code_camera_scene_yardstick(agg):
    """Ring cameras, positions not exact: native error <= max(bar, 2 x the float32 torch_ops error), both against float64."""
    sc = camera_scene(2, 3, 8, 16, 12, 10, seed=11)
    g = upstream(sc, agg)
    want_p, want_x = geometry_reference(sc, agg, g)
    t32_p, t32_x = geometry_reference(sc, agg, g, dtype=torch.float32)
    m_p, m_x, (k_p, k_x) = geometry_magnitudes(sc, agg, g)
    _, _, gp, gx = geometry_host(sc, agg, g)
    for got, want, t32, bar in ((gp, want_p, t32_p, k_p * EPS32 * float(m_p.max())), (gx, want_x, t32_x, k_x * EPS32 * float(m_x.max()))):
        e, e32 = err(got, want), err(t32, want)
        b = bar / max(float(want.abs().max()), float(want.std()), 1e-30)
        print("camera %s: native %.3g, torch float32 %.3g, bar %.3g" % (agg, e, e32, b))
        assert e <= max(b, 2 * e32)


def test_geometry_entry_rejects_what_it_cannot_sum():
    lib = capi.lib()
    assert lib.lt_unproject_aggregate_bwd_geom(None, None, None, None, None, None, None, None, None, None, 0, 1, 1, 4, 1, 1, 1, 0, None) != 0
    dummy = torch.zeros(16)
    p = dummy.data_ptr()
    rc = lib.lt_unproject_aggregate_bwd_geom(p, p, p, None, p, p, None, None, None, p, 1 << 20, 1, 1, 12, 1, 1, 1, 0, None)
    assert rc != 0 and b"power of two" in lib.lt_last_error_string()


# ---- soft-argmax ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("softmax", [True, False])
def test_softargmax_coord_item_code_vs_float64(softmax):
    rng = np.random.RandomState(5)
    B, J, n = 2, 5, 6
    vols = torch.from_numpy(rng.randn(B, J, n, n, n).astype(np.float32) * 3)
    coord = torch.from_numpy(rng.randn(B, n, n, n, 3).astype(np.float32) * 100)
    gk = torch.from_numpy(rng.randn(B, J, 3).astype(np.float32))
    c64 = coord.double().requires_grad_(True)
    kp, probs64 = torch_ops.integrate_tensor_3d_with_coordinates(vols.double(), c64, softmax)
    kp.backward(gk.double())
    probs = probs64.detach().float().reshape(B, J, -1).contiguous()
    got = torch.full((B, n ** 3, 3), float("nan"))
    capi.softargmax3d_coord_bwd_host(probs, gk, got)
    mag = torch.einsum("bjn,bjk->bnk", probs.double().abs(), gk.double().abs())
    assert float(((got.double() - c64.grad.reshape(B, -1, 3)).abs() / ((J + 2) * EPS32 * mag + 1e-30)).max()) <= 1.0


def test_softargmax_coord_rejects_the_2d_mode():
    t = torch.zeros(8)
    assert capi.lib().lt_softargmax3d_coord_bwd(t.data_ptr(), t.data_ptr(), t.data_ptr(), 1, 1, 1, 2, None) != 0
    assert b"mode" in capi.lib().lt_last_error_string()


# ---- DLT --------------------------------------------------------------------------------------------------------------

def proj_reference(P, kp, cf, g):
    """Central differences of the 50-digit forward: d P (V, 3, 4) of g . X.  Moving P[v][0][c] moves A[2v][c] by -c_v, P[v][1][c]
    moves A[2v+1][c] by -c_v, P[v][2][c] moves A[2v][c] by c_v x and A[2v+1][c] by c_v y (the float32 rounding of A as identity)."""
    from test_algebraic_ref_cpu import dlt_rows32
    V = P.shape[0]
    A, _ = dlt_rows32(P, kp, cf)
    c = np.ones(V) if cf is None else cf.astype(np.float64)
    out = np.zeros((V, 3, 4))
    with mpmath.workdps(MP_DPS):
        h = mpmath.mpf(FD_STEP)
        Am = mpmath.matrix(A.tolist())

        def directional(moves):
            res = []
            for sign in (1, -1):
                Ah = Am.copy()
                for r, col, d in moves:
                    Ah[r, col] += sign * h * mpmath.mpf(float(d))
                res.append(mp_point(Ah))
            return float(sum(mpmath.mpf(float(g[i])) * (res[0][i] - res[1][i]) for i in range(3)) / (2 * h))

        for v in range(V):
            x, y = float(kp[v, 0]), float(kp[v, 1])
            for col in range(4):
                out[v, 0, col] = directional([(2 * v, col, -c[v])])
                out[v, 1, col] = directional([(2 * v + 1, col, -c[v])])
                out[v, 2, col] = directional([(2 * v, col, c[v] * x), (2 * v + 1, col, c[v] * y)])
    return out


def proj_bars(P, kp, cf, g, ref):
    """Per-element bars of d P (V, 3, 4), the construction of grad_bars in tests/test_algebraic_ref_cpu.py applied to
    d P[0] = -c G_A[r0], d P[1] = -c G_A[r1], d P[2] = c (x G_A[r0] + y G_A[r1])."""
    A, lam, E = ref["A"], ref["lam"], ref["E"]
    V = P.shape[0]
    s = spreads(ref)
    u = E[:, 0]
    rho = eta(V) * max((s[j] * s[k] + s[j] ** 2 + s[k] ** 2) / max(abs(lam[j] - lam[k]), 1e-300) for j in range(4) for k in range(j + 1, 4))
    rho = 4 * (rho + eigvec_err(ref)[3] / abs(u[3]))
    iw = 1.0 / abs(u[3])
    gu = np.abs(np.concatenate([g.astype(np.float64) * iw, [np.abs(g.astype(np.float64) * u[:3]).sum() * iw * iw]]))
    wabs = sum((gu @ np.abs(E[:, k])) / max(abs(lam[0] - lam[k]), 1e-300) * np.abs(E[:, k]) for k in range(1, 4))
    ua = np.abs(u)
    c = np.ones(V) if cf is None else np.abs(cf.astype(np.float64))
    out = np.zeros((V, 3, 4))
    for v in range(V):
        t = [(np.abs(A[2 * v + r]) @ wabs) * ua + (np.abs(A[2 * v + r]) @ ua) * wabs for r in range(2)]
        out[v, 0], out[v, 1] = c[v] * t[0], c[v] * t[1]
        out[v, 2] = c[v] * (abs(float(kp[v, 0])) * t[0] + abs(float(kp[v, 1])) * t[1])
    return rho * out


def proj_host(P, kp, conf, g):
    gp = torch.full(P.shape, float("nan"))
    capi.triangulate_dlt_proj_bwd_host(torch.from_numpy(P), torch.from_numpy(kp), None if conf is None else torch.from_numpy(conf),
                                       torch.from_numpy(g), gp)
    return gp.numpy()


PROJ_SCENES = ([dict(V=V, noise=2.0, conf=c) for V in (2, 4) for c in (None, "rand")]
               + [dict(V=4, step_deg=1.0, noise=2.0, conf="rand"), dict(V=4, far=True, conf="rand")]
               + [dict(V=4, conf=c) for c in ("graded1e-2", "graded1e-4", "graded1e-6", "zero_view", "tiny")])


@pytest.mark.parametrize("scene", PROJ_SCENES, ids=scene_id)
def test_dlt_proj_item_code_vs_high_precision(scene):
    P, kp, conf, g = make_scene(B=1, J=1, seed=2, **scene)
    gp = proj_host(P, kp, conf, g)
    assert np.isfinite(gp).all()
    Pi, kpi, cfi = item(P, kp, conf, 0, 0)
    ref = dlt_reference(Pi, kpi, cfi)
    worst = err_over_bar(gp[0], proj_reference(Pi, kpi, cfi, g[0, 0]), proj_bars(Pi, kpi, cfi, g[0, 0], ref))
    print("dlt d proj (host) %s: worst err/bar %.3g" % (scene_id(scene), worst))
    assert worst <= 1.0


def test_dlt_proj_sums_the_joints():
    """d P of J joints is the sum of the per-joint d P (float64 partials, one rounding at the end)."""
    P, kp, conf, g = make_scene(V=3, B=2, J=4, seed=6, conf="rand")
    whole = proj_host(P, kp, conf, g)
    parts = sum(proj_host(P, np.ascontiguousarray(kp[:, :, j:j + 1]), np.ascontiguousarray(conf[:, :, j:j + 1]),
                          np.ascontiguousarray(g[:, j:j + 1])).astype(np.float64) for j in range(4))
    assert np.allclose(whole, parts, rtol=4 * ULP32, atol=4 * ULP32 * np.abs(parts).max())


def test_dlt_proj_is_zero_on_an_exact_tie():
    P, kp, conf, g = make_scene(V=3, B=1, J=2, seed=3, conf="zero")
    gp = proj_host(P, kp, conf, g)
    assert np.isfinite(gp).all() and not gp.any()
