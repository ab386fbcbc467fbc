"""The geometry-gradient kernels on the H100 against high-precision references, over their dispatch:
lt_unproject_aggregate_bwd_geom (csrc/backward.cu), lt_triangulate_dlt_proj_bwd (csrc/algebraic.cu) and lt_softargmax3d_coord_bwd.

- Unprojection: a case table over every channel-quad width C / 4 = 1 ... 32 (the warp butterfly of geom_emit and its full-warp
  mask), V across the 64 views view_proj keeps in shared memory, nvox across the 8192-voxel dP chunks and across the geometry
  kernel's grid cap, and the edge maps of tests/test_unproject_cpu.py HOST_SCENES; every case under all four aggregations.
  Exact-geometry scenes hold every element of d proj and d coord to the per-element bars of `geometry_magnitudes`; camera scenes
  to the suite's yardstick, native error <= max(bar, 2 x float32 torch_ops error), both against float64.
  Outputs and the workspace start as a NaN sentinel inside guard bands; the coordinates sit inside NaN guards of one dP chunk, so a
  read past them shows up as NaN.  d proj alone and d coord alone are bit-identical to the same output of the launch writing both,
  and a second launch repeats both bit for bit.  grad_features is accumulated into a non-zero start and compared with the plain
  lt_unproject_aggregate_bwd: bit for bit at nvox = 1, where every feature element and d conf entry receives one addition; elsewhere
  both kernels add with float atomics in no fixed order, so both are held to the yardstick against float64 instead.
- DLT: every scene of tests/test_algebraic_ref_cpu.py SCENES and tests/test_geometry_grad_cpu.py PROJ_SCENES through the device,
  each element held to `proj_bars` around the 50-digit central differences `proj_reference`; item counts across the 128-thread
  CTA, the per-item float64 partials read back from the workspace, the joint merge checked alone (bit for bit: the float64 sum in
  joint order, rounded once), the exact tie and the point at infinity.
- Soft-argmax coordinate backward: nvox across the 256-thread CTA and the grid cap of sm_count x 8 CTAs, J 1 / 17 / 40, B up to
  3000, probabilities of softmax and ReLU volumes from float64 torch_ops, bar (J + 2) 2^-24 sum_j |p g| against float64 einsum.
- Autograd of the three hybrid ops for every subset of inputs requiring grad, with the None slots of each backward, against float64
  autograd of the torch backend; and, in child processes under torch.profiler, which geometry kernels each case launches.

Measured on an H100 80GB HBM3 (700 W power limit), worst err / bar over all cases (printed per case with -s):
- unprojection, exact scenes: d proj 0.099, d coord 0.10; camera scenes at most 0.41 of max(bar, 2 x float32 torch_ops error);
- DLT d P: 0.48 over the 43 scenes; item counts 0.49 (merged samples), items against the host hook 0 float32 ulp-bars;
- coordinate backward: 0.44.
Each of these kernel mutations fails a test here: the warp butterfly stopping one step early, view_proj serving v >= 64 from the
shared copy, the dP merge skipping its last chunk, dp_partial without the min(nvox, ...) clip, dX summing V - 1 views, geom_q with
the (w - 1) / h and (h - 1) / w scales swapped, the DLT merge skipping the last joint, cf on one of the two dP[2] terms, the tie rule
against the largest eigenvalue, and the coordinate backward's grid-stride loop running once.
"""
import itertools
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from lt_b200 import autograd_ops, capi, op, torch_ops
from test_algebraic_ref_cpu import (SCENES, ULP32, dlt_reference, err_over_bar, item, make_scene, point_at_infinity_scene, scene_id)
from test_geometry_grad_cpu import (EPS32, PROJ_SCENES, geometry_magnitudes, geometry_reference, proj_bars, proj_host, proj_reference,
                                    upstream, worst_over_bar)
from test_gpu_unproject import Guarded, guarded_features
from test_unproject_cpu import AGGS, HOST_SCENES, camera_scene, err, exact_scene, reference_grads, tensors

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BAR = 2e-6                      # the plain unprojection backward's bar on exact scenes (tests/test_gpu_unproject.py)
GEOM_CHUNK = 8192               # kGeomChunk of csrc/backward.cu: voxels per dP partial
CHUNK_GUARD = 3 * GEOM_CHUNK    # floats of NaN guard around the coordinates and after the workspace: one chunk of reads


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(t):
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


# ---- unprojection: the case table --------------------------------------------------------------------------------------
# name -> (B, V, C, h, w, nvox, identical views 0 and 1); the names say which branch of the dispatch each case is there for.
UNPROJ_CASES = {
    "C4 V1 nvox1": (2, 1, 4, 4, 4, 1, False),
    "C128 V2 nvox1 C/4=32": (2, 2, 128, 4, 8, 1, False),
    "C8 V3 nvox31": (2, 3, 8, 8, 32, 31, False),
    "C16 V8 C/4=4": (2, 8, 16, 16, 16, 300, False),
    "C32 V3 C/4=8": (3, 3, 32, 32, 8, 500, False),
    "C64 V4 C/4=16": (2, 4, 64, 8, 8, 300, False),
    "C128 V3 C/4=32": (2, 3, 128, 4, 8, 300, False),
    "C4 V63": (2, 63, 4, 4, 4, 100, False),
    "C8 V64": (2, 64, 8, 4, 4, 100, False),
    "C16 V65 V>64": (2, 65, 16, 2, 4, 100, False),
    "C4 V66 V>64": (2, 66, 4, 4, 8, 150, False),
    "C128 V66 V>64 C/4=32": (1, 66, 128, 2, 4, 40, False),
    "C128 V80 d-conf 40 KB": (1, 80, 128, 2, 2, 33, False),
    "C4 V2 nvox8191 one partial chunk": (1, 2, 4, 8, 8, GEOM_CHUNK - 1, False),
    "C8 V3 nvox8192 one full chunk": (1, 3, 8, 8, 8, GEOM_CHUNK, False),
    "C4 V2 nvox8193 multi-chunk partial": (2, 2, 4, 8, 8, GEOM_CHUNK + 1, False),
    "C4 V3 nvox3x8192+17 multi-chunk partial": (2, 3, 4, 16, 16, 3 * GEOM_CHUNK + 17, False),
    "C8 V2 nvox64^3 grid-stride": (1, 2, 8, 16, 16, 64 ** 3, False),
    **{"edge " + k: v for k, v in HOST_SCENES.items()},
}
UNPROJ_PARAMS = [(name, agg) for name in UNPROJ_CASES for agg in AGGS]


def case_scene(name):
    B, V, C, h, w, nvox, ident = UNPROJ_CASES[name]
    return exact_scene(B, V, C, h, w, nvox, seed=sum(map(ord, name)) % 10007, identical_views=ident)


def feature_start(sc):
    """A non-zero start for grad_features, exact in float32 (the kernels accumulate into it)."""
    rng = np.random.RandomState(1)
    return torch.from_numpy((rng.randint(-8, 9, sc.feats.shape) / 16.0).astype(np.float32)).to(DEV)


def geom_device(sc, agg, g, start, want_proj=True, want_coord=True, want_gconf=True):
    """lt_unproject_aggregate_bwd_geom on guarded buffers -> (grad_features, grad_conf or None, d proj (B, V, 3, 4) or None,
    d coord (B, nvox, 3) or None).  Asserts every geometry output written and finite and every guard intact."""
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    F = guarded_features(f)
    X = Guarded((B, nvox, 3), guard=CHUNK_GUARD, fill=c)
    gf = start.clone()
    gc = torch.zeros(B, V, C, device=DEV) if (agg == "conf" and want_gconf) else None
    gp = Guarded((B, V, 12)) if want_proj else None
    gx = Guarded((B, nvox, 3)) if want_coord else None
    ws = Guarded((capi.unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox) // 4,), guard=CHUNK_GUARD)
    capi.unproject_aggregate_bwd_geom(F.t, p.reshape(B, V, 12).contiguous(), X.t, cf if agg == "conf" else None, g.to(DEV).contiguous(),
                                      gf, gc, None if gp is None else gp.t, None if gx is None else gx.t, capi.AGG[agg], ws.t)
    torch.cuda.synchronize()
    assert F.guards_intact() and X.guards_intact() and ws.guards_intact()
    for o in (gp, gx):
        if o is not None:
            assert o.guards_intact() and o.unwritten() == 0 and bool(torch.isfinite(o.t).all())
    return gf, gc, None if gp is None else gp.t.reshape(B, V, 3, 4), None if gx is None else gx.t


def plain_device(sc, agg, g, start, want_gconf=True):
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    B, V, h, w, C = f.shape
    gf = start.clone()
    gc = torch.zeros(B, V, C, device=DEV) if (agg == "conf" and want_gconf) else None
    capi.unproject_aggregate_bwd(f, p.reshape(B, V, 12).contiguous(), c, cf if agg == "conf" else None, g.to(DEV).contiguous(), gf, gc,
                                 capi.AGG[agg])
    torch.cuda.synchronize()
    return gf, gc


@pytest.mark.parametrize("name,agg", UNPROJ_PARAMS, ids=["%s-%s" % p for p in UNPROJ_PARAMS])
def test_unproject_geom_case_vs_float64(name, agg):
    sc = case_scene(name)
    B, V, C, h, w, nvox, ident = UNPROJ_CASES[name]
    g = upstream(sc, agg)
    start = feature_start(sc)
    gf, gc, gp, gx = geom_device(sc, agg, g, start)
    # every element of d proj and d coord within its rounding bar
    want_p, want_x = geometry_reference(sc, agg, g)
    m_p, m_x, (k_p, k_x) = geometry_magnitudes(sc, agg, g)
    wp, wx = worst_over_bar(gp.cpu(), want_p, m_p, k_p), worst_over_bar(gx.cpu(), want_x, m_x, k_x)
    print("unproject geom %-42s %-7s d proj err/bar %.3g, d coord err/bar %.3g" % (name, agg, wp, wx))
    assert wp <= 1.0 and wx <= 1.0, (wp, wx)
    if agg == "max" and ident:
        # views 0 and 1 tie exactly everywhere: the first view takes the gradient, view 1 none at all
        assert not gp[:, 1].any()
    # a second launch, and each output alone: bit for bit
    _, _, gp2, gx2 = geom_device(sc, agg, g, start)
    _, _, gp_only, _ = geom_device(sc, agg, g, start, want_coord=False)
    _, _, _, gx_only = geom_device(sc, agg, g, start, want_proj=False)
    assert same_bits(gp2, gp) and same_bits(gx2, gx) and same_bits(gp_only, gp) and same_bits(gx_only, gx)
    if agg == "conf":   # without the d conf accumulator: the same geometry
        gf_nc, none, gp_nc, gx_nc = geom_device(sc, agg, g, start, want_gconf=False)
        assert none is None and same_bits(gp_nc, gp) and same_bits(gx_nc, gx)
    # feature and confidence gradients: the plain kernel's
    pf, pc = plain_device(sc, agg, g, start)
    if nvox == 1:
        assert same_bits(gf, pf) and (gc is None or same_bits(gc, pc))
        if agg == "conf":
            assert same_bits(gf_nc, pf)
    # elsewhere the atomics' order varies from run to run: the suite's yardstick, max(bar, 2 x float32 torch_ops error)
    want_f, want_c = reference_grads(sc, agg, g)
    y32_f, y32_c = reference_grads(sc, agg, g, dtype=torch.float32)
    for got in (gf, pf):
        assert err(got.cpu().double() - start.cpu().double(), want_f) <= max(BAR, 2 * err(y32_f, want_f))
    if agg == "conf":
        assert max(err(gc, want_c), err(pc, want_c)) <= max(BAR, 2 * err(y32_c, want_c))


CAMERA_CASES = {   # name -> (B, V, C, h, w, n): ring cameras, n^3 voxels
    "camera C32 V4 16x12 n10": (2, 4, 32, 16, 12, 10),
    "camera C8 V65 9x13 n6": (2, 65, 8, 9, 13, 6),
    "camera C128 V3 8x8 n8": (1, 3, 128, 8, 8, 8),
}


@pytest.mark.parametrize("name", list(CAMERA_CASES))
@pytest.mark.parametrize("agg", AGGS)
def test_unproject_geom_camera_scene_yardstick(name, agg):
    B, V, C, h, w, n = CAMERA_CASES[name]
    sc = camera_scene(B, V, C, h, w, n, seed=len(name))
    g = upstream(sc, agg)
    want_p, want_x = geometry_reference(sc, agg, g)
    t32_p, t32_x = geometry_reference(sc, agg, g, dtype=torch.float32)
    m_p, m_x, (k_p, k_x) = geometry_magnitudes(sc, agg, g)
    _, _, gp, gx = geom_device(sc, agg, g, feature_start(sc))
    for what, got, want, t32, bar in (("d proj", gp, want_p, t32_p, k_p * EPS32 * float(m_p.max())),
                                      ("d coord", gx, want_x, t32_x, k_x * EPS32 * float(m_x.max()))):
        e, e32 = err(got, want), err(t32, want)
        b = bar / max(float(want.abs().max()), float(want.std()), 1e-30)
        print("unproject geom %-26s %-7s %s: native %.3g, torch float32 %.3g, bar %.3g" % (name, agg, what, e, e32, b))
        assert e <= max(b, 2 * e32)


def _geom_rc(B, V, C, nvox, agg, ws_bytes, conf=True, grad_conf=True):
    """lt_unproject_aggregate_bwd_geom with placeholder pointers: only for arguments it refuses before any launch."""
    lib = capi.lib()
    dummy = torch.zeros(16, device=DEV)
    p = dummy.data_ptr()
    rc = lib.lt_unproject_aggregate_bwd_geom(p, p, p, p if conf else None, p, p, p if grad_conf else None, p, p, p, ws_bytes, B, V, C, 2, 2,
                                             nvox, agg, None)
    return rc, lib.lt_last_error_string()


def test_unproject_geom_refusals():
    conf = capi.AGG["conf"]
    need = capi.unproject_aggregate_bwd_geom_workspace_bytes
    for C in (12, 20, 24, 36, 96):                                   # C / 4 not a power of two
        rc, msg = _geom_rc(1, 2, C, 10, conf, 1 << 30)
        assert rc != 0 and b"power of two" in msg, C
    rc, msg = _geom_rc(1, 2, 256, 10, conf, 1 << 30)                 # C > 128
    assert rc != 0 and b"power of two" in msg
    rc, msg = _geom_rc(256, 256, 4, 10, capi.AGG["sum"], 1 << 40, conf=False, grad_conf=False)   # B V = 65536
    assert rc != 0 and b"batch too large" in msg
    rc, msg = _geom_rc(1, 81, 128, 10, conf, 1 << 30)                # V C = 10368 floats: over the 40 KB d conf accumulator
    assert rc != 0 and b"too large for the confidence-gradient accumulator" in msg
    rc, msg = _geom_rc(1, 4, 8, 9000, conf, need(1, 4, 9000) - 1)    # one byte short
    assert rc != 0 and b"workspace" in msg


# ---- DLT projection gradient ---------------------------------------------------------------------------------------------
def dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def dlt_proj_device(P, kp, conf, g):
    """lt_triangulate_dlt_proj_bwd on a guarded output and a NaN-filled, guarded workspace -> (d P (B, V, 3, 4), the per-item float64
    partials (B, J, V, 12) it left in the workspace), both numpy."""
    B, V, J = kp.shape[:3]
    out = Guarded(P.shape)
    nbytes = capi.triangulate_dlt_proj_bwd_workspace_bytes(B, V, J)
    ws = Guarded((nbytes // 4,))
    capi.triangulate_dlt_proj_bwd(dev(P), dev(kp), dev(conf), dev(g), out.t, ws.t)
    torch.cuda.synchronize()
    assert out.guards_intact() and out.unwritten() == 0 and ws.guards_intact()
    return out.t.cpu().numpy(), ws.t.cpu().numpy().view(np.float64).reshape(B, J, V, 12)


def merged_in_order(partial):
    """The merge kernel's sum: float64 over the joints in order, rounded once -> (B, V, 3, 4) float32."""
    s = np.zeros(partial.shape[:1] + partial.shape[2:])
    for j in range(partial.shape[1]):
        s = s + partial[:, j]
    return s.astype(np.float32).reshape(partial.shape[0], partial.shape[2], 3, 4)


def item_over_bar(P, kp, conf, g, b, j, got):
    Pi, kpi, cfi = item(P, kp, conf, b, j)
    ref = dlt_reference(Pi, kpi, cfi)
    return err_over_bar(got, proj_reference(Pi, kpi, cfi, g[b, j]), proj_bars(Pi, kpi, cfi, g[b, j], ref))


DLT_SCENES = list({scene_id(s): s for s in SCENES + PROJ_SCENES}.values())


@pytest.mark.parametrize("scene", DLT_SCENES, ids=scene_id)
def test_dlt_proj_bwd_vs_high_precision(scene):
    P, kp, conf, g = make_scene(B=1, J=1, seed=2, **scene)
    gp, partial = dlt_proj_device(P, kp, conf, g)
    assert np.isfinite(gp).all() and np.isfinite(partial).all()
    assert np.array_equal(gp, merged_in_order(partial))
    worst = item_over_bar(P, kp, conf, g, 0, 0, gp[0])
    print("dlt d proj (device) %-44s worst err/bar %.3g" % (scene_id(scene), worst))
    assert worst <= 1.0


def _close_to_host(got, want):
    """Device vs the host hook (the same per-item code; only the device's float64 FMA contraction differs): two float32 ulps, or
    1e-9 of the sample's largest element where a value is the difference of much larger terms."""
    scale = np.abs(want).max(axis=(1, 2, 3), keepdims=True)
    return float(np.max(np.abs(got - want) / (2 * ULP32 * np.abs(want) + 1e-9 * scale + 1e-30)))


@pytest.mark.parametrize("BJ", [(1, 1), (127, 1), (128, 1), (129, 1), (8, 17), (300, 17)], ids=lambda s: "B%dxJ%d" % s)
def test_dlt_proj_bwd_item_counts(BJ):
    """B J = 1, 127, 128, 129, 136 and 5100 items: every output written once, nothing past the end.  The merge alone: the output
    is the float64 joint-order sum of the partials, rounded once.  Sampled items (first, last, either side of 128) against the 50-digit
    reference through their partials; the merged d P of their samples against the float64 sum of the per-joint references within the
    bars summed; every sample against the host hook within a few float32 ulps."""
    B, J = BJ
    P, kp, conf, g = make_scene(V=4, B=B, J=J, seed=B * 1000 + J, conf="rand")
    gp, partial = dlt_proj_device(P, kp, conf, g)
    assert np.isfinite(gp).all() and np.isfinite(partial).all()
    assert np.array_equal(gp, merged_in_order(partial))
    e_host = _close_to_host(gp, proj_host(P, kp, conf, g))
    spots = sorted({i for i in (0, 127, 128, B * J - 1) if i < B * J})
    worst_item = max(item_over_bar(P, kp, conf, g, i // J, i % J, partial[i // J, i % J].reshape(4, 3, 4)) for i in spots)
    worst_merged = 0.0
    for b in sorted({i // J for i in spots}):
        want, bar = np.zeros((4, 3, 4)), np.zeros((4, 3, 4))
        for j in range(J):
            Pi, kpi, cfi = item(P, kp, conf, b, j)
            want += proj_reference(Pi, kpi, cfi, g[b, j])
            bar += proj_bars(Pi, kpi, cfi, g[b, j], dlt_reference(Pi, kpi, cfi))
        worst_merged = max(worst_merged, err_over_bar(gp[b], want, bar))
    print("dlt d proj B=%d J=%d: device vs host %.3g ulp-bars, items err/bar %.3g, merged err/bar %.3g" % (B, J, e_host, worst_item, worst_merged))
    assert e_host <= 1.0 and worst_item <= 1.0 and worst_merged <= 1.0
    gp2, partial2 = dlt_proj_device(P, kp, conf, g)
    assert np.array_equal(gp2.view(np.int32), gp.view(np.int32)) and np.array_equal(partial2.view(np.int64), partial.view(np.int64))


def test_dlt_proj_bwd_is_zero_on_an_exact_tie():
    P, kp, conf, g = make_scene(V=3, B=2, J=5, seed=3, conf="zero")
    gp, partial = dlt_proj_device(P, kp, conf, g)
    assert not gp.any() and not partial.any()


def test_dlt_proj_bwd_point_at_infinity():
    """u[3] = 0 exactly for item (0, 0) (see point_at_infinity_scene): the backward divides by u[3], so that item's partials are NaN
    and with them sample 0's d P.  Its other item's partial and sample 1 are finite and within their bars."""
    P0, kp0, conf0, g0 = point_at_infinity_scene(V=3)
    P1, kp1, conf1, g1 = make_scene(V=3, B=1, J=2, seed=5, conf="rand")
    P, kp, conf, g = (np.concatenate(x) for x in ((P0, P1), (kp0, kp1), (conf0, conf1), (g0, g1)))
    gp, partial = dlt_proj_device(P, kp, conf, g)
    assert np.isnan(gp[0]).all() and np.isnan(partial[0, 0]).all()
    assert np.isfinite(partial[0, 1]).all() and np.isfinite(partial[1]).all() and np.isfinite(gp[1]).all()
    assert item_over_bar(P, kp, conf, g, 0, 1, partial[0, 1].reshape(3, 3, 4)) <= 1.0
    want = sum(proj_reference(*item(P, kp, conf, 1, j), g[1, j]) for j in range(2))
    bar = sum(proj_bars(*item(P, kp, conf, 1, j), g[1, j], dlt_reference(*item(P, kp, conf, 1, j))) for j in range(2))
    assert err_over_bar(gp[1], want, bar) <= 1.0


# ---- soft-argmax coordinate backward -------------------------------------------------------------------------------------
def grid_cap_voxels():
    """Voxels one pass of softargmax_coord_bwd_kernel covers: sm_count x 8 CTAs of 256 threads."""
    return sm_count() * 8 * 256


COORD_CASES = [(3, 17, 1), (2, 40, 255), (2, 17, 256), (3, 1, 257), (2, 40, 257), (1, 17, "cap"), (1, 17, "cap+1"), (2, 1, "cap+1"),
               (1, 40, 64 ** 3 + 1), (3000, 17, 7), (2048, 40, 2)]


def coord_case_nvox(n):
    return {"cap": grid_cap_voxels(), "cap+1": grid_cap_voxels() + 1}.get(n, n)


@pytest.mark.parametrize("softmax", [1, 0], ids=["softmax", "relu"])
@pytest.mark.parametrize("case", COORD_CASES, ids=lambda c: "B%s-J%s-nvox%s" % c)
def test_softargmax_coord_bwd_vs_float64(case, softmax):
    B, J, n = case
    nvox = coord_case_nvox(n)
    gen = torch.Generator(device=DEV).manual_seed(B * 100 + J + nvox % 1000)
    logits = torch.randn((B, J, nvox), generator=gen, device=DEV, dtype=torch.float64) * 4
    coord = torch.randn((B, nvox, 3), generator=gen, device=DEV, dtype=torch.float64) * 500
    _, probs64 = torch_ops.integrate_tensor_3d_with_coordinates(logits, coord, bool(softmax))
    probs = probs64.float().contiguous()
    if not softmax:
        assert bool((probs == 0).any()) or nvox * B * J < 8
    gk = (torch.randn((B, J, 3), generator=gen, device=DEV, dtype=torch.float64)).float()
    out = Guarded((B, nvox, 3))
    capi.softargmax3d_coord_bwd(probs, gk, out.t, B, J, nvox, softmax)
    torch.cuda.synchronize()
    assert out.guards_intact() and out.unwritten() == 0
    want = torch.einsum("bjn,bjk->bnk", probs.double(), gk.double())
    mag = torch.einsum("bjn,bjk->bnk", probs.double().abs(), gk.double().abs())
    worst = float(((out.t.double() - want).abs() / ((J + 2) * EPS32 * mag + 1e-30)).max())
    print("coord bwd B=%d J=%d nvox=%d %s: worst err/bar %.3g" % (B, J, nvox, "softmax" if softmax else "relu", worst))
    assert worst <= 1.0
    again = torch.empty_like(out.t)
    capi.softargmax3d_coord_bwd(probs, gk, again, B, J, nvox, softmax)
    assert same_bits(again, out.t)


def test_softargmax_coord_bwd_refuses_mode_2_on_the_device():
    p = torch.full((1, 2, 8), 0.125, device=DEV)
    with pytest.raises(RuntimeError, match="mode must be 0"):
        capi.softargmax3d_coord_bwd(p, torch.zeros(1, 2, 3, device=DEV), torch.empty(1, 8, 3, device=DEV), 1, 2, 8, 2)


# ---- autograd through the hybrid ops -------------------------------------------------------------------------------------
def subsets(names):
    return [s for r in range(1, len(names) + 1) for s in itertools.combinations(names, r)]


def _unproject_leaves(sc, dtype, want):
    f, p, c, cf = tensors(sc, DEV, dtype)
    B = f.shape[0]
    n = round(c.shape[1] ** (1 / 3))
    leaves = dict(heat=f.permute(0, 1, 4, 2, 3).contiguous(), proj=p, coord=c.reshape(B, n, n, n, 3).contiguous(), conf=cf)
    for k in want:
        leaves[k].requires_grad_(True)
    return leaves


UNPROJ_SLOTS = ("heat", "proj", "coord", "conf")


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("n", [1, 4])
def test_autograd_unproject_every_subset(agg, n):
    """op.unproject_heatmaps(backend="hybrid"): for each subset of (heat, proj, coord, conf) requiring grad, the backward's slots are
    None exactly where no gradient is wanted, and each gradient is that of float64 autograd of the torch backend (per-element bars
    for proj and coord, the plain kernel's bar for heat and conf).  The heat gradient of a subset with proj or coord (the geometry
    kernel) equals that of the plain path: bit for bit at n = 1 (one voxel), within the bar otherwise."""
    sc = exact_scene(2, 3, 8, 8, 8, n ** 3, seed=20 + n)
    B, V, h, w, C = sc.feats.shape
    g = upstream(sc, agg)
    g_vol = g.transpose(1, 2).reshape(B, C, n, n, n).contiguous()
    ref = _unproject_leaves(sc, torch.float64, UNPROJ_SLOTS if agg == "conf" else UNPROJ_SLOTS[:3])
    out = torch_ops.unproject_heatmaps(ref["heat"], ref["proj"], ref["coord"], agg, ref["conf"])
    out.backward(g_vol.to(DEV, torch.float64))
    want_p, want_x = geometry_reference(sc, agg, g)
    m_p, m_x, (k_p, k_x) = geometry_magnitudes(sc, agg, g)
    heat_plain = None
    for want in subsets(UNPROJ_SLOTS if agg == "conf" else UNPROJ_SLOTS[:3]):
        lv = _unproject_leaves(sc, torch.float32, want)
        vol = op.unproject_heatmaps(lv["heat"], lv["proj"], lv["coord"], agg, lv["conf"] if agg == "conf" else None, backend="hybrid")
        grads = vol.grad_fn.apply(g_vol.to(DEV))
        assert len(grads) == 5 and grads[4] is None
        for k, gr in zip(UNPROJ_SLOTS, grads):
            assert (gr is None) == (k not in want), (want, k)
            if gr is None:
                continue
            assert gr.shape == lv[k].shape
            if k == "proj":
                assert worst_over_bar(gr.cpu(), want_p, m_p, k_p) <= 1.0, want
            elif k == "coord":
                assert worst_over_bar(gr.reshape(B, -1, 3).cpu(), want_x, m_x, k_x) <= 1.0, want
            else:
                assert err(gr, ref[k].grad) <= BAR, (want, k, err(gr, ref[k].grad))
        if want == ("heat",):
            heat_plain = grads[0]
        elif "heat" in want and n == 1:
            assert same_bits(grads[0], heat_plain), want


@pytest.mark.parametrize("softmax", [True, False])
def test_autograd_integrate_every_subset(softmax):
    """op.integrate_tensor_3d_with_coordinates(backend="hybrid") for each subset of (volumes, coord): the None slots, and the
    gradients of both outputs' upstream against float64 autograd of torch_ops (yardstick rule)."""
    rng = np.random.RandomState(3)
    B, J, n = 2, 17, 6
    vols = torch.from_numpy(rng.randn(B, J, n, n, n) * 3).to(DEV)
    coord = torch.from_numpy(rng.randn(B, n, n, n, 3) * 100).to(DEV)
    g_kp = torch.from_numpy(rng.randn(B, J, 3)).to(DEV)
    g_vol = torch.from_numpy(rng.randn(B, J, n, n, n) * 1e-2).to(DEV)

    def torch_grads(dt):
        v, c = vols.to(dt).clone().requires_grad_(True), coord.to(dt).clone().requires_grad_(True)
        kp, pr = torch_ops.integrate_tensor_3d_with_coordinates(v, c, softmax)
        return torch.autograd.grad((kp * g_kp.to(dt)).sum() + (pr * g_vol.to(dt)).sum(), (v, c))

    want, yard = torch_grads(torch.float64), torch_grads(torch.float32)
    for sub in subsets(("vol", "coord")):
        v = vols.float().requires_grad_("vol" in sub)
        c = coord.float().requires_grad_("coord" in sub)
        kp, pr = op.integrate_tensor_3d_with_coordinates(v, c, softmax, backend="hybrid")
        grads = kp.grad_fn.apply(g_kp.float(), g_vol.float())
        assert len(grads) == 3 and grads[2] is None
        assert (grads[0] is None) == ("vol" not in sub) and (grads[1] is None) == ("coord" not in sub)
        for got, w, y, k in zip(grads[:2], want, yard, ("vol", "coord")):
            if k in sub:
                e, e32 = err(got, w), err(y, w)
                print("integrate autograd %s %s: native %.3g, torch float32 %.3g" % (sub, k, e, e32))
                assert got.shape == w.shape and e <= max(BAR, 2 * e32), (sub, k, e, e32)


def test_autograd_triangulate_every_subset():
    """multiview.triangulate_batch_of_points(backend="hybrid") for each subset of (proj, points, conf): the None slots and the
    gradients against float64 autograd of the torch backend."""
    from lt_b200 import multiview
    P, kp, conf, g = (torch.from_numpy(a).to(DEV) for a in make_scene(V=4, B=3, J=17, seed=8, conf="rand"))
    p64, k64, c64 = (t.double().requires_grad_(True) for t in (P, kp, conf))
    out = multiview.triangulate_batch_of_points(p64, k64, c64, backend="torch")
    want = torch.autograd.grad((out * g.double()).sum(), (p64, k64, c64))
    for sub in subsets(("proj", "points", "conf")):
        args = [t.clone().requires_grad_(k in sub) for t, k in zip((P, kp, conf), ("proj", "points", "conf"))]
        X = multiview.triangulate_batch_of_points(*args, backend="hybrid")
        grads = X.grad_fn.apply(g)
        assert len(grads) == 3
        for k, gr, w in zip(("proj", "points", "conf"), grads, want):
            assert (gr is None) == (k not in sub), (sub, k)
            if gr is not None:
                assert gr.shape == w.shape and err(gr, w) <= 1e-4, (sub, k, err(gr, w))


# ---- launches ------------------------------------------------------------------------------------------------------------
GEOM_KERNELS = ["unproject_bwd_geom_kernel", "unproject_geom_dp_partial_kernel", "unproject_geom_dp_merge_kernel", "unproject_geom_dx_kernel",
                "softargmax_coord_bwd_kernel", "triangulate_dlt_proj_bwd_kernel", "triangulate_dlt_proj_merge_kernel"]
_NAME = re.compile("|".join(GEOM_KERNELS + ["unproject_bwd_kernel"]))


def _kernel_names(prof):
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    names = []
    for e in sorted(evs, key=lambda e: e.start_ns()):
        m = _NAME.search(e.name())
        if m:
            names.append(m.group(0))
    return names


def profiled_launches():
    """Each unprojection case with both outputs, d proj only and d coord only; each coordinate-backward and DLT item-count case; under
    torch.profiler -> (geometry kernels launched in order, [(case, kernel expected)])."""
    from torch.profiler import ProfilerActivity, profile
    runs, expected = [], []
    geom = GEOM_KERNELS[0]
    for name in UNPROJ_CASES:
        sc = case_scene(name)
        f, p, c, cf = tensors(sc, DEV, torch.float32)
        B, V, h, w, C = f.shape
        nvox = c.shape[1]
        g = torch.zeros(B, nvox, C, device=DEV)
        ws = torch.empty(capi.unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox), dtype=torch.uint8, device=DEV)
        for wp, wx in ((True, True), (True, False), (False, True)):
            gp = torch.empty(B, V, 12, device=DEV) if wp else None
            gx = torch.empty(B, nvox, 3, device=DEV) if wx else None
            runs.append(lambda f=f, p=p.reshape(B, V, 12).contiguous(), c=c, cf=cf, g=g, gp=gp, gx=gx, ws=ws: capi.unproject_aggregate_bwd_geom(
                f, p, c, cf, g, torch.zeros_like(f), torch.zeros_like(cf), gp, gx, capi.AGG["conf"], ws))
            ks = [geom] + (GEOM_KERNELS[1:3] if wp else []) + ([GEOM_KERNELS[3]] if wx else [])
            expected += [("%s proj %d coord %d" % (name, wp, wx), k) for k in ks]
    for B, J, n in COORD_CASES:
        nvox = coord_case_nvox(n)
        probs = torch.full((B, J, nvox), 1.0 / nvox, device=DEV)
        runs.append(lambda probs=probs, B=B, J=J, nvox=nvox: capi.softargmax3d_coord_bwd(probs, torch.ones(B, J, 3, device=DEV),
                                                                                         torch.empty(B, nvox, 3, device=DEV), B, J, nvox, 1))
        expected.append(("coord B%d J%d nvox%d" % (B, J, nvox), GEOM_KERNELS[4]))
    for B, J in ((1, 1), (127, 1), (128, 1), (129, 1), (8, 17), (300, 17)):
        P, kp, conf, g = (dev(a) for a in make_scene(V=4, B=B, J=J, seed=1, conf="rand"))
        ws = torch.empty(capi.triangulate_dlt_proj_bwd_workspace_bytes(B, 4, J), dtype=torch.uint8, device=DEV)
        runs.append(lambda P=P, kp=kp, conf=conf, g=g, ws=ws: capi.triangulate_dlt_proj_bwd(P, kp, conf, g, torch.empty_like(P), ws))
        expected += [("dlt B%d J%d" % (B, J), k) for k in GEOM_KERNELS[5:]]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in runs:
            r()
        torch.cuda.synchronize()
    return _kernel_names(prof), expected


def op_level_launches():
    """One hybrid backward of each op per subset of inputs requiring grad, each under its own profiler window -> {label: geometry and
    plain unprojection backward kernels launched}."""
    from torch.profiler import ProfilerActivity, profile
    sc = exact_scene(2, 3, 8, 8, 8, 64, seed=2)
    P, kp, conf, g = (dev(a) for a in make_scene(V=3, B=2, J=5, seed=1, conf="rand"))
    from lt_b200 import multiview
    out = {}

    def record(label, fn):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        out[label] = _kernel_names(prof)

    for want in subsets(UNPROJ_SLOTS):
        lv = _unproject_leaves(sc, torch.float32, want)
        vol = op.unproject_heatmaps(lv["heat"], lv["proj"], lv["coord"], "conf", lv["conf"], backend="hybrid")
        record("unproject " + "+".join(want), lambda vol=vol: vol.sum().backward())
    for want in subsets(("vol", "coord")):
        v = torch.randn(2, 4, 4, 4, 4, device=DEV).requires_grad_("vol" in want)
        c = torch.randn(2, 4, 4, 4, 3, device=DEV).requires_grad_("coord" in want)
        kp3, _ = op.integrate_tensor_3d_with_coordinates(v, c, True, backend="hybrid")
        record("integrate " + "+".join(want), lambda kp3=kp3: kp3.sum().backward())
    for want in subsets(("proj", "points", "conf")):
        args = [t.clone().requires_grad_(k in want) for t, k in zip((P, kp, conf), ("proj", "points", "conf"))]
        X = multiview.triangulate_batch_of_points(*args, backend="hybrid")
        record("triangulate " + "+".join(want), lambda X=X: X.sum().backward())
    return out


def _child(call):
    """Run `call` of this module in a child process (a profiling session leaves state behind in the process that makes a later
    session miss its first kernel records) -> its JSON result."""
    code = ("import json, sys; sys.path[:0] = %r; import test_gpu_geometry_grad_ref as t; print('RESULT ' + json.dumps(t.%s()))"
            % ([HERE, ROOT], call))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable] + flags + ["-c", code], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])


def test_case_table_launches_every_geometry_kernel():
    """Each case launches the kernels it is named for, in order: the geometry kernel, then the dP partial and merge when d proj is
    wanted and the dX kernel when d coord is; the coordinate backward; the DLT item and merge kernels.  Together: all seven."""
    names, expected = _child("profiled_launches")
    assert len(names) == len(expected), (len(names), len(expected))
    for i, (got, (case, want)) in enumerate(zip(names, expected)):
        assert got == want, (i, case, got, want)
    reached = {}
    for case, k in expected:
        reached.setdefault(k, []).append(case)
    for k in GEOM_KERNELS:
        print("%-34s reached by %d cases, e.g. %s" % (k, len(reached.get(k, [])), reached.get(k, ["none"])[-1]))
    assert set(names) == set(GEOM_KERNELS)
    for branch in ("C/4=32", "V>64", "multi-chunk partial", "one full chunk", "nvox1", "grid-stride", "d-conf 40 KB"):
        named = [name for name in UNPROJ_CASES if branch in name]
        assert named, branch
        for name in named:      # each launch of the case: the geometry kernel, then the dP pair and / or the dX kernel
            assert {k for c, k in expected if c.startswith(name + " proj")} == set(GEOM_KERNELS[:4]), (branch, name)


def test_op_level_geometry_launched_only_when_geometry_needs_grad():
    launched = _child("op_level_launches")
    for label, names in launched.items():
        op_name, want = label.split(" ", 1)
        want = want.split("+")
        if op_name == "unproject":
            geo = "proj" in want or "coord" in want
            assert (GEOM_KERNELS[0] in names) == geo and ("unproject_bwd_kernel" in names) == (not geo), (label, names)
            assert (GEOM_KERNELS[1] in names) == ("proj" in want) and (GEOM_KERNELS[3] in names) == ("coord" in want), (label, names)
        elif op_name == "integrate":
            assert (GEOM_KERNELS[4] in names) == ("coord" in want), (label, names)
        else:
            assert (GEOM_KERNELS[5] in names) == ("proj" in want) and (GEOM_KERNELS[6] in names) == ("proj" in want), (label, names)
    assert len(launched) == 15 + 3 + 7
