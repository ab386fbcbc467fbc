"""Geometry gradients on the H100: lt_unproject_aggregate_bwd_geom, lt_softargmax3d_coord_bwd and lt_triangulate_dlt_proj_bwd on
NaN-guarded buffers, against the float64 references and bars of tests/test_geometry_grad_cpu.py, bit-identical over repeats,
through the hybrid autograd ops, under the sync debug mode and inside a CUDA graph; and a hybrid volumetric training step, whose
geometry needs no gradient, launching no geometry kernel."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import autograd_ops, capi, multiview, op, testing
from test_algebraic_ref_cpu import make_scene
from test_geometry_grad_cpu import (EPS32, geometry_magnitudes, geometry_reference, proj_host, upstream, worst_over_bar)
from test_unproject_cpu import AGGS, camera_scene, err, exact_scene, reference_grads

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GUARD = 64


def guarded(shape, fill=float("nan")):
    """A CUDA tensor of `shape` inside a NaN-filled allocation: (view, whole buffer)."""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), fill, device=DEV)
    return buf[GUARD:GUARD + n].view(shape), buf


def guards_intact(buf):
    return bool(torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all())


def device_geometry(sc, agg, g, grad_features_fill=0.0, want_proj=True, want_coord=True):
    f, p, c, cf = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in sc)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gf = torch.full_like(f, grad_features_fill)
    gc = torch.zeros(B, V, C, device=DEV) if agg == "conf" else None
    gp, gp_buf = guarded((B, V, 12)) if want_proj else (None, None)
    gx, gx_buf = guarded((B, nvox, 3)) if want_coord else (None, None)
    ws = torch.full((capi.unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox),), 255, dtype=torch.uint8, device=DEV)
    capi.unproject_aggregate_bwd_geom(f, p.reshape(B, V, 12).contiguous(), c, cf if agg == "conf" else None, g.to(DEV).contiguous(),
                                      gf, gc, gp, gx, capi.AGG[agg], ws)
    torch.cuda.synchronize()
    for t, buf in ((gp, gp_buf), (gx, gx_buf)):
        if t is not None:
            assert guards_intact(buf) and bool(torch.isfinite(t).all())
    return gf, gc, None if gp is None else gp.reshape(B, V, 3, 4), gx


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("shape", [(2, 3, 8, 8, 32, 300), (3, 2, 4, 32, 8, 300), (2, 5, 16, 4, 4, 200)])
def test_unproject_geom_small_exact_scenes(agg, shape):
    """Every element written, guards intact, within the CPU bars; grad_features accumulated into; the feature / conf gradients
    within the plain kernel's yardstick (2e-6 of scale against float64)."""
    B, V, C, h, w, nvox = shape
    sc = exact_scene(B, V, C, h, w, nvox, seed=B * 100 + V * 10 + C)
    g = upstream(sc, agg)
    want_p, want_x = geometry_reference(sc, agg, g)
    m_p, m_x, (k_p, k_x) = geometry_magnitudes(sc, agg, g)
    gf, gc, gp, gx = device_geometry(sc, agg, g, grad_features_fill=1.0)
    assert worst_over_bar(gp.cpu(), want_p, m_p, k_p) <= 1.0 and worst_over_bar(gx.cpu(), want_x, m_x, k_x) <= 1.0
    want_f, want_c = reference_grads(sc, agg, g)
    assert err(gf.cpu() - 1.0, want_f) <= 2e-6
    if agg == "conf":
        assert err(gc.cpu(), want_c) <= 2e-6
    # either output alone
    _, _, gp2, _ = device_geometry(sc, agg, g, want_coord=False)
    _, _, _, gx2 = device_geometry(sc, agg, g, want_proj=False)
    assert torch.equal(gp2, gp) and torch.equal(gx2, gx)


@pytest.mark.parametrize("agg", AGGS)
def test_unproject_geom_full_size_camera_scene(agg):
    """B = 2, V = 4, 64^3, C = 32: the yardstick against float64 torch_ops on the GPU, and bit-identical repeats."""
    sc = camera_scene(2, 4, 32, 64, 64, 64, seed=3)
    g = upstream(sc, agg) if agg != "max" else torch.from_numpy(np.random.RandomState(7).randn(2, 64 ** 3, 32).astype(np.float32))
    if agg == "max":
        from test_unproject_cpu import max_near_ties
        g = g.masked_fill(max_near_ties(sc, DEV).cpu(), 0.0)
    want_p, want_x = geometry_reference(sc, agg, g, device=DEV)
    t32_p, t32_x = geometry_reference(sc, agg, g, device=DEV, dtype=torch.float32)
    _, _, gp, gx = device_geometry(sc, agg, g)
    for got, want, t32 in ((gp, want_p, t32_p), (gx, want_x, t32_x)):
        e, e32 = err(got, want), err(t32, want)
        print("64^3 %s: native %.3g, torch float32 %.3g" % (agg, e, e32))
        assert e <= max(2e-6, 2 * e32)
    _, _, gp2, gx2 = device_geometry(sc, agg, g)
    assert torch.equal(gp, gp2) and torch.equal(gx, gx2)


@pytest.mark.parametrize("softmax", [0, 1])
def test_softargmax_coord_bwd_device(softmax):
    rng = np.random.RandomState(2)
    B, J, nvox = 3, 17, 64 ** 3
    probs = torch.from_numpy(rng.rand(B, J, nvox).astype(np.float32)).to(DEV)
    gk = torch.from_numpy(rng.randn(B, J, 3).astype(np.float32)).to(DEV)
    out, buf = guarded((B, nvox, 3))
    capi.softargmax3d_coord_bwd(probs, gk, out, B, J, nvox, softmax)
    torch.cuda.synchronize()
    assert guards_intact(buf) and bool(torch.isfinite(out).all())
    want = torch.einsum("bjn,bjk->bnk", probs.double(), gk.double())
    mag = torch.einsum("bjn,bjk->bnk", probs.double().abs(), gk.double().abs())
    assert float(((out.double() - want).abs() / ((J + 2) * EPS32 * mag + 1e-30)).max()) <= 1.0
    out2 = torch.empty_like(out)
    capi.softargmax3d_coord_bwd(probs, gk, out2, B, J, nvox, softmax)
    assert torch.equal(out, out2)


def test_dlt_proj_bwd_device_matches_host_code():
    P, kp, conf, g = make_scene(V=4, B=8, J=17, seed=9, conf="rand")
    want = proj_host(P, kp, conf, g)
    t = [torch.from_numpy(a).to(DEV) for a in (P, kp, conf, g)]
    out, buf = guarded(P.shape)
    ws = torch.empty(capi.triangulate_dlt_proj_bwd_workspace_bytes(8, 4, 17), dtype=torch.uint8, device=DEV)
    capi.triangulate_dlt_proj_bwd(*t, out, ws)
    torch.cuda.synchronize()
    assert guards_intact(buf) and bool(torch.isfinite(out).all())
    # the same float64 solve; the device may contract float64 operations differently: two float32 ulps of each element, or 1e-9 of
    # the largest where an element is the difference of much larger terms (tests/test_gpu_geometry_grad_ref.py holds every element
    # to the 50-digit reference)
    got, want = out.cpu().double().numpy(), want.astype(np.float64)
    assert (np.abs(got - want) <= 2 * 2.0 ** -23 * np.abs(want) + 1e-9 * np.abs(want).max()).all()
    out2 = torch.empty_like(out)
    capi.triangulate_dlt_proj_bwd(*t, out2, ws)
    assert torch.equal(out, out2)


# ---- autograd --------------------------------------------------------------------------------------------------------

def _ops_grads(backend, sc, agg, g_vol, g_kp):
    """unproject -> integrate sharing one coordinate tensor: (d proj, d coord), float64 for torch."""
    dt = torch.float64 if backend == "torch" else torch.float32
    f, p, c, cf = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dt) for a in sc)
    B, V, h, w, C = f.shape
    n = round(c.shape[1] ** (1 / 3))
    p.requires_grad_(True)
    coord = c.reshape(B, n, n, n, 3).requires_grad_(True)
    vol = op.unproject_heatmaps(f.permute(0, 1, 4, 2, 3).contiguous(), p, coord, agg, cf if agg == "conf" else None, backend=backend)
    kp, _ = op.integrate_tensor_3d_with_coordinates(vol * 0.5, coord, True, backend=backend)
    loss = (vol * g_vol.to(dt)).sum() + (kp * g_kp.to(dt)).sum()
    return torch.autograd.grad(loss, (p, coord))


@pytest.mark.parametrize("agg", ["sum", "softmax", "conf"])
def test_autograd_unproject_then_integrate_share_coordinates(agg):
    sc = camera_scene(2, 3, 8, 24, 20, 12, seed=4)
    rng = np.random.RandomState(1)
    g_vol = torch.from_numpy(rng.randn(2, 8, 12, 12, 12).astype(np.float32)).to(DEV)
    g_kp = torch.from_numpy(rng.randn(2, 8, 3).astype(np.float32)).to(DEV)
    want = _ops_grads("torch", sc, agg, g_vol, g_kp)
    got = _ops_grads("hybrid", sc, agg, g_vol, g_kp)
    for a, b in zip(got, want):
        assert a.shape == b.shape
        print("autograd %s: %.3g" % (agg, err(a, b)))
        assert err(a, b) <= 1e-4


def test_autograd_triangulate_proj():
    P, kp, conf, g = (torch.from_numpy(a).to(DEV) for a in make_scene(V=4, B=4, J=17, seed=8, conf="rand"))
    res = []
    for backend, dt in (("torch", torch.float64), ("hybrid", torch.float32)):
        p = P.to(dt).requires_grad_(True)
        out = multiview.triangulate_batch_of_points(p, kp.to(dt), conf.to(dt), backend=backend)
        res.append(torch.autograd.grad((out * g.to(dt)).sum(), p)[0])
    assert res[1].shape == P.shape
    assert err(res[1], res[0]) <= 1e-4, err(res[1], res[0])


def test_hybrid_algebraic_step_trains_the_projections():
    B, V, S, J = 2, 3, 128, 17
    images, batch = testing.make_batch(B, V, image_size=S, seed=11)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    holder = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
    grads = []
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for backend in ("torch", "hybrid"):
            m = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18), device="cpu", backend=backend)
            m.load_state_dict(holder.state_dict())
            m = m.to(DEV).train()
            p = proj.clone().requires_grad_(True)
            kp3d = m(images.to(DEV), p, batch)[0]
            (kp3d ** 2).mean().backward()
            assert p.grad is not None
            grads.append(p.grad)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    print("alg step d proj: %.3g" % err(grads[1], grads[0]))
    assert err(grads[1], grads[0]) <= 1e-3


def _geometry_backward(f, p0, c0, P0, kp, conf):
    """Device tensors in (no host copy: the sync debug mode and the capture forbid one) -> d proj, d coord of the unprojection and
    soft-argmax sharing one coordinate tensor, and d P of the DLT."""
    B = f.shape[0]
    p, c = p0.clone().requires_grad_(True), c0.clone().reshape(B, 4, 4, 4, 3).requires_grad_(True)
    vol = autograd_ops.unproject_heatmaps(f, p, c, "softmax")
    kp3, _ = autograd_ops.integrate_tensor_3d_with_coordinates(vol, c)
    Pd = P0.clone().requires_grad_(True)
    X = autograd_ops.triangulate_batch_of_points(Pd, kp, conf)
    return torch.autograd.grad(vol.sum() + kp3.sum() + X.sum(), (p, c, Pd))


def test_geometry_backwards_no_sync_and_graph_capture():
    sc = exact_scene(2, 3, 8, 8, 8, 64, seed=5)
    f, p0, c0, _ = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in sc)
    f = f.permute(0, 1, 4, 2, 3).contiguous()
    P, kp, conf, _ = (torch.from_numpy(a).to(DEV) for a in make_scene(V=3, B=2, J=5, seed=1, conf="rand"))
    args = (f, p0, c0, P, kp, conf)
    eager = _geometry_backward(*args)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        again = _geometry_backward(*args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        _geometry_backward(*args)                            # warm-up on the side stream
        with torch.cuda.graph(graph, stream=s):
            captured = _geometry_backward(*args)
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    for a, b, c in zip(captured, eager, again):
        assert torch.equal(a, b) and torch.equal(c, b)


GEOM_KERNELS = ("unproject_bwd_geom_kernel", "unproject_geom_", "softargmax_coord_bwd", "triangulate_dlt_proj")

# One hybrid volumetric step (forward and backward) under torch.profiler, printing the CUDA kernel names as JSON.  It runs in a child
# process: a profiling session over an autograd backward leaves profiler state behind in the process, and a later session there
# then misses its first kernel records (tests/test_gpu_unproject.py counts every launch of its window).
_STEP_KERNELS = """
import json, sys
sys.path[:0] = sys.argv[1:3]
import torch
from torch.profiler import ProfilerActivity, profile
import lt_b200
from lt_b200 import testing
dev = "cuda:0"
cfg = testing.make_config(num_layers=18, volume_size=32)
images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
m = lt_b200.VolumetricTriangulationNet(cfg, device=dev, backend="hybrid").to(dev).train()
testing.randomize_weights(m, seed=0, calib_size=64, calib_views=1)
m = m.to(dev).eval()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    kp = m(images.to(dev), None, batch)[0]
    (kp ** 2).mean().backward()
    torch.cuda.synchronize()
evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
print(json.dumps(sorted({e.name() for e in evs})))
"""


def test_hybrid_volumetric_step_launches_no_geometry_kernel():
    """The model's geometry requires no grad: its training step runs the plain unprojection backward and no geometry kernel."""
    import json
    import os
    import subprocess
    import sys
    tests = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _STEP_KERNELS, os.path.dirname(tests), tests]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    names = json.loads(res.stdout.strip().splitlines()[-1])
    assert any("unproject_bwd_kernel" in n for n in names), names
    assert not [n for n in names if any(k in n for k in GEOM_KERNELS)]
