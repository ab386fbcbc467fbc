"""GPU tests of training under torch.use_deterministic_algorithms: the fixed-order unprojection backward
(lt_unproject_aggregate_bwd_det) and V2V's native max-pool backward (lt_maxpool3d_bwd) at op level, and whole training steps at model
level.  The per-element bars of the op-level checks are those of tests/test_deterministic_cpu.py.  The model-level checks run in
one child process with CUBLAS_WORKSPACE_CONFIG set and the flag on, so the flag never reaches the rest of the session."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lt_b200 import capi
from test_deterministic_cpu import term_reference, upstream, pool_cases, pool_input, bits
from test_unproject_cpu import AGGS, exact_scene, camera_scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _dev(sc, agg):
    f, p, c, cf = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in sc)
    B, V = f.shape[:2]
    return f, p.reshape(B, V, 12).contiguous(), c, (cf if agg == "conf" else None)


def det(sc, agg, g, geom=False, ws=None):
    f, p, c, cf = _dev(sc, agg)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gf = torch.zeros_like(f)
    gc = torch.zeros(B, V, C, device=DEV) if agg == "conf" else None
    gp = torch.empty(B, V, 12, device=DEV) if geom else None
    gx = torch.empty(B, nvox, 3, device=DEV) if geom else None
    if ws is None:
        ws = torch.empty(capi.unproject_aggregate_bwd_det_workspace_bytes(B, V, C, h, w, nvox, capi.AGG[agg], geom), dtype=torch.uint8,
                         device=DEV)
    capi.unproject_aggregate_bwd_det(f, p, c, cf, g.to(DEV).contiguous(), gf, gc, gp, gx, capi.AGG[agg], ws)
    return gf, gc, gp, gx


def atomic(sc, agg, g, geom=False):
    f, p, c, cf = _dev(sc, agg)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gf = torch.zeros_like(f)
    gc = torch.zeros(B, V, C, device=DEV) if agg == "conf" else None
    if not geom:
        capi.unproject_aggregate_bwd(f, p, c, cf, g.to(DEV).contiguous(), gf, gc, capi.AGG[agg])
        return gf, gc, None, None
    gp, gx = torch.empty(B, V, 12, device=DEV), torch.empty(B, nvox, 3, device=DEV)
    ws = torch.empty(capi.unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox), dtype=torch.uint8, device=DEV)
    capi.unproject_aggregate_bwd_geom(f, p, c, cf, g.to(DEV).contiguous(), gf, gc, gp, gx, capi.AGG[agg], ws)
    return gf, gc, gp, gx


OP_SCENES = {"V4 C32 32x32 nvox 9001": (2, 4, 32, 32, 32, 9001), "V8 C4 16x16 nvox 4099": (1, 8, 4, 16, 16, 4099),
             "V1 C128 8x16 nvox 1111": (2, 1, 128, 8, 16, 1111), "V2 C32 8x8 one cell": (2, 2, 32, 8, 8, 3000)}


@pytest.mark.parametrize("name", list(OP_SCENES))
@pytest.mark.parametrize("agg", AGGS)
def test_fixed_order_vs_float64_terms_and_atomic(name, agg):
    """Every element within its per-element bar of the float64 terms, and within 2x that bar of the atomic kernel."""
    B, V, C, h, w, nvox = OP_SCENES[name]
    sc = exact_scene(B, V, C, h, w, nvox, seed=B + V + C + h + w + nvox)
    if "one cell" in name:
        sc.coord[:] = np.array([0.25, 0.5, 1.0], np.float32)
    sc.coord[:, ::41, 0] = np.nan
    g = upstream(sc, agg)
    want_f, bar_f, want_c, bar_c = term_reference(sc, agg, g)
    gf, gc, _, _ = (t if t is None else t.cpu().double() for t in det(sc, agg, g))
    af, ac, _, _ = (t if t is None else t.cpu().double() for t in atomic(sc, agg, g))
    assert float(((gf - want_f).abs() - bar_f).max()) <= 0.0
    assert float(((gf - af).abs() - 2 * bar_f).max()) <= 0.0
    if agg == "conf":
        assert float(((gc - want_c).abs() - bar_c).max()) <= 0.0
        assert float(((gc - ac).abs() - 2 * bar_c).max()) <= 0.0


@pytest.mark.parametrize("agg", AGGS)
def test_fixed_order_bit_identical_across_repeats_graphs_streams_and_batches(agg):
    sc = camera_scene(3, 4, 32, 48, 48, 20, seed=2)
    g = upstream(sc, agg)
    first = det(sc, agg, g)
    for _ in range(2):
        again = det(sc, agg, g)
        assert all(a is None or torch.equal(a, b) for a, b in zip(again, first))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        other = det(sc, agg, g)
    torch.cuda.current_stream().wait_stream(side)
    assert all(a is None or torch.equal(a, b) for a, b in zip(other, first))
    # graph replay
    f, p, c, cf = _dev(sc, agg)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    gd = g.to(DEV).contiguous()
    ws = torch.empty(capi.unproject_aggregate_bwd_det_workspace_bytes(B, V, C, h, w, nvox, capi.AGG[agg], False), dtype=torch.uint8, device=DEV)
    gf = torch.zeros_like(f)
    gc = torch.zeros(B, V, C, device=DEV) if agg == "conf" else None
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        gf.zero_()
        if gc is not None:
            gc.zero_()
        capi.unproject_aggregate_bwd_det(f, p, c, cf, gd, gf, gc, None, None, capi.AGG[agg], ws)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(gf, first[0]) and (gc is None or torch.equal(gc, first[1]))
    # per-sample runs
    for b in range(3):
        one = type(sc)(*(a[b:b + 1] for a in sc))
        f1, c1, _, _ = det(one, agg, g[b:b + 1])
        assert torch.equal(f1[0], first[0][b]) and (c1 is None or torch.equal(c1[0], first[1][b]))


@pytest.mark.parametrize("agg", AGGS)
def test_fixed_order_geometry_outputs_bit_equal_geometry_kernel(agg):
    sc = camera_scene(2, 4, 32, 32, 32, 16, seed=6)
    g = upstream(sc, agg)
    gf, gc, gp, gx = det(sc, agg, g, geom=True)
    _, _, ap, ax = atomic(sc, agg, g, geom=True)
    assert torch.equal(gp, ap) and torch.equal(gx, ax)
    pf, pc, _, _ = det(sc, agg, g)
    assert torch.equal(gf, pf) and (gc is None or torch.equal(gc, pc))


@pytest.mark.parametrize("shape,case,cl", list(pool_cases()))
def test_maxpool3d_backward_bit_equal_torch_cuda(shape, case, cl):
    """Against torch's CUDA max_pool3d backward with the flag off (its atomics add one term per element: exact)."""
    x = pool_input(*shape, seed=sum(shape), case=case).to(DEV)
    if cl:
        x = x.contiguous(memory_format=torch.channels_last_3d)
    gy = torch.from_numpy(np.random.RandomState(1).randn(*F.max_pool3d(x, 2, 2).shape).astype(np.float32)).to(DEV)
    gy[0, 0, 0, 0, 0] = -0.0
    xr = x.clone().requires_grad_(True)
    F.max_pool3d(xr, 2, 2).backward(gy)
    gx = torch.full_like(x, float("nan"))
    capi.maxpool3d_bwd(x, gy, gx, 2)
    assert torch.equal(bits(gx), bits(xr.grad))


# ---- model level, in a child process with the flag on -------------------------------------------------------------------

_CHILD = r"""
import json, sys
sys.path[:0] = sys.argv[1:3]
import numpy as np
import torch
torch.use_deterministic_algorithms(True)
import lt_b200
from lt_b200 import testing
import test_gpu_train_step as T
from torch.profiler import ProfilerActivity, profile

torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
Vol, Alg = lt_b200.VolumetricTriangulationNet, lt_b200.AlgebraicTriangulationNet
TORCH_SW = dict(backbone_backend="torch", v2v_backend="torch", norm_backend="torch")
out = {}

def vol_config(agg):
    return testing.make_train_config(testing.make_config(num_layers=18, volume_size=32, aggregation=agg), criterion="MAE", lr=1e-4,
                                     use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01, scale_keypoints_3d=0.1,
                                     process_features_lr=1e-3, volume_net_lr=1e-3, grad_clip=1e-5)

def vol_state(cfg):
    torch.manual_seed(0)
    holder = Vol(cfg, device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=0, calib_size=T.S, calib_views=1)
    return holder.state_dict()

def diffs(a, b, metrics=True):
    bad = [k for k in a[0]["metrics"] if metrics and any(x["metrics"][k] != y["metrics"][k] for x, y in zip(a, b))]
    for part in ("grads", "params", "adam"):
        bad += ["%s %s" % (part, n) for n in a[0][part] if any(not torch.equal(x[part][n], y[part][n]) for x, y in zip(a, b))]
    bad += ["norm %d" % i for i in range(len(a[0]["norm"])) if any(not torch.equal(x["norm"][i], y["norm"][i]) for x, y in zip(a, b))]
    return bad

def graph_flag_eager(make, cfg, state, sw, data, steps=3):
    m = T._model(make, cfg, state, sw, graph=True)
    opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
    rec = []
    for step in range(steps):
        np.random.seed(step)
        _, metrics = testing.reference_train_step(m, opt, cfg, *data)
        rec.append(T._record(m, opt, metrics))
    return rec

for n_views in (2, 4):
    data = T._data(n_views=n_views)
    for agg in ("softmax", "conf_norm"):
        cfg = vol_config(agg)
        st = vol_state(cfg)
        for sw_name, sw in (("native", T.VOL_SWITCHES), ("torch", TORCH_SW)):
            if n_views == 4 and sw_name == "torch":
                continue
            label = "vol V%d %s %s" % (n_views, agg, sw_name)
            a = T._eager(Vol, cfg, st, sw, data)
            b = T._eager(Vol, cfg, st, sw, data)
            out[label + " eager twice"] = diffs(a, b)
            if sw_name == "native" and n_views == 2:
                # TrainStep's metrics are its own device formulas (native criterion, float64 norm sum), not the loop's
                out[label + " TrainStep vs eager"] = diffs(T._graphed(Vol, cfg, st, sw, data), a, metrics=False)
                out[label + " train_graph vs eager"] = diffs(graph_flag_eager(Vol, cfg, st, sw, data), a)

alg_cfg = T._alg_config(True)
alg_st = T._alg_state(True)
data = T._data()
out["alg conf eager twice"] = diffs(T._eager(Alg, alg_cfg, alg_st, T.ALG_SWITCHES, data), T._eager(Alg, alg_cfg, alg_st, T.ALG_SWITCHES, data))

# kernels of one eager step, flag flips recapture, replay without host synchronisation
cfg = vol_config("conf_norm")
st = vol_state(cfg)
data = T._data()
m = T._model(Vol, cfg, st, T.VOL_SWITCHES)
opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
step = lt_b200.TrainStep(m, opt, cfg)
step(*data)
caps = [step.captures]
torch.cuda.synchronize()
prev = torch.cuda.get_sync_debug_mode()
torch.cuda.set_sync_debug_mode("error")
try:
    step(*data)
finally:
    torch.cuda.set_sync_debug_mode(prev)
caps.append(step.captures)
torch.use_deterministic_algorithms(False)
step(*data)
caps.append(step.captures)
torch.use_deterministic_algorithms(True)
step(*data)
caps.append(step.captures)
out["captures"] = caps
m2 = T._model(Vol, cfg, st, T.VOL_SWITCHES)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    kp = m2(data[0], None, data[4])[0]
    (kp ** 2).mean().backward()
    torch.cuda.synchronize()
evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
out["kernels"] = sorted({e.name() for e in evs})
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def child():
    tests = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD, os.path.dirname(tests), tests]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env)
    assert res.returncode == 0, res.stderr[-6000:]
    return json.loads(res.stdout.strip().splitlines()[-1])


def test_volumetric_and_algebraic_steps_repeat_bit_for_bit(child):
    """Three Adam steps run twice from one state: losses, gradients, parameters, Adam state and BatchNorm buffers torch.equal, on the
    native and the torch switches (softmax and conf aggregation, 2 and 4 views), and for the algebraic model with confidences.  At the
    parent commit the volumetric step raises in torch's max_pool3d backward."""
    runs = {k: v for k, v in child.items() if k.endswith("eager twice")}
    assert len(runs) == 7
    assert all(v == [] for v in runs.values()), {k: v[:5] for k, v in runs.items() if v}


def test_graphed_volumetric_steps_bit_identical_to_eager(child):
    """train_graph=True steps equal the eager steps bit for bit through three steps (native switches), losses included; a
    TrainStep's gradients, parameters, Adam state and BatchNorm buffers do too (its metrics come from its own device formulas)."""
    runs = {k: v for k, v in child.items() if "vs eager" in k}
    assert len(runs) == 4
    assert all(v == [] for v in runs.values()), {k: v[:5] for k, v in runs.items() if v}


def test_flag_selects_fixed_order_kernels_and_recaptures(child):
    names = child["kernels"]
    assert not [n for n in names if "unproject_bwd_kernel" in n or "unproject_bwd_geom_kernel" in n], names
    assert any("fo_unproj_bwd_gather_kernel" in n for n in names) and any("pool3d_bwd_kernel" in n for n in names), names
    # capture, replay under set_sync_debug_mode("error") (no host synchronisation), flag off: recapture, flag on: recapture
    assert child["captures"] == [1, 1, 2, 3]
