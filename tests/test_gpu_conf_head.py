"""GPU tests of the confidence heads' native training tail (head_backend="native": autograd_ops.conf_head_tail / view_normalize over
lt_conf_head_tail_fwd / _bwd and lt_view_normalize_fwd / _bwd): the kernels against float64 autograd of the torch formula on the device
with the per-element bars of tests/test_conf_head_cpu.py, repeatability, capture and synchronisation, whole training steps against the
torch head under the weight-noise bars of tests/test_gpu_backbone_train.py, and, in a child process with
torch.use_deterministic_algorithms on and CUBLAS_WORKSPACE_CONFIG unset, bit-identical steps without a cuBLAS kernel."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from lt_b200 import autograd_ops as A
from lt_b200 import capi
from test_conf_head_cpu import U, assert_within, backward_ref, forward_ref, make_head, make_map
from test_gpu_backbone_train import _compare, _no_tf32, _train, _weight_noise

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _run(x, lins, g):
    """The device kernels on x (any strides) -> (out, x0, h1, h2, grad_x, grads)."""
    N, C0 = x.shape[:2]
    (w1, b1), (w2, b2), (w3, b3) = lins
    out, x0, h1, h2 = (torch.empty(N, k, device=DEV) for k in (w3.shape[0], C0, w1.shape[0], w2.shape[0]))
    capi.conf_head_tail(x, *lins, out, x0, h1, h2)
    gx = torch.full_like(x, float("nan"))
    grads = tuple(torch.full_like(t, float("nan")) for lin in lins for t in lin)
    ws = torch.empty(capi.conf_head_tail_bwd_workspace_bytes(N, C0, w1.shape[0], w2.shape[0], w3.shape[0]), dtype=torch.uint8,
                     device=DEV)
    capi.conf_head_tail_bwd(x, w1, w2, w3, x0, h1, h2, out, g, gx, grads, ws)
    return out, x0, h1, h2, gx, grads


def _case(N, H, W, NO, channels_last, scale, seed=0):
    lins = tuple((w.to(DEV), b.to(DEV)) for w, b in make_head(NO=NO, seed=seed + N))
    x = make_map(N, 256, H, W, seed=seed + H * W, channels_last=channels_last).to(DEV)
    g = (torch.randn(N, NO, generator=torch.Generator().manual_seed(seed + 3)) * scale).to(DEV)
    return x, lins, g


@pytest.mark.parametrize("N", [1, 20, 400])
@pytest.mark.parametrize("H,W", [(12, 12), (13, 11), (4, 4)])
@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("NO,scale", [(17, 1e-9), (32, 1e3), (17, 1.0)])
def test_tail_vs_float64_autograd(N, H, W, channels_last, NO, scale):
    x, lins, g = _case(N, H, W, NO, channels_last, scale)
    out, x0, h1, h2, gx, grads = _run(x, lins, g)
    ref, bars = forward_ref(x, lins, x0, h1, h2)
    for name, got in (("x0", x0), ("h1", h1), ("h2", h2), ("y", out)):
        assert_within(name, got, ref[name], bars[name])
    assert gx.stride() == x.stride()
    ref, bars = backward_ref(x, lins, x0, h1, h2, out, g)
    assert_within("dx", gx, ref["dx"], bars["dx"])
    for name, got in zip(("dW1", "db1", "dW2", "db2", "dW3", "db3"), grads):
        assert_within(name, got, ref[name], bars[name])


def test_layouts_bitwise_and_device_equals_host_hook():
    """NCHW and channels_last give the same bits on the device; the forward mean and the MLP equal the host hook's (same fmaf chains)."""
    x, lins, g = _case(20, 13, 11, 32, False, 1.0, seed=5)
    a = _run(x, lins, g)
    b = _run(x.contiguous(memory_format=torch.channels_last), lins, g)
    for t, s in zip(a[:4] + a[5], b[:4] + b[5]):
        assert torch.equal(t, s)
    assert torch.equal(a[4].contiguous(), b[4].contiguous())
    host = capi.conf_head_tail_host(x.cpu(), *[(w.cpu(), bb.cpu()) for w, bb in lins])
    for t, s in zip(a[1:4], host[1:4]):
        assert torch.equal(t.cpu(), s)


@pytest.mark.parametrize("eps", [1e-5, 0.0])
@pytest.mark.parametrize("B,V,C", [(2, 4, 17), (100, 4, 17), (5, 2, 32)])
def test_view_normalize_vs_float64_autograd(eps, B, V, C):
    gen = torch.Generator().manual_seed(B + V)
    c = (torch.rand(B, V, C, generator=gen) + 1e-3).to(DEV)
    g = torch.randn(B, V, C, generator=gen).to(DEV)
    cc = c.clone().requires_grad_(True)
    y = A.view_normalize(cc, eps)
    y.backward(g)
    c64 = c.double().requires_grad_(True)
    y64 = c64 / c64.sum(dim=1, keepdim=True) + eps
    y64.backward(g.double())
    S = c.double().sum(1, keepdim=True)
    assert bool(((y.double() - y64).abs() <= (V + 2) * U * c.double() / S + U * y64.abs()).all())
    bar = U * c64.grad.abs() + 7 * 2.0 ** -52 * (g.double().abs() / S + (g.double() * c.double()).abs().sum(1, keepdim=True) / S ** 2)
    assert bool(((cc.grad.double() - c64.grad).abs() <= bar).all())
    assert torch.equal(c, cc.detach())                  # the forward normalises a copy


def _fn_step(x, lins, g, eps):
    """The two autograd Functions forward and backward: (confidences, grad_x, parameter grads)."""
    xx = x.clone().requires_grad_(True)
    params = [t.clone().requires_grad_(True) for lin in lins for t in lin]
    y = A.ConfHeadTailFn.apply(xx, *params)
    z = A.view_normalize(y.view(-1, 4, y.shape[1]), eps)
    z.backward(g.view(-1, 4, g.shape[1]))
    return [z.detach(), xx.grad] + [p.grad for p in params]


def test_repeats_bitwise_graph_capture_and_no_host_sync():
    x, lins, g = _case(20, 12, 12, 17, True, 1.0, seed=9)
    a = _fn_step(x, lins, g, 1e-5)
    b = _fn_step(x, lins, g, 1e-5)
    assert all(torch.equal(s, t) for s, t in zip(a, b))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _fn_step(x, lins, g, 1e-5)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = _fn_step(x, lins, g, 1e-5)
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(s, t) for s, t in zip(a, c))
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        d = _fn_step(x, lins, g, 1e-5)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    assert all(torch.equal(s, t) for s, t in zip(a, d))


def test_argument_errors_on_device():
    x, lins, g = _case(2, 12, 12, 17, False, 1.0)
    (w1, b1), (w2, b2), (w3, b3) = lins
    out = torch.empty(2, 17, device=DEV)
    with pytest.raises(RuntimeError, match="too small"):
        capi.conf_head_tail(x[:, :, :1], *lins, out, torch.empty(2, 256, device=DEV), torch.empty(2, 512, device=DEV),
                            torch.empty(2, 256, device=DEV))
    ws = torch.empty(8, dtype=torch.uint8, device=DEV)
    res = _run(x, lins, g)
    with pytest.raises(RuntimeError, match="workspace"):
        capi.conf_head_tail_bwd(x, w1, w2, w3, res[1], res[2], res[3], res[0], g, torch.empty_like(x),
                                tuple(torch.empty_like(t) for lin in lins for t in lin), ws)


# ---- model level: one training step, native head against the torch head ---------------------------------------------------
B, V, S, J = 2, 2, 128, 17
TORCH_SW = {}
ALG_NATIVE = dict(backbone_backend="native", norm_backend="native")
VOL_NATIVE = dict(backbone_backend="native", norm_backend="native", v2v_backend="native")


def _models_and_loss(kind, agg=None):
    import lt_b200
    from lt_b200 import testing
    images, batch = testing.make_batch(B, V, image_size=S, seed=11)
    images = images.to(DEV)
    g = torch.Generator().manual_seed(12)
    target = (torch.from_numpy(np.stack([k[:, :3] for k in batch["keypoints_3d"]])).float() + torch.randn(B, J, 3, generator=g) * 50).to(DEV)
    validity = (torch.rand(B, J, 1, generator=g) > 0.2).float().to(DEV)
    if kind == "alg":
        make_cfg = lambda: testing.make_alg_config(num_layers=18, use_confidences=True)        # noqa: E731
        cls = lt_b200.AlgebraicTriangulationNet
        holder = cls(make_cfg(), device="cpu", backend="torch")
        testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
        proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
        head = "backbone.alg_confidences."
    else:
        make_cfg = lambda: testing.make_config(num_layers=18, volume_size=32, aggregation=agg)  # noqa: E731
        cls = lt_b200.VolumetricTriangulationNet
        torch.manual_seed(0)
        holder = cls(make_cfg(), device="cpu", backend="torch")
        testing.randomize_weights(holder, seed=0, calib_size=S, calib_views=1)
        proj = None
        head = "backbone.vol_confidences."

    def step_loss(m):
        kp3d = m(images, proj, batch)[0]
        return (torch.abs(target - kp3d) * validity).sum() / (3 * max(1.0, float(validity.sum())))
    names = [head + n for n in ("head.0.weight", "head.0.bias", "head.2.weight", "head.4.weight", "head.4.bias", "features.4.weight",
                                "features.5.weight", "features.0.weight")] + ["backbone.layer4.1.conv2.weight"]
    return cls, make_cfg, holder.state_dict(), step_loss, names


@pytest.mark.parametrize("kind,agg", [("alg", None), ("vol", "conf"), ("vol", "conf_norm")])
@pytest.mark.parametrize("switches", ["torch", "native"])
def test_training_step_native_head_vs_torch_head(kind, agg, switches):
    cls, make_cfg, sd, step_loss, names = _models_and_loss(kind, agg)
    sw = TORCH_SW if switches == "torch" else (ALG_NATIVE if kind == "alg" else VOL_NATIVE)
    prev = _no_tf32()
    out = {}
    try:
        for run, head, state in (("torch", "torch", sd), ("native", "native", sd), ("noise", "torch", _weight_noise(sd, "backbone"))):
            out[run] = _train(lambda: cls(make_cfg(), device="cpu", backend="hybrid", head_backend=head, **sw), state, step_loss, names)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    _compare(out, names, [1e-4, 1e-3, 1e-3] + [1e-2] * len(names))


# ---- determinism without cuBLAS, in a child process with the flag on and CUBLAS_WORKSPACE_CONFIG unset ------------------------
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
Alg, Vol = lt_b200.AlgebraicTriangulationNet, lt_b200.VolumetricTriangulationNet
out = {}
def diffs(a, b):
    bad = []
    for part in ("grads", "params", "adam"):
        bad += ["%s %s" % (part, n) for n in a[0][part] if any(not torch.equal(x[part][n], y[part][n]) for x, y in zip(a, b))]
    bad += ["norm %d" % i for i in range(len(a[0]["norm"])) if any(not torch.equal(x["norm"][i], y["norm"][i]) for x, y in zip(a, b))]
    return bad
def gemm_kernels(step):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    names = {e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA}
    return sorted(n for n in names if "lt::" not in n and any(k in n.lower() for k in ("gemm", "gemv", "cublas", "cutlass", "splitkreduce")))
cfg, st, data = T._alg_config(True), T._alg_state(True), T._data()
for sw_name, sw in (("native", T.ALG_SWITCHES), ("torch", {})):
    sw = dict(sw, head_backend="native")
    out["TrainStep %s" % sw_name] = diffs(T._graphed(Alg, cfg, st, sw, data, steps=2), T._graphed(Alg, cfg, st, sw, data, steps=2))
    def graph_step():
        m = T._model(Alg, cfg, st, sw, graph=True)
        opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
        np.random.seed(0)
        _, metrics = testing.reference_train_step(m, opt, cfg, *data)
        return [T._record(m, opt, metrics)]
    out["train_graph %s" % sw_name] = diffs(graph_step(), graph_step())
sw = dict(T.ALG_SWITCHES, head_backend="native")
m = T._model(Alg, cfg, st, sw)
opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
out["gemm alg native head"] = gemm_kernels(lambda: testing.reference_train_step(m, opt, cfg, *data))
try:
    m = T._model(Alg, cfg, st, T.ALG_SWITCHES)
    opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
    testing.reference_train_step(m, opt, cfg, *data)
    out["torch head error"] = None
except RuntimeError as exc:
    out["torch head error"] = str(exc)
torch.use_deterministic_algorithms(False)
m = T._model(Alg, cfg, st, T.ALG_SWITCHES)
opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
out["gemm alg torch head, flag off"] = gemm_kernels(lambda: testing.reference_train_step(m, opt, cfg, *data))
vcfg = testing.make_train_config(testing.make_config(num_layers=18, volume_size=32, aggregation="conf_norm"), criterion="MAE", lr=1e-4,
                                 use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01, scale_keypoints_3d=0.1,
                                 process_features_lr=1e-3, volume_net_lr=1e-3, grad_clip=1e-5)
torch.manual_seed(0)
holder = Vol(vcfg, device="cpu", backend="torch")
testing.randomize_weights(holder, seed=0, calib_size=T.S, calib_views=1)
m = T._model(Vol, vcfg, holder.state_dict(), dict(T.VOL_SWITCHES, head_backend="native"))
opt = testing.recipe_optimizer(m, vcfg, eps=1e-3, capturable=True)
np.random.seed(0)
out["gemm vol native head"] = gemm_kernels(lambda: testing.reference_train_step(m, opt, vcfg, *T._data()))
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def child():
    tests = os.path.dirname(os.path.abspath(__file__))
    env = {k: v for k, v in os.environ.items() if k != "CUBLAS_WORKSPACE_CONFIG"}
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD, os.path.dirname(tests), tests]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env)
    assert res.returncode == 0, res.stderr[-6000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    print(json.dumps(out, indent=1))
    return out


def test_native_head_steps_repeat_bit_for_bit_without_cublas_config(child):
    """Two TrainStep steps and one train_graph=True step, each run twice from one state with the flag on and CUBLAS_WORKSPACE_CONFIG
    unset: gradients, parameters, Adam state and BatchNorm buffers torch.equal, with the native and the torch conv / norm switches."""
    runs = {k: v for k, v in child.items() if k.startswith(("TrainStep", "train_graph"))}
    assert len(runs) == 4
    assert all(v == [] for v in runs.values()), {k: v[:5] for k, v in runs.items() if v}


def test_native_head_step_launches_no_cublas_gemm(child):
    assert child["gemm alg native head"] == []
    assert child["gemm alg torch head, flag off"], "the kernel-name filter finds the torch head's cuBLAS GEMMs"


def test_torch_head_under_the_flag_without_cublas_config(child):
    """The torch head's step with the flag on and CUBLAS_WORKSPACE_CONFIG unset: torch builds that check the setting raise cuBLAS's
    RuntimeError naming it; torch 2.11 with CUDA 12.8 on an H100 runs the step (its cuBLAS GEMMs are still launched, see
    test_native_head_step_launches_no_cublas_gemm)."""
    err = child["torch head error"]
    assert err is None or "CUBLAS_WORKSPACE_CONFIG" in err, err


def test_volumetric_native_head_step_gemm_kernels(child):
    """What a volumetric hybrid step with every native switch and the native head still launches from cuBLAS: GEMM kernels only, from
    the step's one matmul outside the heads, the coordinate rotation's einsum (reported in README / DESIGN §7, not changed here)."""
    assert all("gemm" in n.lower() for n in child["gemm vol native head"]), child["gemm vol native head"]
