"""The algebraic-triangulation kernels (csrc/algebraic.cu) on the GPU against high-precision references.

- lt_triangulate_dlt_fwd / _bwd: every scene of tests/test_algebraic_ref_cpu.py against its 50-digit reference and bars; item
  counts around the 128-thread CTA and several thousand items against the host hook and spot items against the reference;
  NaN-prefilled, guarded outputs; bitwise repeats and a CUDA-graph replay; the point at infinity.
- lt_gap_mlp3_fwd (the confidence heads' tail): float64 mean -> Linear -> ReLU -> Linear -> ReLU -> Linear -> sigmoid of the exact
  operands, for float32 and split-fp16 input, with a bar of (summation steps) 2^-24 sum |w||x| per layer carried through.
- lt_view_normalize_fwd: float64 conf / sum_v conf + eps."""
import numpy as np
import pytest
import torch

from lt_b200 import capi
from test_algebraic_ref_cpu import (SCENES, ULP32, check_backward, check_forward, host_backward, host_forward, make_scene,
                                    point_at_infinity_scene, scene_id)
from test_gpu_unproject import Guarded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = 2.0 ** -24


def dev(a):
    return None if a is None else torch.from_numpy(a).to(DEV)


def dlt_forward(P, kp, conf, guard=256):
    out = Guarded((kp.shape[0], kp.shape[2], 3), guard=guard)
    capi.triangulate_dlt(dev(P), dev(kp), dev(conf), out.t)
    torch.cuda.synchronize()
    return out


def dlt_backward(P, kp, conf, g, with_grad_conf=True, guard=256):
    gk = Guarded(kp.shape, guard=guard)
    gc = Guarded(conf.shape, guard=guard) if (conf is not None and with_grad_conf) else None
    capi.triangulate_dlt_bwd(dev(P), dev(kp), dev(conf), dev(g), gk.t, None if gc is None else gc.t)
    torch.cuda.synchronize()
    return gk, gc


# ---- DLT --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("scene", SCENES, ids=scene_id)
def test_dlt_forward_vs_high_precision(scene):
    P, kp, conf, _ = make_scene(B=2, J=4, seed=1, **scene)
    out = dlt_forward(P, kp, conf)
    assert out.guards_intact() and out.unwritten() == 0
    got = out.t.cpu().numpy()
    assert np.isfinite(got).all()
    worst = check_forward(P, kp, conf, got)
    print("dlt forward (device) %s: worst err/bar %.3g" % (scene_id(scene), worst))
    assert worst <= 1.0


@pytest.mark.parametrize("scene", SCENES, ids=scene_id)
def test_dlt_backward_vs_high_precision(scene):
    P, kp, conf, g = make_scene(B=1, J=3, seed=2, **scene)
    gk, gc = dlt_backward(P, kp, conf, g)
    assert gk.guards_intact() and gk.unwritten() == 0
    assert gc is None or (gc.guards_intact() and gc.unwritten() == 0)
    gk_, gc_ = gk.t.cpu().numpy(), None if gc is None else gc.t.cpu().numpy()
    assert np.isfinite(gk_).all() and (gc_ is None or np.isfinite(gc_).all())
    worst = check_backward(P, kp, conf, g, gk_, gc_, [(0, j) for j in range(3)])
    print("dlt backward (device) %s: worst err/bar %.3g" % (scene_id(scene), worst))
    assert worst <= 1.0


def _close_to_host(got, want, per_item_axes):
    """Device vs the host hook (the same per-item code; only the device's float64 FMA contraction differs): one float32 ulp, or
    1e-9 of the item's largest element where a value is the difference of much larger terms."""
    scale = np.abs(want).max(axis=per_item_axes, keepdims=True)
    return float(np.max(np.abs(got - want) / (ULP32 * np.abs(want) + 1e-9 * scale + 1e-30)))


@pytest.mark.parametrize("BJ", [(1, 1), (1, 127), (4, 32), (3, 43), (8, 17), (300, 17)], ids=lambda s: "B%dxJ%d" % s)
def test_dlt_item_counts(BJ):
    """B*J = 1, 127, 128, 129, 136 (config #5) and 5100: tail threads of the 128-thread CTAs and many CTAs, every element written
    once and nothing past the end; all items against the host hook, the first and last items of each CTA against the reference."""
    B, J = BJ
    P, kp, conf, g = make_scene(V=4, B=B, J=J, seed=B * 1000 + J, conf="rand")
    out = dlt_forward(P, kp, conf)
    gk, gc = dlt_backward(P, kp, conf, g)
    for t in (out, gk, gc):
        assert t.guards_intact() and t.unwritten() == 0
    X, gk_, gc_ = out.t.cpu().numpy(), gk.t.cpu().numpy(), gc.t.cpu().numpy()
    hX = host_forward(P, kp, conf)
    hk, hc = host_backward(P, kp, conf, g)
    e = max(_close_to_host(X, hX, (2,)), _close_to_host(gk_, hk, (1, 3)), _close_to_host(gc_, hc, (1,)))
    spots = sorted({i for i in (0, 127, 128, B * J - 1) if i < B * J})
    items = [(i // J, i % J) for i in spots]
    wf = max(check_forward(P[b:b + 1], kp[b:b + 1, :, j:j + 1], conf[b:b + 1, :, j:j + 1], X[b:b + 1, j:j + 1]) for b, j in items)
    wb = check_backward(P, kp, conf, g, gk_, gc_, items)
    print("dlt B=%d J=%d: device vs host %.3g ulp-bars, forward err/bar %.3g, backward err/bar %.3g" % (B, J, e, wf, wb))
    assert e <= 1.0 and wf <= 1.0 and wb <= 1.0


def test_dlt_backward_without_grad_conf():
    """grad_confidences NULL: the key-point gradient is bit-identical to the call that also writes the confidence gradient."""
    P, kp, conf, g = make_scene(V=4, B=5, J=17, seed=7, conf="rand")
    gk0, gc0 = dlt_backward(P, kp, conf, g)
    gk1, gc1 = dlt_backward(P, kp, conf, g, with_grad_conf=False)
    assert gc1 is None and gk1.guards_intact() and gk1.unwritten() == 0
    assert torch.equal(gk0.t.view(torch.int32), gk1.t.view(torch.int32))


def test_dlt_repeats_bitwise_and_replays_in_a_cuda_graph():
    P, kp, conf, g = (dev(a) for a in make_scene(V=4, B=8, J=17, seed=8, conf="graded1e-4"))
    out, gk, gc = torch.empty(8, 17, 3, device=DEV), torch.empty_like(kp), torch.empty_like(conf)

    def step():
        capi.triangulate_dlt(P, kp, conf, out)
        capi.triangulate_dlt_bwd(P, kp, conf, g, gk, gc)
        return [t.clone() for t in (out, gk, gc)]

    first = step()
    for _ in range(3):
        assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(first, step()))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        capi.triangulate_dlt(P, kp, conf, out)
        capi.triangulate_dlt_bwd(P, kp, conf, g, gk, gc)
    # new inputs into the captured buffers
    P2, kp2, conf2, g2 = (dev(a) for a in make_scene(V=4, B=8, J=17, seed=9, conf="rand"))
    for src, dst in ((P2, P), (kp2, kp), (conf2, conf), (g2, g)):
        dst.copy_(src)
    want = step()
    for t in (out, gk, gc):
        t.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(want, (out, gk, gc)))


def test_dlt_point_at_infinity_on_the_device():
    """u[3] = 0 exactly (see point_at_infinity_scene): (+inf, nan, nan) and NaN gradients for that item, as on the host."""
    P, kp, conf, g = point_at_infinity_scene()
    out = dlt_forward(P, kp, conf).t.cpu().numpy()
    assert out[0, 0, 0] == np.inf and np.isnan(out[0, 0, 1:]).all() and np.isfinite(out[0, 1]).all()
    gk, gc = dlt_backward(P, kp, conf, g)
    gk, gc = gk.t.cpu().numpy(), gc.t.cpu().numpy()
    assert np.isnan(gk[0, :, 0]).all() and np.isnan(gc[0, :, 0]).all()
    assert np.isfinite(gk[0, :, 1]).all() and np.isfinite(gc[0, :, 1]).all()


def test_dlt_backward_is_zero_on_an_exact_tie_on_the_device():
    P, kp, conf, g = make_scene(V=3, B=2, J=5, seed=3, conf="zero")
    gk, gc = dlt_backward(P, kp, conf, g)
    assert not gk.t.any() and not gc.t.any()


# ---- confidence-head tail ---------------------------------------------------------------------------------------------

def mlp_reference(x, layers):
    """x (N, P, C0) float64 exact operands -> (out (N, NO), bar (N, NO)).  Each layer's bar: (in + 1) 2^-24 sum |w||x| + |b| for
    its own fmaf chain, plus sum |w| (bar of its input); the sigmoid adds sigma' x bar and 4 float32 ulps of its own."""
    P = x.shape[1]
    h = x.mean(1)
    bar = (P + 1) * U * np.abs(x).mean(1)
    for i, (w, b) in enumerate(layers):
        w, b = w.double().cpu().numpy(), b.double().cpu().numpy()
        z = h @ w.T + b
        bar = (w.shape[1] + 1) * U * (np.abs(h) @ np.abs(w).T + np.abs(b)) + bar @ np.abs(w).T
        if i < 2:
            h = np.maximum(z, 0)
        else:
            s = 1.0 / (1.0 + np.exp(-z))
            return s, s * (1 - s) * bar + 4 * U * s


def mlp_layers(C0, H1, H2, NO, seed):
    g = torch.Generator().manual_seed(seed)
    dims = [(H1, C0), (H2, H1), (NO, H2)]
    return [((torch.randn(o, i, generator=g) * (2.0 / i) ** 0.5).to(DEV), (torch.randn(o, generator=g) * 0.3).to(DEV)) for o, i in dims]


def run_mlp(x, fmt, layers):
    """x (N, P, C0) float32 CUDA; fmt 0 = float32, 1 = split-fp16 made by lt_f32_to_s32.  -> (out, the operands the kernel read)."""
    N, P, C0 = x.shape
    NO = layers[2][0].shape[0]
    if fmt == capi.FMT_S32:
        s = torch.empty(N * P * 2 * C0, dtype=torch.float16, device=DEV)
        capi.f32_to_s32(x.contiguous(), s, N * P, C0)
        exact = torch.empty_like(x)
        capi.s32_to_f32(s, exact, N * P, C0)
        inp = s
    else:
        inp, exact = x.contiguous(), x
    out = Guarded((N, NO))
    capi.gap_mlp3(inp, fmt, N, P, C0, layers[0], layers[1], layers[2], out.t)
    torch.cuda.synchronize()
    assert out.guards_intact() and out.unwritten() == 0
    return out.t.cpu().numpy(), exact.double().cpu().numpy()


MLP_SHAPES = [(4, 1, 256, 512, 256, 17), (4, 9, 256, 512, 256, 17), (3, 1, 256, 512, 256, 32), (3, 9, 256, 512, 256, 32),
              (2, 144, 288, 700, 130, 257), (5, 7, 96, 33, 300, 1), (1, 3, 32, 1, 1, 3)]


@pytest.mark.parametrize("fmt", [capi.FMT_F32, capi.FMT_S32], ids=["f32", "s32"])
@pytest.mark.parametrize("shape", MLP_SHAPES, ids=lambda s: "N%d-P%d-C%d-H%d-H%d-NO%d" % s)
def test_gap_mlp3_vs_float64(shape, fmt):
    N, P, C0, H1, H2, NO = shape
    x = torch.randn(N, P, C0, generator=torch.Generator().manual_seed(P + C0)).to(DEV) * 2
    layers = mlp_layers(C0, H1, H2, NO, seed=C0 + H1)
    got, exact = run_mlp(x, fmt, layers)
    want, bar = mlp_reference(exact, layers)
    worst = float(np.max(np.abs(got - want) / bar))
    print("gap_mlp3 %s fmt %d: worst err/bar %.3g" % (shape, fmt, worst))
    assert worst <= 1.0


def test_gap_mlp3_f32_input_with_c0_off_the_thread_count():
    """C0 = 300 (no multiple of 32: float32 input only), H1 = 257, NO = 300: every loop of the 256-thread CTA has a tail."""
    N, P, C0, H1, H2, NO = 3, 5, 300, 257, 255, 300
    x = torch.randn(N, P, C0, generator=torch.Generator().manual_seed(1)).to(DEV)
    layers = mlp_layers(C0, H1, H2, NO, seed=2)
    got, exact = run_mlp(x, capi.FMT_F32, layers)
    want, bar = mlp_reference(exact, layers)
    assert float(np.max(np.abs(got - want) / bar)) <= 1.0


def test_gap_mlp3_shared_memory_edge():
    """C0 + H1 + H2 = 12288 floats (48 KB of shared memory) is accepted; one more is rejected before any launch."""
    C0, H1, H2, NO = 4096, 4096, 4096, 3
    x = torch.randn(2, 1, C0, generator=torch.Generator().manual_seed(3)).to(DEV)
    layers = mlp_layers(C0, H1, H2, NO, seed=4)
    got, exact = run_mlp(x, capi.FMT_F32, layers)
    want, bar = mlp_reference(exact, layers)
    assert float(np.max(np.abs(got - want) / bar)) <= 1.0
    big = mlp_layers(C0, H1, H2 + 1, NO, seed=4)
    with pytest.raises(RuntimeError, match="hidden sizes too large"):
        capi.gap_mlp3(x, capi.FMT_F32, 2, 1, C0, big[0], big[1], big[2], torch.empty(2, NO, device=DEV))


def test_gap_mlp3_saturated_logits():
    """Logits of +-100 and beyond: exactly 1 and 0, never NaN."""
    C0, H1, H2 = 64, 32, 32
    z = torch.tensor([100.0, -100.0, 1000.0, -1000.0, 88.0, -88.0, 104.0, -104.0], device=DEV)
    layers = mlp_layers(C0, H1, H2, len(z), seed=5)
    layers[2] = (torch.zeros_like(layers[2][0]), z)
    got, _ = run_mlp(torch.randn(2, 3, C0, device=DEV), capi.FMT_F32, layers)
    assert not np.isnan(got).any()
    assert (got[:, [0, 2, 6]] == 1.0).all() and (got[:, [1, 3, 7]] == 0.0).all()
    assert (got[:, 4] <= 1.0).all() and (got[:, 5] >= 0.0).all()


# ---- view normalisation -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("eps", [0.0, 1e-5])
@pytest.mark.parametrize("V", range(1, 9))
@pytest.mark.parametrize("BC", [(1, 127), (2, 64), (3, 43), (1, 255), (4, 64), (1, 257), (17, 17)], ids=lambda s: "B%dxC%d" % s)
def test_view_normalize_vs_float64(BC, V, eps):
    B, C = BC
    rng = np.random.RandomState(V * 100 + C)
    conf = (rng.rand(B, V, C) * 2 + 1e-3).astype(np.float32)
    buf = Guarded((B, V, C), fill=torch.from_numpy(conf))
    capi.view_normalize(buf.t, B, V, C, eps)
    torch.cuda.synchronize()
    assert buf.guards_intact()
    c = conf.astype(np.float64)
    q = c / c.sum(1, keepdims=True)
    want = q + np.float64(np.float32(eps))
    bar = (V + 1) * U * q + U * want                 # the float32 sum of V positive terms, the division, the add
    worst = float(np.max(np.abs(buf.t.cpu().numpy() - want) / bar))
    assert worst <= 1.0, worst


def test_view_normalize_zero_column_is_nan():
    """A column summing to zero gives 0 / 0 = NaN (plus eps), like the reference's conf / conf.sum(1); its neighbours are finite."""
    B, V, C = 2, 4, 130
    conf = np.random.RandomState(0).rand(B, V, C).astype(np.float32) + 0.1
    conf[1, :, 129] = 0
    conf[0, :, 0] = 0
    t = torch.from_numpy(conf).to(DEV)
    capi.view_normalize(t, B, V, C, 1e-5)
    got = t.cpu().numpy()
    assert np.isnan(got[1, :, 129]).all() and np.isnan(got[0, :, 0]).all()
    mask = np.ones((B, C), bool)
    mask[1, 129] = mask[0, 0] = False
    assert np.isfinite(got.transpose(0, 2, 1)[mask]).all()
