"""CPU checks of the confidence heads' native training tail (head_backend="native"): the per-item code of lt_conf_head_tail_fwd /
_bwd and lt_view_normalize_bwd (csrc/algebraic.cu), run on the host through the lt_test_*_host hooks, against a float64 restatement
of the torch formula (ConfidenceHead: MaxPool2d(2) -> ReLU -> mean -> Linear/ReLU/Linear/ReLU/Linear/Sigmoid; the view normalisation
c / sum_v c + eps), and the switch's validation.  No GPU needed.

Bars, per element, u = 2^-24.  Each layer is checked against float64 from the kernel's own float32 input to that layer (the saved
x0, h1, h2, y), so a bar covers one layer's roundings plus the propagated bars of the float32 values it reads:
  x0 = sum_p r_p / P, r >= 0 exact (max and ReLU round nothing): P - 1 additions and one division -> (P + 1) u sum|r| / P.
  a = b + sum_i w_i v_i as one fmaf per input -> (n + 1) u (|b| + sum|w v|), n inputs; h = ReLU(a) rounds nothing.
  y = 1 / (1 + expf(-a)): sigmoid' <= 1/4 carries the bar of a; expf (<= 2 ulp), the add and the division add <= 3 u y.
  d3 = g y (1 - y): three roundings -> 3 u |d3|.
  d2 = [!(h2 <= 0)] W3^T d3 (fmaf chain of NO) -> (NO + 1) u |W3|^T |d3| + |W3|^T bar(d3); likewise d1 and dx0.
  dx = dx0 / P at the arg-max -> bar(dx0) / P + u |dx|.
  dW = sum_n d_n a_n^T, db = sum_n d_n over N rows in order -> (N + 1) u sum|d a| + sum bar(d) |a|.
The backward's reference is autograd's derivative at the kernel's forward point: the hidden ReLU masks are those of the saved h1, h2
(a mask flips only where a float32 forward rounds across 0, a kink where the derivative does not exist), and the pooling stage's
gradient is torch's own float64 autograd of max_pool2d / relu / mean.  Non-finite values must match exactly, position and value.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from lt_b200 import capi

U = 2.0 ** -24


def make_head(C0=256, H1=512, H2=256, NO=17, seed=0, saturate=False):
    """(w1, b1), (w2, b2), (w3, b3) float32 with nn.Linear's default init scale; saturate puts logits far past sigmoid's range."""
    g = torch.Generator().manual_seed(seed)
    lins = []
    for i, o in ((C0, H1), (H1, H2), (H2, NO)):
        k = 1.0 / math.sqrt(i)
        lins.append(((torch.rand(o, i, generator=g) * 2 - 1) * k, (torch.rand(o, generator=g) * 2 - 1) * k))
    if saturate:
        b3 = lins[2][1].clone()
        b3[0::3] = 120.0
        b3[1::3] = -120.0
        lins[2] = (lins[2][0], b3)
    return tuple(lins)


def make_map(N, C0, H, W, seed=1, channels_last=False, ties=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, C0, H, W, generator=g)
    if ties:        # quantised values: many windows hold their maximum twice or more
        x = torch.round(x * 2) / 2
    return x.contiguous(memory_format=torch.channels_last) if channels_last else x


def pool_stage64(x):
    """x0 = mean(relu(max_pool2d(x, 2))) in float64 with its autograd graph: (x64 leaf, x0, relu(pool) values)."""
    x64 = x.double().requires_grad_(True)
    r = F.relu(F.max_pool2d(x64, 2))
    return x64, r.flatten(2).mean(-1), r


def forward_ref(x, lins, x0k, h1k, h2k):
    """Float64 values and bars of every forward output, each layer from the kernel's float32 input."""
    (w1, b1), (w2, b2), (w3, b3) = [(w.double(), b.double()) for w, b in lins]
    _, x0, r = pool_stage64(x)
    P = r.shape[2] * r.shape[3]
    bars = {"x0": (P + 1) * U * r.detach().abs().flatten(2).sum(-1) / P}
    ref = {"x0": x0.detach()}
    for name, v, w, b in (("h1", x0k, w1, b1), ("h2", h1k, w2, b2), ("a3", h2k, w3, b3)):
        v = v.double()
        a = b + v @ w.t()
        bar = (v.shape[1] + 1) * U * (b.abs() + v.abs() @ w.abs().t())
        if name == "a3":
            y = torch.sigmoid(a)
            ref["y"], bars["y"] = y, 0.25 * bar + 3 * U * y
        else:
            ref[name], bars[name] = F.relu(a), bar
    return ref, bars


def backward_ref(x, lins, x0k, h1k, h2k, yk, g):
    """Float64 gradients and bars at the kernel's forward point (see the module docstring)."""
    (w1, _), (w2, _), (w3, _) = [(w.double(), b.double()) for w, b in lins]
    yk, g = yk.double(), g.double()
    m2, m1 = ~(h2k <= 0), ~(h1k <= 0)
    d3 = g * yk * (1 - yk)
    e3 = 3 * U * d3.abs()
    zero = torch.zeros((), dtype=torch.float64)
    d2 = torch.where(m2, d3 @ w3, zero)         # threshold_backward selects; a product with the mask would turn 0 * inf into NaN
    e2 = torch.where(m2, (w3.shape[0] + 1) * U * (d3.abs() @ w3.abs()) + e3 @ w3.abs(), zero)
    d1 = torch.where(m1, d2 @ w2, zero)
    e1 = torch.where(m1, (w2.shape[0] + 1) * U * (d2.abs() @ w2.abs()) + e2 @ w2.abs(), zero)
    dx0 = d1 @ w1
    ex0 = (w1.shape[0] + 1) * U * (d1.abs() @ w1.abs()) + e1 @ w1.abs()
    x64, x0, _ = pool_stage64(x)
    dx, = torch.autograd.grad(x0, x64, dx0)
    # the bar of dx0 lands where its gradient does: the same autograd map applied to the bar (>= 0) routes it to the arg-max
    x64b = x.double().requires_grad_(True)
    edx, = torch.autograd.grad(F.relu(F.max_pool2d(x64b, 2)).flatten(2).mean(-1), x64b, ex0)
    edx = edx + U * dx.abs()
    N = g.shape[0]
    ref, bars = {"dx": dx}, {"dx": edx}
    for name, d, e, a in (("1", d1, e1, x0k), ("2", d2, e2, h1k), ("3", d3, e3, h2k)):
        a = a.double()
        ref["dW" + name] = d.t() @ a
        bars["dW" + name] = (N + 1) * U * (d.abs().t() @ a.abs()) + e.t() @ a.abs()
        ref["db" + name] = d.sum(0)
        bars["db" + name] = (N + 1) * U * d.abs().sum(0) + e.sum(0)
    return ref, bars


def assert_within(name, got, ref, bar):
    got, ref, bar = got.double(), ref.double(), bar.double()
    fin = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(got), fin), "%s: non-finite pattern differs" % name
    same = (got[~fin] == ref[~fin]) | (torch.isnan(got[~fin]) & torch.isnan(ref[~fin]))
    assert bool(same.all()), "%s: non-finite values differ" % name
    err = (got[fin] - ref[fin]).abs()
    worst = float((err - bar[fin]).max()) if err.numel() else -1.0
    assert bool((err <= bar[fin]).all()), "%s: error exceeds the bar by %.3g (max err %.3g)" % (name, worst, float(err.max()))


def check_tail(x, lins, g):
    """Run the host hook and check every output and gradient against the float64 restatement."""
    out, x0, h1, h2, gx, grads = capi.conf_head_tail_host(x, *lins, grad_y=g)
    ref, bars = forward_ref(x, lins, x0, h1, h2)
    for name, got in (("x0", x0), ("h1", h1), ("h2", h2), ("y", out)):
        assert_within(name, got, ref[name], bars[name])
    assert gx.stride() == x.stride()
    ref, bars = backward_ref(x, lins, x0, h1, h2, out, g)
    assert_within("dx", gx, ref["dx"], bars["dx"])
    for name, got in zip(("dW1", "db1", "dW2", "db2", "dW3", "db3"), grads):
        assert_within(name, got, ref[name], bars[name])
    return out, gx, grads


SHAPES = [(3, 12, 12), (2, 13, 11), (1, 4, 4), (2, 3, 2)]


@pytest.mark.parametrize("N,H,W", SHAPES)
@pytest.mark.parametrize("channels_last", [False, True])
def test_tail_matches_float64(N, H, W, channels_last):
    lins = make_head(NO=17, seed=N + H)
    x = make_map(N, 256, H, W, seed=W, channels_last=channels_last)
    g = torch.randn(N, 17, generator=torch.Generator().manual_seed(5))
    check_tail(x, lins, g)


def test_tail_layouts_agree_bitwise():
    """NCHW and channels_last are read in place; the arithmetic is the same, so every output is the same bit for bit."""
    lins = make_head(NO=32, seed=3)
    x = make_map(2, 256, 13, 11, seed=4)
    g = torch.randn(2, 32, generator=torch.Generator().manual_seed(6))
    a = capi.conf_head_tail_host(x, *lins, grad_y=g)
    b = capi.conf_head_tail_host(x.contiguous(memory_format=torch.channels_last), *lins, grad_y=g)
    for t, s in zip(a[:5], b[:5]):
        assert torch.equal(t, s)
    for t, s in zip(a[5], b[5]):
        assert torch.equal(t, s)


def test_saturated_logits_and_scaled_grads():
    lins = make_head(NO=32, seed=7, saturate=True)
    x = make_map(2, 256, 12, 12, seed=8)
    for scale in (1e-9, 1e3):
        g = torch.randn(2, 32, generator=torch.Generator().manual_seed(9)) * scale
        out, _, grads = check_tail(x, lins, g)
        assert bool((out[:, 0::3] == 1).all()) and bool((out[:, 1::3] == 0).all())
        assert bool((grads[4][0::3] == 0).all()) and bool((grads[5][1::3] == 0).all())     # sigma (1 - sigma) = 0 there


def test_ties_and_all_negative_windows():
    lins = make_head(seed=11)
    x = make_map(2, 256, 12, 12, seed=12, ties=True)
    x[0, :40] = -x[0, :40].abs() - 0.5            # every window of these channels negative: pooled ReLU 0, no gradient
    x[1, 7, :4, :4] = 0.5                         # four equal values: the first takes the gradient
    g = torch.randn(2, 17, generator=torch.Generator().manual_seed(13))
    _, gx, _ = check_tail(x, lins, g)
    assert bool((gx[0, :40] == 0).all())
    assert gx[1, 7, 0, 0] != 0 and bool((gx[1, 7, 0, 1] == 0) & (gx[1, 7, 1, 0] == 0) & (gx[1, 7, 1, 1] == 0))


def test_odd_sides_drop_the_tail():
    lins = make_head(seed=14)
    x = make_map(1, 256, 13, 11, seed=15)
    x[:, :, 12, :] = 100.0                        # the dropped last row and column would win every window they were in
    x[:, :, :, 10] = 100.0
    g = torch.randn(1, 17, generator=torch.Generator().manual_seed(16))
    _, gx, _ = check_tail(x, lins, g)
    assert bool((gx[:, :, 12, :] == 0).all()) and bool((gx[:, :, :, 10] == 0).all())


@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_map_values(value):
    """A NaN takes its window (torch's rule) and survives the ReLUs; +inf overflows its row; -inf loses every window it shares."""
    lins = make_head(seed=17)
    x = make_map(3, 256, 12, 12, seed=18)
    x[1, 5, 3, 4] = value
    g = torch.randn(3, 17, generator=torch.Generator().manual_seed(19))
    out, gx, _ = check_tail(x, lins, g)
    assert bool(torch.isfinite(out[0]).all()) and bool(torch.isfinite(out[2]).all())
    if value != value:
        assert bool(torch.isnan(out[1]).all())


@pytest.mark.parametrize("eps", [1e-5, 0.0])
def test_view_normalize_backward(eps):
    g0 = torch.Generator().manual_seed(20)
    c = torch.rand(3, 4, 17, generator=g0) + 1e-3
    g = torch.randn(3, 4, 17, generator=g0)
    got = capi.view_normalize_bwd_host(c, g)
    c64 = c.double().requires_grad_(True)
    y = c64 / c64.sum(dim=1, keepdim=True) + eps
    ref, = torch.autograd.grad(y, c64, g.double())
    S = c.double().sum(1, keepdim=True)
    # float64 sums of V terms and one float32 rounding at the end
    bar = U * ref.abs() + (4 + 3) * 2.0 ** -52 * (g.double().abs() / S + (g.double() * c.double()).abs().sum(1, keepdim=True) / S ** 2)
    assert bool(((got.double() - ref).abs() <= bar).all())


def test_argument_checks():
    lins = make_head(seed=21)
    with pytest.raises(RuntimeError, match="too small"):
        capi.conf_head_tail_host(make_map(1, 256, 1, 5), *lins)
    with pytest.raises(RuntimeError, match="too small"):
        capi.conf_head_tail_host(make_map(1, 256, 5, 1), *lins)
    big = make_head(C0=256, H1=8192, H2=8192, seed=22)
    with pytest.raises(RuntimeError, match="too large"):
        capi.conf_head_tail_host(make_map(1, 256, 4, 4), *big)


def test_conf_head_tail_hook_checks():
    from lt_b200 import autograd_ops, pose_resnet
    head = pose_resnet.ConfidenceHead(512, 17)
    with pytest.raises(ValueError, match="expected a"):
        autograd_ops.conf_head_tail(head, torch.zeros(2, 128, 12, 12))
    with pytest.raises(ValueError, match="too small"):
        autograd_ops.conf_head_tail(head, torch.zeros(2, 256, 1, 12))
    with pytest.raises(RuntimeError, match="CUDA"):
        autograd_ops.conf_head_tail(head, torch.zeros(2, 256, 12, 12))
    with pytest.raises(RuntimeError, match="CUDA"):
        autograd_ops.view_normalize(torch.ones(2, 4, 17), 1e-5)


def _cfg(**kw):
    from lt_b200 import testing
    return testing.make_config(num_layers=18, volume_size=8, **kw)


def test_head_backend_switch_is_checked():
    import lt_b200
    from lt_b200 import testing
    V, Al = lt_b200.VolumetricTriangulationNet, lt_b200.AlgebraicTriangulationNet
    with pytest.raises(ValueError, match="unknown head_backend"):
        V(_cfg(), device="cpu", backend="hybrid", head_backend="cublas")
    with pytest.raises(ValueError, match="unknown head_backend"):
        Al(testing.make_alg_config(num_layers=18), device="cpu", backend="hybrid", head_backend=None)
    for backend in ("torch", "native"):
        with pytest.raises(ValueError, match="head_backend='native' needs backend='hybrid'"):
            V(_cfg(), device="cpu", backend=backend, head_backend="native")
        with pytest.raises(ValueError, match="head_backend='native' needs backend='hybrid'"):
            Al(testing.make_alg_config(num_layers=18), device="cpu", backend=backend, head_backend="native")
    full = dict(backbone_backend="native", norm_backend="native", v2v_backend="native")
    m = V(_cfg(), device="cpu", backend="hybrid", head_backend="native", train_graph=True, **full)
    assert m.head_backend == "native"
    ref = V(_cfg(), device="cpu", backend="hybrid", **full)
    assert ref.head_backend == "torch" and list(m.state_dict().keys()) == list(ref.state_dict().keys())
    a = Al(testing.make_alg_config(num_layers=18), device="cpu", backend="hybrid", head_backend="native")
    assert a.head_backend == "native"


def test_torch_tail_is_the_default():
    """tail=None runs the torch modules exactly as before: the same values bit for bit as the plain module calls."""
    from lt_b200 import pose_resnet
    torch.manual_seed(0)
    head = pose_resnet.ConfidenceHead(64, 17).eval()
    x = torch.randn(2, 64, 12, 12)
    ref = head.head(head.features(x).flatten(2).mean(dim=-1))
    assert torch.equal(head(x), ref)
    # a tail receives the second BatchNorm's output
    seen = []
    head(x, tail=lambda h, t: seen.append(t) or t.sum())
    assert torch.equal(seen[0], head.features[:6](x))
