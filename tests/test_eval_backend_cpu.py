"""eval_backend="native" without a GPU: the constructor rule, which forwards go to the native engine, and the one freshness rule --
every train-mode forward (eager or graphed, with or without gradients) and every TrainStep call invalidates the model's engine and
leaves the training graphs in place.  A stub stands in for the engine."""
import contextlib

import pytest
import torch

import lt_b200
from lt_b200 import testing
from lt_b200.train_graph import _StepEntry


def _vol(**kw):
    return lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=18, volume_size=32), device="cpu", **kw)


def _alg(**kw):
    return lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18, use_confidences=False), device="cpu", **kw)


class _StubEngine:
    def __init__(self):
        self.invalidated = 0

    def invalidate(self):
        self.invalidated += 1


_FakeCuda = type("FakeCuda", (torch.Tensor,), {"is_cuda": property(lambda self: True)})


def _fake_cuda(t):
    """A CPU tensor that reports CUDA: the dispatch checks pass, nothing runs on a device."""
    t = t.clone()
    t.__class__ = _FakeCuda
    return t


@pytest.mark.parametrize("make", [_vol, _alg])
@pytest.mark.parametrize("value", ["torch", "hybrid", "Native", "", True])
def test_unknown_values_raise(make, value):
    with pytest.raises(ValueError, match="eval_backend"):
        make(backend="hybrid", eval_backend=value)


@pytest.mark.parametrize("make", [_vol, _alg])
def test_accepted_with_every_backend_and_switch(make):
    switches = dict(backbone_backend="native", norm_backend="native", head_backend="native")
    if make is _vol:
        switches["v2v_backend"] = "native"
    for kw in (dict(backend="torch"), dict(backend="native"), dict(backend="hybrid"), dict(backend="hybrid", train_graph=True),
               dict(backend="hybrid", train_graph=True, **switches)):
        assert make(eval_backend="native", **kw).eval_backend == "native"
        assert make(**kw).eval_backend is None


@pytest.mark.parametrize("make", [_vol, _alg])
def test_default_never_touches_the_engine(make, monkeypatch):
    """eval_backend=None: an eval forward without gradients runs the torch formulation and creates no engine."""
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    proj = torch.from_numpy(testing.image_projections(batch))
    m = make(backend="torch").eval()
    monkeypatch.setattr(m, "_forward_native", lambda *a: pytest.fail("the native engine ran"))
    with torch.no_grad():
        kp = m(images, proj, batch)[0]
    assert torch.isfinite(kp).all() and m._engine is None


def _routes(m, images, proj, batch, monkeypatch):
    """-> {(training, grad): "native" | "torch"}: where each mode's forward goes."""
    monkeypatch.setattr(m, "_forward_native", lambda *a: "native")
    monkeypatch.setattr(m, "_forward_torch", lambda *a: "torch")
    if isinstance(m, lt_b200.VolumetricTriangulationNet):
        monkeypatch.setattr(m, "_run_device", lambda fn, inputs: pytest.fail("the volumetric _forward_torch is patched"))
    else:
        monkeypatch.setattr(m, "_run_device", lambda fn, inputs: fn(*inputs))
    out = {}
    for training in (True, False):
        m.train(training)
        for grad in (True, False):
            with torch.set_grad_enabled(grad):
                out[(training, grad)] = m(images, proj, batch)
    return out


@pytest.mark.parametrize("make", [_vol, _alg])
@pytest.mark.parametrize("backend", ["torch", "hybrid"])
def test_only_eval_without_grad_goes_to_the_engine(make, backend, monkeypatch):
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    images, proj = _fake_cuda(images), _fake_cuda(torch.from_numpy(testing.image_projections(batch)))
    routes = _routes(make(backend=backend, eval_backend="native"), images, proj, batch, monkeypatch)
    assert routes == {(True, True): "torch", (True, False): "torch", (False, True): "torch", (False, False): "native"}
    routes = _routes(make(backend=backend), images, proj, batch, monkeypatch)
    assert set(routes.values()) == {"torch"}


@pytest.mark.parametrize("make", [_vol, _alg])
def test_native_backend_is_unchanged(make, monkeypatch):
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    images, proj = _fake_cuda(images), _fake_cuda(torch.from_numpy(testing.image_projections(batch)))
    for eval_backend in (None, "native"):
        routes = _routes(make(backend="native", eval_backend=eval_backend), images, proj, batch, monkeypatch)
        assert set(routes.values()) == {"native"}


@pytest.mark.parametrize("make", [_vol, _alg])
def test_cpu_tensors_raise(make):
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    m = make(backend="torch", eval_backend="native").eval()
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        m(images, torch.from_numpy(testing.image_projections(batch)), batch)


@pytest.mark.parametrize("backend", ["native", "torch"])
def test_algebraic_odd_sides(backend, monkeypatch):
    """The tensor-core modes' space-to-depth stem needs even image sides (ValueError before any device work); the exact-fp32 mode's
    stem is an ordinary conv and takes odd sides."""
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    images, proj = _fake_cuda(images[..., :63]), _fake_cuda(torch.from_numpy(testing.image_projections(batch)))

    class _Engine:
        def algebraic_forward(self, *args):
            return "eager"

        def algebraic_forward_graphed(self, *args):
            return ()

    for mode in ("tc", "tc1"):
        m = _alg(backend=backend, eval_backend="native", conv_mode=mode).eval()
        monkeypatch.setattr(m, "engine", lambda: pytest.fail("the engine ran"))
        with torch.no_grad(), pytest.raises(ValueError, match="even image sides"):
            m(images, proj, batch)
    m = _alg(backend=backend, eval_backend="native", conv_mode="simt").eval()
    monkeypatch.setattr(m, "engine", _Engine)
    monkeypatch.setattr(torch.cuda, "device", lambda device: contextlib.nullcontext())
    with torch.no_grad():
        assert m(images, proj, batch) == ("eager" if backend == "native" else ())


@pytest.mark.parametrize("make", [_vol, _alg])
def test_train_mode_forwards_invalidate_the_engine(make):
    """Eager train-mode forwards with and without gradients invalidate the engine; eval forwards on the torch path do not."""
    images, batch = testing.make_batch(2, 2, image_size=64, seed=1)
    proj = torch.from_numpy(testing.image_projections(batch))
    m = make(backend="torch", eval_backend="native")
    eng = m._engine = _StubEngine()
    m.train()
    m(images, proj, batch)
    assert eng.invalidated == 1
    with torch.no_grad():
        m(images, proj, batch)
    assert eng.invalidated == 2
    m.eval()
    m(images, proj, batch)                    # eval with gradients: the torch path, nothing changes
    assert eng.invalidated == 2


@pytest.mark.parametrize("make", [_vol, _alg])
def test_graphed_training_forward_invalidates_the_engine_only(make, monkeypatch):
    images, batch = testing.make_batch(2, 2, image_size=64, seed=1)
    proj = torch.from_numpy(testing.image_projections(batch))
    m = make(backend="hybrid", train_graph=True, eval_backend="native").train()
    m.backend = "torch"                       # CPU: the same forward with torch's ops in place of the native custom ops
    eng = m._engine = _StubEngine()
    sentinel = object()
    m._train_graphs._entries["k"] = sentinel
    replayed = []
    monkeypatch.setattr(m._train_graphs, "run", lambda model, fn, inputs, clone: replayed.append(fn) or fn(*inputs))
    m(images, proj, batch)
    assert len(replayed) == 1 and eng.invalidated == 1
    assert m._train_graphs._entries == {"k": sentinel}


@pytest.mark.parametrize("eval_backend", [None, "native"])
def test_train_step_invalidates_the_engine_only(eval_backend, monkeypatch):
    """A TrainStep call replays Adam and the BatchNorm updates inside its graph: it invalidates the engine and keeps its own graphs and
    the model's train_graph entries.  A stub entry stands in for the captured step."""
    cfg = testing.make_train_config(testing.make_alg_config(num_layers=18, use_confidences=False), criterion="MSESmooth",
                                    mse_smooth_threshold=400)
    m = lt_b200.AlgebraicTriangulationNet(cfg, device="cpu", backend="hybrid", train_graph=True, eval_backend=eval_backend)
    eng = m._engine = _StubEngine()
    sentinel = object()
    m._train_graphs._entries["k"] = sentinel
    step = lt_b200.TrainStep(m, torch.optim.Adam(m.parameters(), lr=1e-4, capturable=True), cfg)
    replays = []

    class _Graph:
        def replay(self):
            replays.append(eng.invalidated)

    def capture(inputs):
        e = _StepEntry()
        e.graph, e.static_in, e.outs, e.metrics, e.grads = _Graph(), [t.clone() for t in inputs], [torch.zeros(1)] * 4, {}, []
        return e

    monkeypatch.setattr(step, "_capture", capture)
    images, batch = testing.make_batch(2, 2, image_size=64, seed=2)
    images, kp, valid, proj = testing.prepare_batch(batch, images, "cpu")
    for n in (1, 2):
        step(_fake_cuda(images), kp, valid, proj, batch)
        assert eng.invalidated == n and replays[-1] == n          # invalidated before the replay
    assert step.captures == 1 and len(step._entries) == 1
    assert m._train_graphs._entries == {"k": sentinel}
