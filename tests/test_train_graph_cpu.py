"""train_graph=True without a GPU: the constructor rules, CPU tensors, and which forwards go to the CUDA graphs."""
import pytest
import torch

import lt_b200
from lt_b200 import testing


def _vol(**kw):
    return lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=18, volume_size=32), device="cpu", **kw)


def _alg(**kw):
    return lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18), device="cpu", **kw)


@pytest.mark.parametrize("make", [_vol, _alg])
@pytest.mark.parametrize("backend", ["torch", "native"])
def test_train_graph_needs_the_hybrid_backend(make, backend):
    with pytest.raises(ValueError, match="train_graph"):
        make(backend=backend, train_graph=True)
    assert make(backend=backend)._train_graphs is None


@pytest.mark.parametrize("make", [_vol, _alg])
def test_train_graph_composes_with_every_switch(make):
    switches = dict(backbone_backend="native", norm_backend="native")
    if make is _vol:
        switches["v2v_backend"] = "native"
    assert make(backend="hybrid", train_graph=True, **switches)._train_graphs is not None
    assert make(backend="hybrid", train_graph=True)._train_graphs is not None


def test_cpu_tensors_raise_in_train_mode():
    images, batch = testing.make_batch(1, 2, image_size=64, seed=0)
    m = _vol(backend="hybrid", train_graph=True).train()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(images, None, batch)
    a = _alg(backend="hybrid", train_graph=True).train()
    with pytest.raises(RuntimeError, match="CUDA"):
        a(images, torch.from_numpy(testing.image_projections(batch)), batch)


@pytest.mark.parametrize("make", [_vol, _alg])
def test_only_training_forwards_with_gradients_replay(make, monkeypatch):
    """Eval and no-grad forwards call the device function directly, as without train_graph; a train-mode forward with gradients
    goes to the capture cache."""
    m = make(backend="hybrid", train_graph=True)
    replayed = []
    monkeypatch.setattr(m._train_graphs, "run", lambda model, fn, inputs, clone: replayed.append(fn) or "graphed")
    fn = lambda *xs: ("eager",) + xs
    m.eval()
    assert m._run_device(fn, (1, 2)) == ("eager", 1, 2)
    with torch.no_grad():
        assert m._run_device(fn, (1,)) == ("eager", 1)
    m.train()
    with torch.no_grad():
        assert m._run_device(fn, (1,)) == ("eager", 1)
    assert not replayed
    assert m._run_device(fn, (1,)) == "graphed" and replayed == [fn]


def test_eval_forward_is_unchanged():
    """The torch formulation on the CPU (the hybrid forward's device function with the torch ops) gives the same outputs with and
    without the train_graph switch of a hybrid model in eval mode."""
    images, batch = testing.make_batch(1, 2, image_size=64, seed=1)
    ref = _vol(backend="torch")
    testing.randomize_weights(ref, seed=2, calib_size=64, calib_views=1)
    m = _vol(backend="hybrid", train_graph=True)
    m.load_state_dict(ref.state_dict())
    m.backend = "torch"                      # CPU: the same forward with torch's ops in place of the native custom ops
    with torch.no_grad():
        a = ref.eval()(images, None, batch)
        b = m.eval()(images, None, batch)
    for x, y in zip(a, b):
        if torch.is_tensor(x):
            assert torch.equal(x, y)


def test_invalidation_drops_the_training_graphs():
    m = _vol(backend="hybrid", train_graph=True)
    m._train_graphs._entries["k"] = object()
    m.to("cpu")
    assert not m._train_graphs._entries
    m._train_graphs._entries["k"] = object()
    m.load_state_dict(m.state_dict())
    assert not m._train_graphs._entries
