"""GPU tests of lt_b200.TrainStep: whole recipe steps from one CUDA graph against the restated eager train.py step
(testing.reference_train_step) from the same state, the capture cache, host-synchronisation freedom and DataLoader-fed steps.

Models, sizes and bars are those of tests/test_gpu_train_graph.py: ResNet-18, 32^3, B = V = 2, capturable Adam with eps = 1e-3,
fp32 convolutions.  A graphed quantity x must satisfy ||x_graphed - x_eager|| <= max(factor * spread, 1e-7 ||x_eager||), where the
spread is the largest difference between three eager runs.  The volumetric step (order-dependent atomics in the unprojection
backward) is held to that bar with factor 10 on its first step, where its metrics, gradients, parameters, Adam state and
BatchNorm buffers are compared; later steps are checked for their num_batches_tracked and finite metrics.  The eager step computes
the criterion with the reference's float32 formula, the graph with the float64 kernel, so the algebraic step on the native
switches is compared bit for bit with an eager step that calls the same native criterion, and its metrics with the reference
formula's within 1e-5 relative."""
import copy

import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import loss as crit, testing
from lt_b200.train_graph import _norm_state

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, V, S = 2, 2, 128
VOL_SWITCHES = dict(backbone_backend="native", v2v_backend="native", norm_backend="native")
ALG_SWITCHES = dict(backbone_backend="native", norm_backend="native")


@pytest.fixture(autouse=True)
def _fp32():
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _vol_config():
    return testing.make_train_config(testing.make_config(num_layers=18, volume_size=32, aggregation="conf_norm"), criterion="MAE",
                                     lr=1e-4, use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01, scale_keypoints_3d=0.1,
                                     process_features_lr=1e-3, volume_net_lr=1e-3, grad_clip=1e-5)


def _alg_config(use_conf):
    return testing.make_train_config(testing.make_alg_config(num_layers=18, use_confidences=use_conf), criterion="MSESmooth",
                                     lr=1e-4, mse_smooth_threshold=400, scale_keypoints_3d=0.1)


@pytest.fixture(scope="module")
def vol_state():
    torch.manual_seed(0)
    holder = lt_b200.VolumetricTriangulationNet(_vol_config(), device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=0, calib_size=S, calib_views=1)
    return holder.state_dict()


def _alg_state(use_conf):
    holder = lt_b200.AlgebraicTriangulationNet(_alg_config(use_conf), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
    return holder.state_dict()


def _data(n_views=V, seed=4, b=B):
    """prepare_batch's tensors and the batch, with some invalid joints; noisy ground truth for the algebraic model."""
    images, batch = testing.make_batch(b, n_views, image_size=S, seed=seed)
    rng = np.random.RandomState(seed)
    for k in batch["keypoints_3d"]:
        k[rng.choice(17, 3, replace=False), 3] = 0.0
        k[:, :3] += rng.normal(0, 40, size=(17, 3))
    return testing.prepare_batch(batch, images, DEV) + (batch,)


def _model(make, config, state, switches, graph=False):
    m = make(config, device="cpu", backend="hybrid", train_graph=graph, **switches)
    m.load_state_dict(state)
    return m.to(DEV).train()


def _record(m, opt, metrics):
    names = [n for n, p in m.named_parameters() if p.requires_grad]
    params = dict(m.named_parameters())
    return {"metrics": {k: float(v) for k, v in metrics.items()},
            "grads": {n: params[n].grad.clone() for n in names},
            "params": {n: p.detach().clone() for n, p in params.items()},
            "adam": {"%s.%s" % (n, k): v.clone() for n in names for k, v in opt.state[params[n]].items()},
            "norm": [b.clone() for b in _norm_state(m)]}


def _eager(make, config, state, switches, data, steps=3, criterion=None):
    """steps of the restated train.py loop from np.random.seed(step); criterion "native" swaps in lt_b200's native criterion."""
    m = _model(make, config, state, switches)
    opt = testing.recipe_optimizer(m, config, eps=1e-3, capturable=True)
    orig = testing.reference_keypoints_loss
    if criterion == "native":
        testing.reference_keypoints_loss = lambda kind, p, g, v, t=400: crit.keypoints_loss(kind, p, g, v, t, backend="native")
    try:
        rec = []
        for step in range(steps):
            np.random.seed(step)
            _, metrics = testing.reference_train_step(m, opt, config, *data)
            rec.append(_record(m, opt, metrics))
    finally:
        testing.reference_keypoints_loss = orig
    torch.cuda.synchronize()
    return rec


def _graphed(make, config, state, switches, data, steps=3):
    m = _model(make, config, state, switches)
    opt = testing.recipe_optimizer(m, config, eps=1e-3, capturable=True)
    step_fn = lt_b200.TrainStep(m, opt, config)
    rec = []
    for step in range(steps):
        np.random.seed(step)
        _, metrics = step_fn(*data)
        r = _record(m, opt, metrics)
        norms = sum(float(p.grad.norm()) ** 2 for p in m.parameters() if p.requires_grad) ** 0.5
        assert abs(r["metrics"]["grad_norm_times_lr"] - config.opt.lr * norms) <= 1e-6 * config.opt.lr * norms
        rec.append(r)
    assert step_fn.captures == 1
    torch.cuda.synchronize()
    return rec


def _within(label, g, e, others, factor, floor=1e-7):
    g, e = g.double(), e.double()
    runs = [e] + [o.double() for o in others]
    spread = max(float((a - b).norm()) for i, a in enumerate(runs) for b in runs[i + 1:])
    d = float((g - e).norm())
    bar = max(factor * spread, floor * float(e.norm()))
    assert d <= bar, "%s: ||graphed - eager|| %.3e > bar %.3e (eager spread %.3e)" % (label, d, bar, spread)


def _compare(graphed, eagers, factor, bar_steps, floor=1e-7, parts=("grads", "params", "adam")):
    for step, g in enumerate(graphed):
        e, others = eagers[0][step], [r[step] for r in eagers[1:]]
        assert g["metrics"].keys() == e["metrics"].keys()
        assert all(np.isfinite(x) for x in g["metrics"].values()), step
        for i, (gb, eb) in enumerate(zip(g["norm"], e["norm"])):
            if eb.dtype == torch.int64:
                assert torch.equal(gb, eb), "num_batches_tracked %d after step %d" % (i, step)
        if step >= bar_steps:
            continue
        for k in e["metrics"]:
            _within("metric %s" % k, torch.tensor(g["metrics"][k]), torch.tensor(e["metrics"][k]),
                    [torch.tensor(o["metrics"][k]) for o in others], factor, floor)
        for part in parts:
            assert g[part].keys() == e[part].keys()
            for n in e[part]:
                _within("%s %s step %d" % (part, n, step), g[part][n], e[part][n], [o[part][n] for o in others], factor, floor)
        for i, eb in enumerate(e["norm"]):
            if eb.dtype != torch.int64:
                _within("norm buffer %d" % i, g["norm"][i], eb, [o["norm"][i] for o in others], factor, floor)


def test_volumetric_step_matches_train_py(vol_state):
    data = _data()
    cfg = _vol_config()
    make = lt_b200.VolumetricTriangulationNet
    eagers = [_eager(make, cfg, vol_state, VOL_SWITCHES, data) for _ in range(3)]
    graphed = _graphed(make, cfg, vol_state, VOL_SWITCHES, data)
    assert set(graphed[0]["metrics"]) == {"MAE", "volumetric_ce_loss", "total_loss", "grad_norm_times_lr", "l2", "base_point_l2"}
    _compare(graphed, eagers, factor=10, bar_steps=1)


def test_one_view_volumetric_step(vol_state):
    """With one view the eager steps repeat bit for bit (no cross-view atomics), so the bar is a relative floor: the graph's 1-view
    transform is a torch.where where train.py indexes with a boolean mask, which sums the base joint's gradient in another order.
    Gradients and Adam moments are not compared: the biases in front of a BatchNorm have gradients that are zero up to rounding."""
    data = _data(n_views=1, seed=6)
    cfg = _vol_config()
    make = lt_b200.VolumetricTriangulationNet
    eagers = [_eager(make, cfg, vol_state, VOL_SWITCHES, data, steps=1, criterion="native") for _ in range(3)]
    _compare(_graphed(make, cfg, vol_state, VOL_SWITCHES, data, steps=1), eagers, factor=10, bar_steps=1, floor=1e-5,
             parts=("params",))


@pytest.mark.parametrize("use_conf", [True, False])
def test_algebraic_step_matches_train_py(use_conf):
    data = _data(seed=11)
    cfg = _alg_config(use_conf)
    state = _alg_state(use_conf)
    make = lt_b200.AlgebraicTriangulationNet
    same_kernels = _eager(make, cfg, state, ALG_SWITCHES, data, criterion="native")
    reference = _eager(make, cfg, state, ALG_SWITCHES, data)
    graphed = _graphed(make, cfg, state, ALG_SWITCHES, data)
    assert set(graphed[0]["metrics"]) == {"MSESmooth", "total_loss", "grad_norm_times_lr", "l2"}
    for step, (g, e, r) in enumerate(zip(graphed, same_kernels, reference)):
        for part in ("grads", "params", "adam"):
            for n in e[part]:
                assert torch.equal(g[part][n], e[part][n]), "%s %s after step %d" % (part, n, step)
        assert all(torch.equal(a, b) for a, b in zip(g["norm"], e["norm"])), step
        for k in ("MSESmooth", "total_loss", "l2"):
            assert g["metrics"][k] == e["metrics"][k] or abs(g["metrics"][k] - r["metrics"][k]) <= 1e-5 * abs(r["metrics"][k]), k
            assert abs(g["metrics"][k] - r["metrics"][k]) <= 1e-5 * abs(r["metrics"][k]), k
        assert abs(g["metrics"]["grad_norm_times_lr"] - e["metrics"]["grad_norm_times_lr"]) <= 1e-6 * e["metrics"]["grad_norm_times_lr"]


def test_capture_cache_and_first_replay():
    cfg = _alg_config(True)
    state = _alg_state(True)
    m = _model(lt_b200.AlgebraicTriangulationNet, cfg, state, ALG_SWITCHES)
    opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
    step = lt_b200.TrainStep(m, opt, cfg)
    data = {b: _data(seed=5, b=b) for b in (1, 2)}
    step(*data[2])
    assert step.captures == 1
    assert all(float(s["step"]) == 1 for s in opt.state.values())            # the first replay was the first update
    for _ in range(2):
        step(*data[2])
    assert step.captures == 1
    step(*data[1])
    assert step.captures == 2
    step(*data[2])
    assert step.captures == 2
    opt.param_groups[0]["lr"] = 2e-4
    step(*data[2])
    assert step.captures == 3
    opt.load_state_dict(copy.deepcopy(opt.state_dict()))           # new state tensors
    step(*data[2])
    assert step.captures == 4
    m.to(DEV)
    step(*data[2])
    assert step.captures == 5
    w = m.backbone.alg_confidences.head[0].weight
    w.requires_grad_(False)
    step(*data[2])
    assert step.captures == 6
    w.requires_grad_(True)
    step(*data[2])
    assert step.captures == 7                      # the capture above replaced the graphs of the same input shapes
    m.eval()
    m.train()
    m.zero_grad()
    _, metrics = step(*data[2])
    assert step.captures == 7 and bool(torch.isfinite(metrics["total_loss"]))
    assert all(p.grad is not None for p in m.parameters() if p.requires_grad)


def test_replay_without_host_synchronisation(vol_state):
    data = _data()
    cfg = _vol_config()
    m = _model(lt_b200.VolumetricTriangulationNet, cfg, vol_state, VOL_SWITCHES)
    step = lt_b200.TrainStep(m, testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True), cfg)
    step(*data)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        _, metrics = step(*data)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert step.captures == 1 and bool(torch.isfinite(metrics["total_loss"]))


class _Images(torch.utils.data.Dataset):
    def __init__(self, images):
        self.images = images

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return self.images[i]


def test_dataloader_fed_steps():
    """A DataLoader with a worker and a pin-memory thread feeds the images, as in train.py; the steps equal directly fed ones."""
    cfg = _alg_config(True)
    state = _alg_state(True)
    _, kp, valid, proj, batch = _data(seed=8)
    images = [testing.make_batch(B, V, image_size=S, seed=30 + i)[0] for i in range(3)]
    runs = []
    for fed in (False, True):
        m = _model(lt_b200.AlgebraicTriangulationNet, cfg, state, ALG_SWITCHES)
        step = lt_b200.TrainStep(m, testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True), cfg)
        it = iter(torch.utils.data.DataLoader(_Images(images), batch_size=None, num_workers=1, pin_memory=True)) if fed else None
        out = []
        for i in range(3):
            x = next(it).to(DEV, non_blocking=True) if fed else images[i].to(DEV)
            out.append(step(x, kp, valid, proj, batch)[1]["total_loss"])
        assert step.captures == 1
        runs.append(torch.stack(out))
    assert torch.equal(runs[0], runs[1])
