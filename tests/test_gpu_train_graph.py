"""GPU tests of CUDA-graph training (`train_graph=True`): graphed steps against eager steps from the same state, the capture cache,
host-synchronisation freedom, anomaly mode, DataLoader-fed steps and output lifetime.

The bar is measured, not assumed: the eager steps run three times from the same state, and every quantity x of the graphed run must
satisfy ||x_graphed - x_eager|| <= max(2 max ||x_eager - x_eager'||, 1e-7 ||x_eager||) over the pairs of eager runs (L2 norms per
tensor).  The unprojection backward's atomics spread the backbone gradients between eager runs; norms over three pairs estimate
that spread better than a maximum over one pair.  Adam runs with eps = 1e-3: with the default 1e-8 its first step is lr * sign(g),
which turns any last-bit difference of a near-zero gradient element (for example cuDNN choosing another algorithm under capture)
into a parameter difference of 2 lr; with eps = 1e-3 a parameter moves by at most the change of its gradient.  What the native
kernels compute bit for bit (the first forward's outputs and the running statistics it writes) must be bit-identical graphed.
Convolutions and BatchNorm on torch run in full fp32, as in the other parity tests.

The algebraic steps on the native switches hold to that bar with a factor of 2 (they are bit-identical through three steps).  The
algebraic steps on the torch switches (cuDNN may choose other, order-dependent algorithms under capture) and the volumetric steps get a factor of 10, and only the first step is held to the bar: its backward has order-dependent atomics, and equal
eager launches reproduce much of their order while graph replay, with other timing, does not, so eager repeats under-sample that
spread.  From the second step on, that first-step difference is amplified by the step's ReLU and BatchNorm decisions: on an H100 the
graphed second-step gradients of the native switches were up to 20x the eager-only spread.  Later steps are checked for their
BatchNorm step counts, their capture count and finite losses.  With the torch switches the volumetric first-step gradients are not
compared at all: cuDNN's choices under capture put single V2V weight gradients at up to 14x the eager spread in one run and inside
it in the next, so only the first step's loss, forward outputs and running statistics are held to the bar there.
"""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import loss as ce, testing
from lt_b200.train_graph import _norm_state

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, V, S = 2, 2, 128
NATIVE = dict(backbone_backend="native", v2v_backend="native", norm_backend="native")


def _vol_config():
    return testing.make_config(num_layers=18, volume_size=32, aggregation="conf_norm")


@pytest.fixture(scope="module")
def vol_state():
    torch.manual_seed(0)
    holder = lt_b200.VolumetricTriangulationNet(_vol_config(), device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=0, calib_size=S, calib_views=1)
    return holder.state_dict()


@pytest.fixture(scope="module")
def vol_data():
    images, batch = testing.make_batch(B, V, image_size=S, seed=4)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    return images.to(DEV), batch, gt[..., :3], gt[..., 3:]


def _vol_model(state, switches, graph, **kw):
    m = lt_b200.VolumetricTriangulationNet(_vol_config(), device="cpu", backend="hybrid", train_graph=graph, **switches, **kw)
    m.load_state_dict(state)
    return m.to(DEV).train()


def _vol_loss(data, out, loss_fn):
    _, batch, kp_gt, valid = data
    kp, _, vols, _, _, coord, _ = out
    mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
    return 0.1 * mae + 0.01 * loss_fn(coord, vols, kp_gt, valid)


def _train(m, forward, step_loss, steps=3):
    """steps Adam steps from np.random.seed(step): per step the loss, the parameter gradients, the parameters and BatchNorm state
    after the step; the first step's forward outputs."""
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, eps=1e-3)
    names = [n for n, p in m.named_parameters() if p.requires_grad]
    rec = []
    for step in range(steps):
        np.random.seed(step)
        opt.zero_grad(set_to_none=True)
        out = forward(m, step)
        loss = step_loss(out)
        loss.backward()
        params = dict(m.named_parameters())
        r = {"loss": loss.detach().clone(), "grads": {n: params[n].grad.clone() for n in names if params[n].grad is not None}}
        if step == 0:
            r["outs"] = [None if o is None else o.detach().clone() for o in out if torch.is_tensor(o) or o is None]
        opt.step()
        r["params"] = {n: p.detach().clone() for n, p in params.items()}
        r["norm"] = [b.clone() for b in _norm_state(m)]
        rec.append(r)
    torch.cuda.synchronize()
    return rec


def _within(label, g, e, others, factor, exact=False):
    """||g - e|| <= max(factor max ||a - b|| over the pairs of eager runs (e, *others), 1e-7 ||e||)."""
    g, e = g.double(), e.double()
    runs = [e] + [o.double() for o in others]
    d = float((g - e).norm())
    spread = max(float((a - b).norm()) for i, a in enumerate(runs) for b in runs[i + 1:])
    bar = max(factor * spread, 1e-7 * float(e.norm()))
    assert g.shape == e.shape, label
    if exact:
        assert torch.equal(g, e), "%s: not bit-identical (||diff|| %.3e)" % (label, d)
    assert d <= bar, "%s: ||graphed - eager|| %.3e > bar %.3e (eager spread %.3e)" % (label, d, bar, spread)
    return d, bar


def _compare(graphed, eagers, exact_outputs, factor=2, bar_steps=None, grads=True):
    """Every quantity of the first bar_steps steps (all by default) within the bar; num_batches_tracked exact and losses finite in all."""
    worst = 0.0
    for step, g in enumerate(graphed):
        assert bool(torch.isfinite(g["loss"])), "loss of step %d" % step
        if bar_steps is not None and step >= bar_steps:
            for i, (gb, eb) in enumerate(zip(g["norm"], eagers[0][step]["norm"])):
                if eb.dtype == torch.int64:
                    assert torch.equal(gb, eb), "num_batches_tracked %d after step %d" % (i, step)
            continue
        e, others = eagers[0][step], [r[step] for r in eagers[1:]]
        checks = [("loss", g["loss"], e["loss"], [o["loss"] for o in others])]
        assert g["grads"].keys() == e["grads"].keys()
        if grads:
            checks += [("grad " + n, g["grads"][n], e["grads"][n], [o["grads"][n] for o in others]) for n in e["grads"]]
            checks += [("param " + n, g["params"][n], e["params"][n], [o["params"][n] for o in others]) for n in e["params"]]
        for i, (gb, eb) in enumerate(zip(g["norm"], e["norm"])):
            if eb.dtype == torch.int64:
                assert torch.equal(gb, eb), "num_batches_tracked %d after step %d" % (i, step)
            else:
                # the first step's running statistics come from the first forward, which the native kernels compute bit for bit
                checks.append(("norm buffer %d" % i, gb, eb, [o["norm"][i] for o in others]))
                if exact_outputs and step == 0:
                    assert torch.equal(gb, eb), "norm buffer %d after the first step" % i
        if step == 0:
            for i, go in enumerate(g["outs"]):
                if e["outs"][i] is not None:
                    checks.append(("output %d" % i, go, e["outs"][i], [o["outs"][i] for o in others]))
                    if exact_outputs:
                        assert torch.equal(go, e["outs"][i]), "output %d of the first forward" % i
        for label, a, b, c in checks:
            d, bar = _within("%s step %d" % (label, step), a, b, c, factor)
            worst = max(worst, d / bar if bar else 0.0)
    print("worst ||graphed - eager|| / bar: %.3f" % worst)


@pytest.fixture(autouse=True)
def _fp32():
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


def _vol_forward(data):
    images, batch = data[:2]
    return lambda m, step: m(images, None, batch)


@pytest.mark.parametrize("switches", ["native", "torch"])
def test_volumetric_graphed_steps_match_eager(vol_state, vol_data, switches):
    sw = NATIVE if switches == "native" else {}
    loss_fn = ce.VolumetricCELoss(backend="native")
    step_loss = lambda out: _vol_loss(vol_data, out, loss_fn)
    runs = [_train(_vol_model(vol_state, sw, graph), _vol_forward(vol_data), step_loss) for graph in (False, False, False, True)]
    _compare(runs[-1], runs[:-1], exact_outputs=switches == "native", factor=10, bar_steps=1, grads=switches == "native")


def _alg_config(use_conf, softmax):
    cfg = testing.make_alg_config(num_layers=18, use_confidences=use_conf)
    cfg.model.heatmap_softmax = softmax
    return cfg


@pytest.mark.parametrize("use_conf,softmax,switches", [(True, True, "native"), (True, False, "native"), (False, True, "native"),
                                                       (False, False, "native"), (True, True, "torch")])
def test_algebraic_graphed_steps_match_eager(use_conf, softmax, switches):
    sw = dict(backbone_backend="native", norm_backend="native") if switches == "native" else {}
    Va, J = 3, 17
    images, batch = testing.make_batch(B, Va, image_size=S, seed=11)
    images = images.to(DEV)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    g = torch.Generator().manual_seed(12)
    target = (torch.from_numpy(np.stack([k[:, :3] for k in batch["keypoints_3d"]])).float() + torch.randn(B, J, 3, generator=g) * 50).to(DEV)
    validity = (torch.rand(B, J, 1, generator=g) > 0.2).float()
    denom = 3 * max(1.0, float(validity.sum()))
    validity = validity.to(DEV)
    holder = lt_b200.AlgebraicTriangulationNet(_alg_config(use_conf, softmax), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
    sd = holder.state_dict()

    def model(graph):
        m = lt_b200.AlgebraicTriangulationNet(_alg_config(use_conf, softmax), device="cpu", backend="hybrid", train_graph=graph, **sw)
        m.load_state_dict(sd)
        return m.to(DEV).train()
    forward = lambda m, step: m(images, proj, batch)
    step_loss = lambda out: (torch.abs(target - out[0]) * validity).sum() / denom
    runs = [_train(model(graph), forward, step_loss) for graph in (False, False, False, True)]
    if switches == "native":
        _compare(runs[-1], runs[:-1], exact_outputs=True)
    else:
        _compare(runs[-1], runs[:-1], exact_outputs=False, factor=10, bar_steps=1)


def test_capture_cache():
    """On the algebraic model with the native switches: a 32^3 V2V net cannot take B = 1 in train mode (its deepest BatchNorm would
    see one value per channel)."""
    holder = lt_b200.AlgebraicTriangulationNet(_alg_config(True, True), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
    state = holder.state_dict()
    m = lt_b200.AlgebraicTriangulationNet(_alg_config(True, True), device="cpu", backend="hybrid", train_graph=True,
                                          backbone_backend="native", norm_backend="native")
    m.load_state_dict(state)
    m = m.to(DEV).train()
    graphs = m._train_graphs
    data = {}
    for b in (1, 2):
        images, batch = testing.make_batch(b, V, image_size=S, seed=5)
        data[b] = (images.to(DEV), torch.from_numpy(testing.image_projections(batch)).to(DEV), batch)

    def step(b=2):
        kp = m(*data[b])[0]
        (kp * 1e-3).sum().backward()

    for _ in range(3):
        step()
        assert graphs.captures == 1
    step(1)
    assert graphs.captures == 2
    step()
    step(1)
    assert graphs.captures == 2
    m.to(DEV)
    step()
    assert graphs.captures == 3
    m.load_state_dict(state)
    step()
    assert graphs.captures == 4
    w = m.backbone.alg_confidences.head[0].weight
    w.requires_grad_(False)
    step()
    assert graphs.captures == 5
    w.requires_grad_(True)
    step()                                                 # back to the mask of the entry captured after load_state_dict
    assert graphs.captures == 5
    w.data = w.data.clone()
    step()
    assert graphs.captures == 6
    m.eval()
    with torch.no_grad():
        kp_eval = m(*data[2])[0]
    assert kp_eval.grad_fn is None and graphs.captures == 6
    m.train()
    step()
    assert graphs.captures == 6


def test_replay_without_host_synchronisation(vol_state, vol_data):
    images, batch = vol_data[:2]
    m = _vol_model(vol_state, NATIVE, True)
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        kp, features, volumes = m(images, None, batch)[:3]
        ((kp * 1e-3).sum() + volumes.mean()).backward()
        torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m.zero_grad(set_to_none=True)
        kp, features, volumes = m(images, None, batch)[:3]
        ((kp * 1e-3).sum() + volumes.mean()).backward()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert m._train_graphs.captures == 1
    assert m.volume_net.output_layer.weight.grad is not None


def test_anomaly_mode(vol_state, vol_data):
    loss_fn = ce.VolumetricCELoss(backend="native")
    step_loss = lambda out: _vol_loss(vol_data, out, loss_fn)
    eager = [_train(_vol_model(vol_state, NATIVE, False), _vol_forward(vol_data), step_loss) for _ in range(3)]
    m = _vol_model(vol_state, NATIVE, True)
    with torch.autograd.detect_anomaly():
        graphed = _train(m, _vol_forward(vol_data), step_loss)
    assert m._train_graphs.captures == 1
    _compare(graphed, eager, exact_outputs=True, factor=10, bar_steps=1)


class _Images(torch.utils.data.Dataset):
    def __init__(self, images):
        self.images = images

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return self.images[i]


def test_dataloader_fed_steps(vol_state, vol_data):
    """A DataLoader with a worker and a pin-memory thread feeds the steps, as in train.py; the capture happens on the first step."""
    batch = vol_data[1]
    images = [testing.make_batch(B, V, image_size=S, seed=20 + i)[0] for i in range(3)]
    loss_fn = ce.VolumetricCELoss(backend="native")
    step_loss = lambda out: _vol_loss(vol_data, out, loss_fn)
    eager = [_train(_vol_model(vol_state, NATIVE, False), lambda m, step: m(images[step].to(DEV), None, batch), step_loss)
             for _ in range(3)]
    loader = torch.utils.data.DataLoader(_Images(images), batch_size=None, num_workers=1, pin_memory=True)
    it = iter(loader)
    m = _vol_model(vol_state, NATIVE, True)
    graphed = _train(m, lambda m, step: m(next(it).to(DEV, non_blocking=True), None, batch), step_loss)
    assert m._train_graphs.captures == 1
    _compare(graphed, eager, exact_outputs=True, factor=10, bar_steps=1)


def test_output_lifetime(vol_state, vol_data):
    images, batch = vol_data[:2]
    for clone in (True, False):
        m = _vol_model(vol_state, NATIVE, True)
        m.clone_outputs = clone
        outs = []
        for step in range(2):
            np.random.seed(step)
            kp, features, volumes = m(images, None, batch)[:3]
            (kp * 1e-3).sum().backward()
            outs.append((kp, kp.detach().clone(), volumes))
        torch.cuda.synchronize()
        (kp0, kp0_at_step, vol0), (kp1, _, vol1) = outs
        assert not torch.equal(kp0_at_step, kp1)           # another rotation, so other key points
        if clone:
            assert torch.equal(kp0, kp0_at_step) and kp0.data_ptr() != kp1.data_ptr() and vol0.data_ptr() != vol1.data_ptr()
        else:
            assert kp0.data_ptr() == kp1.data_ptr() and vol0.data_ptr() == vol1.data_ptr() and torch.equal(kp0, kp1)
