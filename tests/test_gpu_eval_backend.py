"""GPU tests of eval_backend="native": the eval forward of a hybrid model after training equals, bit for bit, a fresh backend="native"
model loaded with its state dict; it stays fresh across TrainStep calls, graphed training forwards (only BatchNorm statistics change)
and eager optimizer steps; evaluations leave training bit-identical; one graph per input shape and refresh; replays without host
synchronisation; accuracy against the hybrid eager eval with TF32 off; the native backend's errors.

ResNet-18 (ResNet-50 for the accuracy test), 128^2, 32^3 grid, B = V = 2."""
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from conftest import rel_err
import lt_b200
from lt_b200 import testing
from lt_b200.train_graph import _norm_state
from test_gpu_forward import TOL

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
B, V, S, N = 2, 2, 128, 32
VOL_NATIVE = dict(backbone_backend="native", v2v_backend="native", norm_backend="native", head_backend="native")
ALG_NATIVE = dict(backbone_backend="native", norm_backend="native", head_backend="native")
Vol, Alg = lt_b200.VolumetricTriangulationNet, lt_b200.AlgebraicTriangulationNet


def _vol_config(agg="conf_norm", kind="mpii", num_layers=18):
    return testing.make_train_config(testing.make_config(num_layers=num_layers, volume_size=N, aggregation=agg, kind=kind),
                                     criterion="MAE", lr=1e-4, use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01,
                                     scale_keypoints_3d=0.1)


def _alg_config(use_conf=True, softmax=True, num_layers=18):
    cfg = testing.make_train_config(testing.make_alg_config(num_layers=num_layers, use_confidences=use_conf), criterion="MSESmooth",
                                    lr=1e-4, mse_smooth_threshold=400, scale_keypoints_3d=0.1)
    cfg.model.heatmap_softmax = softmax
    return cfg


_STATES = {}


def _state(make, cfg):
    """Calibrated seeded weights of the model `cfg` describes, made once per configuration."""
    key = (make.__name__, json.dumps(cfg.model, sort_keys=True, default=str))
    if key not in _STATES:
        holder = make(cfg, device="cpu", backend="torch")
        if make is Vol:
            testing.randomize_weights(holder, seed=0, calib_size=S, calib_views=1)
        else:
            testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
        _STATES[key] = holder.state_dict()
    return _STATES[key]


def _model(make, cfg, switches, **kw):
    m = make(cfg, device="cpu", backend="hybrid", eval_backend="native", **switches, **kw)
    m.load_state_dict(_state(make, cfg))
    return m.to(DEV).train()


def _data(b=B, seed=4, views=V):
    """(images, keypoints_3d, validity, image-space projections, batch) as TrainStep and the models take them."""
    images, batch = testing.make_batch(b, views, image_size=S, seed=seed)
    return testing.prepare_batch(batch, images, DEV) + (batch,)


def _eval(m, data):
    """m's eval forward without gradients; m goes back to its mode."""
    was = m.training
    m.eval()
    with torch.no_grad():
        out = m(data[0], data[3], data[4])
    m.train(was)
    return out


def _fresh_native(make, cfg, m):
    r = make(cfg, device="cpu", backend="native")
    r.load_state_dict(m.state_dict())
    return r.to(DEV).eval()


def _assert_same(got, want, label):
    assert len(got) == len(want), label
    for i, (a, b) in enumerate(zip(got, want)):
        if a is None or b is None:
            assert a is None and b is None, "%s: output %d" % (label, i)
        elif torch.is_tensor(a):
            assert a.shape == b.shape and a.dtype == b.dtype and torch.equal(a, b), "%s: output %d differs" % (label, i)
        else:                                                        # the volumetric model's cuboids
            assert len(a) == len(b) and all(np.array_equal(c.position, d.position) and np.array_equal(c.sides, d.sides)
                                            for c, d in zip(a, b)), "%s: cuboids" % label


def _check_fresh(make, cfg, m, data, label):
    """m's eval forward equals a fresh native model of m's current state dict, with finite key points -> the outputs."""
    out = _eval(m, data)
    _assert_same(out, _eval(_fresh_native(make, cfg, m), data), label)
    assert bool(torch.isfinite(out[0]).all()), label
    return out


def _loss(out):
    return (out[0] * 1e-3).sum() + (out[2].mean() if len(out) == 7 else 0.0)


@pytest.fixture(autouse=True)
def _fp32():
    prev = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


CASES = [(Vol, dict(agg="softmax", kind="mpii")), (Vol, dict(agg="conf_norm", kind="coco")),
         (Alg, dict(use_conf=True, softmax=True)), (Alg, dict(use_conf=True, softmax=False)),
         (Alg, dict(use_conf=False, softmax=True)), (Alg, dict(use_conf=False, softmax=False))]


@pytest.mark.parametrize("switches", ["native", "torch"])
@pytest.mark.parametrize("make,kw", CASES, ids=["vol-softmax-mpii", "vol-conf_norm-coco", "alg-conf-softmax", "alg-conf-relu",
                                               "alg-softmax", "alg-relu"])
def test_eval_after_training_equals_a_native_model(make, kw, switches):
    cfg = (_vol_config if make is Vol else _alg_config)(**kw)
    sw = (VOL_NATIVE if make is Vol else ALG_NATIVE) if switches == "native" else {}
    m = _model(make, cfg, sw)
    data = _data()
    opt = torch.optim.Adam(m.parameters(), lr=1e-4, eps=1e-3)
    for step in range(2):
        np.random.seed(step)
        opt.zero_grad(set_to_none=True)
        _loss(m(data[0], data[3], data[4])).backward()
        opt.step()
    out = _check_fresh(make, cfg, m, data, "after two training steps")
    assert len(out) == (7 if make is Vol else 4)
    if make is Vol:
        assert (out[3] is not None) == (kw["agg"] == "conf_norm")


@pytest.mark.parametrize("switches", ["native", "torch"])
@pytest.mark.parametrize("make", [Vol, Alg], ids=["vol", "alg"])
def test_eval_sees_every_update(make, switches):
    """eval -> TrainStep call -> eval -> graphed training forward and backward (BatchNorm statistics only: replayed, and written through
    pointers on the native switches) -> eval -> eager Adam step (tensor versions) -> eval.  Each eval equals a fresh native model of the
    state dict at that point and differs from the eval before it."""
    cfg = _vol_config() if make is Vol else _alg_config()
    sw = (VOL_NATIVE if make is Vol else ALG_NATIVE) if switches == "native" else {}
    m = _model(make, cfg, sw, train_graph=True)
    data = _data()
    opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
    step = lt_b200.TrainStep(m, opt, cfg)
    outs = [_check_fresh(make, cfg, m, data, "before training")]
    np.random.seed(0)
    step(*data)
    outs.append(_check_fresh(make, cfg, m, data, "after a TrainStep call"))
    norm = [b.clone() for b in _norm_state(m)]
    params = [p.detach().clone() for p in m.parameters()]
    np.random.seed(1)
    m.zero_grad(set_to_none=True)
    _loss(m(data[0], data[3], data[4])).backward()
    assert m._train_graphs.captures == 1
    assert all(torch.equal(p, q) for p, q in zip(m.parameters(), params))
    assert not all(torch.equal(a, b) for a, b in zip(_norm_state(m), norm))
    outs.append(_check_fresh(make, cfg, m, data, "after a graphed training forward"))
    with warnings.catch_warnings():
        warnings.filterwarnings("ignore", message=".*capturable=True.*")
        opt.step()
    outs.append(_check_fresh(make, cfg, m, data, "after an eager optimizer step"))
    for i in range(1, len(outs)):
        assert not torch.equal(outs[i][0], outs[i - 1][0]), "eval %d repeats eval %d" % (i, i - 1)


def _steps_with_and_without_evals(make, cfg, sw, steps=3):
    """steps TrainStep calls from np.random.seed(step), with and without an eval forward after each -> the mismatching quantities
    (parameters, Adam state, BatchNorm buffers) of the two runs."""
    data = _data()
    rec = []
    for evals in (False, True):
        m = _model(make, cfg, sw)
        opt = testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True)
        step = lt_b200.TrainStep(m, opt, cfg)
        for s in range(steps):
            np.random.seed(s)
            step(*data)
            if evals:
                _eval(m, data)
        torch.cuda.synchronize()
        r = {"param " + n: p.detach().clone() for n, p in m.named_parameters()}
        r.update({"adam %s %s" % (n, k): v.clone() for n, p in m.named_parameters() for k, v in opt.state.get(p, {}).items()})
        r.update({"norm %d" % i: b.clone() for i, b in enumerate(_norm_state(m))})
        rec.append(r)
    assert rec[0].keys() == rec[1].keys()
    return [k for k in rec[0] if not torch.equal(rec[0][k], rec[1][k])]


def test_evals_leave_algebraic_training_unchanged():
    assert _steps_with_and_without_evals(Alg, _alg_config(), ALG_NATIVE) == []


_CHILD = r"""
import json, sys
sys.path[:0] = [sys.argv[1], sys.argv[2]]
import torch
torch.use_deterministic_algorithms(True)
import test_gpu_eval_backend as T
print(json.dumps(T._steps_with_and_without_evals(T.Vol, T._vol_config(), T.VOL_NATIVE)))
"""


def test_evals_leave_deterministic_volumetric_training_unchanged():
    """Under torch.use_deterministic_algorithms(True) (a child process: the flag is global) the volumetric steps repeat bit for bit,
    so the evaluations between them must change nothing."""
    tests = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHILD, os.path.dirname(tests), tests]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=1500, env=env)
    assert res.returncode == 0, res.stderr[-6000:]
    assert json.loads(res.stdout.strip().splitlines()[-1]) == []


@pytest.mark.parametrize("make", [Vol, Alg], ids=["vol", "alg"])
def test_one_capture_per_shape_and_refresh(make):
    cfg = _vol_config() if make is Vol else _alg_config()
    m = _model(make, cfg, VOL_NATIVE if make is Vol else ALG_NATIVE)
    eng = m.engine()
    full, short = _data(), _data(b=1, seed=5)                     # a short last batch
    for _ in range(2):
        _eval(m, full)
    assert eng.captures == 1
    for _ in range(2):
        _eval(m, short)
        _eval(m, full)
    assert eng.captures == 2
    with torch.no_grad():
        m(full[0], full[3], full[4])                            # a train-mode forward refreshes the engine
    assert eng.captures == 2 and not eng._graphs
    for _ in range(2):
        _eval(m, full)
    assert eng.captures == 3
    _eval(m, short)
    assert eng.captures == 4
    assert m.engine() is eng


@pytest.mark.parametrize("make", [Vol, Alg], ids=["vol", "alg"])
def test_replayed_eval_without_host_synchronisation(make):
    cfg = _vol_config() if make is Vol else _alg_config()
    m = _model(make, cfg, VOL_NATIVE if make is Vol else ALG_NATIVE)
    data = _data()
    want = _eval(m, data)
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = _eval(m, data)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert m.engine().captures == 1
    _assert_same(got, want, "replay")


@pytest.mark.parametrize("make", [Vol, Alg], ids=["vol", "alg"])
def test_accuracy_against_the_hybrid_eager_eval(make):
    """With TF32 off, the native eval is within test_gpu_forward's "tc" bars (features, volumes and heat maps, key points in mm) of the
    hybrid eager eval of the same weights (an eval forward with gradients, on the torch switches); the confidences, the algebraic model's
    2-D key points (4 views) and the coordinate volumes within test_gpu_algebraic's bars against its oracle."""
    cfg = _vol_config(agg="conf_norm", num_layers=50) if make is Vol else _alg_config(num_layers=50)
    m = _model(make, cfg, {}).eval()
    data = _data(views=2 if make is Vol else 4)
    with torch.no_grad():
        native = m(data[0], data[3], data[4])
    eager = [o.detach() if torch.is_tensor(o) else o for o in m(data[0], data[3], data[4])]
    t_feat, _, t_vol, t_kp = TOL["tc"]
    if make is Vol:
        e = dict(features=rel_err(native[1].cpu().numpy(), eager[1].cpu().numpy()),
                 volumes=rel_err(native[2].cpu().numpy(), eager[2].cpu().numpy()),
                 kp=float((native[0] - eager[0]).abs().max()), conf=float((native[3] - eager[3]).abs().max()))
        print("volumetric native vs hybrid eager: %s" % e)
        assert e["features"] < t_feat and e["volumes"] < t_vol and e["kp"] < t_kp and e["conf"] < 1e-4
        assert float((native[5] - eager[5]).abs().max()) < 1e-2 and torch.equal(native[6], eager[6])     # mm
    else:
        e = dict(heat=rel_err(native[2].cpu().numpy(), eager[2].cpu().numpy()), kp3d=float((native[0] - eager[0]).abs().max()),
                 kp2d=float((native[1] - eager[1]).abs().max()), conf=float((native[3] - eager[3]).abs().max()))
        print("algebraic native vs hybrid eager: %s" % e)
        assert e["heat"] < t_vol and e["kp3d"] < t_kp and e["kp2d"] < 0.02 and e["conf"] < 1e-4


@pytest.mark.parametrize("make", [Vol, Alg], ids=["vol", "alg"])
def test_errors(make):
    cfg = _vol_config() if make is Vol else _alg_config()
    m = _model(make, cfg, {}).eval()
    images, _, _, proj, batch = _data()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="CUDA"):
            m(images.cpu(), proj.cpu(), batch)
        with pytest.raises(ValueError, match="even image sides"):
            m(images[..., :S - 1], proj, batch)


class _Images(torch.utils.data.Dataset):
    def __init__(self, images):
        self.images = images

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return self.images[i]


@pytest.mark.parametrize("make", [Vol, Alg], ids=["vol", "alg"])
def test_dataloader_fed_eval_passes(make):
    """As train.py's validation pass: a DataLoader with a worker and pin_memory=True feeds the eval forwards after a TrainStep call,
    twice; the first forward of each pass captures while the pin-memory thread prefetches batches of another size than the
    training batch.  Every forward equals a replay of the same batch fed directly, bit for bit."""
    cfg = _vol_config() if make is Vol else _alg_config()
    m = _model(make, cfg, VOL_NATIVE if make is Vol else ALG_NATIVE)
    step = lt_b200.TrainStep(m, testing.recipe_optimizer(m, cfg, eps=1e-3, capturable=True), cfg)
    train = _data()
    val = [testing.make_batch(3, V, image_size=S, seed=40 + i) for i in range(4)]
    proj = [torch.from_numpy(testing.image_projections(batch)).to(DEV) for _, batch in val]
    for epoch in range(2):
        np.random.seed(epoch)
        step(*train)
        loader = torch.utils.data.DataLoader(_Images([images for images, _ in val]), batch_size=None, num_workers=1, pin_memory=True)
        got = [_eval(m, (x.to(DEV, non_blocking=True), None, None, proj[i], val[i][1])) for i, x in enumerate(loader)]
        assert len(got) == len(val) and m.engine().captures == epoch + 1
        for i, (images, batch) in enumerate(val):
            _assert_same(got[i], _eval(m, (images.to(DEV), None, None, proj[i], batch)), "epoch %d, batch %d" % (epoch, i))
        assert m.engine().captures == epoch + 1
