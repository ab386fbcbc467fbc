"""GPU tests of the native training BatchNorm (norm_backend="native": autograd_ops.batch_norm -> lt_batch_norm_fwd / _bwd): each
configuration against float64 autograd of F.batch_norm (+ add) (+ ReLU) on the device, every BatchNorm of a training step redone from
the data a float64 copy of the model records, and whole training steps against the same steps on cuDNN in full fp32."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from conftest import rel_err
from lt_b200 import autograd_ops as A
from test_gpu_backbone_train import _compare, _no_tf32, _train, _weight_noise

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BAR = 1e-6
QUANTITIES = ("y", "dx", "dr", "dw", "db", "rm", "rv")

# name -> (input shape, relu, residual): 2-D and 3-D, C from 16 to 2048, odd sides, M from 2 to ~10^6
CONFIGS = {
    "2d C16 relu": ((2, 16, 13, 11), True, False),
    "2d C32 relu res": ((3, 32, 13, 11), True, True),
    "2d C64": ((2, 64, 9, 7), False, False),
    "2d C256 res": ((2, 256, 7, 5), False, True),
    "2d C2048 relu res": ((4, 2048, 3, 3), True, True),
    "2d C2048 M=2": ((2, 2048, 1, 1), True, False),
    "2d C64 relu M=1e6": ((4, 64, 500, 500), True, False),
    "3d C16 relu": ((2, 16, 9, 9, 9), True, False),
    "3d C32 relu res": ((2, 32, 9, 9, 9), True, True),
    "3d C128 relu res": ((3, 128, 5, 5, 5), True, True),
    "3d C64": ((2, 64, 3, 5, 7), False, False),
    "3d C32 relu res M=1.3e6": ((5, 32, 64, 64, 64), True, True),
}


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last if t.dim() == 4 else torch.channels_last_3d)


def _problem(shape, residual, seed, mean=0.0, dy_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    C = shape[1]
    bn = (nn.BatchNorm2d if len(shape) == 4 else nn.BatchNorm3d)(C, momentum=0.1)
    with torch.no_grad():
        bn.weight.copy_(1.0 + 0.3 * torch.randn(C, generator=g))
        bn.bias.copy_(0.2 * torch.randn(C, generator=g))
        bn.running_mean.copy_(0.1 * torch.randn(C, generator=g))
        bn.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    scale = torch.rand((1, C) + (1,) * (len(shape) - 2), generator=g) * 2 + 0.1
    x = (torch.randn(shape, generator=g) * scale + mean + 0.5 * torch.randn((1, C) + (1,) * (len(shape) - 2), generator=g))
    r = torch.randn(shape, generator=g) if residual else None
    gy = torch.randn(shape, generator=g) * 1e-3 * dy_scale
    return bn, x.to(DEV), None if r is None else r.to(DEV), gy.to(DEV)


def _run(bn, x, r, gy, relu, train, how):
    """how: "native" (fp32 kernels), "cudnn" (fp32 torch) or "f64" (float64 torch autograd)."""
    m = copy.deepcopy(bn).to(DEV).train(train)
    dt = torch.float64 if how == "f64" else torch.float32
    m = m.to(dt)
    xx = _cl(x.to(dt)).requires_grad_(True)
    rr = None if r is None else _cl(r.to(dt)).requires_grad_(True)
    if how == "native":
        y = A.batch_norm(m, xx, relu=relu, residual=rr)
    else:
        y = m(xx)
        if rr is not None:
            y = y + rr
        if relu:
            y = F.relu(y)
    y.backward(gy.to(dt))
    return {"y": y.detach(), "dx": xx.grad, "dr": None if rr is None else rr.grad, "dw": m.weight.grad, "db": m.bias.grad,
            "rm": m.running_mean, "rv": m.running_var, "nbt": int(m.num_batches_tracked)}


def _errs(res, ref):
    return {q: None if res[q] is None else rel_err(res[q].double().cpu().numpy(), ref[q].double().cpu().numpy()) for q in QUANTITIES}


def _check(bn, x, r, gy, relu, train, label):
    """rel_err is relative to the reference's own magnitude, so a scaled dY is compared as it is."""
    ref = _run(bn, x, r, gy, relu, train, "f64")
    nat = _run(bn, x, r, gy, relu, train, "native")
    cud = _run(bn, x, r, gy, relu, train, "cudnn")
    en, ec = _errs(nat, ref), _errs(cud, ref)
    if train and x.numel() // x.shape[1] == 2:
        # two values per channel normalise to -1 and +1 whatever x is, so the exact dx is zero and any fp32 dx is rounding noise of
        # x - mean (one ulp of x against |x1 - x2| / 2), for cuDNN as for the native kernels: there is nothing to compare
        en["dx"] = None
    print("%-28s %s" % (label, "  ".join("%s %s/%s" % (q, "-" if en[q] is None else "%.1e" % en[q], "-" if ec[q] is None else "%.1e" % ec[q])
                                         for q in QUANTITIES)))
    for q in QUANTITIES:
        if en[q] is not None:
            assert en[q] <= max(BAR, 2 * ec[q]), (label, q, en[q], ec[q])
    assert nat["nbt"] == ref["nbt"] == (1 if train else 0)
    return nat


@pytest.mark.parametrize("name", list(CONFIGS))
def test_config_vs_float64_autograd(name):
    shape, relu, res = CONFIGS[name]
    bn, x, r, gy = _problem(shape, res, len(name))
    _check(bn, x, r, gy, relu, True, name)


@pytest.mark.parametrize("name", ["2d C32 relu res", "3d C128 relu res", "2d C64", "2d C2048 M=2"])
def test_eval_mode_vs_float64_autograd(name):
    shape, relu, res = CONFIGS[name]
    bn, x, r, gy = _problem(shape, res, 7)
    nat = _check(bn, x, r, gy, relu, False, name + " eval")
    assert torch.equal(nat["rm"].cpu(), bn.running_mean) and torch.equal(nat["rv"].cpu(), bn.running_var)


@pytest.mark.parametrize("name", ["2d C32 relu res", "3d C16 relu", "2d C2048 relu res"])
def test_mean_far_above_std(name):
    """mean = 10^3 std per channel: plain fp32 sums of squares would cancel."""
    shape, relu, res = CONFIGS[name]
    bn, x, r, gy = _problem(shape, res, 3, mean=1e3 * 1.0)
    _check(bn, x, r, gy, relu, True, name + " mean 1e3")


@pytest.mark.parametrize("factor", [1e-9, 1e3])
@pytest.mark.parametrize("name", ["2d C32 relu res", "3d C128 relu res", "2d C64"])
def test_gradients_scale_with_the_output_gradient(name, factor):
    shape, relu, res = CONFIGS[name]
    bn, x, r, gy = _problem(shape, res, 5, dy_scale=factor)
    _check(bn, x, r, gy, relu, True, "%s dY x %g" % (name, factor))


@pytest.mark.parametrize("name", ["2d C32 relu res", "3d C32 relu res", "2d C2048 relu res", "2d C64 relu M=1e6"])
def test_forward_and_backward_are_bitwise_repeatable(name):
    shape, relu, res = CONFIGS[name]
    bn, x, r, gy = _problem(shape, res, 9)
    a = _run(bn, x, r, gy, relu, True, "native")
    b = _run(bn, x, r, gy, relu, True, "native")
    for q in QUANTITIES:
        assert (a[q] is None and b[q] is None) or torch.equal(a[q], b[q]), q


@pytest.mark.parametrize("train", [True, False])
def test_no_host_synchronisation(train):
    bn, x, r, gy = _problem((2, 64, 13, 11), True, 1)
    _run(bn, x, r, gy, True, train, "native")            # library load, workspace
    m = copy.deepcopy(bn).to(DEV).train(train)
    xx = _cl(x).requires_grad_(True)
    rr = _cl(r).requires_grad_(True)
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = A.batch_norm(m, xx, relu=True, residual=rr)
        y.backward(gy)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    torch.cuda.synchronize()
    assert xx.grad is not None and rr.grad is not None and m.weight.grad is not None


def test_error_paths():
    bn = nn.BatchNorm2d(16).to(DEV).train()
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        A.batch_norm(bn.cpu(), torch.zeros(2, 16, 3, 3))
    bn = bn.to(DEV)
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        A.batch_norm(bn, torch.zeros(2, 16, 3, 3, device=DEV), residual=torch.zeros(2, 16, 3, 3))
    for m, shape in ((nn.BatchNorm2d(16, momentum=None), (2, 16, 3, 3)), (nn.BatchNorm2d(16, affine=False), (2, 16, 3, 3)),
                     (nn.BatchNorm3d(16, track_running_stats=False), (2, 16, 2, 2, 2)), (nn.BatchNorm2d(18), (2, 18, 3, 3)),
                     (nn.BatchNorm2d(16), (1, 16, 1, 1))):
        with pytest.raises(ValueError):
            A.batch_norm(m.to(DEV).train(), torch.zeros(shape, device=DEV))


# ---- every BatchNorm of a training step, on the data it meets there ------------------------------------------------------------

def _recording_norm(cap):
    """A float64 `norm` hook: records a copy of the module as it was before the call, its input, residual and output gradient."""
    def norm(m, x, relu=False, residual=None):
        entry = [copy.deepcopy(m), x.detach(), None if residual is None else residual.detach(), relu, None]
        cap.append(entry)
        y = F.batch_norm(x, m.running_mean, m.running_var, m.weight, m.bias, m.training, m.momentum, m.eps)
        if residual is not None:
            y = y + residual
        y = F.relu(y) if relu else y
        y.register_hook(lambda g: entry.__setitem__(4, g.detach()))
        return y
    return norm


def _redo_every_bn(cap, label):
    assert cap and all(e[4] is not None for e in cap)
    prev = _no_tf32()
    try:
        worst = 0.0
        for i, (m, x, r, relu, g) in enumerate(cap):
            tag = "%s bn %d C%d %s" % (label, i, m.num_features, tuple(x.shape[2:]))
            # the float64 reference of the fp32 data both fp32 runs see
            x, g = x.float().double(), g.float().double()
            r = None if r is None else r.float().double()
            m = copy.deepcopy(m).float().double()
            ref = _run(m, x, r, g, relu, True, "f64")
            nat = _run(m, x, r, g, relu, True, "native")
            cud = _run(m, x, r, g, relu, True, "cudnn")
            en, ec = _errs(nat, ref), _errs(cud, ref)
            for q in QUANTITIES:
                if en[q] is not None:
                    worst = max(worst, en[q] / max(BAR, 2 * ec[q]))
                    assert en[q] <= max(BAR, 2 * ec[q]), (tag, q, en[q], ec[q])
        print("%s: %d BatchNorms, worst error / bar %.2f" % (label, len(cap), worst))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.mark.parametrize("layers,style", [(18, "simple"), (50, "simple"), (50, "caffe")])
def test_every_backbone_bn_on_its_training_step_data_vs_float64(layers, style):
    import lt_b200
    from lt_b200 import testing
    cfg = testing.make_alg_config(num_layers=layers, use_confidences=True)
    cfg.model.backbone.style = style
    holder = lt_b200.AlgebraicTriangulationNet(cfg, device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=128)
    n64 = holder.backbone.to(DEV).train().double()
    g = torch.Generator().manual_seed(layers)
    x = torch.randn(4, 3, 128, 128, generator=g).to(DEV).double()
    cap = []
    heat, _, alg, _ = n64(x, None, _recording_norm(cap))
    ((heat * torch.randn(heat.shape, generator=g).to(DEV).double()).sum() * 1e-3 +
     (alg * torch.randn(alg.shape, generator=g).to(DEV).double()).sum() * 1e-2).backward()
    assert len(cap) == sum(isinstance(m, nn.BatchNorm2d) for m in n64.modules())
    _redo_every_bn(cap, "resnet%d %s" % (layers, style))


def test_every_v2v_bn_on_its_training_step_data_vs_float64():
    from lt_b200.v2v import V2VModel
    torch.manual_seed(3)
    net = V2VModel(32, 17).to(DEV).train().double()
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 32, 32, 32, 32, generator=g).to(DEV).double()
    cap = []
    out = net(x, None, _recording_norm(cap))
    (out * torch.randn(out.shape, generator=g).to(DEV).double()).sum().mul(1e-3).backward()
    assert len(cap) == sum(isinstance(m, nn.BatchNorm3d) for m in net.modules())
    _redo_every_bn(cap, "v2v 32^3")


# ---- whole training steps against cuDNN fp32 --------------------------------------------------------------------------------------

def _train_keeping_buffers(make_model, state, step_loss, names):
    made = []

    def make():
        made.append(make_model())
        return made[-1]
    res = _train(make, state, step_loss, names)
    bufs = dict(made[-1].named_buffers())
    running = torch.cat([b.detach().double().flatten() for n, b in bufs.items() if "running" in n])
    tracked = {n: int(b) for n, b in bufs.items() if n.endswith("num_batches_tracked")}
    return res, running, tracked


def _compare_with_buffers(out, names, bars, state):
    _compare({k: v[0] for k, v in out.items()}, names, bars)
    ref = out["torch"][1]
    moved = {k: float((out[k][1] - ref).norm() / ref.norm()) for k in ("native", "noise")}
    bar = max(1e-4, 3 * moved["noise"])
    print("%-60s native %.2e  weight noise %.2e  bar %.2e" % ("running statistics (relative L2)", moved["native"], moved["noise"], bar))
    assert moved["native"] <= bar
    want = {n: int(state[n]) + 2 for n in out["torch"][2]}     # two train-mode steps from the state's counters
    assert out["native"][2] == out["torch"][2] == want


def test_algebraic_training_step_matches_cudnn():
    """ResNet-50 bottleneck with confidences, native convolutions and BatchNorm against cuDNN fp32, with the weight-noise bars of
    tests/test_gpu_backbone_train.py, plus the running statistics of every BatchNorm after the two steps."""
    import lt_b200
    from lt_b200 import testing
    B, V, S, J = 2, 2, 128, 17
    images, batch = testing.make_batch(B, V, image_size=S, seed=11)
    images = images.to(DEV)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    g = torch.Generator().manual_seed(12)
    target = (torch.from_numpy(np.stack([k[:, :3] for k in batch["keypoints_3d"]])).float() + torch.randn(B, J, 3, generator=g) * 50).to(DEV)
    validity = (torch.rand(B, J, 1, generator=g) > 0.2).float().to(DEV)

    def config():
        cfg = testing.make_alg_config(num_layers=50, use_confidences=True)
        cfg.model.backbone.style = "simple"
        return cfg
    holder = lt_b200.AlgebraicTriangulationNet(config(), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=13, calib_size=S)
    sd = holder.state_dict()

    def step_loss(m):
        kp3d = m(images, proj, batch)[0]
        return (torch.abs(target - kp3d) * validity).sum() / (3 * max(1.0, float(validity.sum())))
    names = ["backbone.conv1.weight", "backbone.bn1.weight", "backbone.layer2.0.conv1.weight", "backbone.layer2.0.bn3.bias",
             "backbone.layer2.0.downsample.1.weight", "backbone.layer4.2.conv2.weight", "backbone.deconv_layers.1.weight",
             "backbone.deconv_layers.6.weight", "backbone.final_layer.weight", "backbone.alg_confidences.features.0.weight",
             "backbone.alg_confidences.features.5.weight"]
    prev = _no_tf32()
    out = {}
    try:
        for run, native, state in (("torch", False, sd), ("native", True, sd), ("noise", False, _weight_noise(sd, "backbone"))):
            kw = dict(backbone_backend="native", norm_backend="native") if native else {}
            out[run] = _train_keeping_buffers(
                lambda: lt_b200.AlgebraicTriangulationNet(config(), device="cpu", backend="hybrid", **kw), state, step_loss, names)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    _compare_with_buffers(out, names, [1e-4, 1e-3, 1e-3] + [1e-2] * len(names), sd)


def test_volumetric_training_step_with_all_three_native_backends_matches_cudnn():
    """ResNet-18, 32^3, B = 2, conf aggregation, recipe loss 0.1 MAE + 0.01 CE, Adam: native convolutions of both nets and native
    BatchNorm against cuDNN fp32."""
    import lt_b200
    from lt_b200 import loss as ce, testing
    B, V, S = 2, 2, 128
    images, batch = testing.make_batch(B, V, image_size=S, seed=4)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]

    def config():
        return testing.make_config(num_layers=18, volume_size=32, aggregation="conf_norm")
    torch.manual_seed(0)
    holder = lt_b200.VolumetricTriangulationNet(config(), device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=0, calib_size=S, calib_views=1)
    sd = holder.state_dict()
    loss_fn = ce.VolumetricCELoss(backend="native")

    def step_loss(m):
        kp, _, vols, _, _, coord, _ = m(images, None, batch)
        mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
        return 0.1 * mae + 0.01 * loss_fn(coord, vols, kp_gt, valid)
    names = ["backbone.conv1.weight", "backbone.bn1.weight", "backbone.layer3.0.conv1.weight", "backbone.layer4.1.bn2.bias",
             "backbone.deconv_layers.3.weight", "backbone.vol_confidences.features.0.weight", "process_features.0.weight",
             "volume_net.front_layers.0.block.0.weight", "volume_net.front_layers.0.block.1.weight",
             "volume_net.encoder_decoder.mid_res.res_branch.4.bias", "volume_net.output_layer.weight"]
    prev = _no_tf32()
    out = {}
    try:
        for run, native, state in (("torch", False, sd), ("native", True, sd), ("noise", False, _weight_noise(sd, "backbone"))):
            kw = dict(backbone_backend="native", v2v_backend="native", norm_backend="native") if native else {}
            out[run] = _train_keeping_buffers(
                lambda: lt_b200.VolumetricTriangulationNet(config(), device="cpu", backend="hybrid", **kw), state, step_loss, names)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    _compare_with_buffers(out, names, [1e-4, 1e-3, 1e-3] + [1e-2] * len(names), sd)
