"""CPU checks of the native training BatchNorm (norm_backend="native": autograd_ops.batch_norm over csrc/norm.cu), no GPU needed: the
option's rules, the `norm` hook of the backbone and the V2V net (every BatchNorm routed once with the right ReLU / residual flags, and
a hook computing the torch formula reproduces the hook-free forward and its gradients), the module attributes the hook rejects, and
the argument checks of the C entry points.  The kernels themselves are covered by tests/test_gpu_norm_train.py."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import lt_b200
from lt_b200 import autograd_ops as A
from lt_b200 import capi, pose_resnet, testing
from lt_b200.v2v import V2VModel


def _torch_norm(record):
    """A `norm` hook that records (module, relu, has residual) and computes relu(BatchNorm(x) + residual) with torch."""
    def norm(m, x, relu=False, residual=None):
        record.append((m, relu, residual is not None))
        y = F.batch_norm(x, m.running_mean, m.running_var, m.weight, m.bias, m.training, m.momentum, m.eps)
        if residual is not None:
            y = y + residual
        return F.relu(y) if relu else y
    return norm


def _pose_flags(name, kind):
    """(relu, residual) the hook must receive for the backbone BatchNorm `name`."""
    parts = name.split(".")
    if "downsample" in parts or "confidences" in name:
        return False, False
    if name.startswith("layer"):
        return True, parts[-1] == ("bn2" if kind == "basic" else "bn3")
    return True, False          # stem bn1, deconv stack


def _v2v_flags(name):
    if "skip_con" in name:
        return False, False
    return True, name.endswith("res_branch.4")


def _check_routing(net, record, flags):
    names = {id(m): n for n, m in net.named_modules()}
    bns = [n for n, m in net.named_modules() if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm3d))]
    seen = [names[id(m)] for m, _, _ in record]
    assert sorted(seen) == sorted(bns) and len(seen) == len(set(seen))
    for m, relu, res in record:
        assert (relu, res) == flags(names[id(m)]), names[id(m)]


def _check_grads(net, hooked, ref, got):
    """The parameter gradients of sum(out.square().sum()) agree bit for bit between the two forwards."""
    sum(o.square().sum() for o in ref).backward()
    sum(o.square().sum() for o in got).backward()
    for (n, p), (_, q) in zip(net.named_parameters(), hooked.named_parameters()):
        assert p.grad is not None and torch.equal(p.grad, q.grad), n


@pytest.mark.parametrize("layers,style", [(18, "simple"), (50, "simple"), (50, "caffe")])
@pytest.mark.parametrize("train", [False, True])
def test_norm_hook_routes_every_backbone_batchnorm(layers, style, train):
    cfg = testing.make_config(num_layers=layers, style=style).model.backbone
    cfg.alg_confidences = cfg.vol_confidences = True
    torch.manual_seed(layers)
    net = pose_resnet.get_pose_net(cfg, device="cpu").train(train)
    with torch.no_grad():
        for m in net.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.running_mean.normal_(0.0, 0.1)
                m.running_var.uniform_(0.5, 2.0)
    hooked = copy.deepcopy(net)
    x = torch.randn(2, 3, 128, 128)
    record = []
    with torch.set_grad_enabled(train):
        ref = net(x)
        got = hooked(x, None, _torch_norm(record))
    for a, b in zip(ref, got):
        assert torch.equal(a, b)
    _check_routing(hooked, record, lambda n: _pose_flags(n, net.kind))
    for (n, a), (_, b) in zip(net.named_buffers(), hooked.named_buffers()):
        if not n.endswith("num_batches_tracked"):       # the recording hook leaves the counter to the real one
            assert torch.equal(a, b), n
    if train:
        _check_grads(net, hooked, ref, got)


@pytest.mark.parametrize("train", [False, True])
def test_norm_hook_routes_every_v2v_batchnorm(train):
    torch.manual_seed(5)
    net = V2VModel(4, 5).train(train)
    hooked = copy.deepcopy(net)
    x = torch.randn(2, 4, 32, 32, 32)         # two samples: the 1^3 map of level 5 has one value per channel each
    record = []
    with torch.set_grad_enabled(train):
        ref = net(x)
        got = hooked(x, None, _torch_norm(record))
    assert torch.equal(ref, got)
    _check_routing(hooked, record, _v2v_flags)
    if train:
        _check_grads(net, hooked, [ref], [got])


def test_norm_hook_with_conv_hook_keeps_gradients():
    """Both hooks at once on a Res3DBlock with a skip conv: autograd through the fake `norm` equals the hook-free gradients."""
    from lt_b200.v2v import Res3DBlock
    torch.manual_seed(2)
    blk = Res3DBlock(8, 16).train()
    hooked = copy.deepcopy(blk)
    x = torch.randn(2, 8, 5, 4, 3, requires_grad=True)
    xh = x.detach().clone().requires_grad_(True)
    blk(x).square().sum().backward()
    hooked(xh, lambda m, t: m(t), _torch_norm([])).square().sum().backward()
    assert torch.equal(x.grad, xh.grad)
    for (n, p), (_, q) in zip(blk.named_parameters(), hooked.named_parameters()):
        assert torch.equal(p.grad, q.grad), n


def _cfg():
    c = testing.make_config(num_layers=18, volume_size=32)
    c.model.use_confidences = True
    return c


def test_norm_backend_option_is_checked():
    V, Al = lt_b200.VolumetricTriangulationNet, lt_b200.AlgebraicTriangulationNet
    full = dict(backbone_backend="native", v2v_backend="native")
    with pytest.raises(ValueError, match="unknown norm_backend"):
        V(_cfg(), device="cpu", backend="hybrid", norm_backend="cudnn", **full)
    with pytest.raises(ValueError, match="unknown norm_backend"):
        Al(_cfg(), device="cpu", backend="hybrid", backbone_backend="native", norm_backend="fused")
    for backend in ("torch", "native"):
        with pytest.raises(ValueError, match="needs"):
            V(_cfg(), device="cpu", backend=backend, norm_backend="native")
        with pytest.raises(ValueError, match="needs"):
            Al(_cfg(), device="cpu", backend=backend, norm_backend="native")
    with pytest.raises(ValueError, match="norm_backend='native' needs backend='hybrid' and backbone_backend='native' and v2v_backend"):
        V(_cfg(), device="cpu", backend="hybrid", backbone_backend="native", norm_backend="native")
    with pytest.raises(ValueError, match="norm_backend='native' needs"):
        V(_cfg(), device="cpu", backend="hybrid", v2v_backend="native", norm_backend="native")
    with pytest.raises(ValueError, match="norm_backend='native' needs backend='hybrid' and backbone_backend='native'"):
        Al(_cfg(), device="cpu", backend="hybrid", norm_backend="native")
    m = V(_cfg(), device="cpu", backend="hybrid", norm_backend="native", **full)
    ref = V(_cfg(), device="cpu", backend="hybrid", **full)
    assert (m.norm_backend, ref.norm_backend) == ("native", "torch")
    assert list(m.state_dict().keys()) == list(ref.state_dict().keys())
    assert [n for n, _ in m.named_modules()] == [n for n, _ in ref.named_modules()]
    m = Al(_cfg(), device="cpu", backend="hybrid", backbone_backend="native", norm_backend="native")
    ref = Al(_cfg(), device="cpu", backend="hybrid")
    assert m.norm_backend == "native" and list(m.state_dict().keys()) == list(ref.state_dict().keys())


@pytest.mark.parametrize("module,shape", [
    (nn.BatchNorm2d(8, momentum=None), (2, 8, 3, 3)),
    (nn.BatchNorm2d(8, affine=False), (2, 8, 3, 3)),
    (nn.BatchNorm3d(8, track_running_stats=False), (2, 8, 3, 3, 3)),
    (nn.BatchNorm2d(6), (2, 6, 3, 3)),                  # C % 4 != 0
    (nn.BatchNorm2d(8), (1, 8, 1, 1)),                  # one value per channel in train mode
    (nn.BatchNorm2d(8), (2, 4, 3, 3)),                  # channel count differs from the module's
])
def test_hook_rejects_what_the_kernels_do_not_implement(module, shape):
    with pytest.raises(ValueError):
        A.batch_norm(module.train(), torch.zeros(shape))


def test_hook_needs_cuda_tensors():
    with pytest.raises(RuntimeError, match="CUDA tensors"):
        A.batch_norm(nn.BatchNorm2d(8).train(), torch.zeros(2, 8, 3, 3), relu=True)
    with pytest.raises(RuntimeError, match="CUDA tensors"):       # eval mode: one value per channel is fine, the device is not
        A.batch_norm(nn.BatchNorm3d(8).eval(), torch.zeros(1, 8, 1, 1, 1))


def test_workspace_query():
    assert capi.batch_norm_workspace_bytes(0, 64) == 0
    assert capi.batch_norm_workspace_bytes(100, 6) == 0
    small, big = capi.batch_norm_workspace_bytes(2, 16), capi.batch_norm_workspace_bytes(20 * 96 * 96, 2048)
    assert 0 < small < big
    assert big <= 8 << 20                               # bounded whatever M is
    assert capi.batch_norm_workspace_bytes(10 ** 9, 2048) == big


def test_c_entry_points_check_arguments_before_touching_a_device():
    buf = torch.zeros(64)
    p = buf.data_ptr()
    lib = capi.lib()
    ws = capi.batch_norm_workspace_bytes(8, 16)

    def fwd(*, x=p, M=8, C=16, training=1, ws_bytes=ws):
        return lib.lt_batch_norm_fwd(x, None, p, p, p, p, p, p, p, M, C, 1e-5, 0.1, training, 1, p, ws_bytes, None)

    def bwd(*, x=p, y=p, M=8, C=16, training=1, relu=1):
        return lib.lt_batch_norm_bwd(x, y, p, p, p, p, p, None, p, p, M, C, training, relu, p, ws, None)

    for call, msg in ((lambda: fwd(x=None), b"null pointer"), (lambda: fwd(M=0), b"bad sizes"), (lambda: fwd(C=-4), b"bad sizes"),
                      (lambda: fwd(C=18), b"C % 4 != 0"), (lambda: fwd(M=1), b"M >= 2"), (lambda: fwd(ws_bytes=ws - 1), b"workspace too small"),
                      (lambda: bwd(x=None), b"null pointer"), (lambda: bwd(y=None), b"null pointer"), (lambda: bwd(M=0), b"bad sizes"),
                      (lambda: bwd(C=6), b"C % 4 != 0"), (lambda: bwd(M=1), b"M >= 2")):
        assert call() == -1
        assert msg in lib.lt_last_error_string(), lib.lt_last_error_string()
    assert lib.lt_batch_norm_fwd(p + 4, None, p, p, p, p, p, p, p, 8, 16, 1e-5, 0.1, 1, 1, p, ws, None) == -1
    assert b"16-byte aligned" in lib.lt_last_error_string()
