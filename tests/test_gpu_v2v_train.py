"""GPU tests of the native V2V training convolutions (autograd_ops.ConvNdFn / ConvTranspose3dFn: forward and data gradient on the
forward conv kernels, weight gradient on csrc/conv_wgrad.cu) against torch autograd in float64 on the device, and of a training
step of the volumetric model with v2v_backend="native" against the cuDNN V2V."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from lt_b200 import autograd_ops as A
from lt_b200 import capi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL_OUT = 2e-5      # output and data gradient: the forward layer bar (tests/test_gpu_tc.py)
TOL_W = 1e-4        # weight and bias gradients

# (cin, cout, k, (D, H, W), N): every V2V Conv3d type at 8^3 - 16^3, B = 2; 8 x 9 x 10 etc. give M tiles of 128 positions that
# do not divide the grid
CONV_CASES = [
    (32, 16, 7, (9, 10, 16), 2),    # front_layers[0]; its data gradient is 7^3 16 -> 32 on LT_CONV_TC_FOLD
    (16, 32, 3, (8, 9, 10), 2),     # Res3DBlock(16, 32)
    (16, 32, 1, (8, 8, 9), 2),      # its skip
    (32, 32, 3, (8, 12, 16), 2),    # full width (W >= 16): forward and data gradient on LT_CONV_TC_FOLD
    (32, 32, 3, (9, 8, 10), 2),
    (32, 64, 3, (8, 8, 8), 2),
    (64, 64, 3, (8, 9, 8), 2),
    (64, 128, 3, (8, 8, 10), 2),
    (128, 128, 3, (8, 8, 8), 2),
    (32, 64, 1, (9, 8, 8), 2),
    (64, 128, 1, (8, 8, 8), 2),
    (32, 32, 1, (10, 8, 8), 2),     # back_layers[1], [2]
    (32, 17, 1, (8, 8, 12), 2),     # output_layer
]
DECONV_CASES = [(128, 128, (8, 8, 8), 2), (128, 64, (8, 9, 8), 2), (64, 32, (8, 8, 10), 2)]


def _record_impls():
    launched = []
    orig = capi.conv_nd
    capi.conv_nd = lambda d, *a: (launched.append(a[-1]), orig(d, *a))[1]
    return launched, orig


def _run_native(x, w, b, fn, gy):
    xn = x.clone().to(memory_format=torch.channels_last_3d).requires_grad_(True)
    wn, bn = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = fn(xn, wn, bn)
    y.backward(gy)
    torch.cuda.synchronize()
    return y.detach(), xn.grad, wn.grad, bn.grad


def _run_ref(x, w, b, fn, gy):
    xd, wd, bd = [t.double().requires_grad_(True) for t in (x, w, b)]
    y = fn(xd, wd, bd)
    y.backward(gy.double())
    return y.detach(), xd.grad, wd.grad, bd.grad


def _check(native, ref, label):
    errs = [rel_err(a.double().cpu().numpy(), r.cpu().numpy()) for a, r in zip(native, ref)]
    print("%s: out %.2e dX %.2e dW %.2e db %.2e" % ((label,) + tuple(errs)))
    assert errs[0] < TOL_OUT and errs[1] < TOL_OUT, errs
    assert errs[2] < TOL_W and errs[3] < TOL_W, errs


def _conv_problem(case, seed):
    cin, cout, k, dims, N = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, *dims, generator=g)
    w = torch.randn(cout, cin, k, k, k, generator=g) * (2.0 / (cin * k ** 3)) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    gy = torch.randn(N, cout, *dims, generator=g) * 1e-3
    return [t.to(DEV) for t in (x, w, b, gy)]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv3d_layer_vs_float64_autograd(case):
    k = case[2]
    x, w, b, gy = _conv_problem(case, sum(case[:3]))
    launched, orig = _record_impls()
    try:
        native = _run_native(x, w, b, lambda x_, w_, b_: A.conv3d(x_, w_, b_, (k // 2,) * 3), gy)
    finally:
        capi.conv_nd = orig
    ref = _run_ref(x, w, b, lambda x_, w_, b_: F.conv3d(x_, w_, b_, 1, k // 2), gy)
    _check(native, ref, "conv3d %s" % (case,))
    cin, cout, _, dims, _ = case
    fold_fwd = k in (3, 7) and dims[2] >= 16 and _round32(cin) == 32 and cout == 32
    fold_dgrad = k in (3, 7) and dims[2] >= 16 and _round32(cout) == 32 and cin == 32
    assert launched == [capi.CONV_TC_FOLD if fold_fwd else capi.CONV_TC, capi.CONV_TC_FOLD if fold_dgrad else capi.CONV_TC]
    if case == (32, 32, 3, (8, 12, 16), 2) or k == 7:
        assert launched[1] == capi.CONV_TC_FOLD


def _round32(c):
    return (c + 31) // 32 * 32


def _deconv_problem(case, seed):
    cin, cout, dims, N = case
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, cin, *dims, generator=g)
    w = torch.randn(cin, cout, 2, 2, 2, generator=g) * (1.0 / cin) ** 0.5
    b = torch.randn(cout, generator=g) * 0.1
    gy = torch.randn(N, cout, *[2 * s for s in dims], generator=g) * 1e-3
    return [t.to(DEV) for t in (x, w, b, gy)]


@pytest.mark.parametrize("case", DECONV_CASES)
def test_conv_transpose3d_layer_vs_float64_autograd(case):
    x, w, b, gy = _deconv_problem(case, sum(case[:2]))
    native = _run_native(x, w, b, A.conv_transpose3d, gy)
    ref = _run_ref(x, w, b, lambda x_, w_, b_: F.conv_transpose3d(x_, w_, b_, 2), gy)
    _check(native, ref, "conv_transpose3d %s" % (case,))


@pytest.mark.parametrize("factor", [1e-9, 1e3])
@pytest.mark.parametrize("which", ["conv7", "conv3", "deconv"])
def test_gradients_scale_with_the_output_gradient(which, factor):
    """dY far below fp16's normal range (1e-12 here) keeps its bits through the power-of-two scale of lt_f32_to_s32_scaled."""
    if which == "deconv":
        x, w, b, gy = _deconv_problem(DECONV_CASES[1], 5)
        fn, ref_fn = A.conv_transpose3d, lambda x_, w_, b_: F.conv_transpose3d(x_, w_, b_, 2)
    else:
        case = CONV_CASES[0] if which == "conv7" else CONV_CASES[3]
        k = case[2]
        x, w, b, gy = _conv_problem(case, 6)
        fn = lambda x_, w_, b_: A.conv3d(x_, w_, b_, (k // 2,) * 3)
        ref_fn = lambda x_, w_, b_: F.conv3d(x_, w_, b_, 1, k // 2)
    native = _run_native(x, w, b, fn, gy * factor)
    ref = _run_ref(x, w, b, ref_fn, gy)
    _check((native[0],) + tuple(t / factor for t in native[1:]), ref, "%s dY x %g" % (which, factor))


@pytest.mark.parametrize("which", ["conv", "deconv"])
def test_backward_is_bitwise_deterministic(which):
    if which == "conv":
        x, w, b, gy = _conv_problem((64, 64, 3, (12, 12, 12), 2), 9)
        fn = lambda x_, w_, b_: A.conv3d(x_, w_, b_, (1, 1, 1))
    else:
        x, w, b, gy = _deconv_problem((128, 64, (8, 8, 8), 2), 9)
        fn = A.conv_transpose3d
    r1 = _run_native(x, w, b, fn, gy)
    r2 = _run_native(x, w, b, fn, gy)
    for a, c in zip(r1, r2):
        assert torch.equal(a, c)


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError):
        A.conv3d(torch.zeros(1, 32, 4, 4, 4), torch.zeros(32, 32, 3, 3, 3), None, (1, 1, 1))
    with pytest.raises(RuntimeError):
        A.conv_transpose3d(torch.zeros(1, 64, 2, 2, 2), torch.zeros(64, 32, 2, 2, 2), None)


def test_module_training_step_matches_cudnn_v2v():
    """ResNet-18, 32^3, B = 2, train mode (batch-statistics BatchNorm), recipe loss 0.1 MAE + 0.01 CE, Adam: the step with the
    native V2V convolutions against the same step on cuDNN in full fp32.  Both runs draw the same rotations (NumPy seed reset).

    A randomly initialised V2V with batch-statistics BatchNorm amplifies last-bit differences: on the H100 the first-step losses
    agreed to 2.6e-6 while the first layer's weight gradient differed by 6e-2 and the second-step loss by 6e-3.  So each quantity is
    held to max(fixed bar, 3 x the difference that a 1e-6 relative perturbation of the V2V weights -- the size of one native layer's
    error -- causes in the cuDNN run)."""
    import lt_b200
    from lt_b200 import loss as ce, testing
    B, V, S, lr = 2, 2, 64, 1e-3
    images, batch = testing.make_batch(B, V, image_size=S, seed=4)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    torch.manual_seed(0)
    holder = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=18, volume_size=32), device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=0, calib_size=S, calib_views=1)
    sd = holder.state_dict()
    g = torch.Generator().manual_seed(1)
    sd_noisy = {k: (v * (1 + 1e-6 * torch.randn(v.shape, generator=g)) if k.startswith("volume_net") and k.endswith("weight") else v)
                for k, v in sd.items()}
    loss_fn = ce.VolumetricCELoss(backend="native")
    names = ["volume_net.front_layers.0.block.0.weight", "volume_net.encoder_decoder.decoder_upsample2.block.0.weight",
             "volume_net.output_layer.weight", "process_features.0.weight", "backbone.layer4.1.conv2.weight"]
    tf32 = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    res = {}
    try:
        for run, v2v, state in (("torch", "torch", sd), ("native", "native", sd), ("noise", "torch", sd_noisy)):
            m = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=18, volume_size=32), device=DEV, backend="hybrid",
                                                   v2v_backend=v2v)
            m.load_state_dict(state)
            m = m.to(DEV).train()
            opt = torch.optim.Adam(m.parameters(), lr=lr)
            losses = []
            for step in range(2):
                np.random.seed(step)
                opt.zero_grad(set_to_none=True)
                kp, _, vols, _, _, coord, _ = m(images, None, batch)
                mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
                loss = 0.1 * mae + 0.01 * loss_fn(coord, vols, kp_gt, valid)
                loss.backward()
                losses.append(float(loss.detach()))
                if step == 0:
                    params = dict(m.named_parameters())
                    grads = {n: params[n].grad.detach().clone() for n in names}
                    before = torch.cat([p.detach().flatten() for p in m.parameters()])
                opt.step()
                if step == 0:
                    update = torch.cat([p.detach().flatten() for p in m.parameters()]) - before
            res[run] = (losses, grads, update)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32
    l_t, g_t, p_t = res["torch"]

    def diffs(run):
        l, gr, p = res[run]
        moved = float((p - p_t).norm() / p_t.norm())     # the first Adam step, ~lr sign(g) per element
        return ([abs(l[0] - l_t[0]) / abs(l_t[0]), abs(l[1] - l_t[1]) / abs(l_t[1]), moved] +
                [rel_err(gr[n].cpu().numpy(), g_t[n].cpu().numpy()) for n in names])
    nat, noise = diffs("native"), diffs("noise")
    bars = [1e-4, 1e-3, 1e-3] + [1e-2] * len(names)
    labels = ["loss step 1", "loss step 2", "first Adam update (relative L2)"] + ["grad " + n for n in names]
    for lab, dn, dz, bar in zip(labels, nat, noise, bars):
        print("%-70s native %.2e  weight noise %.2e  bar %.2e" % (lab, dn, dz, max(bar, 3 * dz)))
    for lab, dn, dz, bar in zip(labels, nat, noise, bars):
        assert dn <= max(bar, 3 * dz), lab
