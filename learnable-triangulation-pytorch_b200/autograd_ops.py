"""Differentiable wrappers of the native custom ops (`backend="hybrid"`): the forward is the same hand-written kernel the
inference path uses, the backward is `csrc/backward.cu` (lt_unproject_aggregate_bwd, lt_softargmax3d_bwd) and
`csrc/algebraic.cu` (lt_triangulate_dlt_bwd).

This is the first stage of SURVEY section 8f row 1: with it the reference training loop (`train.py:159-243`,
`total_loss.backward()` at :236) runs the custom ops on the native kernels while the convolutions stay on torch/cuDNN
autograd.  Volumetric model: the unprojection + aggregation and the 3-D soft-argmax -- the ops the reference implements as
Python loops over (sample, view) pairs with ~10 passes over a (V, C, N^3) staging tensor.  Algebraic model: the 2-D
soft-argmax (op.py:11-47, both branches) and the confidence-weighted DLT, which the reference runs as one torch.svd per
(sample, joint) (multiview.py:171-183).  Gradients: feature maps / heat-maps, `conf` and algebraic confidences, V2V logits,
2-D key points, and -- when they require grad, as at op level where a caller may refine cameras or learn a cuboid -- projection
matrices (unprojection, DLT) and coordinate volumes (unprojection, 3-D soft-argmax).  The models' geometry comes from numpy and
requires no grad, so their training steps launch no geometry kernel.
"""
import torch
import torch.nn.functional as F

from . import capi, engine
from .engine import _round_up


class UnprojectHeatmapsFn(torch.autograd.Function):
    """op.unproject_heatmaps (reference op.py:99-166), NCHW features in, NCDHW volume out."""

    @staticmethod
    def forward(ctx, heatmaps, proj_matricies, coord_volumes, vol_confidences, agg):
        B, V, C, h, w = heatmaps.shape
        vol_shape = tuple(coord_volumes.shape[1:4])
        nvox = vol_shape[0] * vol_shape[1] * vol_shape[2]
        feats_cl = heatmaps.detach().float().permute(0, 1, 3, 4, 2).contiguous()          # (B, V, h, w, C)
        proj = proj_matricies.detach().float().contiguous()
        coord = coord_volumes.detach().float().reshape(B, nvox, 3).contiguous()
        conf = None
        if agg == capi.AGG["conf"]:
            conf = vol_confidences.detach().float().reshape(B, V, C).contiguous()
        out_cl = torch.empty((B, nvox, C), dtype=torch.float32, device=heatmaps.device)
        capi.unproject_aggregate(feats_cl, proj, coord, conf, out_cl, capi.FMT_F32, agg)
        ctx.save_for_backward(feats_cl, proj, coord, conf if conf is not None else torch.empty(0, device=heatmaps.device))
        ctx.agg, ctx.vol_shape, ctx.has_conf = agg, vol_shape, conf is not None
        ctx.conf_shape = None if vol_confidences is None else tuple(vol_confidences.shape)
        ctx.geom_shapes = (tuple(proj_matricies.shape), tuple(coord_volumes.shape))
        return out_cl.permute(0, 2, 1).reshape(B, C, *vol_shape).contiguous()

    @staticmethod
    def backward(ctx, grad_out):
        feats_cl, proj, coord, conf = ctx.saved_tensors
        conf = conf if ctx.has_conf else None
        B, V, h, w, C = feats_cl.shape
        nvox = coord.shape[1]
        g_cl = grad_out.float().reshape(B, C, nvox).permute(0, 2, 1).contiguous()          # (B, nvox, C)
        grad_feats = torch.zeros_like(feats_cl)
        need_conf = ctx.has_conf and ctx.needs_input_grad[3]
        grad_conf = torch.zeros((B, V, C), dtype=torch.float32, device=feats_cl.device) if need_conf else None
        need_proj, need_coord = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        grad_proj = grad_coord = None
        if torch.are_deterministic_algorithms_enabled():
            # the fixed-order backward (no float atomics), whatever warn_only says: same terms, one summation order
            dev = feats_cl.device
            grad_proj = torch.empty((B, V, 12), dtype=torch.float32, device=dev) if need_proj else None
            grad_coord = torch.empty((B, nvox, 3), dtype=torch.float32, device=dev) if need_coord else None
            ws = torch.empty(capi.unproject_aggregate_bwd_det_workspace_bytes(B, V, C, h, w, nvox, ctx.agg, need_proj or need_coord),
                             dtype=torch.uint8, device=dev)
            capi.unproject_aggregate_bwd_det(feats_cl, proj, coord, conf, g_cl, grad_feats, grad_conf, grad_proj, grad_coord, ctx.agg, ws)
            proj_shape, coord_shape = ctx.geom_shapes
            grad_proj = grad_proj.reshape(proj_shape) if need_proj else None
            grad_coord = grad_coord.reshape(coord_shape) if need_coord else None
        elif need_proj or need_coord:
            dev = feats_cl.device
            grad_proj = torch.empty((B, V, 12), dtype=torch.float32, device=dev) if need_proj else None
            grad_coord = torch.empty((B, nvox, 3), dtype=torch.float32, device=dev) if need_coord else None
            ws = torch.empty(capi.unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox), dtype=torch.uint8, device=dev)
            capi.unproject_aggregate_bwd_geom(feats_cl, proj, coord, conf, g_cl, grad_feats, grad_conf, grad_proj, grad_coord, ctx.agg, ws)
            proj_shape, coord_shape = ctx.geom_shapes
            grad_proj = grad_proj.reshape(proj_shape) if need_proj else None
            grad_coord = grad_coord.reshape(coord_shape) if need_coord else None
        else:
            capi.unproject_aggregate_bwd(feats_cl, proj, coord, conf, g_cl, grad_feats, grad_conf, ctx.agg)
        # grad_feats is the kernels' accumulation target even when the heat-maps need no gradient; it is returned only if they do
        grad_heat = grad_feats.permute(0, 1, 4, 2, 3) if ctx.needs_input_grad[0] else None   # (B, V, C, h, w) view
        return grad_heat, grad_proj, grad_coord, (grad_conf.reshape(ctx.conf_shape) if need_conf else None), None


class MaxPool3dFn(torch.autograd.Function):
    """F.max_pool3d(x, k, k) with the native fixed-order backward (lt_maxpool3d_bwd): what V2V's pooling runs under
    torch.use_deterministic_algorithms, where torch has no deterministic CUDA max_pool3d backward.  The forward is torch's."""

    @staticmethod
    def forward(ctx, x, k):
        ctx.save_for_backward(x)
        ctx.k = k
        return F.max_pool3d(x, k, k)

    @staticmethod
    def backward(ctx, grad_y):
        x, = ctx.saved_tensors
        if x.dtype != torch.float32:
            raise TypeError("the native max-pool backward takes float32 (got %s)" % x.dtype)
        grad_x = torch.empty_like(x)
        capi.maxpool3d_bwd(x, grad_y, grad_x, ctx.k)
        return grad_x, None


class IntegrateTensor3dFn(torch.autograd.Function):
    """op.integrate_tensor_3d_with_coordinates (reference op.py:84-96): (keypoints, normalised volumes)."""

    @staticmethod
    def forward(ctx, volumes, coord_volumes, softmax):
        B, J = volumes.shape[:2]
        nvox = volumes[0, 0].numel()
        logits = volumes.detach().float().contiguous()
        coord = coord_volumes.detach().float().reshape(B, nvox, 3).contiguous()
        out = torch.empty_like(logits)
        keypoints = torch.empty((B, J, 3), dtype=torch.float32, device=volumes.device)
        ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, nvox) // 4 + 1, dtype=torch.float32, device=volumes.device)
        capi.softargmax3d(logits, J * nvox, 1, nvox, coord, out, keypoints, ws, B, J, nvox, 1.0, softmax)
        ctx.save_for_backward(out, coord)
        ctx.softmax = bool(softmax)
        ctx.coord_shape = tuple(coord_volumes.shape)
        return keypoints, out

    @staticmethod
    def backward(ctx, grad_kp, grad_vol):
        probs, coord = ctx.saved_tensors
        B, J = probs.shape[:2]
        nvox = coord.shape[1]
        dev = probs.device
        g_kp = (grad_kp if grad_kp is not None else torch.zeros((B, J, 3), device=dev)).float().contiguous()
        g_vol = None if grad_vol is None else grad_vol.float().contiguous()
        grad_logits = grad_coord = None
        if ctx.needs_input_grad[0]:
            grad_logits = torch.empty_like(probs)
            scratch = torch.empty(B * J, dtype=torch.float32, device=dev)
            capi.softargmax3d_bwd(probs, coord, g_kp, g_vol, grad_logits, scratch, B, J, nvox, 1.0, ctx.softmax)
        if ctx.needs_input_grad[1]:
            grad_coord = torch.empty((B, nvox, 3), dtype=torch.float32, device=dev)
            capi.softargmax3d_coord_bwd(probs.reshape(B, J, nvox), g_kp, grad_coord, B, J, nvox, ctx.softmax)
            grad_coord = grad_coord.reshape(ctx.coord_shape)
        return grad_logits, grad_coord, None


class IntegrateTensor2dFn(torch.autograd.Function):
    """op.integrate_tensor_2d (reference op.py:11-47): (B, J, h, w) -> (coordinates (B, J, 2) [x, y in pixels], heat-maps)."""

    @staticmethod
    def forward(ctx, heatmaps, softmax):
        B, J, h, w = heatmaps.shape
        dev = heatmaps.device
        logits = heatmaps.detach().float().contiguous()
        grid = engine.pixel_grid(B, h, w, dev)
        out = torch.empty_like(logits)
        kp = torch.empty((B, J, 3), dtype=torch.float32, device=dev)
        ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, h * w) // 4 + 1, dtype=torch.float32, device=dev)
        mode = 1 if softmax else 2          # 2: ReLU heat-maps, centre of mass divided by the mass (op.py:25-41)
        capi.softargmax3d(logits, J * h * w, 1, h * w, grid, out, kp, ws, B, J, h * w, 1.0, mode)
        ctx.save_for_backward(out, grid)
        ctx.mode = mode
        return kp[:, :, :2].contiguous(), out

    @staticmethod
    def backward(ctx, grad_kp, grad_heat):
        probs, grid = ctx.saved_tensors
        B, J, h, w = probs.shape
        dev = probs.device
        g_kp = torch.zeros((B, J, 3), dtype=torch.float32, device=dev)
        if grad_kp is not None:
            g_kp[:, :, :2] = grad_kp
        g_heat = None if grad_heat is None else grad_heat.float().contiguous()
        grad_logits = torch.empty_like(probs)
        scratch = torch.empty(2 * B * J, dtype=torch.float32, device=dev)
        capi.softargmax3d_bwd(probs, grid, g_kp, g_heat, grad_logits, scratch, B, J, h * w, 1.0, ctx.mode)
        return grad_logits, None


class TriangulateDltFn(torch.autograd.Function):
    """multiview.triangulate_batch_of_points (reference multiview.py:141-183): (B, V, 3, 4), (B, V, J, 2), (B, V, J) or None
    -> (B, J, 3).  Gradients reach the key points, the confidences and the projection matrices."""

    @staticmethod
    def forward(ctx, proj_matricies, points, confidences):
        B, V, J = points.shape[:3]
        proj = proj_matricies.detach().float().contiguous()
        kp = points.detach().float().contiguous()
        conf = None if confidences is None else confidences.detach().float().contiguous()
        out = torch.empty((B, J, 3), dtype=torch.float32, device=points.device)
        capi.triangulate_dlt(proj, kp, conf, out)
        ctx.save_for_backward(proj, kp, conf if conf is not None else torch.empty(0, device=points.device))
        ctx.has_conf = conf is not None
        return out

    @staticmethod
    def backward(ctx, grad_out):
        proj, kp, conf = ctx.saved_tensors
        conf = conf if ctx.has_conf else None
        need_conf = ctx.has_conf and ctx.needs_input_grad[2]
        g = grad_out.float().contiguous()
        grad_kp = grad_conf = grad_proj = None
        if ctx.needs_input_grad[1] or need_conf:
            grad_kp = torch.empty_like(kp)
            grad_conf = torch.empty_like(conf) if need_conf else None
            capi.triangulate_dlt_bwd(proj, kp, conf, g, grad_kp, grad_conf)
        if ctx.needs_input_grad[0]:
            B, V, J = kp.shape[:3]
            grad_proj = torch.empty_like(proj)
            ws = torch.empty(capi.triangulate_dlt_proj_bwd_workspace_bytes(B, V, J), dtype=torch.uint8, device=proj.device)
            capi.triangulate_dlt_proj_bwd(proj, kp, conf, g, grad_proj, ws)
        return grad_proj, (grad_kp if ctx.needs_input_grad[1] else None), grad_conf


class VolumetricCEFn(torch.autograd.Function):
    """VolumetricCELoss (reference loss.py:52-80) on csrc/loss.cu: probs (B, J, nvox), coord (B, nvox, 3), keypoints_gt (B, J, 3),
    validity (B, J), all float32 CUDA -> 0-dim loss.  Only the volumes get a gradient: the reference's argmin is detached, and the
    coordinates, ground truth and validity are data."""

    @staticmethod
    def forward(ctx, probs, coord, keypoints_gt, validity):
        B, J, nvox = probs.shape
        dev = probs.device
        p = probs.detach().contiguous()
        v = validity.detach().contiguous()
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        index = torch.empty((B, J), dtype=torch.int32, device=dev)
        picked = torch.empty((B, J), dtype=torch.float32, device=dev)
        ws = torch.empty(capi.volumetric_ce_workspace_bytes(B, J, nvox), dtype=torch.uint8, device=dev)
        capi.volumetric_ce(p, coord.detach().contiguous(), keypoints_gt.detach().contiguous(), v, loss, index, picked, ws)
        ctx.save_for_backward(index, picked, v)
        ctx.nvox = nvox
        ctx.mark_non_differentiable(index, picked)
        return loss.reshape(()), index, picked

    @staticmethod
    def backward(ctx, grad_loss, grad_index, grad_picked):
        index, picked, v = ctx.saved_tensors
        B, J = index.shape
        grad = torch.empty((B, J, ctx.nvox), dtype=torch.float32, device=index.device)
        capi.volumetric_ce_bwd(grad_loss.float().reshape(1).contiguous(), index, picked, v, grad)
        return grad, None, None, None


def volumetric_ce_loss(probs, coord, keypoints_gt, validity):
    """-> (0-dim loss, index (B, J) int32, picked (B, J)); probs etc. as VolumetricCEFn."""
    return VolumetricCEFn.apply(probs, coord, keypoints_gt, validity)


class KeypointsLossFn(torch.autograd.Function):
    """The keypoint criteria (reference loss.py:7-49) on csrc/loss.cu: pred, gt (n, dim), validity (n,), float32 CUDA -> 0-dim loss.
    `kind` is a capi.KEYPOINTS_LOSS name.  Only pred gets a gradient; the ground truth and the validity are data."""

    @staticmethod
    def forward(ctx, pred, gt, validity, kind, threshold):
        p = pred.detach().contiguous()
        loss = torch.empty(1, dtype=torch.float32, device=p.device)
        norm = torch.empty(1, dtype=torch.float64, device=p.device)
        capi.keypoints_loss(p, gt, validity, loss, norm, kind, threshold)
        ctx.save_for_backward(p, gt, validity, norm)
        ctx.kind, ctx.threshold = kind, threshold
        return loss.reshape(())

    @staticmethod
    def backward(ctx, grad_loss):
        p, gt, validity, norm = ctx.saved_tensors
        grad = torch.empty_like(p)
        capi.keypoints_loss_bwd(grad_loss.float().reshape(1).contiguous(), p, gt, validity, norm, grad, ctx.kind, ctx.threshold)
        return grad, None, None, None, None


def keypoints_loss(pred, gt, validity, kind, threshold=400.0):
    """-> 0-dim loss; pred, gt (n, dim) and validity (n,) as KeypointsLossFn (gt and validity contiguous)."""
    return KeypointsLossFn.apply(pred, gt, validity, kind, threshold)


def integrate_tensor_2d(heatmaps, softmax=True):
    return IntegrateTensor2dFn.apply(heatmaps, softmax)


def triangulate_batch_of_points(proj_matricies_batch, points_batch, confidences_batch=None):
    return TriangulateDltFn.apply(proj_matricies_batch, points_batch, confidences_batch)


def unproject_heatmaps(heatmaps, proj_matricies, coord_volumes, volume_aggregation_method="sum", vol_confidences=None):
    agg = capi.AGG["conf" if volume_aggregation_method.startswith("conf") else volume_aggregation_method]
    return UnprojectHeatmapsFn.apply(heatmaps, proj_matricies, coord_volumes, vol_confidences, agg)


def integrate_tensor_3d_with_coordinates(volumes, coord_volumes, softmax=True):
    return IntegrateTensor3dFn.apply(volumes, coord_volumes, softmax)


# ---- Convolutions for training (v2v_backend="native", backbone_backend="native"): forward and data gradient on the forward conv
# kernels, weight gradient on csrc/conv_wgrad.cu.  Activations are float32 channels_last(_3d) tensors, so the kernels read and write
# them in place of a transpose and torch's BatchNorm / ReLU / pooling / adds run on them unchanged.  A 2-D map is a 3-D one with D = 1.

class _Filter:
    """The nn.Conv attributes engine.pack_conv reads, for a filter that is not (or not only) a module's own."""

    def __init__(self, weight, bias, stride, padding):
        self.weight, self.bias = weight, bias
        self.kernel_size, self.stride, self.padding = tuple(weight.shape[2:]), tuple(stride), tuple(padding)


_WORKSPACE = {}


def _workspace(device, nbytes):
    """Scratch of the weight-gradient and BatchNorm launches of one device (launches on one stream are ordered); it grows on demand."""
    ws = _WORKSPACE.get(device)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 32 << 20), dtype=torch.uint8, device=device)
        _WORKSPACE[device] = ws
    return ws


def _as3(t, fill):
    """A 2-D conv attribute (h, w) as its 3-D form (fill, h, w); 3-tuples pass unchanged."""
    t = tuple(t)
    return (fill,) * (3 - len(t)) + t


def _cl(x):
    """(N, C, [D,] H, W) -> contiguous float32 (N, D, H, W, C), D = 1 for 2-D maps (a view for channels_last(_3d) input)."""
    if not x.is_cuda:
        raise RuntimeError("lt_b200 native training convolutions need CUDA tensors (got %s)" % x.device)
    if x.dim() == 4:
        return x.float().contiguous(memory_format=torch.channels_last).permute(0, 2, 3, 1).unsqueeze(1)
    return x.float().contiguous(memory_format=torch.channels_last_3d).permute(0, 2, 3, 4, 1)


def _from_cl(out, c, nd):
    """(N, D, H, W, C') channels-last -> the (N, c, [D,] H, W) view of its first c channels (nd = 2 drops D = 1)."""
    out = out[..., :c]
    return out[:, 0].permute(0, 3, 1, 2) if nd == 2 else out.permute(0, 4, 1, 2, 3)


def _to_s32(x_cl, cp, absmax_bits=None, inv_scale=None):
    """(N, D, H, W, C) float32 -> split-fp16 (N, D, H, W, 2 cp), scaled by the power of two that absmax_bits selects."""
    out = torch.empty(x_cl.shape[:4] + (2 * cp,), dtype=torch.float16, device=x_cl.device)
    capi.f32_to_s32_scaled(x_cl, out, x_cl[..., 0].numel(), x_cl.shape[4], cp, absmax_bits, inv_scale)
    return out


def conv3d_wgrad_desc(N, dims, cin, cout, k, padding, stride=(1, 1, 1)):
    """The forward launch of a convolution (3-D form: a 2-D one has D = 1) as lt_conv_wgrad_fwd reads it: split-fp16 input and
    output gradient, 32-channel padded."""
    cin_p, cout_p, out_dims = _round_up(cin, 32), _round_up(cout, 32), engine.conv_out_dims(dims, k, stride, padding)
    return engine.conv_desc(N, dims, cin_p, cout_p, k, stride, padding, out_dims, out_dims, cout_p, capi.FMT_S32, capi.FMT_S32)


def conv_transpose3d_desc(N, dims, cin, cout):
    """ConvTranspose3d(k=2, s=2) as the engine's one grouped 1x1x1 GEMM: N = 8 cout, block g = a 4 + b 2 + c to output phase (a, b, c)."""
    D, H, W = dims
    return engine.conv_desc(N, dims, cin, 8 * cout, (1, 1, 1), (1, 1, 1), (0, 0, 0), dims, (2 * D, 2 * H, 2 * W), cout, capi.FMT_S32,
                            capi.FMT_S32, out_scale=(2, 2, 2), out_groups=(2, 2, 2))


def conv3d_dgrad_filter(weight_shape, padding):
    """Data gradient of a stride-1 'same' convolution (Cout, Cin, [kd,] kh, kw) as a forward conv of dY: lt_conv_gather_weights_fwd
    source (base, (s_td, s_th, s_tw, s_ci, s_co)) of the filter flipped in space with Cin and Cout swapped -- element (td, th, tw,
    ci' = co, co' = ci) = w[co][ci][kd-1-td][kh-1-th][kw-1-tw] -- and the conv's (k, stride, pad, cin', cout') in 3-D form.  With
    1x1 filters it is the transposed filter of any stride."""
    cout, cin = weight_shape[:2]
    kd, kh, kw = _as3(weight_shape[2:], 1)
    T = kd * kh * kw
    return (T - 1, (-kh * kw, -kw, -1, cin * T, T)), (kd, kh, kw), (1, 1, 1), _as3(padding, 0), cout, cin


def conv_s2_dgrad_filter(weight_shape, stride):
    """Data gradient of a 3-tap stride-2 pad-1 convolution (Cout, Cin, [kd,] kh, kw) as ONE grouped forward conv of dY.

    Along a stride-2 axis, input phase a of dX reads dY positions {m, m+1} only: a = 0 takes tap 1 at m, a = 1 takes tap 2 at m
    and tap 0 at m+1.  So all phases together are a 2-tap stride-1 pad-0 conv of dY (reads past the end arrive as TMA zero fill)
    with one Cin-wide column block per phase, block g = (a ogh + b) ogw + c written to input phase (a, b, c) at output scale 2.
    Tap u of phase a reads kernel index 1 + 2u (a = 0) or 2 - 2u (a = 1) of the filter zero-padded to 4 along every stride-2 axis:
    index 3 is the zero of the tap phase 0 does not use.  Returns ([lt_conv_gather_weights_fwd (base, strides) per block, into the
    padded filter], k, pad, groups, cin', cout') in 3-D form."""
    cout, cin = weight_shape[:2]
    k3, s3 = _as3(weight_shape[2:], 1), _as3(stride, 1)
    kp = tuple(4 if s == 2 else kk for kk, s in zip(k3, s3))          # the padded filter's extents
    tap_stride = (kp[1] * kp[2], kp[2], 1)
    T = kp[0] * kp[1] * kp[2]
    phases = [((1, 2), (2, -2)) if s == 2 else ((0, 0),) for s in s3]  # per axis and phase: (first kernel index, step per tap)
    srcs = []
    for pa in phases[0]:
        for pb in phases[1]:
            for pc in phases[2]:
                base = pa[0] * tap_stride[0] + pb[0] * tap_stride[1] + pc[0] * tap_stride[2]
                srcs.append((base, (pa[1] * tap_stride[0], pb[1] * tap_stride[1], pc[1] * tap_stride[2], cin * T, T)))
    k = tuple(2 if s == 2 else 1 for s in s3)
    return srcs, k, (0, 0, 0), tuple(2 if s == 2 else 1 for s in s3), cout, cin


def pad_s2_filter(weight, stride):
    """The filter zero-padded to 4 taps along every stride-2 axis (conv_s2_dgrad_filter's source)."""
    pads = []
    for s in reversed(_as3(stride, 1)[3 - (weight.dim() - 2):]):
        pads += [0, 1 if s == 2 else 0]
    return torch.nn.functional.pad(weight, pads)


def conv_transpose3d_dgrad_filter(weight_shape):
    """Data gradient of ConvTranspose3d(k=2, s=2) (Cin, Cout, 2, 2, 2): dX[o][ci] = sum_{t, co} dY[2 o + t][co] w[ci][co][t], a 2^3
    stride-2 pad-0 conv of dY with element (td, th, tw, ci' = co, co' = ci) = w[ci][co][td][th][tw]."""
    cin, cout = weight_shape[:2]
    return (0, (4, 2, 1, 8, cout * 8)), (2, 2, 2), (2, 2, 2), (0, 0, 0), cout, cin


def conv_transpose2d_k4s2_dgrad_filter(weight_shape):
    """Data gradient of ConvTranspose2d(k=4, s=2, p=1) (Cin, Cout, 4, 4): dX[i] = sum_{ky, co} dY[2 i - 1 + ky][co] w[ci][co][ky], a
    4x4 stride-2 pad-1 conv of dY with element (th, tw, ci' = co, co' = ci) = w[ci][co][th][tw] (no flip); 3-D form."""
    cin, cout = weight_shape[:2]
    return (0, (0, 4, 1, 16, cout * 16)), (1, 4, 4), (1, 2, 2), (0, 1, 1), cout, cin


def _grad_s32(grad_out, cp):
    """dL/dy -> (split-fp16 of S dL/dy, (N, D, H, W, C) float32 view, absmax bits, 1 / S on the device): S = 2^(9 - floor(log2 max|g|))."""
    g = _cl(grad_out)
    amax = torch.empty(1, dtype=torch.int32, device=g.device)
    capi.absmax(g, amax)
    inv = torch.empty(1, dtype=torch.float32, device=g.device)
    return _to_s32(g, cp, amax, inv), g, amax, inv


def _wgrad(desc, x_s, g_s, amax, cin, cout, taps, groups=1):
    """lt_conv_wgrad_fwd of the forward call `desc` -> float32 [taps][cin][groups cout]."""
    gw = torch.empty((taps, cin, groups * cout), dtype=torch.float32, device=x_s.device)
    ws = _workspace(x_s.device, capi.conv_wgrad_workspace_bytes(desc))
    capi.conv_wgrad(desc, x_s, g_s, amax, cin, cout, gw, ws)
    return gw


def conv_kind(k, stride, padding):
    """The supported geometry of a convolution in 3-D form: "same" (stride 1, odd kernel, padding k // 2), "s2k1" (1x1, stride 2 on
    the strided axes) or "s2k3" (3 taps, stride 2, padding 1 on the strided axes; 1x1 on the others); ValueError otherwise."""
    if all(s == 1 for s in stride):
        if all(kk % 2 == 1 and p == kk // 2 for kk, p in zip(k, padding)):
            return "same"
    elif all(s in (1, 2) for s in stride):
        strided = {(kk, p) for kk, s, p in zip(k, stride, padding) if s == 2}
        plain_ok = all(kk == 1 and p == 0 for kk, s, p in zip(k, stride, padding) if s == 1)
        if plain_ok and strided == {(1, 0)}:
            return "s2k1"
        if plain_ok and strided == {(3, 1)}:
            return "s2k3"
    raise ValueError("native conv: stride-1 'same' convolutions (odd kernel, padding k // 2), 1x1 stride 2 and 3-tap stride-2 "
                     "pad-1 convolutions only, got k=%s stride=%s padding=%s" % (tuple(k), tuple(stride), tuple(padding)))


def conv_s2_dgrad(g_s, weight, stride, in_dims, inv, out=None):
    """dX (N, D, H, W, Cin) float32 of a 3-tap stride-2 pad-1 conv from the split-fp16 scaled output gradient g_s (1 / scale on the
    device in `inv`): ONE grouped launch (conv_s2_dgrad_filter) writing every input phase over its own extent; into `out` if given."""
    cin = weight.shape[1]
    srcs, k, pad, groups, ci, co = conv_s2_dgrad_filter(weight.shape, stride)
    wp = pad_s2_filter(weight.detach().float(), stride).contiguous()
    pk = engine.pack_filter([(wp, base, strides) for base, strides in srcs], k, (1, 1, 1), pad, ci, co, None, None, out_fmt=capi.FMT_F32)
    out = engine.Act(g_s.shape[0], *in_dims, cin, capi.FMT_F32, g_s.device) if out is None else engine.Act.view(out)
    engine.launch_conv(engine.Act.view(g_s), pk, out, out_dims=g_s.shape[1:4], out_scale=groups, out_groups=groups, scale_mul=inv)
    return out.data


class ConvNdFn(torch.autograd.Function):
    """nn.Conv2d / nn.Conv3d on the tensor-core kernels, fp32-grade in all three passes, for the geometries of conv_kind (every conv
    of v2v.py and of the backbone but its stem).  forward: lt_conv_nd_fwd (scale 1 / S, shift = bias).  Data gradient, as forward
    convs of the output gradient: stride 1 -- the filter flipped in space with Cin / Cout swapped (re-gathered by
    lt_conv_gather_weights_fwd with negated tap strides); 1x1 stride 2 -- the transposed filter into the even phase of dX (the
    other phases are zero); 3-tap stride 2 -- one grouped launch writing every input phase (conv_s2_dgrad_filter).  Weight
    gradient: lt_conv_wgrad_fwd on the forward's descriptor; bias gradient: torch's sum of the output gradient.  The float32 input
    is saved (the tensor torch keeps anyway) and split to fp16 pairs again in the backward."""

    @staticmethod
    def forward(ctx, x, weight, bias, stride, padding):
        nd = weight.dim() - 2
        cout, cin = weight.shape[:2]
        k, st, pad = _as3(weight.shape[2:], 1), _as3(stride, 1), _as3(padding, 0)
        kind = conv_kind(k, st, pad)
        if kind == "s2k3" and cin % 32:
            raise ValueError("native conv: 3-tap stride-2 convolutions need Cin % 32 == 0 (grouped data gradient), got %d" % cin)
        x_cl = _cl(x)
        in_dims = tuple(x_cl.shape[1:4])
        if kind == "s2k3" and any(n < 2 for n, s in zip(in_dims, st) if s == 2):
            raise ValueError("native conv: 3-tap stride-2 convolutions need map sides of at least 2, got %s" % (in_dims,))
        cin_p = _round_up(cin, 32)
        x_s = _to_s32(x_cl, cin_p)
        pk = engine.pack_conv(_Filter(weight.detach(), None if bias is None else bias.detach(), stride, padding), None, cin_pad=cin_p,
                              out_fmt=capi.FMT_F32)
        out = engine.Act(x.shape[0], *engine.conv_out_dims(in_dims, k, st, pad), _round_up(cout, 4), capi.FMT_F32, x.device)
        engine.launch_conv(engine.Act.view(x_s), pk, out)
        ctx.save_for_backward(x, weight)
        ctx.geom = (k, st, pad, kind, in_dims)
        return _from_cl(out.data, cout, nd)

    @staticmethod
    def backward(ctx, grad_out):
        x, weight = ctx.saved_tensors
        k, st, pad, kind, in_dims = ctx.geom
        nd = weight.dim() - 2
        cout, cin = weight.shape[:2]
        T = k[0] * k[1] * k[2]
        cout_p = _round_up(cout, 32)
        g_s, g, amax, inv = _grad_s32(grad_out, cout_p)
        N = g.shape[0]
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            w = weight.detach().float().contiguous()
            if kind == "s2k3":
                out = conv_s2_dgrad(g_s, w, st, in_dims, inv)
            else:
                (base, strides), kk, _, pd, ci, co = conv3d_dgrad_filter(weight.shape, pad)
                pk = engine.pack_filter((w, base, strides), kk, (1, 1, 1), pd, ci, co, None, None, out_fmt=capi.FMT_F32)
                # s2k1: dX is zero off the even phase
                out = engine.Act(N, *in_dims, _round_up(cin, 4), capi.FMT_F32, g.device, zero=kind == "s2k1")
                engine.launch_conv(engine.Act.view(g_s), pk, out, out_scale=st, scale_mul=inv)
                out = out.data
            gx = _from_cl(out, cin, nd)
        if ctx.needs_input_grad[1]:
            x_s = _to_s32(_cl(x), _round_up(cin, 32))
            d = conv3d_wgrad_desc(N, in_dims, cin, cout, k, pad, st)
            gw = _wgrad(d, x_s, g_s, amax, cin, cout, T).reshape(T, cin, cout).permute(2, 1, 0).reshape(weight.shape).contiguous()
        if ctx.needs_input_grad[2]:
            gb = g.sum(dim=(0, 1, 2, 3))
        return gx, gw, gb, None, None



class ConvTranspose3dFn(torch.autograd.Function):
    """nn.ConvTranspose3d(k=2, s=2, p=0) (v2v.py Upsample3DBlock) with Cout % 32 == 0: the forward is the engine's one grouped 1x1x1
    GEMM (N = 8 Cout, each 32-channel block written to its phase of the output lattice); the data gradient is a 2^3 stride-2
    convolution of the output gradient (Cin' = Cout, Cout' = Cin) on conv_tc_kernel; the weight gradient is lt_conv_wgrad_fwd over
    the forward's grouped GEMM."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        cin, cout = weight.shape[:2]
        if tuple(weight.shape[2:]) != (2, 2, 2) or cout % 32 or cin % 32:
            raise ValueError("native ConvTranspose3d: kernel 2, stride 2 and channel counts that are multiples of 32 only, got %s"
                             % (tuple(weight.shape),))
        x_cl = _cl(x)
        N, D, H, W = x_cl.shape[:4]
        x_s = _to_s32(x_cl, cin)
        pk = engine.pack_deconv3d_k2s2(_Filter(weight.detach(), None if bias is None else bias.detach(), (2, 2, 2), (0, 0, 0)), None)
        y = engine.deconv3d_k2s2(engine.Act.view(x_s), pk, capi.FMT_S32, relu=False)
        out = torch.empty((N, 2 * D, 2 * H, 2 * W, cout), dtype=torch.float32, device=x.device)
        capi.s32_to_f32(y.data, out, y.pixels, cout)
        ctx.save_for_backward(x, weight)
        return out.permute(0, 4, 1, 2, 3)

    @staticmethod
    def backward(ctx, grad_out):
        x, weight = ctx.saved_tensors
        cin, cout = weight.shape[:2]
        g_s, g, amax, inv = _grad_s32(grad_out, cout)
        N, D, H, W = x.shape[0], x.shape[2], x.shape[3], x.shape[4]
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            w = weight.detach().float().contiguous()
            (base, strides), k, stride, pad, ci, co = conv_transpose3d_dgrad_filter(weight.shape)
            pk = engine.pack_filter((w, base, strides), k, stride, pad, ci, co, None, None, out_fmt=capi.FMT_F32)
            out = engine.Act(N, D, H, W, cin, capi.FMT_F32, g.device)
            engine.launch_conv(engine.Act.view(g_s), pk, out, scale_mul=inv)
            gx = out.data.permute(0, 4, 1, 2, 3)
        if ctx.needs_input_grad[1]:
            x_s = _to_s32(_cl(x), cin)
            gw = _wgrad(conv_transpose3d_desc(N, (D, H, W), cin, cout), x_s, g_s, amax, cin, cout, 1, groups=8)       # [1][ci][g cout + co], g = a 4 + b 2 + c
            gw = gw.reshape(cin, 8, cout).permute(0, 2, 1).reshape(cin, cout, 2, 2, 2).contiguous()
        if ctx.needs_input_grad[2]:
            gb = g.sum(dim=(0, 1, 2, 3))
        return gx, gw, gb


def conv_transpose2d_k4s2_desc(N, dims, cin, cout, py, px):
    """Phase (py, px) of ConvTranspose2d(k=4, s=2, p=1) as the forward launches it (the engine's 2x2 stride-1 conv into the
    (py, px) sub-lattice of the 2H x 2W output), 3-D form with split-fp16 output gradient: lt_conv_wgrad_fwd's descriptor."""
    _, H, W = dims
    cin_p, cout_p = _round_up(cin, 32), _round_up(cout, 32)
    _, pad = engine.deconv2d_k4s2_phase(py, px, cout)
    return engine.conv_desc(N, dims, cin_p, cout_p, (1, 2, 2), (1, 1, 1), pad, dims, (1, 2 * H, 2 * W), cout_p, capi.FMT_S32, capi.FMT_S32,
                            out_scale=(1, 2, 2), out_off=(0, py, px))


def conv_transpose2d_k4s2_wgrad_scatter(gw, py, px):
    """Weight gradient [4 taps (i, j)][cin][cout] of phase (py, px) -> its (cin, cout, 2, 2) share of dW at kernel rows / columns
    1 - py + 2 (1 - i) and 1 - px + 2 (1 - j) (tap i reads ky = 3 - py - 2i): assign to dW[:, :, 1 - py::2, 1 - px::2]."""
    cin, cout = gw.shape[1:]
    return gw.reshape(2, 2, cin, cout).flip(0, 1).permute(2, 3, 0, 1)


class ConvTranspose2dK4Fn(torch.autograd.Function):
    """nn.ConvTranspose2d(k=4, s=2, p=1) (the backbone's deconv_layers) on the tensor-core kernels: the forward is the inference
    engine's four 2x2 stride-1 phase launches into one float32 output; the data gradient is a 4x4 stride-2 pad-1 conv of the output
    gradient with the filter unflipped (Cin' = Cout, Cout' = Cin); the weight gradient is one lt_conv_wgrad_fwd per phase, each of the
    16 taps belonging to exactly one phase."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        cin, cout = weight.shape[:2]
        x_s = _to_s32(_cl(x), _round_up(cin, 32))
        phases = engine.pack_deconv2d_k4s2(_Filter(weight.detach(), None if bias is None else bias.detach(), (2, 2), (1, 1)), None,
                                           out_fmt=capi.FMT_F32)
        out = engine.deconv2d_k4s2(engine.Act.view(x_s), phases, capi.FMT_F32, relu=False)
        ctx.save_for_backward(x, weight)
        return _from_cl(out.data, cout, 2)

    @staticmethod
    def backward(ctx, grad_out):
        x, weight = ctx.saved_tensors
        cin, cout = weight.shape[:2]
        N, _, H, W = x.shape
        cout_p = _round_up(cout, 32)
        g_s, g, amax, inv = _grad_s32(grad_out, cout_p)
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            w = weight.detach().float().contiguous()
            (base, strides), k, stride, pad, ci, co = conv_transpose2d_k4s2_dgrad_filter(weight.shape)
            pk = engine.pack_filter((w, base, strides), k, stride, pad, ci, co, None, None, out_fmt=capi.FMT_F32)
            out = engine.Act(N, 1, H, W, _round_up(cin, 4), capi.FMT_F32, g.device)
            engine.launch_conv(engine.Act.view(g_s), pk, out, scale_mul=inv)
            gx = _from_cl(out.data, cin, 2)
        if ctx.needs_input_grad[1]:
            x_s = _to_s32(_cl(x), _round_up(cin, 32))
            gw = torch.empty((cin, cout, 4, 4), dtype=torch.float32, device=g.device)
            for py in (0, 1):
                for px in (0, 1):
                    gp = _wgrad(conv_transpose2d_k4s2_desc(N, (1, H, W), cin, cout, py, px), x_s, g_s, amax, cin, cout, 4)
                    gw[:, :, 1 - py::2, 1 - px::2] = conv_transpose2d_k4s2_wgrad_scatter(gp, py, px)
        if ctx.needs_input_grad[2]:
            gb = g.sum(dim=(0, 1, 2, 3))
        return gx, gw, gb


def stem_wgrad_desc(N, H, W, cout):
    """The stem's 4x4 stride-1 conv (front pad 2) over the (N, H/2, W/2, 32) space-to-depth input, 3-D form, as lt_conv_wgrad_fwd
    reads it."""
    dims = (1, H // 2, W // 2)
    return engine.conv_desc(N, dims, 32, _round_up(cout, 32), (1, 4, 4), (1, 1, 1), (0, 2, 2), dims, dims, _round_up(cout, 32), capi.FMT_S32,
                            capi.FMT_S32)


def stem_wgrad_index(device):
    """For every element (c, ky, kx) of a (3, 7, 7) stem filter, its row (tap (a, b), s2d channel) in the [16][12] rows of the
    s2d conv's weight gradient: ky = 2a + r - 1, kx = 2b + s - 1, channel (r 2 + s) 3 + c (engine.stem_s2d_filter).  Every element
    has exactly one such row; the 45 rows whose ky or kx falls outside [0, 7) are dropped."""
    c = torch.arange(3, device=device).view(3, 1, 1)
    ky = torch.arange(7, device=device).view(1, 7, 1)
    kx = torch.arange(7, device=device).view(1, 1, 7)
    a, r = (ky + 1) // 2, (ky + 1) % 2
    b, s = (kx + 1) // 2, (kx + 1) % 2
    return ((a * 4 + b) * 12 + (r * 2 + s) * 3 + c).reshape(-1)


class StemConvFn(torch.autograd.Function):
    """The backbone's 7x7 stride-2 pad-3 stem on 3-channel images, as the tensor-core inference runs it: lt_stem_s2d_fwd packs the
    images into the 2x2 space-to-depth split-fp16 input, then a 4x4 stride-1 conv (engine.pack_stem_s2d).  Weight gradient:
    lt_conv_wgrad_fwd of that 4x4 conv (12 real input channels), mapped back to (Cout, 3, 7, 7).  No image gradient."""

    @staticmethod
    def forward(ctx, images, weight, bias):
        if not images.is_cuda:
            raise RuntimeError("lt_b200 native training convolutions need CUDA tensors (got %s)" % images.device)
        N, C, H, W = images.shape
        cout = weight.shape[0]
        img = images.detach().float().contiguous()
        x_s = torch.empty((N, 1, H // 2, W // 2, 64), dtype=torch.float16, device=images.device)
        capi.stem_s2d(img, x_s, N, C, H, W)
        pk = engine.pack_stem_s2d(_Filter(weight.detach(), None if bias is None else bias.detach(), (2, 2), (3, 3)), None,
                                  out_fmt=capi.FMT_F32)
        out = engine.Act(N, 1, H // 2, W // 2, _round_up(cout, 4), capi.FMT_F32, images.device)
        engine.launch_conv(engine.Act.view(x_s), pk, out, out_dims=(1, H // 2, W // 2))
        ctx.save_for_backward(img, weight)
        return _from_cl(out.data, cout, 2)

    @staticmethod
    def backward(ctx, grad_out):
        img, weight = ctx.saved_tensors
        N, C, H, W = img.shape
        cout = weight.shape[0]
        g_s, g, amax, inv = _grad_s32(grad_out, _round_up(cout, 32))
        gw = gb = None
        if ctx.needs_input_grad[1]:
            x_s = torch.empty((N, 1, H // 2, W // 2, 64), dtype=torch.float16, device=img.device)
            capi.stem_s2d(img, x_s, N, C, H, W)
            gs = _wgrad(stem_wgrad_desc(N, H, W, cout), x_s, g_s, amax, 12, cout, 16)           # [tap a 4 + b][s2d channel][cout]
            gw = gs.reshape(16 * 12, cout)[stem_wgrad_index(img.device)].t().reshape(cout, 3, 7, 7).contiguous()
        if ctx.needs_input_grad[2]:
            gb = g.sum(dim=(0, 1, 2, 3))
        return None, gw, gb


def conv3d(x, weight, bias=None, padding=(0, 0, 0)):
    """F.conv3d(x, weight, bias, 1, padding) for stride-1 'same' filters on the native training kernels."""
    return ConvNdFn.apply(x, weight, bias, (1, 1, 1), tuple(padding))


def conv2d(x, weight, bias=None, stride=(1, 1), padding=(0, 0)):
    """F.conv2d(x, weight, bias, stride, padding) for the geometries of conv_kind on the native training kernels."""
    return ConvNdFn.apply(x, weight, bias, tuple(stride), tuple(padding))


def conv_transpose3d(x, weight, bias=None):
    """F.conv_transpose3d(x, weight, bias, stride=2) for 2^3 filters on the native training kernels."""
    return ConvTranspose3dFn.apply(x, weight, bias)


def conv_transpose2d_k4s2(x, weight, bias=None):
    """F.conv_transpose2d(x, weight, bias, stride=2, padding=1) for 4x4 filters on the native training kernels."""
    if tuple(weight.shape[2:]) != (4, 4):
        raise ValueError("native ConvTranspose2d: 4x4 filters only, got %s" % (tuple(weight.shape),))
    return ConvTranspose2dK4Fn.apply(x, weight, bias)


def stem_conv(images, weight, bias=None):
    """F.conv2d(images, weight, bias, 2, 3) for a (Cout, 3, 7, 7) stem filter on the native training kernels (no image gradient)."""
    if tuple(weight.shape[1:]) != (3, 7, 7) or images.dim() != 4 or images.shape[1] != 3:
        raise ValueError("native stem: 3-channel images and (Cout, 3, 7, 7) filters only, got %s and %s"
                         % (tuple(images.shape), tuple(weight.shape)))
    if images.shape[2] % 2 or images.shape[3] % 2:
        raise ValueError("native stem: even image sides only (space-to-depth input), got %dx%d" % tuple(images.shape[2:]))
    if images.requires_grad and torch.is_grad_enabled():
        raise ValueError("native stem: image gradients are not computed; the images must not require grad")
    return StemConvFn.apply(images, weight, bias)


def v2v_conv(module, x):
    """A Conv3d / ConvTranspose3d module of the V2V net applied through the native functions (the module's own parameters)."""
    if isinstance(module, torch.nn.ConvTranspose3d):
        if tuple(module.stride) != (2, 2, 2) or tuple(module.padding) != (0, 0, 0) or tuple(module.output_padding) != (0, 0, 0):
            raise ValueError("native ConvTranspose3d: stride 2, no padding only")
        return conv_transpose3d(x, module.weight, module.bias)
    if tuple(module.stride) != (1, 1, 1) or module.groups != 1 or tuple(module.dilation) != (1, 1, 1):
        raise ValueError("native Conv3d: stride 1, no groups, no dilation only")
    return conv3d(x, module.weight, module.bias, module.padding)


def backbone_conv(module, x):
    """A Conv2d / ConvTranspose2d module of the 2-D backbone (pose_resnet.py), its confidence heads or `process_features` applied
    through the native functions (the module's own parameters): the 7x7 stride-2 stem on 3-channel images, stride-1 'same',
    1x1 stride-2 and 3x3 stride-2 pad-1 convs, and k4 s2 p1 transposed convs.  ValueError for anything else."""
    if isinstance(module, torch.nn.ConvTranspose2d):
        if (tuple(module.kernel_size) != (4, 4) or tuple(module.stride) != (2, 2) or tuple(module.padding) != (1, 1)
                or tuple(module.output_padding) != (0, 0) or module.groups != 1 or tuple(module.dilation) != (1, 1)
                or module.padding_mode != "zeros"):
            raise ValueError("native ConvTranspose2d: kernel 4, stride 2, padding 1, no output padding, groups or dilation only")
        return conv_transpose2d_k4s2(x, module.weight, module.bias)
    if not isinstance(module, torch.nn.Conv2d) or module.groups != 1 or tuple(module.dilation) != (1, 1):
        raise ValueError("native Conv2d: no groups, no dilation only")
    if isinstance(module.padding, str):
        raise ValueError("native Conv2d: numeric padding only, got %r" % (module.padding,))
    if module.padding_mode != "zeros":
        raise ValueError("native Conv2d: zero padding only, got padding_mode=%r" % (module.padding_mode,))
    if tuple(module.kernel_size) == (7, 7) and tuple(module.stride) == (2, 2) and tuple(module.padding) == (3, 3):
        return stem_conv(x, module.weight, module.bias)
    conv_kind(_as3(module.kernel_size, 1), _as3(module.stride, 1), _as3(module.padding, 0))
    return conv2d(x, module.weight, module.bias, module.stride, module.padding)


# ---- BatchNorm for training (norm_backend="native"): batch statistics, the ReLU after the BatchNorm and the residual add of a residual
# unit on csrc/norm.cu, over the float32 channels-last maps the native convolutions produce.

class BatchNormActFn(torch.autograd.Function):
    """act(BatchNorm(x) (+ residual)) with act = ReLU or identity, for (N, C, [D,] H, W) float32 maps with C % 4 == 0: lt_batch_norm_fwd
    and lt_batch_norm_bwd.  Train mode normalises with the batch statistics and updates the running buffers in place; eval mode uses
    the running buffers.  x, the output (with ReLU, for its mask) and the per-channel mean / invstd are saved: the output is the tensor
    the next convolution keeps anyway, so nothing extra is stored.  The output is channels_last(_3d), so the next native conv reads it
    as a view."""

    @staticmethod
    def forward(ctx, x, weight, bias, residual, running_mean, running_var, eps, momentum, training, relu):
        nd = x.dim() - 2
        C = x.shape[1]
        x_cl = _cl(x)
        M = x_cl.numel() // C
        r_cl = None if residual is None else _cl(residual)
        y_cl = torch.empty_like(x_cl)
        mean = torch.empty(C, dtype=torch.float32, device=x.device)
        invstd = torch.empty_like(mean)
        ws = _workspace(x.device, capi.batch_norm_workspace_bytes(M, C))
        capi.batch_norm(x_cl, r_cl, weight.detach().float().contiguous(), bias.detach().float().contiguous(), running_mean, running_var,
                        mean, invstd, y_cl, M, C, eps, momentum, training, relu, ws)
        y = _from_cl(y_cl, C, nd)
        ctx.save_for_backward(x, y if relu else None, mean, invstd, weight)
        ctx.cfg = (M, C, nd, bool(training), bool(relu))
        return y

    @staticmethod
    def backward(ctx, grad_out):
        x, y, mean, invstd, weight = ctx.saved_tensors
        M, C, nd, training, relu = ctx.cfg
        x_cl = _cl(x)
        g_cl = _cl(grad_out)
        gx = torch.empty_like(x_cl)
        gr = torch.empty_like(x_cl) if ctx.needs_input_grad[3] else None
        gw = torch.empty(C, dtype=torch.float32, device=x.device)
        gb = torch.empty_like(gw)
        ws = _workspace(x.device, capi.batch_norm_workspace_bytes(M, C))
        capi.batch_norm_bwd(x_cl, _cl(y) if relu else None, g_cl, weight.detach().float().contiguous(), mean, invstd, gx, gr, gw, gb, M, C,
                            training, relu, ws)
        return (_from_cl(gx, C, nd), gw, gb, None if gr is None else _from_cl(gr, C, nd), None, None, None, None, None, None)


def batch_norm(module, x, relu=False, residual=None):
    """`norm` hook of pose_resnet.PoseResNet / v2v.V2VModel: relu(module(x) + residual) (ReLU and residual optional) for an
    nn.BatchNorm2d / BatchNorm3d on the native kernels, reading eps, momentum, training, the affine parameters and the running buffers
    from the module; num_batches_tracked is incremented on the device in train mode, as nn.BatchNorm does.  ValueError for what the
    kernels do not implement: momentum=None (cumulative average), affine=False, track_running_stats=False, C % 4 != 0, fewer than 2
    values per channel in train mode; RuntimeError for CPU tensors."""
    if module.momentum is None:
        raise ValueError("native BatchNorm: momentum=None (cumulative moving average) is not supported")
    if not module.affine:
        raise ValueError("native BatchNorm: affine=False is not supported")
    if not module.track_running_stats:
        raise ValueError("native BatchNorm: track_running_stats=False is not supported")
    C = module.num_features
    if C % 4:
        raise ValueError("native BatchNorm: the channel count must be a multiple of 4, got %d" % C)
    if x.dim() not in (4, 5) or x.shape[1] != C:
        raise ValueError("native BatchNorm: expected a (N, %d, [D,] H, W) map, got %s" % (C, tuple(x.shape)))
    if residual is not None and tuple(residual.shape) != tuple(x.shape):
        raise ValueError("native BatchNorm: residual %s differs from the input %s" % (tuple(residual.shape), tuple(x.shape)))
    if module.training and x.numel() // C < 2:
        raise ValueError("native BatchNorm: expected more than 1 value per channel when training, got input size %s" % (tuple(x.shape),))
    if not x.is_cuda or (residual is not None and not residual.is_cuda):
        raise RuntimeError("lt_b200 native BatchNorm needs CUDA tensors (got %s)" % x.device)
    if module.training:
        module.num_batches_tracked.add_(1)
    return BatchNormActFn.apply(x, module.weight, module.bias, residual, module.running_mean, module.running_var, module.eps,
                                module.momentum, module.training, relu)


# ---- The confidence heads' tail for training (head_backend="native"): csrc/algebraic.cu's lt_conf_head_tail_fwd / _bwd and
# lt_view_normalize_fwd / _bwd.  No cuBLAS: the head's Linear layers and their gradients are fixed-order kernels of the project.

class ConfHeadTailFn(torch.autograd.Function):
    """MaxPool2d(2) -> ReLU -> mean over the pooled positions -> Linear + ReLU -> Linear + ReLU -> Linear + Sigmoid of a (N, C0, H, W)
    float32 map of any element strides (NCHW or channels_last, read in place): lt_conf_head_tail_fwd, which keeps the mean x0 and the
    hidden activations h1, h2 for lt_conf_head_tail_bwd.  Gradients reach the map and the six Linear parameters."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2, w3, b3):
        N, dev = x.shape[0], x.device
        lins = tuple((w.detach().float().contiguous(), b.detach().float().contiguous()) for w, b in ((w1, b1), (w2, b2), (w3, b3)))
        out, x0, h1, h2 = (torch.empty((N, k), dtype=torch.float32, device=dev)
                           for k in (lins[2][0].shape[0], x.shape[1], lins[0][0].shape[0], lins[1][0].shape[0]))
        capi.conf_head_tail(x.detach(), *lins, out, x0, h1, h2)
        ctx.save_for_backward(x, lins[0][0], lins[1][0], lins[2][0], x0, h1, h2, out)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        x, w1, w2, w3, x0, h1, h2, y = ctx.saved_tensors
        N, C0 = x0.shape
        dev = x.device
        grad_x = torch.empty_like(x)
        grads = tuple(torch.empty(shape, dtype=torch.float32, device=dev)
                      for shape in (w1.shape, w1.shape[:1], w2.shape, w2.shape[:1], w3.shape, w3.shape[:1]))
        ws = torch.empty(capi.conf_head_tail_bwd_workspace_bytes(N, C0, w1.shape[0], w2.shape[0], w3.shape[0]), dtype=torch.uint8,
                         device=dev)
        capi.conf_head_tail_bwd(x.detach(), w1, w2, w3, x0, h1, h2, y, grad_out.float().contiguous(), grad_x, grads, ws)
        return (grad_x,) + grads


def conf_head_tail(head, x):
    """The `tail` hook of pose_resnet.ConfidenceHead: its second max pool, ReLU, global mean and `head` MLP applied to the second
    BatchNorm's output x through ConfHeadTailFn.  ValueError for a map the kernels do not take; RuntimeError for CPU tensors."""
    lin = [m for m in head.head if isinstance(m, torch.nn.Linear)]
    if x.dim() != 4 or x.shape[1] != lin[0].in_features:
        raise ValueError("native confidence head: expected a (N, %d, H, W) map, got %s" % (lin[0].in_features, tuple(x.shape)))
    if x.shape[2] < 2 or x.shape[3] < 2:
        raise ValueError("native confidence head: a %dx%d map is too small for the 2x2 max pool" % tuple(x.shape[2:]))
    if x.dtype != torch.float32:
        raise TypeError("native confidence head: float32 maps only (got %s)" % x.dtype)
    if not x.is_cuda:
        raise RuntimeError("lt_b200 native confidence head needs CUDA tensors (got %s)" % x.device)
    return ConfHeadTailFn.apply(x, lin[0].weight, lin[0].bias, lin[1].weight, lin[1].bias, lin[2].weight, lin[2].bias)


class ViewNormalizeFn(torch.autograd.Function):
    """conf / conf.sum(dim=1, keepdim=True) + eps for (B, V, C) float32 confidences: lt_view_normalize_fwd on a copy (the backward
    reads the un-normalised values), lt_view_normalize_bwd."""

    @staticmethod
    def forward(ctx, conf, eps):
        c = conf.detach().float().contiguous()
        out = c.clone()
        B, V, C = c.shape
        capi.view_normalize(out, B, V, C, eps)
        ctx.save_for_backward(c)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        c, = ctx.saved_tensors
        grad = torch.empty_like(c)
        capi.view_normalize_bwd(c, grad_out.float().contiguous(), grad)
        return grad, None


def view_normalize(conf, eps):
    """(B, V, C) confidences normalised over the views (dim 1), plus eps, on the native kernels."""
    if conf.dim() != 3:
        raise ValueError("view_normalize: expected (B, V, C) confidences, got %s" % (tuple(conf.shape),))
    if not conf.is_cuda:
        raise RuntimeError("lt_b200 native view normalisation needs CUDA tensors (got %s)" % conf.device)
    return ViewNormalizeFn.apply(conf, eps)
