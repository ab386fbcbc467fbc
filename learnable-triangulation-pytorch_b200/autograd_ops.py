"""Differentiable wrappers of the native custom ops (`backend="hybrid"`): the forward is the same hand-written kernel the
inference path uses, the backward is `csrc/backward.cu` (lt_unproject_aggregate_bwd, lt_softargmax3d_bwd) and
`csrc/algebraic.cu` (lt_triangulate_dlt_bwd).

This is the first stage of SURVEY section 8f row 1: with it the reference training loop (`train.py:159-243`,
`total_loss.backward()` at :236) runs the custom ops on the native kernels while the convolutions stay on torch/cuDNN
autograd.  Volumetric model: the unprojection + aggregation and the 3-D soft-argmax -- the ops the reference implements as
Python loops over (sample, view) pairs with ~10 passes over a (V, C, N^3) staging tensor.  Algebraic model: the 2-D
soft-argmax (op.py:11-47, both branches) and the confidence-weighted DLT, which the reference runs as one torch.svd per
(sample, joint) (multiview.py:171-183).  Gradients: feature maps / heat-maps, `conf` and algebraic confidences, V2V logits,
2-D key points; projection matrices and coordinate volumes carry none (they do not in the reference either: they come from
numpy camera data).
"""
import torch

from . import capi


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
        capi.unproject_aggregate_bwd(feats_cl, proj, coord, conf, g_cl, grad_feats, grad_conf, ctx.agg)
        grad_heat = grad_feats.permute(0, 1, 4, 2, 3)                                       # (B, V, C, h, w) view
        return grad_heat, None, None, (grad_conf.reshape(ctx.conf_shape) if need_conf else None), None


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
        return keypoints, out

    @staticmethod
    def backward(ctx, grad_kp, grad_vol):
        probs, coord = ctx.saved_tensors
        B, J = probs.shape[:2]
        nvox = coord.shape[1]
        dev = probs.device
        g_kp = (grad_kp if grad_kp is not None else torch.zeros((B, J, 3), device=dev)).float().contiguous()
        g_vol = None if grad_vol is None else grad_vol.float().contiguous()
        grad_logits = torch.empty_like(probs)
        scratch = torch.empty(B * J, dtype=torch.float32, device=dev)
        capi.softargmax3d_bwd(probs, coord, g_kp, g_vol, grad_logits, scratch, B, J, nvox, 1.0, ctx.softmax)
        return grad_logits, None, None


def pixel_grid(B, h, w, device):
    """(B, h*w, 3) float32 coordinates (x, y, 0) of the pixels of an h x w map: the 2-D soft-argmax runs on the 3-D kernels."""
    ys, xs = torch.meshgrid(torch.arange(h, device=device, dtype=torch.float32), torch.arange(w, device=device, dtype=torch.float32),
                            indexing="ij")
    return torch.stack([xs, ys, torch.zeros_like(xs)], dim=-1).reshape(1, h * w, 3).expand(B, h * w, 3).contiguous()


class IntegrateTensor2dFn(torch.autograd.Function):
    """op.integrate_tensor_2d (reference op.py:11-47): (B, J, h, w) -> (coordinates (B, J, 2) [x, y in pixels], heat-maps)."""

    @staticmethod
    def forward(ctx, heatmaps, softmax):
        B, J, h, w = heatmaps.shape
        dev = heatmaps.device
        logits = heatmaps.detach().float().contiguous()
        grid = pixel_grid(B, h, w, dev)
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
    -> (B, J, 3).  Gradients reach the key points and the confidences, not the projection matrices."""

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
        grad_kp = torch.empty_like(kp)
        grad_conf = torch.empty_like(conf) if need_conf else None
        capi.triangulate_dlt_bwd(proj, kp, conf, grad_out.float().contiguous(), grad_kp, grad_conf)
        return None, (grad_kp if ctx.needs_input_grad[1] else None), grad_conf


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


def integrate_tensor_2d(heatmaps, softmax=True):
    return IntegrateTensor2dFn.apply(heatmaps, softmax)


def triangulate_batch_of_points(proj_matricies_batch, points_batch, confidences_batch=None):
    return TriangulateDltFn.apply(proj_matricies_batch, points_batch, confidences_batch)


def unproject_heatmaps(heatmaps, proj_matricies, coord_volumes, volume_aggregation_method="sum", vol_confidences=None):
    agg = capi.AGG["conf" if volume_aggregation_method.startswith("conf") else volume_aggregation_method]
    return UnprojectHeatmapsFn.apply(heatmaps, proj_matricies, coord_volumes, vol_confidences, agg)


def integrate_tensor_3d_with_coordinates(volumes, coord_volumes, softmax=True):
    return IntegrateTensor3dFn.apply(volumes, coord_volumes, softmax)


# ---- V2V convolutions for training (v2v_backend="native"): forward and data gradient on the forward conv kernels, weight gradient on
# csrc/conv_wgrad.cu.  Activations are float32 channels_last_3d tensors, so the kernels read and write them in place of a transpose
# and torch's BatchNorm / ReLU / pooling / adds run on them unchanged.

class _Filter:
    """The nn.Conv attributes engine.pack_conv reads, for a filter that is not (or not only) a module's own."""

    def __init__(self, weight, bias, stride, padding):
        self.weight, self.bias = weight, bias
        self.kernel_size, self.stride, self.padding = tuple(weight.shape[2:]), tuple(stride), tuple(padding)


_WORKSPACE = {}


def _workspace(device, nbytes):
    """Scratch shared by the split-K conv launches and the weight gradient of one device (launches on one stream are ordered)."""
    ws = _WORKSPACE.get(device)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(max(nbytes, 32 << 20), dtype=torch.uint8, device=device)
        _WORKSPACE[device] = ws
    return ws


def _round_up(v, m):
    return (v + m - 1) // m * m


def _cl(x):
    """(N, C, D, H, W) -> contiguous float32 (N, D, H, W, C) (a view for channels_last_3d input)."""
    if not x.is_cuda:
        raise RuntimeError("lt_b200 native V2V convolutions need CUDA tensors (got %s)" % x.device)
    return x.float().contiguous(memory_format=torch.channels_last_3d).permute(0, 2, 3, 4, 1)


def _to_s32(x_cl, cp, absmax_bits=None, inv_scale=None):
    """(N, D, H, W, C) float32 -> split-fp16 (N, D, H, W, 2 cp), scaled by the power of two that absmax_bits selects."""
    out = torch.empty(x_cl.shape[:4] + (2 * cp,), dtype=torch.float16, device=x_cl.device)
    capi.f32_to_s32_scaled(x_cl, out, x_cl[..., 0].numel(), x_cl.shape[4], cp, absmax_bits, inv_scale)
    return out


def conv_desc(N, in_dims, cin_p, cout_p, k, stride, pad, out_dims, out_c, out_fmt, out_scale=(1, 1, 1), out_full=None, groups=(1, 1, 1)):
    """lt_conv_desc of a split-fp16-input launch without ReLU or residual; out_full: the output tensor's grid (default out_dims)."""
    fd, fh, fw = out_full or out_dims
    return capi.ConvDesc(N=N, ID=in_dims[0], IH=in_dims[1], IW=in_dims[2], Cin=cin_p, OD=out_dims[0], OH=out_dims[1], OW=out_dims[2],
                         Cout=cout_p, KD=k[0], KH=k[1], KW=k[2], sd=stride[0], sh=stride[1], sw=stride[2], pd=pad[0], ph=pad[1], pw=pad[2],
                         FD=fd, FH=fh, FW=fw, FC=out_c, osd=out_scale[0], osh=out_scale[1], osw=out_scale[2], relu=0, residual=capi.RES_NONE,
                         in_format=capi.FMT_S32, out_format=out_fmt, ogd=groups[0], ogh=groups[1], ogw=groups[2])


def conv3d_wgrad_desc(N, dims, cin, cout, k, padding):
    """The forward launch of a stride-1 Conv3d as lt_conv_wgrad_fwd reads it: split-fp16 input and output gradient, 32-channel padded."""
    return conv_desc(N, dims, _round_up(cin, 32), _round_up(cout, 32), k, (1, 1, 1), padding, dims, _round_up(cout, 32), capi.FMT_S32)


def conv_transpose3d_desc(N, dims, cin, cout):
    """ConvTranspose3d(k=2, s=2) as the engine's one grouped 1x1x1 GEMM: N = 8 cout, block g = a 4 + b 2 + c to output phase (a, b, c)."""
    D, H, W = dims
    return conv_desc(N, dims, cin, 8 * cout, (1, 1, 1), (1, 1, 1), (0, 0, 0), dims, cout, capi.FMT_S32, out_scale=(2, 2, 2),
                     out_full=(2 * D, 2 * H, 2 * W), groups=(2, 2, 2))


def conv3d_dgrad_filter(weight_shape, padding):
    """Data gradient of a stride-1 'same' Conv3d (Cout, Cin, kd, kh, kw) as a forward conv of dY: lt_conv_gather_weights_fwd source
    (base, (s_td, s_th, s_tw, s_ci, s_co)) of the filter flipped in space with Cin and Cout swapped -- element (td, th, tw, ci' = co,
    co' = ci) = w[co][ci][kd-1-td][kh-1-th][kw-1-tw] -- and the conv's (k, stride, pad, cin', cout')."""
    cout, cin, kd, kh, kw = weight_shape
    T = kd * kh * kw
    return (T - 1, (-kh * kw, -kw, -1, cin * T, T)), (kd, kh, kw), (1, 1, 1), tuple(padding), cout, cin


def conv_transpose3d_dgrad_filter(weight_shape):
    """Data gradient of ConvTranspose3d(k=2, s=2) (Cin, Cout, 2, 2, 2): dX[o][ci] = sum_{t, co} dY[2 o + t][co] w[ci][co][t], a 2^3
    stride-2 pad-0 conv of dY with element (td, th, tw, ci' = co, co' = ci) = w[ci][co][td][th][tw]."""
    cin, cout = weight_shape[:2]
    return (0, (4, 2, 1, 8, cout * 8)), (2, 2, 2), (2, 2, 2), (0, 0, 0), cout, cin


def _launch(x_s, cin_p, pk, out_dims, out_c, scale, shift, out_fmt=capi.FMT_F32, out_scale=(1, 1, 1), out_full=None, groups=(1, 1, 1)):
    """One lt_conv_nd_fwd of packed filter `pk` over split-fp16 x_s; the full-resolution 3^3 / 7^3 layers take LT_CONV_TC_FOLD as in
    the inference engine."""
    N, D, H, W = x_s.shape[:4]
    fd, fh, fw = out_full or out_dims
    c_store = out_c if out_fmt == capi.FMT_F32 else 2 * out_c
    out = torch.empty((N, fd, fh, fw, c_store), dtype=torch.float32 if out_fmt == capi.FMT_F32 else torch.float16, device=x_s.device)
    d = conv_desc(N, (D, H, W), cin_p, pk.cout_p, pk.k, pk.stride, pk.pad, out_dims, out_c, out_fmt, out_scale, out_full, groups)
    ws = _workspace(x_s.device, 0)
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    impl, weight = capi.CONV_TC, pk.w
    if pk.w_fold is not None and W >= 16 and out_c == 32 and out_fmt == capi.FMT_F32:
        impl, weight = capi.CONV_TC_FOLD, pk.w_fold
        d.Cout = pk.cout
    capi.conv_nd(d, x_s, weight, scale, shift, None, out, impl)
    return out, d


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


class Conv3dFn(torch.autograd.Function):
    """nn.Conv3d with stride 1 and "same" padding (every Conv3d of v2v.py) on the tensor-core kernels, fp32-grade in all three passes.
    forward: lt_conv_nd_fwd (scale 1 / S, shift = bias); data gradient: the same kernels over the output gradient with the filter
    flipped in space and Cin / Cout swapped (re-gathered by lt_conv_gather_weights_fwd with negated tap strides); weight gradient:
    lt_conv_wgrad_fwd; bias gradient: torch's sum of the output gradient."""

    @staticmethod
    def forward(ctx, x, weight, bias, padding):
        from .engine import pack_conv
        cout, cin, kd, kh, kw = weight.shape
        if tuple(padding) != (kd // 2, kh // 2, kw // 2) or not (kd % 2 and kh % 2 and kw % 2):
            raise ValueError("native Conv3d: stride 1 'same' convolutions only (odd kernel, padding k // 2), got k=%s padding=%s"
                             % ((kd, kh, kw), tuple(padding)))
        x_cl = _cl(x)
        cin_p = _round_up(cin, 32)
        x_s = _to_s32(x_cl, cin_p)
        pk = pack_conv(_Filter(weight.detach(), None if bias is None else bias.detach(), (1, 1, 1), padding), None, cin_pad=cin_p,
                       out_fmt=capi.FMT_F32)
        out, _ = _launch(x_s, cin_p, pk, x_cl.shape[1:4], _round_up(cout, 4), pk.scale, pk.shift)
        ctx.save_for_backward(x_s, weight)
        ctx.padding = tuple(padding)
        return out[..., :cout].permute(0, 4, 1, 2, 3)

    @staticmethod
    def backward(ctx, grad_out):
        from .engine import pack_filter
        x_s, weight = ctx.saved_tensors
        cout, cin, kd, kh, kw = weight.shape
        T = kd * kh * kw
        cout_p = _round_up(cout, 32)
        g_s, g, amax, inv = _grad_s32(grad_out, cout_p)
        N, D, H, W = g.shape[:4]
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            w = weight.detach().float().contiguous()
            (base, strides), k, stride, pad, ci, co = conv3d_dgrad_filter(weight.shape, ctx.padding)
            pk = pack_filter((w, base, strides), k, stride, pad, ci, co, None, None, out_fmt=capi.FMT_F32)
            out, _ = _launch(g_s, cout_p, pk, (D, H, W), _round_up(cin, 4), pk.scale * inv, pk.shift)
            gx = out[..., :cin].permute(0, 4, 1, 2, 3)
        if ctx.needs_input_grad[1]:
            d = conv3d_wgrad_desc(N, (D, H, W), cin, cout, (kd, kh, kw), ctx.padding)
            gw = _wgrad(d, x_s, g_s, amax, cin, cout, T).reshape(kd, kh, kw, cin, cout).permute(4, 3, 0, 1, 2).contiguous()
        if ctx.needs_input_grad[2]:
            gb = g.sum(dim=(0, 1, 2, 3))
        return gx, gw, gb, None


class ConvTranspose3dFn(torch.autograd.Function):
    """nn.ConvTranspose3d(k=2, s=2, p=0) (v2v.py Upsample3DBlock) with Cout % 32 == 0: the forward is the engine's one grouped 1x1x1
    GEMM (N = 8 Cout, each 32-channel block written to its phase of the output lattice); the data gradient is a 2^3 stride-2
    convolution of the output gradient (Cin' = Cout, Cout' = Cin) on conv_tc_kernel; the weight gradient is lt_conv_wgrad_fwd over
    the forward's grouped GEMM."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        from .engine import pack_deconv3d_k2s2
        cin, cout = weight.shape[:2]
        if tuple(weight.shape[2:]) != (2, 2, 2) or cout % 32 or cin % 32:
            raise ValueError("native ConvTranspose3d: kernel 2, stride 2 and channel counts that are multiples of 32 only, got %s"
                             % (tuple(weight.shape),))
        x_cl = _cl(x)
        N, D, H, W = x_cl.shape[:4]
        x_s = _to_s32(x_cl, cin)
        pk = pack_deconv3d_k2s2(_Filter(weight.detach(), None if bias is None else bias.detach(), (2, 2, 2), (0, 0, 0)), None)
        y_s, _ = _launch(x_s, cin, pk, (D, H, W), cout, pk.scale, pk.shift, out_fmt=capi.FMT_S32, out_scale=(2, 2, 2),
                         out_full=(2 * D, 2 * H, 2 * W), groups=(2, 2, 2))
        out = torch.empty((N, 2 * D, 2 * H, 2 * W, cout), dtype=torch.float32, device=x.device)
        capi.s32_to_f32(y_s, out, out[..., 0].numel(), cout)
        ctx.save_for_backward(x_s, weight)
        return out.permute(0, 4, 1, 2, 3)

    @staticmethod
    def backward(ctx, grad_out):
        from .engine import pack_filter
        x_s, weight = ctx.saved_tensors
        cin, cout = weight.shape[:2]
        g_s, g, amax, inv = _grad_s32(grad_out, cout)
        N, D, H, W = x_s.shape[:4]
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            w = weight.detach().float().contiguous()
            (base, strides), k, stride, pad, ci, co = conv_transpose3d_dgrad_filter(weight.shape)
            pk = pack_filter((w, base, strides), k, stride, pad, ci, co, None, None, out_fmt=capi.FMT_F32)
            out, _ = _launch(g_s, cout, pk, (D, H, W), cin, pk.scale * inv, pk.shift)
            gx = out.permute(0, 4, 1, 2, 3)
        if ctx.needs_input_grad[1]:
            gw = _wgrad(conv_transpose3d_desc(N, (D, H, W), cin, cout), x_s, g_s, amax, cin, cout, 1, groups=8)       # [1][ci][g cout + co], g = a 4 + b 2 + c
            gw = gw.reshape(cin, 8, cout).permute(0, 2, 1).reshape(cin, cout, 2, 2, 2).contiguous()
        if ctx.needs_input_grad[2]:
            gb = g.sum(dim=(0, 1, 2, 3))
        return gx, gw, gb


def conv3d(x, weight, bias=None, padding=(0, 0, 0)):
    """F.conv3d(x, weight, bias, 1, padding) for stride-1 'same' filters on the native training kernels."""
    return Conv3dFn.apply(x, weight, bias, tuple(padding))


def conv_transpose3d(x, weight, bias=None):
    """F.conv_transpose3d(x, weight, bias, stride=2) for 2^3 filters on the native training kernels."""
    return ConvTranspose3dFn.apply(x, weight, bias)


def v2v_conv(module, x):
    """A Conv3d / ConvTranspose3d module of the V2V net applied through the native functions (the module's own parameters)."""
    if isinstance(module, torch.nn.ConvTranspose3d):
        if tuple(module.stride) != (2, 2, 2) or tuple(module.padding) != (0, 0, 0) or tuple(module.output_padding) != (0, 0, 0):
            raise ValueError("native ConvTranspose3d: stride 2, no padding only")
        return conv_transpose3d(x, module.weight, module.bias)
    if tuple(module.stride) != (1, 1, 1) or module.groups != 1 or tuple(module.dilation) != (1, 1, 1):
        raise ValueError("native Conv3d: stride 1, no groups, no dilation only")
    return conv3d(x, module.weight, module.bias, module.padding)
