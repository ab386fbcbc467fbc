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
