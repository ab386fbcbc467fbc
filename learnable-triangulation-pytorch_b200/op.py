"""Op-level drop-ins for the two custom ops of the volumetric path.

Same names / argument meaning / error behaviour as `/root/reference/mvn/utils/op.py`:
`unproject_heatmaps` (:99-166) and `integrate_tensor_3d_with_coordinates` (:84-96).
CUDA tensors without grad go to the hand-written kernels through the C ABI; anything else must
ask for another formulation explicitly -- there is no silent fallback: backend="torch" (or
LT_B200_BACKEND=torch) is the autograd/CPU torch formulation, backend="hybrid" keeps the native
forward kernels and adds their native backward (autograd_ops.py, csrc/backward.cu) for training.
"""
import os

import torch

from . import autograd_ops, capi, engine, torch_ops

_AGGS = ("sum", "max", "softmax", "conf", "conf_norm")


def _resolve_backend(backend, *tensors):
    backend = backend or os.environ.get("LT_B200_BACKEND", "native")
    if backend == "torch":
        return "torch"
    if backend not in ("native", "hybrid"):
        raise ValueError("unknown backend {!r}".format(backend))
    if backend == "hybrid":
        if not all(t.is_cuda for t in tensors if t is not None):
            raise RuntimeError("lt_b200 hybrid ops need CUDA tensors")
        return "hybrid"
    if not all(t.is_cuda for t in tensors if t is not None):
        raise RuntimeError("lt_b200 native ops need CUDA tensors; pass backend='torch' (or LT_B200_BACKEND=torch) "
                           "for the autograd/CPU formulation")
    if torch.is_grad_enabled() and any(t.requires_grad for t in tensors if t is not None):
        raise RuntimeError("lt_b200 native ops are inference-only; use backend='torch' when gradients are required")
    return "native"


def unproject_heatmaps(heatmaps, proj_matricies, coord_volumes, volume_aggregation_method="sum", vol_confidences=None,
                       backend=None):
    if not (volume_aggregation_method in _AGGS or volume_aggregation_method.startswith("conf")):
        raise ValueError("Unknown volume_aggregation_method: {}".format(volume_aggregation_method))
    which = _resolve_backend(backend, heatmaps, proj_matricies, coord_volumes, vol_confidences)
    if which == "torch":
        return torch_ops.unproject_heatmaps(heatmaps, proj_matricies, coord_volumes, volume_aggregation_method, vol_confidences)
    if which == "hybrid":
        return autograd_ops.unproject_heatmaps(heatmaps, proj_matricies, coord_volumes, volume_aggregation_method, vol_confidences)
    B, V, C, h, w = heatmaps.shape
    vol_shape = tuple(coord_volumes.shape[1:4])
    nvox = vol_shape[0] * vol_shape[1] * vol_shape[2]
    feats_cl = heatmaps.float().permute(0, 1, 3, 4, 2).contiguous()            # (B, V, h, w, C)
    agg = capi.AGG["conf" if volume_aggregation_method.startswith("conf") else volume_aggregation_method]
    conf = None
    if agg == capi.AGG["conf"]:
        conf = vol_confidences.float().reshape(B, V, C).contiguous()
    out_cl = torch.empty((B, nvox, C), dtype=torch.float32, device=heatmaps.device)
    capi.unproject_aggregate(feats_cl, proj_matricies.float().contiguous(), coord_volumes.float().reshape(B, nvox, 3).contiguous(),
                             conf, out_cl, capi.FMT_F32, agg)
    out = torch.empty((B, C, nvox), dtype=torch.float32, device=heatmaps.device)
    capi.cl_to_cf(out_cl, out, B, nvox, C, C)
    return out.view(B, C, *vol_shape)


def integrate_tensor_3d_with_coordinates(volumes, coord_volumes, softmax=True, backend=None):
    which = _resolve_backend(backend, volumes, coord_volumes)
    if which == "torch":
        return torch_ops.integrate_tensor_3d_with_coordinates(volumes, coord_volumes, softmax)
    if which == "hybrid":
        return autograd_ops.integrate_tensor_3d_with_coordinates(volumes, coord_volumes, softmax)
    B, J = volumes.shape[:2]
    nvox = volumes[0, 0].numel()
    logits = volumes.float().contiguous()
    coord = coord_volumes.float().reshape(B, nvox, 3).contiguous()
    out = torch.empty_like(logits)
    keypoints = torch.empty((B, J, 3), dtype=torch.float32, device=volumes.device)
    ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, nvox) // 4 + 1, dtype=torch.float32, device=volumes.device)
    capi.softargmax3d(logits, J * nvox, 1, nvox, coord, out, keypoints, ws, B, J, nvox, 1.0, softmax)
    return keypoints, out


def integrate_tensor_2d(heatmaps, softmax=True, backend=None):
    """Drop-in for reference op.py:11-47: (B, J, h, w) -> coordinates (B, J, 2) [x, y in pixels], normalised heatmaps."""
    which = _resolve_backend(backend, heatmaps)
    if which == "torch":
        return torch_ops.integrate_tensor_2d(heatmaps, softmax)
    if which == "hybrid":
        return autograd_ops.integrate_tensor_2d(heatmaps, softmax)
    B, J, h, w = heatmaps.shape
    dev = heatmaps.device
    grid = engine.pixel_grid(B, h, w, dev)
    logits = heatmaps.float().contiguous()
    out = torch.empty_like(logits)
    kp = torch.empty((B, J, 3), dtype=torch.float32, device=dev)
    ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, h * w) // 4 + 1, dtype=torch.float32, device=dev)
    # softmax=False: ReLU heat-maps, centre of mass divided by the mass (op.py:25-41) = mode 2 of lt_softargmax3d_fwd
    capi.softargmax3d(logits, J * h * w, 1, h * w, grid, out, kp, ws, B, J, h * w, 1.0, 1 if softmax else 2)
    return kp[:, :, :2].contiguous(), out
