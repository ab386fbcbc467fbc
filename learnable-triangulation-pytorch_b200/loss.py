"""Drop-ins for the reference's training criteria (mvn/models/loss.py): the keypoint criteria KeypointsMSELoss,
KeypointsMSESmoothLoss, KeypointsMAELoss and KeypointsL2Loss (loss.py:7-49, train.py:217, 246) and VolumetricCELoss (loss.py:52-80),
the cross-entropy term of the volumetric training recipe (`use_volumetric_ce_loss`, train.py:222-230).

On CUDA tensors the losses run on csrc/loss.cu.  The keypoint criteria (`lt_keypoints_loss_fwd` / `_bwd`) sum their terms in
float64 in one CTA and keep the divisor dim * max(1, sum v) on the device, where the reference reads sum v to the host with
`.item()` (and MSESmooth's boolean-mask index synchronises again): they can run inside a CUDA graph.  The cross-entropy loss
(`lt_volumetric_ce_fwd` / `lt_volumetric_ce_bwd`): one pass over each sample's coordinate volume finds the nearest voxel of every
joint, and the backward writes the sparse gradient of the volumes in one pass.  The reference instead builds (J, N^3, 3) difference
tensors per sample, copies the argmin to the host, and indexes one voxel per (sample, joint) with Python ints, whose backward
zero-fills and accumulates a volume-sized gradient for every term.

Backend: the `backend` argument, else LT_B200_BACKEND, else "native".  "torch" is the vectorised torch formulation
(torch_ops.keypoints_loss / torch_ops.volumetric_ce_loss, for CPU tensors and as a checker).  These ops always have their native
backward, so "native" and "hybrid" both run the kernels, with or without grad.  CPU tensors on those backends raise; nothing falls
back silently.
"""
import os

from torch import nn

from . import autograd_ops, torch_ops


def _resolve_backend(backend, *tensors):
    backend = backend or os.environ.get("LT_B200_BACKEND", "native")
    if backend == "torch":
        return "torch"
    if backend not in ("native", "hybrid"):
        raise ValueError("unknown backend {!r}".format(backend))
    if not all(t.is_cuda for t in tensors):
        raise RuntimeError("lt_b200 native ops need CUDA tensors; pass backend='torch' (or LT_B200_BACKEND=torch) "
                           "for the CPU formulation")
    return "native"


def _check_shapes(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity):
    if volumes_batch_pred.dim() != 5:
        raise ValueError("volumes_batch_pred must be (B, J, X, Y, Z), got {}".format(tuple(volumes_batch_pred.shape)))
    B, J = volumes_batch_pred.shape[:2]
    grid = tuple(volumes_batch_pred.shape[2:])
    if tuple(coord_volumes_batch.shape) != (B,) + grid + (3,):
        raise ValueError("coord_volumes_batch must be {} to match the volumes, got {}".format((B,) + grid + (3,),
                                                                                             tuple(coord_volumes_batch.shape)))
    if tuple(keypoints_gt.shape) != (B, J, 3):
        raise ValueError("keypoints_gt must be {}, got {}".format((B, J, 3), tuple(keypoints_gt.shape)))
    if keypoints_binary_validity.dim() != 3 or tuple(keypoints_binary_validity.shape[:2]) != (B, J) \
            or keypoints_binary_validity.shape[2] < 1:
        raise ValueError("keypoints_binary_validity must be (B, J, k >= 1) with (B, J) = {}, got {}".format(
            (B, J), tuple(keypoints_binary_validity.shape)))


def volumetric_ce_loss(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity, backend=None):
    """Functional form of VolumetricCELoss.forward: 0-dim loss; the gradient reaches volumes_batch_pred only."""
    _check_shapes(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity)
    which = _resolve_backend(backend, coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity)
    if which == "torch":
        return torch_ops.volumetric_ce_loss(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity)
    B, J = volumes_batch_pred.shape[:2]
    probs = volumes_batch_pred.float().reshape(B, J, -1)
    coord = coord_volumes_batch.detach().float().reshape(B, -1, 3).contiguous()     # logical (X, Y, Z) order, any strides
    kp = keypoints_gt.detach().float().contiguous()
    validity = keypoints_binary_validity.detach()[..., 0].float().contiguous()      # the reference's validity[0]
    return autograd_ops.volumetric_ce_loss(probs, coord, kp, validity)[0]


class VolumetricCELoss(nn.Module):
    """Same constructor and forward as the reference's VolumetricCELoss (loss.py:52-80); `backend` is optional (see module doc)."""

    def __init__(self, backend=None):
        super().__init__()
        self.backend = backend

    def forward(self, coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity):
        return volumetric_ce_loss(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity,
                                  backend=self.backend)


def _check_keypoint_shapes(pred, gt, validity):
    if pred.dim() != 3 or pred.shape[-1] < 1:
        raise ValueError("keypoints_pred must be (B, J, dim), got {}".format(tuple(pred.shape)))
    if gt.shape != pred.shape:
        raise ValueError("keypoints_gt must be {} to match keypoints_pred, got {}".format(tuple(pred.shape), tuple(gt.shape)))
    if tuple(validity.shape) not in (tuple(pred.shape[:2]), tuple(pred.shape[:2]) + (1,)):
        raise ValueError("keypoints_binary_validity must be (B, J, 1) or (B, J) with (B, J) = {}, got {}".format(
            tuple(pred.shape[:2]), tuple(validity.shape)))


def keypoints_loss(kind, keypoints_pred, keypoints_gt, keypoints_binary_validity, threshold=400, backend=None):
    """Functional form of the keypoint criteria: `kind` is "mse", "mse_smooth", "mae" or "l2"; -> 0-dim loss.  The gradient reaches
    keypoints_pred only (the ground truth and the validity are data)."""
    _check_keypoint_shapes(keypoints_pred, keypoints_gt, keypoints_binary_validity)
    which = _resolve_backend(backend, keypoints_pred, keypoints_gt, keypoints_binary_validity)
    validity = keypoints_binary_validity.detach().reshape(keypoints_pred.shape[:2] + (1,))
    if which == "torch":
        return torch_ops.keypoints_loss(keypoints_pred, keypoints_gt.detach(), validity, kind, threshold)
    B, J, dim = keypoints_pred.shape
    return autograd_ops.keypoints_loss(keypoints_pred.float().reshape(B * J, dim), keypoints_gt.detach().float().reshape(B * J, dim)
                                       .contiguous(), validity.float().reshape(B * J).contiguous(), kind, float(threshold))


class _KeypointsLoss(nn.Module):
    kind = None

    def __init__(self, backend=None):
        super().__init__()
        self.backend = backend

    def forward(self, keypoints_pred, keypoints_gt, keypoints_binary_validity):
        return keypoints_loss(self.kind, keypoints_pred, keypoints_gt, keypoints_binary_validity,
                              threshold=getattr(self, "threshold", 400), backend=self.backend)


class KeypointsMSELoss(_KeypointsLoss):
    """sum (gt - pred)^2 v / (dim * max(1, sum v)), as the reference's KeypointsMSELoss (loss.py:7-15); `backend` is optional (see
    module doc).  The gradient reaches keypoints_pred only."""
    kind = "mse"


class KeypointsMSESmoothLoss(_KeypointsLoss):
    """KeypointsMSELoss with every d = (gt - pred)^2 v > threshold replaced by d^0.1 * threshold^0.9, as the reference's
    KeypointsMSESmoothLoss(threshold=400) (loss.py:17-28); `backend` is optional (see module doc).  The gradient reaches
    keypoints_pred only."""
    kind = "mse_smooth"

    def __init__(self, threshold=400, backend=None):
        super().__init__(backend)
        self.threshold = threshold


class KeypointsMAELoss(_KeypointsLoss):
    """sum |gt - pred| v / (dim * max(1, sum v)), as the reference's KeypointsMAELoss (loss.py:31-39); `backend` is optional (see
    module doc).  The gradient reaches keypoints_pred only."""
    kind = "mae"


class KeypointsL2Loss(_KeypointsLoss):
    """sum over points of sqrt(sum_d (gt - pred)^2 v) / max(1, sum v), as the reference's KeypointsL2Loss (loss.py:42-49), the
    training metric `l2`; `backend` is optional (see module doc).  Its gradient, which reaches keypoints_pred only, is torch's
    through the reference formula: NaN where a point's residual has length zero (every invalid point among them)."""
    kind = "l2"
