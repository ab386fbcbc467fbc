"""Drop-in for the reference's VolumetricCELoss (mvn/models/loss.py:52-80), the cross-entropy term of the volumetric training recipe
(`use_volumetric_ce_loss`, train.py:222-230).

On CUDA tensors the loss runs on csrc/loss.cu (`lt_volumetric_ce_fwd` / `lt_volumetric_ce_bwd`): one pass over each sample's
coordinate volume finds the nearest voxel of every joint, and the backward writes the sparse gradient of the volumes in one pass.
The reference instead builds (J, N^3, 3) difference tensors per sample, copies the argmin to the host, and indexes one voxel per
(sample, joint) with Python ints, whose backward zero-fills and accumulates a volume-sized gradient for every term.

Backend: the `backend` argument, else LT_B200_BACKEND, else "native".  "torch" is the vectorised torch formulation
(torch_ops.volumetric_ce_loss, for CPU tensors and as a checker).  This op always has its native backward, so "native" and
"hybrid" both run the kernels, with or without grad.  CPU tensors on those backends raise; nothing falls back silently.
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
