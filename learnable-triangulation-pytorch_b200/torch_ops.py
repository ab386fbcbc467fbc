"""Autograd-capable torch formulations of the two custom ops (backend="torch").

Used when gradients are needed (training is a "next" row, SURVEY.md section 8f) and for host-logic
tests on machines without a GPU.  They are vectorised over batch and views (no Python loops over
B*V like the reference) and are NOT the product inference path: the native backend never routes
through this file.
"""
import torch
import torch.nn.functional as F


def sample_views(heatmaps, proj_matricies, coord_volumes):
    """Per-view bilinear samples of every voxel, (B, V, C, nvox), invalid-depth voxels zeroed (op.py:113-147)."""
    B, V, C, h, w = heatmaps.shape
    pts = coord_volumes.reshape(B, 1, -1, 3)
    ones = torch.ones_like(pts[..., :1])
    proj = torch.cat([pts, ones], dim=-1) @ proj_matricies.transpose(-1, -2)       # (B, V, N, 3)
    z = proj[..., 2]
    invalid = z <= 0.0
    z = torch.where(z == 0.0, torch.ones_like(z), z)
    xy = proj[..., :2] / z.unsqueeze(-1)
    # reference quirk (op.py:128-129): x is normalised by the map height, y by the width
    gx = 2 * (xy[..., 0] / h - 0.5)
    gy = 2 * (xy[..., 1] / w - 0.5)
    grid = torch.stack([gx, gy], dim=-1).reshape(B * V, -1, 1, 2)
    sampled = F.grid_sample(heatmaps.reshape(B * V, C, h, w), grid, align_corners=True)   # (BV, C, N, 1)
    sampled = sampled.reshape(B, V, C, -1)
    return sampled.masked_fill(invalid.unsqueeze(2), 0.0)


def partial_aggregate(sampled, volume_aggregation_method, vol_confidences=None):
    """This rank's share of the view aggregation, (B, P, C, nvox): softmax -> (sum s e^s, sum e^s) [unshifted]."""
    if volume_aggregation_method == "softmax":
        e = torch.exp(sampled)
        return torch.stack([(sampled * e).sum(1), e.sum(1)], dim=1)
    if volume_aggregation_method == "max":
        return sampled.max(1)[0].unsqueeze(1)
    if volume_aggregation_method.startswith("conf"):
        B, V, C = sampled.shape[:3]
        return (sampled * vol_confidences.reshape(B, V, C, 1)).sum(1).unsqueeze(1)
    return sampled.sum(1).unsqueeze(1)


def finalize_aggregate(partial, volume_aggregation_method):
    return partial[:, 0] / partial[:, 1] if volume_aggregation_method == "softmax" else partial[:, 0]


def unproject_heatmaps(heatmaps, proj_matricies, coord_volumes, volume_aggregation_method="sum", vol_confidences=None):
    """Same contract as reference op.py:99-166, batched."""
    B, V, C, h, w = heatmaps.shape
    vol_shape = coord_volumes.shape[1:4]
    sampled = sample_views(heatmaps, proj_matricies, coord_volumes)
    if volume_aggregation_method.startswith("conf"):
        out = (sampled * vol_confidences.reshape(B, V, C, 1)).sum(1)
    elif volume_aggregation_method == "sum":
        out = sampled.sum(1)
    elif volume_aggregation_method == "max":
        out = sampled.max(1)[0]
    elif volume_aggregation_method == "softmax":
        out = (sampled * torch.softmax(sampled, dim=1)).sum(1)
    else:
        raise ValueError("Unknown volume_aggregation_method: {}".format(volume_aggregation_method))
    return out.reshape(B, C, *vol_shape)


def integrate_tensor_3d_with_coordinates(volumes, coord_volumes, softmax=True):
    """Same contract as reference op.py:84-96."""
    B, J = volumes.shape[:2]
    flat = volumes.reshape(B, J, -1)
    flat = torch.softmax(flat, dim=2) if softmax else F.relu(flat)
    coords = flat @ coord_volumes.reshape(B, -1, 3)
    return coords, flat.reshape(volumes.shape)


def integrate_tensor_2d(heatmaps, softmax=True):
    """Same contract as reference op.py:11-47."""
    B, J, h, w = heatmaps.shape
    flat = heatmaps.reshape(B, J, -1)
    flat = torch.softmax(flat, dim=2) if softmax else F.relu(flat)
    hm = flat.reshape(B, J, h, w)
    mass_x, mass_y = hm.sum(dim=2), hm.sum(dim=3)
    x = (mass_x * torch.arange(w, device=hm.device, dtype=hm.dtype)).sum(dim=2, keepdim=True)
    y = (mass_y * torch.arange(h, device=hm.device, dtype=hm.dtype)).sum(dim=2, keepdim=True)
    if not softmax:
        x = x / mass_x.sum(dim=2, keepdim=True)
        y = y / mass_y.sum(dim=2, keepdim=True)
    return torch.cat((x, y), dim=2), hm


def volumetric_ce_index(coord_volumes, keypoints_gt):
    """(B, J) flat index of the voxel nearest to each ground-truth point: the distances and torch.argmin of loss.py:68-71, for all
    samples at once and without copying the indices to the host."""
    B = coord_volumes.shape[0]
    dists = torch.sqrt(((coord_volumes.reshape(B, 1, -1, 3) - keypoints_gt.unsqueeze(2)) ** 2).sum(-1))   # (B, J, nvox)
    return torch.argmin(dists, dim=-1)


def volumetric_ce_loss(coord_volumes_batch, volumes_batch_pred, keypoints_gt, keypoints_binary_validity):
    """Same contract as reference loss.py:52-80 (VolumetricCELoss.forward), vectorised: one argmin over (B, J, nvox), one gather,
    one sum; no host synchronisation."""
    B, J = volumes_batch_pred.shape[:2]
    index = volumetric_ce_index(coord_volumes_batch.detach(), keypoints_gt.detach())
    p = volumes_batch_pred.reshape(B, J, -1).gather(2, index.unsqueeze(-1)).squeeze(-1)
    terms = keypoints_binary_validity[..., 0] * (-torch.log(p + 1e-6))
    return terms.sum() / (B * J)


def triangulate_batch_of_points(proj_matricies_batch, points_batch, confidences_batch=None):
    """Weighted DLT, batched (reference multiview.py:141-183 loops over samples and joints and calls torch.svd each time)."""
    B, V, J = points_batch.shape[:3]
    if confidences_batch is None:
        confidences_batch = torch.ones(B, V, J, dtype=points_batch.dtype, device=points_batch.device)
    P = proj_matricies_batch.unsqueeze(2)                                     # (B, V, 1, 3, 4)
    A = P[..., 2:3, :] * points_batch.unsqueeze(-1) - P[..., :2, :]          # (B, V, J, 2, 4)
    A = A * confidences_batch.unsqueeze(-1).unsqueeze(-1)
    A = A.permute(0, 2, 1, 3, 4).reshape(B, J, 2 * V, 4)
    _, _, vh = torch.linalg.svd(A.double(), full_matrices=False)
    X = vh[..., 3, :]
    return (X[..., :3] / X[..., 3:4]).to(points_batch.dtype)


def keypoints_loss(pred, gt, validity, kind, threshold=400.0):
    """The keypoint criteria of the reference (loss.py:7-49) with the divisor max(1, sum v) kept on the device: no host
    synchronisation.  pred, gt (B, J, dim), validity (B, J, 1); `kind` is one of "mse", "mse_smooth", "mae", "l2".  MSESmooth's
    replaced branch is a torch.where whose untaken pow sees 1, so its gradient is the reference's index_put gradient."""
    r = gt - pred
    divisor = torch.clamp(validity.sum(), min=1)
    if kind == "l2":
        return torch.sqrt((r ** 2 * validity).sum(dim=2)).sum() / divisor
    if kind == "mae":
        terms = torch.abs(r) * validity
    else:
        terms = r ** 2 * validity
        if kind == "mse_smooth":
            over = terms > threshold
            terms = torch.where(over, torch.where(over, terms, torch.ones_like(terms)) ** 0.1 * threshold ** 0.9, terms)
        elif kind != "mse":
            raise ValueError("unknown keypoints loss kind {!r}".format(kind))
    return terms.sum() / (pred.shape[-1] * divisor)
