"""Pinhole cameras and projective helpers (host side, float64 numpy).

Mirror of the part of `/root/reference/mvn/utils/multiview.py` the volumetric path
touches: `Camera` (:5-52), homogeneous helpers (:55-86), point projection (:89-110).
`stack_projections` is the vectorised replacement of the per-camera deepcopy +
`update_after_resize` + `.projection` loop in `triangulation.py:272-278`.
"""
import numpy as np
import torch


class Camera:
    """K, R, t pinhole camera; same attributes/methods as the reference class."""

    def __init__(self, R, t, K, dist=None, name=""):
        self.R = np.array(R).copy()
        assert self.R.shape == (3, 3)
        self.t = np.array(t).copy()
        assert self.t.size == 3
        self.t = self.t.reshape(3, 1)
        self.K = np.array(K).copy()
        assert self.K.shape == (3, 3)
        self.dist = None if dist is None else np.array(dist).copy().flatten()
        self.name = name

    def update_after_crop(self, bbox):
        left, upper, _, _ = bbox
        self.K[0, 2] -= left
        self.K[1, 2] -= upper

    def update_after_resize(self, image_shape, new_image_shape):
        (h, w), (nh, nw) = image_shape, new_image_shape
        self.K[0, 0], self.K[0, 2] = self.K[0, 0] * (nw / w), self.K[0, 2] * (nw / w)
        self.K[1, 1], self.K[1, 2] = self.K[1, 1] * (nh / h), self.K[1, 2] * (nh / h)

    @property
    def extrinsics(self):
        return np.hstack([self.R, self.t])

    @property
    def projection(self):
        return self.K.dot(self.extrinsics)


def stack_projections(cameras, image_shape=None, new_image_shape=None):
    """cameras[v][b] (the collate layout, datasets/utils.py:26) -> float32 (B, V, 3, 4) array of K'[R|t].

    If shapes are given, the intrinsics are rescaled image->heatmap exactly like
    `Camera.update_after_resize` (multiview.py:33-44) *without* touching the caller's
    objects (the reference deep-copies them, triangulation.py:272).  All arithmetic is
    float64, cast to float32 last, as in the reference.
    """
    n_views, batch = len(cameras), len(cameras[0])
    K = np.empty((batch, n_views, 3, 3), dtype=np.float64)
    E = np.empty((batch, n_views, 3, 4), dtype=np.float64)
    for v in range(n_views):
        for b in range(batch):
            cam = cameras[v][b]
            K[b, v] = cam.K
            E[b, v, :, :3] = cam.R
            E[b, v, :, 3] = np.asarray(cam.t).reshape(3)
    if image_shape is not None:
        (h, w), (nh, nw) = image_shape, new_image_shape
        K[..., 0, 0] = K[..., 0, 0] * (nw / w)
        K[..., 1, 1] = K[..., 1, 1] * (nh / h)
        K[..., 0, 2] = K[..., 0, 2] * (nw / w)
        K[..., 1, 2] = K[..., 1, 2] * (nh / h)
    return np.matmul(K, E).astype(np.float32)


def euclidean_to_homogeneous(points):
    if isinstance(points, np.ndarray):
        return np.hstack([points, np.ones((len(points), 1))])
    if torch.is_tensor(points):
        return torch.cat([points, points.new_ones((points.shape[0], 1))], dim=1)
    raise TypeError("Works only with numpy arrays and PyTorch tensors.")


def homogeneous_to_euclidean(points):
    if isinstance(points, np.ndarray):
        return (points.T[:-1] / points.T[-1]).T
    if torch.is_tensor(points):
        return (points.transpose(1, 0)[:-1] / points.transpose(1, 0)[-1]).transpose(1, 0)
    raise TypeError("Works only with numpy arrays and PyTorch tensors.")


def project_3d_points_to_image_plane_without_distortion(proj_matrix, points_3d, convert_back_to_euclidean=True):
    if isinstance(proj_matrix, np.ndarray) and isinstance(points_3d, np.ndarray):
        result = euclidean_to_homogeneous(points_3d) @ proj_matrix.T
    elif torch.is_tensor(proj_matrix) and torch.is_tensor(points_3d):
        result = euclidean_to_homogeneous(points_3d) @ proj_matrix.t()
    else:
        raise TypeError("Works only with numpy arrays and PyTorch tensors.")
    return homogeneous_to_euclidean(result) if convert_back_to_euclidean else result


def triangulate_batch_of_points(proj_matricies_batch, points_batch, confidences_batch=None, backend=None):
    """Drop-in for reference multiview.py:171-183: (B, V, 3, 4), (B, V, J, 2), (B, V, J) -> (B, J, 3)."""
    from . import autograd_ops, capi, op as _op, torch_ops
    which = _op._resolve_backend(backend, proj_matricies_batch, points_batch, confidences_batch)
    if which == "torch":
        return torch_ops.triangulate_batch_of_points(proj_matricies_batch, points_batch, confidences_batch)
    if which == "hybrid":
        # native forward and backward kernels in the autograd graph (gradients to the points and the confidences)
        return autograd_ops.triangulate_batch_of_points(proj_matricies_batch, points_batch, confidences_batch)
    B, V, J = points_batch.shape[:3]
    out = torch.empty((B, J, 3), dtype=torch.float32, device=points_batch.device)
    conf = None if confidences_batch is None else confidences_batch.float().contiguous()
    capi.triangulate_dlt(proj_matricies_batch.float().contiguous(), points_batch.float().contiguous(), conf, out)
    return out
