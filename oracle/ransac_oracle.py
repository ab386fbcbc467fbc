"""CPU oracle of the RANSAC triangulation baseline: a restatement of the reference's RANSACTriangulationNet
(mvn/models/triangulation.py:17-128) in numpy / scipy, with the view pairs as an input instead of Python's `random`.

The pairs are what `sorted(random.sample(view_set, 2))` draws (triangulation.py:85); lt_b200.triangulation.draw_view_pairs draws
them in the reference's order.  Besides the reference's results this reports what the tests need: the refined point at tight
tolerances (the minimiser itself, not scipy's default stopping point) and each view's inlier margin |err - eps| per draw.
"""
import numpy as np
import torch
from scipy.optimize import least_squares, minimize

from . import vol_oracle

TIGHT = dict(xtol=1e-15, ftol=1e-15, gtol=1e-15)


def dlt(proj, points):
    """multiview.py:113-138: rows x P[2] - P[0], y P[2] - P[1] (numpy promotes int64 points and float32 matrices to float64), the
    right singular vector of the smallest singular value, dehomogenised."""
    proj, points = np.asarray(proj), np.asarray(points)
    A = np.zeros((2 * len(proj), 4))
    for j in range(len(proj)):
        A[j * 2 + 0] = points[j][0] * proj[j][2, :] - proj[j][0, :]
        A[j * 2 + 1] = points[j][1] * proj[j][2, :] - proj[j][1, :]
    _, _, vh = np.linalg.svd(A, full_matrices=False)
    X = vh[3, :]
    return X[:3] / X[3]


def reprojection_errors(X, points, proj):
    """multiview.py:186-193 for one point: 0.5 |p_v - pi_v(X)| per view (float64)."""
    Xh = np.append(np.asarray(X, dtype=np.float64), 1.0)
    err = []
    for p, P in zip(points, proj):
        uvw = Xh @ np.asarray(P).T
        err.append(0.5 * np.sqrt(np.sum((p - uvw[:2] / uvw[2]) ** 2)))
    return np.array(err)


def huber_cost(X, points, proj):
    """The cost least_squares(loss='huber') minimises: 1/2 sum rho(f^2), rho(z) = z (z <= 1), 2 sqrt(z) - 1 above."""
    z = reprojection_errors(X, points, proj) ** 2
    return 0.5 * float(np.sum(np.where(z <= 1, z, 2 * np.sqrt(z) - 1)))


def refine(X0, points, proj, tight=False):
    """triangulation.py:114-126: least_squares(loss='huber', method='trf') of the inliers' reprojection errors from X0, at scipy's
    default tolerances; or the minimiser itself (tight=True): least_squares at TIGHT tolerances, then polished by a derivative-free
    Nelder-Mead on huber_cost, since scipy's finite-difference Jacobian of the error norms is rank-deficient and can stall short of
    the minimum when a view lies far out in the Huber branch."""
    res = least_squares(lambda x: reprojection_errors(x, points, proj), np.array(X0), loss="huber", method="trf",
                        **(TIGHT if tight else {}))
    if not tight:
        return res.x
    pol = minimize(huber_cost, res.x, args=(points, proj), method="Nelder-Mead",
                   options=dict(xatol=1e-9, fatol=1e-15, maxiter=20000, maxfev=40000))
    return pol.x if pol.fun < huber_cost(res.x, points, proj) else res.x


def triangulate_ransac(proj, points, pairs, reprojection_error_epsilon=15, direct_optimization=True, tight=True):
    """triangulation.py:72-128 with the drawn pairs (n_iters, 2) given.  -> dict: dlt (the inlier DLT), refined (scipy default;
    None without direct_optimization), tight (TIGHT tolerances; None without direct_optimization), inliers (sorted list), margins
    (n_iters, V) of |err - eps|.  tight=False skips the tight solve (only what the reference computes)."""
    proj, points = np.asarray(proj), np.asarray(points)
    assert len(proj) == len(points) and len(points) >= 2                       # :73-74
    view_set = set(range(len(points)))
    inlier_set = set()
    margins = []
    for sampled in pairs:                                                       # :84-97
        sampled = sorted(int(v) for v in sampled)
        X = dlt(proj[sampled], points[sampled])
        err = reprojection_errors(X, points, proj)
        margins.append(np.abs(err - reprojection_error_epsilon))
        new_inlier_set = set(sampled)
        for view in view_set:
            if err[view] < reprojection_error_epsilon:
                new_inlier_set.add(view)
        if len(new_inlier_set) > len(inlier_set):
            inlier_set = new_inlier_set
    if len(inlier_set) == 0:                                                    # :100-101
        inlier_set = view_set.copy()
    inliers = sorted(inlier_set)
    X = dlt(proj[inliers], points[inliers])                                     # :103-107
    out = dict(dlt=X, refined=None, tight=None, inliers=inliers, margins=np.array(margins).reshape(len(pairs), len(points)))
    if direct_optimization:
        out["refined"] = refine(X, points[inliers], proj[inliers])
        if tight:
            out["tight"] = refine(X, points[inliers], proj[inliers], tight=True)
    return out


def triangulate_batch(proj, keypoints_2d, pairs, reprojection_error_epsilon=15, direct_optimization=True, tight=True):
    """The per-(sample, joint) loop of triangulation.py:58-65: proj (B, V, 3, 4) float32, keypoints_2d (B, V, J, 2) int64, pairs
    (B, J, n_iters, 2) -> dict of (B, J, 3) float64 arrays dlt / refined / tight, inliers [B][J] lists, margins (B, J, n_iters, V)."""
    B, V, J = np.asarray(keypoints_2d).shape[:3]
    items = [[triangulate_ransac(proj[b], keypoints_2d[b, :, j], pairs[b, j], reprojection_error_epsilon, direct_optimization, tight)
              for j in range(J)] for b in range(B)]
    out = {"inliers": [[it["inliers"] for it in row] for row in items],
           "margins": np.array([[it["margins"] for it in row] for row in items])}
    for key in ("dlt", "refined", "tight"):
        out[key] = None if items[0][0][key] is None else np.array([[it[key] for it in row] for row in items])
    return out


def keypoints_2d_from_heatmaps(heatmaps, image_shape):
    """triangulation.py:44-52: the first maximal index per map (torch.max; a NaN counts as the maximum), x = idx % w, y = idx // w,
    scaled by the float32 image / map ratio and truncated into int64.  heatmaps (B, V, J, h, w) -> (B, V, J, 2) int64."""
    hm = torch.as_tensor(np.asarray(heatmaps))
    B, V, J, h, w = hm.shape
    _, idx = torch.max(hm.reshape(B, V, J, -1), dim=-1)
    kp = torch.stack([idx % w, idx // w], dim=-1)
    out = torch.zeros_like(kp)
    out[..., 0] = kp[..., 0] * (image_shape[1] / w)
    out[..., 1] = kp[..., 1] * (image_shape[0] / h)
    return out.numpy()


@torch.no_grad()
def ransac_forward(sd, images, proj, pairs, direct_optimization=True, reprojection_error_epsilon=15, style="simple"):
    """Eval-mode RANSACTriangulationNet.forward (triangulation.py:27-70) on the CPU with the drawn pairs given.
    -> heatmaps (B, V, J, h, w) float32, keypoints_2d (B, V, J, 2) int64, and triangulate_batch's dict."""
    sd = vol_oracle._sub({k: v.detach().float().cpu() for k, v in sd.items()}, "backbone.")
    images = images.detach().float().cpu()
    B, V = images.shape[:2]
    H, W = images.shape[3:]
    heat, _ = vol_oracle.pose_resnet_forward(sd, images.reshape(B * V, 3, H, W), style)
    heat = heat.reshape(B, V, *heat.shape[1:]).numpy()
    kp2d = keypoints_2d_from_heatmaps(heat, (H, W))
    return heat, kp2d, triangulate_batch(np.asarray(proj, dtype=np.float32), kp2d, pairs, reprojection_error_epsilon,
                                         direct_optimization)
