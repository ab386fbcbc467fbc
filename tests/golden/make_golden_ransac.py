"""Generate tests/golden/ransac.npz from the UNMODIFIED reference's RANSACTriangulationNet (mvn/models/triangulation.py:17-128).

Needs a checkout of the reference (karfly/learnable-triangulation-pytorch); the tests only read the stored fixture:
    LT_REFERENCE=<path to the reference checkout> python tests/golden/make_golden_ransac.py
The reference samples a `set` with random.sample (triangulation.py:85), which Python >= 3.11 refuses.  This script wraps
random.sample so that a set is passed as sorted(set), which is what Python <= 3.10 did with the reference's set of small ints; the
wrapper lives here only.  It also logs the drawn pairs and the inlier lists triangulate_ransac returns.  Nothing is copied from the
reference.
"""
import math
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ["LT_REFERENCE"])

from lt_b200 import testing  # noqa: E402
from lt_b200.triangulation import RANSACTriangulationNet  # noqa: E402
from mvn.models.triangulation import RANSACTriangulationNet as RefNet  # noqa: E402

_sample = random.sample
DRAWN = []


def _sample_py310(population, k, **kw):
    """random.sample as Python <= 3.10 ran it on a set (tuple of the set; sorted for small ints), logging what it drew."""
    if isinstance(population, (set, frozenset)):
        population = sorted(population)
    out = _sample(population, k, **kw)
    DRAWN.append(sorted(out))
    return out


random.sample = _sample_py310

N_ITERS = 10
SEED = 1234


def cameras(V, narrow=False, image_size=384):
    """(V, 3, 4) float32: make_cameras' ring, or V cameras 1 degree apart on it (narrow baseline)."""
    cams = ([testing.make_cameras(1, image_size=image_size, phase=0.3 + math.radians(1.0) * v)[0] for v in range(V)] if narrow
            else testing.make_cameras(V, image_size=image_size))
    return np.stack([c.projection for c in cams]).astype(np.float32)


def project(P, X):
    uvw = np.append(X, 1.0) @ P.astype(np.float64).T
    return uvw[:2] / uvw[2]


def scene(V, J, outliers, narrow=False, seed=0):
    """proj (1, V, 3, 4) float32, int64 points (1, V, J, 2): points ~ N(0, 300^2) + (0, 0, 900) mm, 2 px noise, truncated; views
    V-1, V-2, ... of `outliers` moved 60-200 px away in every joint."""
    rng = np.random.RandomState(seed)
    P = cameras(V, narrow)
    kp = np.zeros((1, V, J, 2), np.int64)
    for j in range(J):
        X = rng.randn(3) * 300 + [0, 0, 900]
        for v in range(V):
            p = project(P[v], X) + rng.randn(2) * 2
            if v >= V - outliers:
                p += rng.uniform(60, 200, 2) * rng.choice([-1, 1], 2)
            kp[0, v, j] = np.trunc(p)
    return P[None], kp


def boundary_scene(J=6, seed=7):
    """V = 3, one projection matrix per joint: view 2's error against the DLT of views (0, 1) is 15 +- 1e-3 px (alternating), set
    through its u translation P[2][0, 3] and checked after the float32 rounding."""
    rng = np.random.RandomState(seed)
    P0 = cameras(3)
    Ps, kps = [], []
    for j in range(J):
        X = rng.randn(3) * 300 + [0, 0, 900]
        P = P0.copy()
        kp = np.stack([np.trunc(project(P[v], X) + rng.randn(2) * 2) for v in range(3)]).astype(np.int64)
        Xd = RefDLT(P[:2], kp[:2])
        kp[2] = np.round(project(P[2], Xd)) + [30, 0]
        target = 15.0 + (1e-3 if j % 2 == 0 else -1e-3)
        e = kp[2] - project(P[2], Xd)
        delta = e[0] - math.sqrt(4 * target ** 2 - e[1] ** 2)       # shift of pi_x that puts 0.5 |e| at target
        w = float(np.append(Xd, 1.0) @ P[2, 2].astype(np.float64))
        P[2, 0, 3] = np.float32(float(P[2, 0, 3]) + delta * w)
        err = 0.5 * np.linalg.norm(kp[2] - project(P[2], RefDLT(P[:2], kp[:2])))
        assert 0.5e-3 < abs(err - 15.0) < 1.5e-3, err
        Ps.append(P)
        kps.append(kp)
    # one sample per joint: (J, 3, 3, 4) projections, (J, 3, 1, 2) points
    return np.stack(Ps), np.stack(kps)[:, :, None]


def RefDLT(P, kp):
    from mvn.utils import multiview
    return multiview.triangulate_point_from_multiple_views_linear(P, kp)


def run_reference(tag, proj, kp, out):
    """triangulate_ransac of the reference on every (sample, joint), with and without direct_optimization, from the same seed."""
    B, V, J = kp.shape[:3]
    res = {}
    for direct in (False, True):
        random.seed(SEED)
        del DRAWN[:]
        pts, inl = np.zeros((B, J, 3)), np.zeros((B, J), np.int64)
        for b in range(B):
            for j in range(J):
                X, inliers = RefNet.triangulate_ransac(None, proj[b], kp[b, :, j], n_iters=N_ITERS, direct_optimization=direct)
                pts[b, j] = X
                inl[b, j] = sum(1 << int(v) for v in inliers)
        res[direct] = (pts, inl, np.array(DRAWN, np.int32).reshape(B, J, N_ITERS, 2))
    assert np.array_equal(res[False][2], res[True][2]) and np.array_equal(res[False][1], res[True][1])
    out[tag + "_proj"], out[tag + "_kp"], out[tag + "_pairs"], out[tag + "_inliers"] = proj, kp, res[True][2], res[True][1]
    out[tag + "_dlt"], out[tag + "_refined"] = res[False][0], res[True][0]
    print("%s: V=%d, inlier counts %s" % (tag, V, sorted({bin(int(m)).count("1") for m in res[True][1].ravel()})))


def gen_scenes(out):
    for tag, args in {"ring2": (2, 8, 0), "ring3_two_inliers": (3, 8, 1), "ring4": (4, 8, 0), "ring4_out1": (4, 8, 1),
                      "ring4_out2": (4, 8, 2), "ring8_out2": (8, 6, 2), "ring31_out2": (31, 4, 2)}.items():
        run_reference(tag, *scene(*args, seed=len(tag)), out)
    for tag, args in {"narrow4": (4, 8, 0), "narrow4_out1": (4, 8, 1)}.items():
        run_reference(tag, *scene(*args, narrow=True, seed=len(tag)), out)
    run_reference("boundary", *boundary_scene(), out)


def gen_model(out):
    """One RANSACTriangulationNet.forward of the reference: ResNet-18, B = 2, V = 4, 48 x 80 images (maps 16 x 24: W / w = 10 / 3),
    seeded weights, with and without direct_optimization; the pairs it drew, the inlier lists and random's state afterwards."""
    B, V, H, W = 2, 4, 48, 80
    holder = RANSACTriangulationNet(testing.make_ransac_config(num_layers=18), device="cpu", backend="torch")
    testing.randomize_ransac_weights(holder, seed=11, calib_size=64)
    g = torch.Generator().manual_seed(12)
    images = torch.randn(B, V, 3, H, W, generator=g)
    proj = torch.from_numpy(np.stack([cameras(V, image_size=W)] * B))
    out["model_proj"] = proj.numpy()          # the images are regenerated from the seed (torch.randn, generator seed 12)
    out["model_state_dict_keys"] = np.array(sorted(holder.state_dict().keys()))
    for direct in (False, True):
        ref = RefNet(testing.make_ransac_config(num_layers=18, direct_optimization=direct), device="cpu")
        ref.load_state_dict(holder.state_dict(), strict=True)
        ref.eval()
        inliers = []
        orig = ref.triangulate_ransac

        def logged(*a, **kw):
            X, inl = orig(*a, **kw)
            inliers.append(sum(1 << int(v) for v in inl))
            return X, inl

        ref.triangulate_ransac = logged
        random.seed(SEED)
        del DRAWN[:]
        with torch.no_grad():
            kp3d, kp2d, heat, conf = ref(images, proj, None)
        tag = "model_direct" if direct else "model_dlt"
        out[tag + "_keypoints_3d"], out[tag + "_inliers"] = kp3d.numpy(), np.array(inliers, np.int64).reshape(B, 17)
        out[tag + "_pairs"] = np.array(DRAWN, np.int32).reshape(B, 17, N_ITERS, 2)
        out[tag + "_random_state"] = np.array(random.getstate()[1], np.int64)
        if not direct:
            out["model_keypoints_2d"], out["model_heatmaps"] = kp2d.numpy(), heat.numpy()
            assert kp2d.dtype == torch.int64 and not conf.any()
        else:
            assert np.array_equal(kp2d.numpy(), out["model_keypoints_2d"]) and np.array_equal(heat.numpy(), out["model_heatmaps"])
        print("%s: keypoints_3d[0, :2] %s, inlier counts %s" % (tag, kp3d[0, :2].numpy(), sorted({bin(m).count("1") for m in inliers})))
    out["model_seed"] = np.array([SEED])


if __name__ == "__main__":
    out = {"n_iters": np.array([N_ITERS]), "seed": np.array([SEED])}
    gen_scenes(out)
    gen_model(out)
    path = os.path.join(HERE, "ransac.npz")
    np.savez_compressed(path, **out)
    print("ransac.npz", os.path.getsize(path))
