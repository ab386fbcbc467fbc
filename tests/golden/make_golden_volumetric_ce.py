"""Generate tests/golden/volumetric_ce.npz from the UNMODIFIED reference's VolumetricCELoss (mvn/models/loss.py:52-80).

Needs a checkout of the reference (karfly/learnable-triangulation-pytorch); the tests only read the stored fixture:
    LT_REFERENCE=<path to the reference checkout> python tests/golden/make_golden_volumetric_ce.py
It imports the reference read-only, feeds it seeded synthetic inputs and stores the inputs and outputs as .npz.  Nothing is
copied from the reference.  The other fixtures in this directory come from make_golden.py.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.environ["LT_REFERENCE"])

from mvn.models.loss import VolumetricCELoss as RefCE  # noqa: E402


def _rotation(axis, theta):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(theta) * K + (1 - np.cos(theta)) * K @ K


def gen_volumetric_ce():
    """VolumetricCELoss of the reference, with its gradient w.r.t. the volumes, B = 2, J = 17, 12^3:
    case "rot": a rotated cuboid, joints 0-1 of each sample far outside it (the nearest voxel lies on the boundary);
    case "view": the same coordinates seen through a permuted and flipped view (coord.transpose(0, 1, 3, 2, 4)[:, ::-1], the
      transfer_cmu_to_human36m shape of triangulation.py:336-339), made contiguous;
    case "lattice": an axis-aligned grid with integer coordinates (exactly representable), joint 3 of sample 0 exactly midway
      between two neighbouring voxels (a tie: the lower flat index wins) and a NaN ground-truth point at (1, 5) (every distance
      NaN: index 0).  Validity is 0 for joint 7 of sample 0 in all cases.
    Stored per case: coord, keypoints, the reference's argmin index (from the nonzero pattern of its gradient and the same
    distances), its loss and its gradient at the picked voxels (zero elsewhere, checked here)."""
    rng = np.random.RandomState(2024)
    B, J, n = 2, 17, 12
    vols = torch.softmax(torch.from_numpy((rng.randn(B, J, n ** 3) * 2).astype(np.float32)), -1).reshape(B, J, n, n, n)
    validity = np.ones((B, J, 1), dtype=np.float32)
    validity[0, 7] = 0.0
    idx = np.arange(n, dtype=np.float64)
    g = np.stack(np.meshgrid(idx, idx, idx, indexing="ij"), -1)
    base = np.array([[120.0, -340.0, 910.0], [-75.0, 260.0, 880.0]])
    rot = np.stack([(g * (2500.0 / (n - 1)) - 1250.0) @ _rotation([1, 2, 3], 0.4 + b).T + base[b] for b in range(B)]).astype(np.float32)
    kp = (base[:, None] + rng.uniform(-1100, 1100, size=(B, J, 3))).astype(np.float32)
    kp[:, 0] = base + [4000.0, 0.0, 0.0]
    kp[:, 1] = base + [-2500.0, 3000.0, -1800.0]
    lattice = (g * 100.0 + [-600.0, -500.0, 300.0]).astype(np.float32)[None].repeat(B, 0)
    kp_l = (lattice[:, 0, 0, 0][:, None] + rng.randint(0, n - 1, size=(B, J, 3)) * 100.0 + 37.0).astype(np.float32)
    kp_l[0, 3] = lattice[0, 4, 6, 2] + [50.0, 0.0, 0.0]           # midway between voxels (4, 6, 2) and (5, 6, 2)
    kp_l[1, 5] = np.nan
    cases = {"rot": (rot, kp), "view": (np.ascontiguousarray(rot.transpose(0, 1, 3, 2, 4)[:, ::-1]), kp), "lattice": (lattice, kp_l)}
    out = {"volumes": vols.numpy(), "validity": validity}
    for tag, (coord, k) in cases.items():
        v = vols.clone().requires_grad_(True)
        loss = RefCE()(torch.from_numpy(coord), v, torch.from_numpy(k), torch.from_numpy(validity))
        loss.backward()
        grad = v.grad.reshape(B, J, -1)
        ct, kt = torch.from_numpy(coord), torch.from_numpy(k)
        index = np.stack([torch.argmin(torch.sqrt(((ct[b].unsqueeze(0) - kt[b].reshape(J, 1, 1, 1, 3)) ** 2).sum(-1)).reshape(J, -1),
                                       dim=-1).numpy() for b in range(B)])
        nz = grad.numpy() != 0
        assert nz.sum() == (validity[..., 0] != 0).sum()
        for b in range(B):
            for j in range(J):
                assert (np.flatnonzero(nz[b, j]) == ([index[b, j]] if validity[b, j, 0] else [])).all()
        out[tag + "_coord"], out[tag + "_keypoints"] = coord, k
        out[tag + "_index"] = index
        out[tag + "_loss"] = np.array([loss.item()], dtype=np.float32)
        out[tag + "_grad_at_index"] = np.take_along_axis(grad.numpy(), index[..., None], 2)[..., 0]
        print("volumetric_ce[%s]: loss %.6f, index %s" % (tag, loss.item(), index[0, :6]))
    assert out["lattice_index"][0, 3] == (4 * n + 6) * n + 2 and out["lattice_index"][1, 5] == 0
    np.savez_compressed(os.path.join(HERE, "volumetric_ce.npz"), **out)


if __name__ == "__main__":
    gen_volumetric_ce()
    print("volumetric_ce.npz", os.path.getsize(os.path.join(HERE, "volumetric_ce.npz")))
