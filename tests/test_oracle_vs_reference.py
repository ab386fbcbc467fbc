"""Oracle and host mirror vs the reference itself: the reference's outputs on these seeded inputs are stored in
tests/golden/reference_pins.npz (tests/golden/make_golden.py); large outputs are pinned on a fixed, seeded sample."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err
from oracle import vol_oracle as O
from lt_b200 import pose_resnet, testing, torch_ops, v2v

UNPROJECT_SHAPES = [(1, 2, 3, 9, 13, 5), (2, 8, 4, 12, 12, 6), (1, 9, 2, 8, 6, 4)]


@pytest.fixture(scope="module")
def pins():
    return np.load(os.path.join(GOLDEN, "reference_pins.npz"))


def unproject_inputs(shape):
    B, V, C, h, w, n = shape
    rng = np.random.RandomState(B * 100 + V)
    heat = rng.randn(B, V, C, h, w).astype(np.float32)
    cams = testing.make_cameras(V, image_size=48, radius=3000.0)
    proj = np.stack([np.stack([O.projection_after_resize(c.K, c.R, c.t, (48, 48), (h, w)) for c in cams])] * B)
    coord = np.stack([O.coord_volume(rng.randn(3) * 100 + [0, 0, 900], 2600.0, n) for _ in range(B)])
    conf = rng.rand(B, V, C).astype(np.float32)
    return heat, proj, coord, conf


def v2v_and_backbone_inputs(v2v_cls=v2v.V2VModel, get_pose_net=pose_resnet.get_pose_net):
    """Seeded V2V (BN statistics randomised) + input, then a ResNet-34 backbone + input, drawn in this order."""
    torch.manual_seed(0)
    v = v2v_cls(32, 17).eval()
    for m in v.modules():
        if isinstance(m, torch.nn.BatchNorm3d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    x = torch.randn(1, 32, 32, 32, 32)
    cfg = testing.AttrDict(num_layers=34, style="simple", num_joints=17, alg_confidences=False, vol_confidences=False,
                           init_weights=False)
    bb = get_pose_net(cfg, device="cpu").eval()
    xi = torch.randn(2, 3, 64, 64)
    return v, x, bb, xi


def _pinned(pins, name, got):
    idx, want = pins[name + "_idx"], pins[name + "_val"]
    return rel_err(np.asarray(got).ravel()[idx], want)


@pytest.mark.parametrize("shape", UNPROJECT_SHAPES)
@pytest.mark.parametrize("agg", ["sum", "max", "softmax", "conf"])
def test_unproject_random(pins, shape, agg):
    heat, proj, coord, conf = unproject_inputs(shape)
    want = pins["unproject_%d_%s" % (UNPROJECT_SHAPES.index(shape), agg)]
    assert rel_err(O.unproject_heatmaps(heat, proj, coord, agg, conf), want) < 2e-5
    got_t = torch_ops.unproject_heatmaps(torch.from_numpy(heat), torch.from_numpy(proj), torch.from_numpy(coord), agg,
                                         torch.from_numpy(conf)).numpy()
    assert rel_err(got_t, want) < 2e-5


def test_coord_volume_and_projection_bit_exact(pins):
    base = np.array([123.4, -56.7, 910.1])
    mine = O.coord_volume(base, 2500.0, 32)
    assert mine.shape == (32, 32, 32, 3)
    assert np.array_equal(mine.ravel()[pins["coord_idx"]], pins["coord_val"])
    images, batch = testing.make_batch(1, 2, image_size=64, seed=5)
    cam = batch["cameras"][1][0]
    assert np.array_equal(O.projection_after_resize(cam.K, cam.R, cam.t, (64, 64), (16, 16)), pins["projection"])


def test_v2v_and_backbone_functional_restatement(pins):
    v, x, bb, xi = v2v_and_backbone_inputs()
    assert _pinned(pins, "v2v", O.v2v_forward(v.state_dict(), x)) < 1e-5
    ohm, ofe = O.pose_resnet_forward(bb.state_dict(), xi)
    assert _pinned(pins, "feats", ofe) < 1e-5 and _pinned(pins, "heat", ohm) < 1e-5
