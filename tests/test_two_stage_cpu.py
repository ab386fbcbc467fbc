"""TwoStageTriangulationNet without a GPU: the constructor's checks, the forward's refusals, stale-graph invalidation and the lazy
cuboids against the ones the volumetric model builds on the host from the same key points."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import capi, testing
from lt_b200.triangulation import LazyCuboids


def _models(kind="mpii", num_joints=17, use_gt_pelvis=False, alg_backend="native", vol_backend="native", alg_joints=None,
            cuboid_side=2500.0):
    alg = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=18, num_joints=alg_joints or num_joints), device="cpu",
                                            backend=alg_backend)
    cfg = testing.make_config(num_layers=18, volume_size=16, kind=kind, num_joints=num_joints, use_gt_pelvis=use_gt_pelvis,
                              cuboid_side=cuboid_side)
    vol = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend=vol_backend)
    return alg.eval(), vol.eval()


def test_constructor_accepts_native_models_and_registers_them():
    alg, vol = _models()
    m = lt_b200.TwoStageTriangulationNet(alg, vol)
    assert m.algebraic is alg and m.volumetric is vol and m.clone_outputs and not m.training
    keys = m.state_dict().keys()
    assert {"algebraic." + k for k in alg.state_dict()} | {"volumetric." + k for k in vol.state_dict()} == set(keys)
    lt_b200.TwoStageTriangulationNet(*_models(kind="coco"))


@pytest.mark.parametrize("kw, match", [
    (dict(alg_backend="torch"), "algebraic model has backend='torch'"),
    (dict(vol_backend="hybrid"), "volumetric model has backend='hybrid'"),
    (dict(use_gt_pelvis=True), "use_gt_pelvis=False"),
    (dict(alg_joints=16), "different joint counts"),
    (dict(kind="h36m"), "unknown skeleton kind"),
    (dict(kind="mpii", num_joints=6), "reads joint 6"),
    (dict(kind="coco", num_joints=12), "reads joint 12"),
])
def test_constructor_value_errors(kw, match):
    with pytest.raises(ValueError, match=match):
        lt_b200.TwoStageTriangulationNet(*_models(**kw))


def test_constructor_refuses_other_types_and_split_devices():
    alg, vol = _models()
    with pytest.raises(ValueError, match="takes an AlgebraicTriangulationNet"):
        lt_b200.TwoStageTriangulationNet(vol, alg)
    with pytest.raises(ValueError, match="one device"):
        lt_b200.TwoStageTriangulationNet(alg.to("meta"), vol)


def test_forward_refusals():
    m = lt_b200.TwoStageTriangulationNet(*_models())
    images, batch = testing.make_batch(1, 2, image_size=64)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.train()
        with torch.no_grad():
            m(images, None, batch)
    m.eval()
    m.volumetric.train()
    with pytest.raises(RuntimeError, match="inference-only"), torch.no_grad():
        m(images, None, batch)
    m.eval()
    with pytest.raises(RuntimeError, match="inference-only"):
        m(images, None, batch)
    with pytest.raises(RuntimeError, match="needs CUDA tensors"), torch.no_grad():
        m(images, None, batch)


class _Engine:
    """Stands in for NativeEngine: counts invalidations."""

    def __init__(self):
        self.epoch = 0

    def invalidate(self):
        self.epoch += 1


def test_invalidation_reaches_both_engines_and_the_graphs():
    m = lt_b200.TwoStageTriangulationNet(*_models())
    m.algebraic._engine, m.volumetric._engine = _Engine(), _Engine()
    m._graphs["entry"] = object()
    m.load_state_dict(m.state_dict())
    assert m._graphs == {} and m.algebraic._engine.epoch >= 1 and m.volumetric._engine.epoch >= 1
    m._graphs["entry"] = object()
    m.float()
    assert m._graphs == {} and m.algebraic._engine.epoch >= 2 and m.volumetric._engine.epoch >= 2
    # a submodule's own load_state_dict: its engine moves on, which changes the version the composite keys its graphs on
    before = m.volumetric._engine.epoch
    m.volumetric.load_state_dict(m.volumetric.state_dict())
    assert m.volumetric._engine.epoch == before + 1


def test_graph_key_follows_submodule_weights(monkeypatch):
    monkeypatch.setattr(capi, "lib", lambda: None)
    m = lt_b200.TwoStageTriangulationNet(*_models())
    va, vv = m.algebraic.engine()._param_version(), m.volumetric.engine()._param_version()
    m.algebraic.load_state_dict(m.algebraic.state_dict())
    assert m.algebraic.engine()._param_version() != va and m.volumetric.engine()._param_version() == vv
    m.volumetric.load_state_dict(m.volumetric.state_dict())
    assert m.volumetric.engine()._param_version() != vv


@pytest.mark.parametrize("kind, side", [("mpii", 2500.0), ("coco", 2345.6), ("coco", 2500)])
def test_lazy_cuboids_equal_host_built(kind, side):
    """The two-pass protocol: float32 key points as numpy -> _host_geometry's float64 cuboids.  LazyCuboids from the float32 base
    points (what lt_cuboid_from_keypoints_fwd writes as `center`) must give the same Cuboid3D positions and sides bit for bit."""
    B, J = 5, 17
    rng = np.random.RandomState(3)
    kp = (rng.randn(B, J, 3) * 700 + [13.7, -250.1, 900.3]).astype(np.float32)
    _, vol = _models(kind=kind, cuboid_side=side)
    batch = {"cameras": [testing.make_cameras(2, image_size=64)[v:v + 1] * B for v in range(2)], "pred_keypoints_3d": kp}
    _, base, position, step, _, host = vol._host_geometry(batch, B, (64, 64), (16, 16))
    if kind == "coco":
        center = (kp[:, 11] + kp[:, 12]) / np.float32(2)
    else:
        center = kp[:, 6]
    assert np.array_equal(center.astype(np.float64), base)
    lazy = LazyCuboids(torch.from_numpy(center), side)
    assert len(lazy) == B and lazy._items is None             # len() does not build (or copy) anything
    for b in range(B):
        assert lazy[b].position.dtype == host[b].position.dtype == np.float64
        assert np.array_equal(lazy[b].position, host[b].position) and np.array_equal(lazy[b].sides, host[b].sides)
    assert np.array_equal(np.stack([c.position for c in lazy]), position)
    assert list(lazy[1:3]) == lazy._items[1:3]
