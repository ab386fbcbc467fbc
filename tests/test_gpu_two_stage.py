"""TwoStageTriangulationNet on the GPU against the two-pass protocol it replaces: the native algebraic forward, its key points copied
to the host (.cpu().numpy()) as batch['pred_keypoints_3d'], then the native volumetric forward.  The inference kernels use no float
atomics and the hand-off kernel forms exactly the host's values, so every output must match bit for bit."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import capi, pipeline, testing

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _bits(t):
    """Bit pattern of a float32 tensor or array (NaN-safe exact comparison)."""
    a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    return np.ascontiguousarray(a).view(np.int32 if a.dtype == np.float32 else np.int64)


def _same(a, b):
    return np.array_equal(_bits(a), _bits(b))


def _models(layers=18, kind="mpii", agg="softmax", side=2500.0, transfer=False, use_confidences=True, size=128, n=32, seed=0):
    alg = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=layers, use_confidences=use_confidences), device="cpu")
    testing.randomize_backbone_weights(alg, seed=seed, calib_size=min(size, 128))
    cfg = testing.make_config(num_layers=layers, volume_size=n, aggregation=agg, use_gt_pelvis=False, kind=kind, cuboid_side=side)
    cfg.model.transfer_cmu_to_human36m = transfer
    vol = lt_b200.VolumetricTriangulationNet(cfg, device="cpu")
    testing.randomize_weights(vol, seed=seed + 1, calib_size=min(size, 128))
    if agg.startswith("conf"):
        g = torch.Generator().manual_seed(seed + 2)
        for lin in (vol.backbone.vol_confidences.head[i] for i in (0, 2, 4)):
            lin.weight.data = torch.randn(lin.weight.shape, generator=g) * (1.0 / lin.weight.shape[1]) ** 0.5
    return alg.to(DEV).eval(), vol.to(DEV).eval()


def _data(B, V, size, seed, phase=0.3):
    images, batch = testing.make_batch(B, V, image_size=size, seed=seed)
    cams = testing.make_cameras(V, size, phase=phase)
    batch["cameras"] = [[lt_b200.Camera(c.R, c.t, c.K) for _ in range(B)] for c in cams]
    del batch["pred_keypoints_3d"]
    return images.to(DEV), torch.from_numpy(testing.image_projections(batch)).to(DEV), batch


def _two_pass(alg, vol, images, proj, batch):
    kp_alg = alg(images, proj, batch)[0]
    return kp_alg, vol(images, None, dict(batch, pred_keypoints_3d=kp_alg.cpu().numpy()))


def _assert_identical(got, want):
    kp, features, volumes, conf, cuboids, coord, base = got
    kp_w, features_w, volumes_w, conf_w, cuboids_w, coord_w, base_w = want
    for name, a, b in (("keypoints", kp, kp_w), ("features", features, features_w), ("volumes", volumes, volumes_w),
                       ("coord", coord, coord_w), ("base_points", base, base_w)):
        assert tuple(a.shape) == tuple(b.shape) and _same(a, b), name
    assert (conf is None) == (conf_w is None) and (conf is None or _same(conf, conf_w))
    assert len(cuboids) == len(cuboids_w)
    for c, w in zip(cuboids, cuboids_w):
        assert c.position.dtype == w.position.dtype == np.float64
        assert _same(c.position, w.position) and _same(c.sides, w.sides)


@pytest.mark.parametrize("kind", ["mpii", "coco"])
@pytest.mark.parametrize("side", [2500.0, 2345.6])
def test_cuboid_kernel_equals_host_geometry(kind, side):
    """lt_cuboid_from_keypoints_fwd against _base_points / _host_geometry on float32 key points, with magnitudes whose coco sums
    round in float32 and a side whose half is not a float32."""
    rng = np.random.RandomState(7)
    B, J = 300, 17
    kp = (rng.randn(B, J, 3) * np.array([1.0, 1e3, 3e5])[rng.randint(0, 3, size=(B, 1, 1))] + rng.randn(B, 1, 3) * 977).astype(np.float32)
    kp[0, 11:13] = [[1e30, -3e-38, 0.1], [3e30, 7e-39, 0.2]]
    center = torch.empty((B, 3), dtype=torch.float32, device=DEV)
    position = torch.empty_like(center)
    capi.cuboid_from_keypoints(torch.from_numpy(kp).to(DEV), kind, side, center, position)
    cfg = testing.make_config(num_layers=18, volume_size=16, kind=kind, use_gt_pelvis=False, cuboid_side=side)
    vol = lt_b200.VolumetricTriangulationNet(cfg, device="cpu")
    batch = {"cameras": [testing.make_cameras(1)[:1] * B], "pred_keypoints_3d": kp}
    _, base, pos, _, _, _ = vol._host_geometry(batch, B, (64, 64), (16, 16))
    assert _same(center, base.astype(np.float32)) and np.array_equal(center.cpu().numpy().astype(np.float64), base)
    assert _same(position, pos.astype(np.float32))
    with pytest.raises(RuntimeError, match="bad size"):
        capi.cuboid_from_keypoints(torch.zeros((B, 12 if kind == "coco" else 6, 3), device=DEV), kind, side, center, position)


CASES = {
    "r18-mpii-softmax": dict(layers=18, kind="mpii", agg="softmax", side=2500.0, B=2, V=3),
    "r18-coco-conf_norm-side2345.6-cmu": dict(layers=18, kind="coco", agg="conf_norm", side=2345.6, transfer=True, B=2, V=3),
    "r50-mpii-conf_norm-side2345.6": dict(layers=50, kind="mpii", agg="conf_norm", side=2345.6, B=2, V=4),
    "r50-coco-softmax-cmu-noconf": dict(layers=50, kind="coco", agg="softmax", transfer=True, use_confidences=False, B=3, V=2),
    "r152-config2": dict(layers=152, kind="mpii", agg="softmax", side=2500.0, B=8, V=4, size=384, n=64),
}


@pytest.mark.parametrize("case", list(CASES))
def test_bit_identical_to_two_pass(case):
    c = dict(CASES[case])
    B, V, size = c.pop("B"), c.pop("V"), c.get("size", 128)
    alg, vol = _models(**c)
    model = lt_b200.TwoStageTriangulationNet(alg, vol)
    images, proj, batch = _data(B, V, size, seed=3)
    with torch.no_grad():
        kp_alg, want = _two_pass(alg, vol, images, proj, batch)
        got = model(images, proj, batch)
        got_derived = model(images, None, batch)        # image-space projections from batch['cameras']
    assert torch.isfinite(kp_alg).all() and torch.isfinite(got[0]).all()
    _assert_identical(got, want)
    _assert_identical(got_derived, want)
    assert len(model._graphs) == 1


def test_replay_follows_new_inputs_and_leaves_the_eager_algebraic_forward_alone():
    alg, vol = _models(layers=18, kind="coco", agg="softmax")
    model = lt_b200.TwoStageTriangulationNet(alg, vol)
    images, proj, batch = _data(2, 3, 128, seed=4)
    images2, proj2, batch2 = _data(2, 3, 128, seed=5, phase=1.1)
    with torch.no_grad():
        eager = alg(images, proj, batch)
        first = model(images, proj, batch)
        second = model(images2, proj2, batch2)
        eager_after = alg(images, proj, batch)
        _, want2 = _two_pass(alg, vol, images2, proj2, batch2)
        _, want1 = _two_pass(alg, vol, images, proj, batch)
    _assert_identical(second, want2)
    _assert_identical(first, want1)                       # the first call's outputs are clones: the replay did not touch them
    assert not _same(first[0], second[0])
    for a, b in zip(eager, eager_after):
        assert _same(a, b)
    assert len(model._graphs) == 1


def test_outputs_follow_reloaded_weights():
    alg, vol = _models(layers=18)
    model = lt_b200.TwoStageTriangulationNet(alg, vol)
    images, proj, batch = _data(2, 3, 128, seed=6)
    with torch.no_grad():
        before = model(images, proj, batch)
        sd = alg.state_dict()
        sd["backbone.final_layer.weight"] = sd["backbone.final_layer.weight"] * 1.5
        alg.load_state_dict(sd)
        after_alg = model(images, proj, batch)
        _, want = _two_pass(alg, vol, images, proj, batch)
        _assert_identical(after_alg, want)
        assert not _same(after_alg[6], before[6])         # the pelvis moved with the algebraic weights
        sd = vol.state_dict()
        sd["volume_net.output_layer.weight"] = sd["volume_net.output_layer.weight"] * 0.75
        vol.load_state_dict(sd)
        after_vol = model(images, proj, batch)
        _, want = _two_pass(alg, vol, images, proj, batch)
    _assert_identical(after_vol, want)
    assert not _same(after_vol[2], after_alg[2])


def test_forward_does_not_synchronise():
    alg, vol = _models(layers=18, agg="conf_norm")
    model = lt_b200.TwoStageTriangulationNet(alg, vol)
    images, _, batch = _data(2, 3, 128, seed=8)
    images2, proj2, batch2 = _data(2, 3, 128, seed=9, phase=0.9)
    with torch.no_grad():
        model(images, None, batch)                         # capture (synchronises once)
        torch.cuda.synchronize()
        prev = torch.cuda.get_sync_debug_mode()
        torch.cuda.set_sync_debug_mode("error")
        try:
            out = model(images2, None, batch2)
            model.clone_outputs = False
            out_static = model(images2, None, batch2)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
            model.clone_outputs = True
        _, want = _two_pass(alg, vol, images2, proj2, batch2)
    _assert_identical(out, want)                           # reading the cuboids synchronises, outside the checked region
    _assert_identical(out_static, want)


def test_inference_stream_equals_direct_calls():
    B, V, S = 2, 3, 128
    alg, vol = _models(layers=18)
    model = lt_b200.TwoStageTriangulationNet(alg, vol)
    batches, want = [], []
    for i in range(3):
        images, _, batch = _data(B, V, S, seed=30 + i, phase=0.3 + 0.2 * i)
        batch["images"] = np.ascontiguousarray(images.permute(0, 1, 3, 4, 2).cpu().numpy())
        batches.append(batch)
        with torch.no_grad():
            want.append(model(images, None, batch)[0].cpu().numpy())
    got = list(pipeline.InferenceStream(model).run(batches))
    assert len(got) == 3
    for g, w in zip(got, want):
        assert g.shape == (B, 17, 3) and _same(g, w)
