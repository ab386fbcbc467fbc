"""Module-level GPU parity: the drop-in VolumetricTriangulationNet (native backend, through the C ABI) against the
golden vectors of the unmodified reference, the CPU oracle, and -- at BASELINE config #2 sizes -- between its own
exact-fp32 and tensor-core modes (size-independent property: both must agree, argmax indices bit-exact)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err
from oracle import vol_oracle as O
import lt_b200
from lt_b200 import testing

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# (features, unprojected/logits, volumes) relative tolerances; keypoints in mm
# keypoints: 0.5 mm = 2e-4 of the 2500 mm cuboid (the contract is 1e-3 relative)
TOL = {"simt": (1e-4, 2e-4, 1e-3, 0.5), "tc": (2e-4, 5e-4, 1e-3, 0.5), "tc1": (5e-2, 2e-1, None, None)}


@pytest.fixture(scope="module")
def r50_case():
    B, V, S, n = 2, 2, 128, 32
    cfg = testing.make_config(num_layers=50, volume_size=n)
    model = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend="torch")
    testing.randomize_weights(model, seed=1, calib_size=S)
    images, batch = testing.make_batch(B, V, image_size=S, seed=3)
    return model.state_dict(), images, batch, n


def _native(sd, n, mode, graph, num_layers=50):
    m = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=num_layers, volume_size=n), device=DEV,
                                           backend="native", conv_mode=mode, use_cuda_graph=graph)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval()


@pytest.mark.parametrize("mode,graph", [("simt", False), ("simt", True), ("tc", False), ("tc", True), ("tc1", False)])
def test_forward_matches_reference_vectors(r50_case, mode, graph):
    sd, images, batch, n = r50_case
    g = np.load(os.path.join(GOLDEN, "forward_r50.npz"))
    model = _native(sd, n, mode, graph)
    with torch.no_grad():
        for _ in range(2 if graph else 1):       # second call replays the captured graph
            kp, feats, vols, conf, cuboids, coords, base = model(images.to(DEV), None, batch)
    torch.cuda.synchronize()
    t_feat, t_mid, t_vol, t_kp = TOL[mode]
    assert conf is None and len(cuboids) == images.shape[0]
    assert tuple(kp.shape) == (2, 17, 3) and tuple(feats.shape) == (2, 2, 32, 32, 32) and tuple(vols.shape) == (2, 17, n, n, n)
    assert np.allclose(base.cpu().numpy(), g["base_points"])
    assert np.array_equal(coords[:, ::5, ::5, ::5].cpu().numpy(), g["coord_sub"])            # bit-exact geometry
    e_feat = rel_err(feats[:, :, ::4, ::3, ::3].cpu().numpy(), g["features_sub"])
    print("mode=%s graph=%s features rel err %.3e" % (mode, graph, e_feat))
    assert e_feat < t_feat
    if t_vol is not None:
        e_vol = rel_err(vols[:, :, ::3, ::3, ::3].cpu().numpy(), g["volumes_sub"])
        e_kp = float(np.abs(kp.cpu().numpy() - g["keypoints"]).max())
        print("mode=%s volumes rel err %.3e keypoints max abs err %.4f mm" % (mode, e_vol, e_kp))
        assert e_vol < t_vol and e_kp < t_kp
        assert np.array_equal(vols.reshape(2, 17, -1).argmax(-1).cpu().numpy(), g["volumes_argmax"])    # bit-exact indices


@pytest.mark.parametrize("mode", ["simt", "tc"])
def test_stages_match_oracle(r50_case, mode):
    """Intermediates (unprojected volume, V2V logits) against the CPU oracle run on the same inputs."""
    sd, images, batch, n = r50_case
    base = np.stack([k[6, :3] for k in batch["keypoints_3d"]])
    kp_o, feats_o, vols_o, coords_o, inter = O.volumetric_forward(sd, images, batch["cameras"], base, volume_size=n,
                                                                  return_intermediates=True)
    model = _native(sd, n, mode, False)
    eng = model.engine()
    eng.prepare()
    B, V = images.shape[:2]
    with torch.no_grad():
        feats = eng.backbone_features(images.to(DEV).reshape(B * V, *images.shape[2:]))
        f_nchw = feats.data.view(B, V, feats.H, feats.W, feats.C).permute(0, 1, 4, 2, 3)
        assert rel_err(f_nchw.cpu().numpy(), feats_o.numpy()) < TOL[mode][0]
        proj = torch.from_numpy(inter["proj"]).to(DEV)
        coord = coords_o.to(DEV).contiguous()
        vol = eng.unproject(feats, B, V, proj, coord, lt_b200.capi.AGG["softmax"])
        from test_gpu_ops import act_to_nchw
        assert rel_err(act_to_nchw(vol).cpu().numpy(), inter["unprojected"]) < TOL[mode][1]
        logits = eng.v2v(vol)
        got = act_to_nchw(logits, 17).cpu().numpy()
        e = rel_err(got, inter["logits"])
        print("mode=%s logits rel err %.3e" % (mode, e))
        assert e < TOL[mode][1]


def test_config2_sizes_tensor_core_vs_exact_fp32():
    """ResNet-152, 4 views 384x384, 64^3 grid (BASELINE config #2 shapes, B=2): tensor-core path vs exact-fp32 path."""
    B, V, S, n = 2, 4, 384, 64
    cfg = testing.make_config(num_layers=152, volume_size=n)
    ref = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend="torch")
    testing.randomize_weights(ref, seed=2, calib_size=S, calib_views=1)
    sd = ref.state_dict()
    images, batch = testing.make_batch(B, V, image_size=S, seed=4)
    outs = {}
    for mode in ("simt", "tc"):
        model = _native(sd, n, mode, True, num_layers=152)
        with torch.no_grad():
            outs[mode] = model(images.to(DEV), None, batch)
        del model
        torch.cuda.empty_cache()
    a, b = outs["tc"], outs["simt"]
    assert torch.equal(a[5], b[5])                                                     # coordinate volumes
    e_feat, e_vol = rel_err(a[1].cpu().numpy(), b[1].cpu().numpy()), rel_err(a[2].cpu().numpy(), b[2].cpu().numpy())
    e_kp = float((a[0] - b[0]).abs().max())
    print("config2 shapes: features %.3e volumes %.3e keypoints %.4f mm" % (e_feat, e_vol, e_kp))
    assert e_feat < 3e-4 and e_vol < 1e-3 and e_kp < 0.5
    assert torch.equal(a[2].reshape(B, 17, -1).argmax(-1), b[2].reshape(B, 17, -1).argmax(-1))
    # size-independent properties of the softmaxed volumes / soft-argmax
    s = a[2].reshape(B, 17, -1).sum(-1)
    assert float((s - 1).abs().max()) < 1e-4
    lo, hi = a[5].reshape(B, -1, 3).min(1)[0], a[5].reshape(B, -1, 3).max(1)[0]
    assert bool(((a[0] >= lo[:, None]) & (a[0] <= hi[:, None])).all()), "expected coordinates must lie inside the cuboid"


def test_config2_full_size_vs_oracle():
    """BASELINE config #2 at full size (ResNet-152, 4 views 384x384, 64^3 grid, calibrated weights, B=1): the native tensor-core
    path against the CPU oracle's restatement of reference triangulation.py:245-355 on the same inputs -- features, unprojected
    volume, V2V logits, softmaxed volumes <= 1e-3 relative, keypoints <= 1e-3 of the cuboid, arg-max voxels bit-equal."""
    from oracle import parity
    B, V, S, n = 1, 4, 384, 64
    cfg = testing.make_config(num_layers=152, volume_size=n)
    holder = lt_b200.VolumetricTriangulationNet(cfg, device=DEV, backend="torch")
    testing.randomize_weights(holder, seed=2, calib_size=S, calib_views=1)
    sd = {k: v.detach().cpu() for k, v in holder.state_dict().items()}
    del holder
    torch.cuda.empty_cache()
    images, batch = testing.make_batch(B, V, image_size=S, seed=4)
    oracle_out, secs = parity.oracle_forward(sd, images, batch, n)
    model = _native(sd, n, "tc", False, num_layers=152)
    with torch.no_grad():
        out = model(images.to(DEV), None, batch)
    res = parity.compare_outputs(out, oracle_out)
    res.update(parity.compare_stages(model, images, batch, oracle_out, DEV))
    print("config2 full size vs oracle (%.1f s CPU): %s" % (secs, res))
    assert res["coord_volumes_bit_exact"] and res["argmax_equal"]
    assert res["features_rel"] < 1e-3 and res["unprojected_rel"] < 1e-3 and res["logits_rel"] < 1e-3 and res["volumes_rel"] < 1e-3
    assert res["keypoints_mm"] < 1e-3 * parity.CUBOID_MM
