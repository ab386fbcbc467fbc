"""The RANSAC triangulation baseline on the CPU: the oracle against the reference's stored results, the native kernel's per-item code
(lt_test_triangulate_ransac_host) and the torch backend against the oracle, and the module's plumbing.

Bars: inlier sets must agree wherever every view's margin |err - 15| exceeds 1e-6 px; DLT points within 1e-6 mm plus the float32
rounding of the output on the ring scenes; refined points on the well-posed ring scenes within 1e-3 mm of the oracle's tight solve
and 1 mm of scipy's default stopping point (the reference), see WELL_POSED."""
import os
import random
import sys
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import ransac_oracle as R
import lt_b200
from lt_b200 import capi, testing
from lt_b200.triangulation import draw_view_pairs, triangulate_ransac_batch

G = np.load(os.path.join(GOLDEN, "ransac.npz"))
SCENES = sorted({k[:-len("_proj")] for k in G.files if k.endswith("_proj") and not k.startswith("model")})
N_ITERS = int(G["n_iters"][0])
MARGIN = 1e-6


def f32_round(x):
    """Half an ulp of float32 at |x|: what storing a float64 result as float32 may move it by."""
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64) / 2


def masks(inliers, V):
    return np.array([[sum(1 << v for v in row_j) for row_j in row] for row in inliers], np.int64)


def host(proj, kp, pairs, direct):
    B, V, J = kp.shape[:3]
    out = torch.empty((B, J, 3), dtype=torch.float32)
    inl = torch.empty((B, J), dtype=torch.int64)
    capi.triangulate_ransac_host(torch.from_numpy(np.ascontiguousarray(proj, np.float32)), torch.from_numpy(np.ascontiguousarray(kp)),
                                 torch.from_numpy(np.ascontiguousarray(pairs, np.int32)), pairs.shape[2], 15.0, direct, out, inl)
    return out.numpy(), inl.numpy()


@pytest.fixture(scope="module")
def oracle():
    return {s: R.triangulate_batch(G[s + "_proj"], G[s + "_kp"], G[s + "_pairs"]) for s in SCENES}


# ---- 1. the oracle reproduces the reference -------------------------------------------------------------------------------

@pytest.mark.parametrize("scene", SCENES)
def test_oracle_reproduces_reference(scene, oracle):
    o = oracle[scene]
    V = G[scene + "_kp"].shape[1]
    assert np.array_equal(masks(o["inliers"], V), G[scene + "_inliers"])
    for got, want in ((o["dlt"], G[scene + "_dlt"]), (o["refined"], G[scene + "_refined"])):
        assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()


def test_pairs_are_the_references_draws():
    """draw_view_pairs after random.seed gives the pairs the reference drew, and leaves random in the same state."""
    B, V, J = 2, 4, 17
    random.seed(int(G["model_seed"][0]))
    pairs = draw_view_pairs(B, J, V, N_ITERS)
    assert np.array_equal(pairs, G["model_dlt_pairs"])
    assert np.array_equal(np.array(random.getstate()[1], np.int64), G["model_dlt_random_state"])
    for s in SCENES:          # every scene was drawn from the same seed, items in order
        B, V, J = G[s + "_kp"].shape[:3]
        random.seed(int(G["seed"][0]))
        assert np.array_equal(draw_view_pairs(B, J, V, N_ITERS), G[s + "_pairs"]), s


# ---- 2. the kernel's item code against the oracle --------------------------------------------------------------------------

def _clear(o):
    """(B, J) bool: items whose every margin exceeds MARGIN."""
    return (o["margins"] > MARGIN).all(axis=(2, 3))


@pytest.mark.parametrize("scene", SCENES)
def test_host_item_code_vs_oracle(scene, oracle):
    o = oracle[scene]
    proj, kp, pairs = G[scene + "_proj"], G[scene + "_kp"], G[scene + "_pairs"]
    V = kp.shape[1]
    clear = _clear(o)
    assert clear.all(), "every stored scene keeps its margins above %g px" % MARGIN
    for direct in (False, True):
        got, inl = host(proj, kp, pairs, direct)
        assert np.array_equal(inl[clear], masks(o["inliers"], V)[clear])
        if not direct:
            err = np.abs(got - o["dlt"])
            if scene.startswith("narrow"):
                # the narrow-baseline rig: the DLT's conditioning bar of test_algebraic_ref_cpu (eta |A|^2 / gap, over |u3|)
                bar = np.array([[_dlt_bar(proj[b], kp[b, :, j], o["inliers"][b][j]) for j in range(kp.shape[2])]
                                for b in range(kp.shape[0])])
            else:
                bar = np.full_like(err, 1e-6)
            assert (err <= bar + f32_round(o["dlt"])).all(), (scene, float((err - bar).max()))
        else:
            _check_refined(scene, proj, kp, o, got)


# the 4-to-31-view ring scenes with 3 or more inliers: a well-posed minimum, where the refined point is pinned in millimetres.  On
# two inliers, the narrow baseline and a view far out in the Huber branch the cost is flat for metres or has several local minima,
# scipy stops wherever its tolerances end and the native refinement may settle elsewhere; there only finiteness is checked.
WELL_POSED = ("ring4", "ring4_out1", "ring8_out2", "ring31_out2")


def _check_refined(scene, proj, kp, o, got):
    """On WELL_POSED scenes: every refined point costs no more than the oracle's tight solve, lies within 1e-3 mm of it and within
    1 mm of the reference's (scipy default) result."""
    B, V, J = kp.shape[:3]
    assert np.isfinite(got).all()
    if scene not in WELL_POSED:
        return
    for b in range(B):
        for j in range(J):
            inl = o["inliers"][b][j]
            mine = R.huber_cost(got[b, j].astype(np.float64), kp[b, inl, j], proj[b, inl])
            tight = R.huber_cost(o["tight"][b, j], kp[b, inl, j], proj[b, inl])
            assert mine <= tight + 1e-9 * (1 + tight), (scene, b, j, mine, tight)
    if scene in WELL_POSED:
        assert (np.abs(got - o["tight"]) <= 1e-3 + f32_round(o["tight"])).all(), (scene, float(np.abs(got - o["tight"]).max()))
        assert np.abs(got - G[scene + "_refined"]).max() < 1.0


def _dlt_bar(P, kp, inliers):
    """Per-coordinate first-order error bound of the float64 DLT of the inlier rows (test_algebraic_ref_cpu's forward_bar)."""
    from test_algebraic_ref_cpu import dlt_reference, forward_bar
    P = P[inliers].astype(np.float32)
    # the ref module builds float32 rows; the RANSAC rows are float64 and exact-product, so its bar bounds them too
    ref = dlt_reference(P, kp[inliers].astype(np.float32), None)
    return forward_bar(ref) + 1e-6


def test_host_item_code_is_deterministic_and_follows_the_first_largest_set():
    """The 2-inlier scene: every draw gives a set of two, so the first drawn pair must win."""
    s = "ring3_two_inliers"
    got, inl = host(G[s + "_proj"], G[s + "_kp"], G[s + "_pairs"], True)
    got2, inl2 = host(G[s + "_proj"], G[s + "_kp"], G[s + "_pairs"], True)
    assert np.array_equal(got, got2) and np.array_equal(inl, inl2)
    first = G[s + "_pairs"][..., 0, :]
    assert np.array_equal(inl, (1 << first[..., 0].astype(np.int64)) | (1 << first[..., 1].astype(np.int64)))


def test_host_hook_rejects_bad_sizes():
    buf = torch.zeros(64)
    p = buf.data_ptr()
    lib = capi.lib()
    assert lib.lt_test_triangulate_ransac_host(p, p, p, 1, 65, 1, 10, 15.0, 1, p, None) != 0
    assert b"at most 64" in lib.lt_last_error_string()
    assert lib.lt_test_triangulate_ransac_host(p, p, p, 1, 1, 1, 10, 15.0, 1, p, None) != 0
    assert b"bad sizes" in lib.lt_last_error_string()
    assert lib.lt_triangulate_ransac_fwd(p, None, p, 1, 4, 1, 10, 15.0, 1, p, None, None) != 0
    assert b"null pointer" in lib.lt_last_error_string()
    assert lib.lt_heatmap_argmax_fwd(p, 16, p, p, p, 1 << 20, 1, 17, 8, 8, 1.0, 1.0, None) != 0
    assert b"bad sizes" in lib.lt_last_error_string()


# ---- 3. the torch backend against the reference's forward -------------------------------------------------------------------

def _model(direct, backend="torch"):
    holder = lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=18, direct_optimization=direct), device="cpu",
                                            backend=backend)
    return testing.randomize_ransac_weights(holder, seed=11, calib_size=64)


def _images():
    return torch.randn(2, 4, 3, 48, 80, generator=torch.Generator().manual_seed(12))


@pytest.mark.parametrize("direct", [False, True])
def test_torch_backend_matches_reference_forward(direct):
    model = _model(direct)
    proj = torch.from_numpy(G["model_proj"])
    tag = "model_direct" if direct else "model_dlt"
    random.seed(int(G["model_seed"][0]))
    with torch.no_grad():
        kp3d, kp2d, heat, conf = model(_images(), proj, None)
    assert np.array_equal(np.array(random.getstate()[1], np.int64), G[tag + "_random_state"])
    assert kp2d.dtype == torch.int64 and np.array_equal(kp2d.numpy(), G["model_keypoints_2d"])
    assert np.abs(heat.numpy() - G["model_heatmaps"]).max() <= 1e-5 * np.abs(G["model_heatmaps"]).max()
    assert conf.dtype == torch.float32 and conf.shape == (2, 4, 17) and not conf.any()
    o = R.triangulate_batch(G["model_proj"], kp2d.numpy(), G[tag + "_pairs"], direct_optimization=direct)
    clear = _clear(o)
    assert np.array_equal(masks(o["inliers"], 4)[clear], G[tag + "_inliers"][clear])
    _, inl = triangulate_ransac_batch(proj, kp2d, torch.from_numpy(G[tag + "_pairs"]), 15, direct)
    got_masks = (inl.numpy().astype(np.int64) << np.arange(4)).sum(-1)
    assert np.array_equal(got_masks[clear], G[tag + "_inliers"][clear])
    if direct:
        # arbitrary key points of random weights: the refinement is checked by its cost (see _check_refined)
        _check_refined(tag, G["model_proj"], kp2d.numpy(), o, kp3d.numpy())
    else:
        err = np.abs(kp3d.numpy() - o["dlt"])[clear]
        assert (err <= 1e-6 + 1e-9 * np.abs(o["dlt"][clear]) + f32_round(o["dlt"][clear])).all(), float(err.max())
        assert np.abs(kp3d.numpy() - G[tag + "_keypoints_3d"])[clear].max() < 1e-3


def test_torch_backend_on_the_golden_scenes(oracle):
    for s in SCENES:
        X, inl = triangulate_ransac_batch(torch.from_numpy(G[s + "_proj"]), torch.from_numpy(G[s + "_kp"]),
                                          torch.from_numpy(G[s + "_pairs"]), 15, True)
        got_masks = (inl.numpy().astype(np.int64) << np.arange(inl.shape[-1])).sum(-1)
        assert np.array_equal(got_masks, G[s + "_inliers"]), s
        _check_refined(s, G[s + "_proj"], G[s + "_kp"], oracle[s], X.numpy())


# ---- 4. plumbing ------------------------------------------------------------------------------------------------------------

def test_constructor_side_effects_and_state_dict_keys():
    cfg = testing.make_ransac_config(num_layers=18)
    cfg.model.backbone.alg_confidences = True
    cfg.model.backbone.vol_confidences = True
    model = lt_b200.RANSACTriangulationNet(cfg, device="cpu", backend="torch")
    assert cfg.model.backbone.alg_confidences is False and cfg.model.backbone.vol_confidences is False
    assert model.n_iters == 10 and model.reprojection_error_epsilon == 15 and model.direct_optimization is True
    assert sorted(model.state_dict().keys()) == list(G["model_state_dict_keys"])
    assert isinstance(model, lt_b200.triangulation._EngineOwner)


def test_native_backend_error_paths():
    model = lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=18), device="cpu")
    assert model.backend == "native" or os.environ.get("LT_B200_BACKEND")
    model.backend = "native"
    images = torch.zeros(1, 4, 3, 64, 64)
    proj = torch.zeros(1, 4, 3, 4)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):
        model.eval()(images, proj, None)
    model.train()
    with pytest.raises(RuntimeError):
        model(images, proj, None)
    with pytest.raises(AssertionError):
        model(torch.zeros(1, 1, 3, 64, 64), proj[:, :1], None)
    with pytest.raises(AssertionError):
        _model(True)(torch.zeros(1, 1, 3, 64, 64), proj[:, :1], None)
    with pytest.raises(ValueError):
        lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=18), device="cpu", backend="hybrid")


def test_install_patches_the_ransac_model(monkeypatch):
    names = ["mvn_stub", "mvn_stub.models", "mvn_stub.models.triangulation", "mvn_stub.models.loss", "mvn_stub.utils",
             "mvn_stub.utils.op"]
    mods = {n: types.ModuleType(n) for n in names}
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    lt_b200.install(mods["mvn_stub"])
    assert mods["mvn_stub.models.triangulation"].RANSACTriangulationNet is lt_b200.RANSACTriangulationNet
