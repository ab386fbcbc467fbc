"""The RANSAC baseline's kernels on the GPU: the heat-map arg-max against torch.max bit for bit, the RANSAC kernel against its host
item code (lt_test_triangulate_ransac_host, the same operations: ransac.cu contracts no multiply-add), and the native model against
the CPU oracle on seeded weights."""
import os
import random

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import ransac_oracle as R
import lt_b200
from lt_b200 import capi, testing

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = np.load(os.path.join(GOLDEN, "ransac.npz"))
SCENES = sorted({k[:-len("_proj")] for k in G.files if k.endswith("_proj") and not k.startswith("model")})


def argmax_native(logits_cl, J, H, W):
    N, h, w, C = logits_cl.shape
    heat = torch.empty((N, J, h, w), dtype=torch.float32, device=DEV)
    kp = torch.empty((N, J, 2), dtype=torch.int64, device=DEV)
    ws = torch.empty(capi.heatmap_argmax_workspace_bytes(N, J, h, w) // 4, dtype=torch.float32, device=DEV)
    capi.heatmap_argmax(logits_cl, C, heat, kp, ws, N, J, h, w, W / w, H / h)
    return heat, kp


def argmax_torch(heat, H, W):
    N, J, h, w = heat.shape
    _, idx = torch.max(heat.reshape(N, J, -1), dim=-1)
    kp = torch.stack([idx % w, idx // w], dim=-1)
    out = torch.zeros_like(kp)
    out[..., 0] = kp[..., 0] * (W / w)
    out[..., 1] = kp[..., 1] * (H / h)
    return out


@pytest.mark.parametrize("N,J,C,h,w,H,W", [(8, 17, 32, 24, 24, 96, 96), (3, 17, 32, 23, 37, 80, 150), (2, 5, 16, 1, 1, 2, 2),
                                           (4, 40, 64, 41, 29, 130, 118), (2, 17, 32, 16, 24, 48, 80), (32, 17, 32, 96, 96, 384, 384)])
def test_argmax_matches_torch_max(N, J, C, h, w, H, W):
    g = torch.Generator().manual_seed(N * 1000 + h)
    logits = torch.randn((N, h, w, C), generator=g)
    logits = torch.round(logits * 4) / 4                          # many exact ties
    if h * w > 4:
        logits[0, 0, 0, 0] = float("nan")                           # NaN counts as the maximum
        logits[0, h - 1, w - 1, 0] = float("nan")                   # two NaNs: the first wins
        logits[0, h // 2, w // 2, 1] = float("inf")
        logits[1, :, :, 2] = 7.0                                     # all equal: index 0
        logits[1, :, :, 3] = -float("inf")
        logits[1, h - 1, w - 1, 4 % J] = 50.0                       # maximum at the last pixel
    logits = logits.to(DEV).contiguous()
    heat, kp = argmax_native(logits, J, H, W)
    want_heat = logits.permute(0, 3, 1, 2)[:, :J].contiguous()
    assert torch.equal(heat.view(torch.int32), want_heat.view(torch.int32))
    assert torch.equal(kp, argmax_torch(want_heat, H, W))


def _kernel(proj, kp, pairs, direct):
    B, V, J = kp.shape[:3]
    out = torch.empty((B, J, 3), dtype=torch.float32, device=DEV)
    inl = torch.empty((B, J), dtype=torch.int64, device=DEV)
    p, k, pr = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (proj.astype(np.float32), kp, pairs.astype(np.int32)))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        capi.triangulate_ransac(p, k, pr, pairs.shape[2], 15.0, direct, out, inl)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    return out.cpu().numpy(), inl.cpu().numpy()


def _host(proj, kp, pairs, direct):
    B, V, J = kp.shape[:3]
    out = torch.empty((B, J, 3), dtype=torch.float32)
    inl = torch.empty((B, J), dtype=torch.int64)
    capi.triangulate_ransac_host(torch.from_numpy(np.ascontiguousarray(proj, np.float32)), torch.from_numpy(np.ascontiguousarray(kp)),
                                 torch.from_numpy(np.ascontiguousarray(pairs, np.int32)), pairs.shape[2], 15.0, direct, out, inl)
    return out.numpy(), inl.numpy()


@pytest.mark.parametrize("scene", SCENES)
@pytest.mark.parametrize("direct", [False, True])
def test_ransac_kernel_matches_host_item_code(scene, direct):
    proj, kp, pairs = G[scene + "_proj"], G[scene + "_kp"], G[scene + "_pairs"]
    got, inl = _kernel(proj, kp, pairs, direct)
    want, inl_h = _host(proj, kp, pairs, direct)
    assert np.array_equal(inl, inl_h) and np.array_equal(inl, G[scene + "_inliers"])
    assert np.abs(got.astype(np.float64) - want).max() <= 1e-6, float(np.abs(got - want).max())
    again, inl2 = _kernel(proj, kp, pairs, direct)
    assert np.array_equal(again.view(np.int32), got.view(np.int32)) and np.array_equal(inl2, inl)


def test_ransac_kernel_large_batch_matches_host():
    rng = np.random.RandomState(5)
    B, V, J = 100, 4, 17
    P = np.stack([np.stack([c.projection for c in testing.make_cameras(V)]).astype(np.float32)] * B)
    X = rng.randn(B, J, 3) * 300 + [0, 0, 900]
    uvw = np.einsum("bvij,bkj->bvki", P.astype(np.float64), np.concatenate([X, np.ones((B, J, 1))], -1))
    kp = np.trunc(uvw[..., :2] / uvw[..., 2:3] + rng.randn(B, V, J, 2) * 2).astype(np.int64)
    kp[::3, 1] += 90
    pairs = np.sort(np.stack([rng.choice(V, 2, replace=False) for _ in range(B * J * 10)]).reshape(B, J, 10, 2), -1).astype(np.int32)
    for direct in (False, True):
        got, inl = _kernel(P, kp, pairs, direct)
        want, inl_h = _host(P, kp, pairs, direct)
        assert np.array_equal(inl, inl_h) and np.abs(got.astype(np.float64) - want).max() <= 1e-6


@pytest.mark.parametrize("mode", ["tc", "simt"])
def test_native_model_vs_oracle(mode):
    B, V, H, W = 2, 4, 48, 80
    holder = lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=18), device="cpu", backend="torch")
    testing.randomize_ransac_weights(holder, seed=11, calib_size=64)
    model = lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=18), device=DEV, backend="native", conv_mode=mode)
    model.load_state_dict(holder.state_dict(), strict=True)
    model = model.to(DEV).eval()
    images = torch.randn(B, V, 3, H, W, generator=torch.Generator().manual_seed(12))
    proj = torch.from_numpy(G["model_proj"])
    random.seed(int(G["model_seed"][0]))
    with torch.no_grad():
        kp3d, kp2d, heat, conf = model(images.to(DEV), proj.to(DEV), None)
    assert np.array_equal(np.array(random.getstate()[1], np.int64), G["model_direct_random_state"])
    heat_o, kp2d_o, o = R.ransac_forward(holder.state_dict(), images, G["model_proj"], G["model_direct_pairs"])
    heat = heat.cpu().numpy()
    herr = np.abs(heat - heat_o).max()
    assert herr <= 1e-3 * np.abs(heat_o).max(), herr
    assert kp2d.dtype == torch.int64 and conf.dtype == torch.float32 and not conf.any()
    top2 = np.sort(heat_o.reshape(B, V, 17, -1), -1)[..., -2:]
    sure = (top2[..., 1] - top2[..., 0]) > 2 * herr                                  # (B, V, J)
    kp2d = kp2d.cpu().numpy()
    assert np.array_equal(kp2d[sure], kp2d_o[sure])
    items = sure.all(axis=1)                                                           # (B, J): every view's peak is unambiguous
    assert items.sum() >= 17
    assert np.array_equal(kp2d_o, G["model_keypoints_2d"])
    o_inl = np.array([[sum(1 << v for v in r) for r in row] for row in o["inliers"]])
    assert np.array_equal(o_inl[items], G["model_direct_inliers"][items])
    # the native key points against the native item code on the native key points, and against the reference where the peaks agree
    want, inl = _host(G["model_proj"], kp2d, G["model_direct_pairs"], True)
    assert np.abs(kp3d.cpu().numpy().astype(np.float64) - want).max() <= 1e-6
    assert np.array_equal(inl[items], G["model_direct_inliers"][items])
    d = np.abs(kp3d.cpu().numpy() - G["model_direct_keypoints_3d"])[items]
    print("ransac[%s]: heat err %.2e, %d/%d items unambiguous, kp3d vs reference max %.3g mm, median %.3g mm"
          % (mode, herr, items.sum(), items.size, d.max(), np.median(d)))
