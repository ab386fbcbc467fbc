"""Times of the RANSAC baseline's native kernels and model forward on the GPU, beside the CPU oracle on the same inputs.

    python tools/ransac_timing.py [--out DIR]

lt_triangulate_ransac_fwd (with and without the refinement) and lt_heatmap_argmax_fwd by CUDA events over repeated launches, the
native RANSACTriangulationNet forward (ResNet-152, 384 x 384, tc mode, default weights) by CUDA events, at B in {8, 100}, V = 4, J = 17; the CPU
oracle (numpy DLT + scipy refinement per item, as the reference runs it) on a subset of the items, scaled per item.  Prints the card
name and power limit with the numbers and writes them as JSON under --out."""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import capi, testing  # noqa: E402
from lt_b200.triangulation import draw_view_pairs  # noqa: E402
from oracle import ransac_oracle as R  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def events(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def scene(B, V, J, seed=0):
    rng = np.random.RandomState(seed)
    P = np.stack([np.stack([c.projection for c in testing.make_cameras(V)]).astype(np.float32)] * B)
    X = rng.randn(B, J, 3) * 300 + [0, 0, 900]
    uvw = np.einsum("bvij,bkj->bvki", P.astype(np.float64), np.concatenate([X, np.ones((B, J, 1))], -1))
    kp = np.trunc(uvw[..., :2] / uvw[..., 2:3] + rng.randn(B, V, J, 2) * 2).astype(np.int64)
    kp[::3, 1] += 90                                         # an outlier view in every third sample
    random.seed(seed)
    return P, kp, draw_view_pairs(B, J, V, 10)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ransac_timing measures on a GPU"
    res = {"card": card()}
    print("card, power limit:", res["card"])
    V, J = 4, 17
    for B in (8, 100):
        P, kp, pairs = scene(B, V, J)
        p, k, pr = (torch.from_numpy(a).to(DEV) for a in (P, kp, pairs))
        out = torch.empty((B, J, 3), dtype=torch.float32, device=DEV)
        r = {}
        for direct in (False, True):
            r["ransac_kernel_ms_direct%d" % direct] = events(lambda: capi.triangulate_ransac(p, k, pr, 10, 15.0, direct, out), 200)
        h = w = 96
        logits = torch.randn((B * V, h, w, 32), device=DEV)
        heat = torch.empty((B * V, J, h, w), device=DEV)
        kp2 = torch.empty((B * V, J, 2), dtype=torch.int64, device=DEV)
        ws = torch.empty(capi.heatmap_argmax_workspace_bytes(B * V, J, h, w) // 4, device=DEV)
        ms = events(lambda: capi.heatmap_argmax(logits, 32, heat, kp2, ws, B * V, J, h, w, 4.0, 4.0), 200)
        nbytes = 4.0 * B * V * h * w * (32 + J)
        r["argmax_ms"], r["argmax_GBps"] = ms, nbytes / ms / 1e6
        n_cpu = min(B, 8)
        t = time.perf_counter()
        R.triangulate_batch(P[:n_cpu], kp[:n_cpu], pairs[:n_cpu], direct_optimization=True, tight=False)
        r["oracle_cpu_ms_per_item"] = (time.perf_counter() - t) * 1e3 / (n_cpu * J)
        r["oracle_cpu_ms_batch_estimate"] = r["oracle_cpu_ms_per_item"] * B * J
        res["B%d" % B] = r
        print("B=%d V=%d J=%d: %s" % (B, V, J, json.dumps({k2: round(v, 4) for k2, v in r.items()})))
    # the native model forward, ResNet-152 at 384 x 384 (the eval config), B = 8
    model = lt_b200.RANSACTriangulationNet(testing.make_ransac_config(num_layers=152), device=DEV, backend="native").to(DEV).eval()
    for B in (8, 100):
        images, batch = testing.make_batch(B, V, image_size=384, seed=1, device=DEV)
        proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
        with torch.no_grad():
            fwd = events(lambda: model(images, proj, batch), 10)
        res["model_forward_ms_B%d" % B] = fwd
        print("RANSACTriangulationNet forward (ResNet-152, 384^2, B=%d, V=%d): %.3f ms" % (B, V, fwd))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ransac_timing.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
