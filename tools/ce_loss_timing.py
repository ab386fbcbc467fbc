#!/usr/bin/env python
"""Time the volumetric cross-entropy loss (VolumetricCELoss, csrc/loss.cu) on the GPU against the per-sample, per-joint
formulation of the reference (the loss restated in tests/test_volumetric_ce_cpu.py).

    python tools/ce_loss_timing.py [--iters N] [--steps N] [--rounds N] [--no-step] [--json OUT]

Prints the card name and power limit, then:
  1. CUDA-event medians of loss forward + backward, reference formulation vs native, at B in {5, 8}, J = 17, 64^3;
  2. each native kernel's achieved bytes/s against 3.35 TB/s (H100 SXM HBM3 data-sheet figure): the search reads the coordinate
     volume once (12 B per voxel per sample), the backward writes the full gradient (4 B per element);
  3. one recipe-shaped training step (ResNet-152 volumetric model, backend="hybrid", B = 5, V = 4, 384^2, train mode,
     0.1 * MAE + 0.01 * CE, Adam step) with each loss, the two alternated --rounds times; median step time per round.
Needs a CUDA device; it does not fall back to anything.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lt_b200  # noqa: E402
from lt_b200 import capi, loss as ce, testing  # noqa: E402
from test_volumetric_ce_cpu import oracle_volumetric_ce_loss  # noqa: E402

DEV = "cuda:0"
HBM_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def problem(B, J, n, seed=0):
    g = torch.Generator().manual_seed(seed)
    ax = torch.linspace(-1250.0, 1250.0, n)
    coord = torch.stack(torch.meshgrid(ax, ax, ax, indexing="ij"), -1).expand(B, n, n, n, 3) + torch.randn(B, 1, 1, 1, 3, generator=g) * 100
    vols = torch.softmax(torch.randn(B, J, n ** 3, generator=g) * 3, -1).reshape(B, J, n, n, n)
    kp = torch.randn(B, J, 3, generator=g) * 400
    valid = torch.ones(B, J, 1)
    return [t.contiguous().to(DEV) for t in (coord, vols, kp, valid)]


def event_median(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def loss_timing(iters):
    rows = []
    for B in (5, 8):
        coord, vols, kp, valid = problem(B, 17, 64)

        def step(fn):
            v = vols.clone().requires_grad_(True)
            fn(coord, v, kp, valid).backward()
        native = ce.VolumetricCELoss(backend="native")
        t_ref = event_median(lambda: step(oracle_volumetric_ce_loss), max(3, iters // 10))
        t_nat = event_median(lambda: step(native), iters)
        # the clone of the volumes is part of both timings; report it so it can be subtracted
        t_clone = event_median(lambda: vols.clone(), iters)
        rows.append({"B": B, "J": 17, "grid": 64, "reference_ms": t_ref, "native_ms": t_nat, "clone_ms": t_clone,
                     "speedup": t_ref / t_nat})
        print("loss fwd+bwd B=%d J=17 64^3: reference formulation %.3f ms, native %.3f ms (%.0fx); volumes clone in both %.3f ms"
              % (B, t_ref, t_nat, t_ref / t_nat, t_clone))
    return rows


def kernel_timing(iters):
    rows = []
    for B in (5, 8):
        J, n = 17, 64
        nvox = n ** 3
        coord, vols, kp, valid = problem(B, J, n)
        probs, c, v = vols.reshape(B, J, nvox), coord.reshape(B, nvox, 3), valid[..., 0].contiguous()
        loss = torch.empty(1, device=DEV)
        index = torch.empty((B, J), dtype=torch.int32, device=DEV)
        picked = torch.empty((B, J), device=DEV)
        ws = torch.empty(capi.volumetric_ce_workspace_bytes(B, J, nvox), dtype=torch.uint8, device=DEV)
        grad = torch.empty_like(probs)
        g = torch.ones(1, device=DEV)
        t_f = event_median(lambda: capi.volumetric_ce(probs, c, kp, v, loss, index, picked, ws), iters)
        t_b = event_median(lambda: capi.volumetric_ce_bwd(g, index, picked, v, grad), iters)
        bytes_f, bytes_b = B * nvox * 12, B * J * nvox * 4
        rows.append({"B": B, "fwd_ms": t_f, "fwd_bytes": bytes_f, "fwd_TBps": bytes_f / t_f / 1e9,
                     "bwd_ms": t_b, "bwd_bytes": bytes_b, "bwd_TBps": bytes_b / t_b / 1e9})
        print("kernels B=%d: forward (memset + search + finish) %.4f ms, %.2f TB/s = %.0f %% of 3.35; backward %.4f ms, %.2f TB/s = %.0f %%"
              % (B, t_f, bytes_f / t_f / 1e9, 100 * bytes_f / t_f / 1e9 / 3.35, t_b, bytes_b / t_b / 1e9,
                 100 * bytes_b / t_b / 1e9 / 3.35))
    return rows


def training_step_timing(steps, rounds):
    B, V, S = 5, 4, 384
    torch.manual_seed(0)
    model = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=152, volume_size=64), device=DEV,
                                               backend="hybrid").to(DEV).train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-4)
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    losses = {"native": ce.VolumetricCELoss(backend="native"), "reference": oracle_volumetric_ce_loss}

    def step(which):
        opt.zero_grad(set_to_none=True)
        kp, _, vols, _, _, coord, _ = model(images, None, batch)
        mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
        (0.1 * mae + 0.01 * losses[which](coord, vols, kp_gt, valid)).backward()
        opt.step()

    res = {"native": [], "reference": []}
    for r in range(rounds):
        for which in ("reference", "native"):
            t = event_median(lambda: step(which), steps, warmup=2)
            res[which].append(t)
            print("training step round %d, %s CE: median %.2f ms over %d steps" % (r, which, t, steps))
    summary = {k: statistics.median(v) for k, v in res.items()}
    print("training step (ResNet-152, B=5, V=4, 384^2, hybrid, Adam): reference CE %.2f ms, native CE %.2f ms (median of rounds)"
          % (summary["reference"], summary["native"]))
    return {"rounds": res, "median": summary}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ce_loss_timing.py needs a CUDA device")
    name, limit = card()
    print("device: %s, power limit %s" % (name, limit))
    out = {"device": name, "power_limit": limit, "loss": loss_timing(a.iters), "kernels": kernel_timing(a.iters)}
    if not a.no_step:
        out["training_step"] = training_step_timing(a.steps, a.rounds)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
