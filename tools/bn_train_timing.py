#!/usr/bin/env python
"""Time the native training BatchNorm (norm_backend="native": autograd_ops.batch_norm, csrc/norm.cu) against torch's BatchNorm + ReLU
(+ add).

    python tools/bn_train_timing.py [--iters N] [--steps N] [--rounds N] [--no-step] [--json OUT]

Prints the card name, power limit and max SM clock, then:
  1. per BatchNorm class at recipe shapes -- the ResNet-152 backbone's BN + ReLU and BN + add + ReLU at each stage resolution
     (B*V = 20, 384^2) and the V2V net's at 64^3 / 32^3 (B = 5): CUDA-event medians of the fused native forward + backward and of
     torch's BatchNorm + ReLU (+ add) on the same channels-last fp32 tensors, with the bytes the native passes move (counted from the
     shapes) over the native time against the H100 SXM's 3.35 TB/s;
  2. the backbone (ResNet-152, B*V = 20, 384^2) and V2V (B = 5, 64^3) forward + backward with the native convolutions, norm_backend
     torch vs native, alternated --rounds times, with the peak memory of each;
  3. the recipe volumetric training step (ResNet-152, B = 5, V = 4, 384^2, 64^3, 0.1 MAE + 0.01 CE, Adam) with all three native
     backends against the native convolutions with torch BatchNorm.
Needs a CUDA device; it does not fall back to anything.
"""
import argparse
import json
import os
import statistics
import sys
from collections import defaultdict

import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import lt_b200  # noqa: E402
from lt_b200 import autograd_ops as A, loss as ce, pose_resnet, testing  # noqa: E402
from lt_b200.v2v import V2VModel  # noqa: E402
from v2v_train_timing import DEV, card, event_median  # noqa: E402

HBM_PEAK = 3.35e12      # H100 SXM data sheet

# label -> (shape, relu, residual): the BatchNorm classes of the recipe's two nets
CLASSES = {
    "backbone stem 192^2 C64 bn+relu": ((20, 64, 192, 192), True, False),
    "backbone layer1 96^2 C64 bn+relu": ((20, 64, 96, 96), True, False),
    "backbone layer1 96^2 C256 bn+add+relu": ((20, 256, 96, 96), True, True),
    "backbone layer2 48^2 C128 bn+relu": ((20, 128, 48, 48), True, False),
    "backbone layer2 48^2 C512 bn+add+relu": ((20, 512, 48, 48), True, True),
    "backbone layer3 24^2 C256 bn+relu": ((20, 256, 24, 24), True, False),
    "backbone layer3 24^2 C1024 bn+add+relu": ((20, 1024, 24, 24), True, True),
    "backbone layer4 12^2 C512 bn+relu": ((20, 512, 12, 12), True, False),
    "backbone layer4 12^2 C2048 bn+add+relu": ((20, 2048, 12, 12), True, True),
    "backbone deconv 96^2 C256 bn+relu": ((20, 256, 96, 96), True, False),
    "v2v 64^3 C32 bn+relu": ((5, 32, 64, 64, 64), True, False),
    "v2v 64^3 C32 bn+add+relu": ((5, 32, 64, 64, 64), True, True),
    "v2v 32^3 C64 bn+add+relu": ((5, 64, 32, 32, 32), True, True),
}


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last if t.dim() == 4 else torch.channels_last_3d)


def native_bytes(shape, relu, res):
    """Bytes the native passes move: forward statistics (x) + apply (x, r -> y); backward reduce (x, g, y) + apply (x, g, y -> dx, dr)."""
    e = 4 * int(np.prod(shape))
    return e * ((1) + (2 + res) + (2 + relu) + (3 + relu + res))


def class_timing(iters, rounds):
    out = {}
    for label, (shape, relu, res) in CLASSES.items():
        C = shape[1]
        bn = (nn.BatchNorm2d if len(shape) == 4 else nn.BatchNorm3d)(C).to(DEV).train()
        x = _cl(torch.randn(shape, device=DEV)).requires_grad_(True)
        r = _cl(torch.randn(shape, device=DEV)).requires_grad_(True) if res else None
        g = _cl(torch.randn(shape, device=DEV))

        def native():
            A.batch_norm(bn, x, relu=relu, residual=r).backward(g)

        def torch_ref():
            y = bn(x)
            if r is not None:
                y = y + r
            (F.relu(y, inplace=True) if relu else y).backward(g)
        times = defaultdict(list)
        for _ in range(rounds):
            for name, fn in (("native", native), ("torch", torch_ref)):
                times[name].append(event_median(fn, iters))
        med = {k: statistics.median(v) for k, v in times.items()}
        nbytes = native_bytes(shape, relu, res)
        bw = nbytes / (med["native"] * 1e-3)
        print("%-42s native %7.3f ms  torch %7.3f ms  x%.2f   native %.0f GB/s = %.0f%% of 3.35 TB/s  (spread native %.3f-%.3f)"
              % (label, med["native"], med["torch"], med["torch"] / med["native"], bw / 1e9, 100 * bw / HBM_PEAK,
                 min(times["native"]), max(times["native"])))
        out[label] = {"rounds_ms": dict(times), "median_ms": med, "native_bytes": nbytes, "native_GBps": bw / 1e9}
        del x, r, g, bn
        torch.cuda.empty_cache()
    return out


def _alternate(iters, rounds, runs, label):
    res, mem = defaultdict(list), {}
    for r in range(rounds):
        for key, step in runs.items():
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            res[key].append(event_median(step, iters))
            mem[key] = torch.cuda.max_memory_allocated() / 2 ** 30
            print("%s round %d, %s: %.2f ms" % (label, r, key, res[key][-1]))
    med = {k: statistics.median(v) for k, v in res.items()}
    print("%s, median of rounds: " % label + ", ".join("%s %.2f ms [%.2f-%.2f] (peak %.2f GiB)" % (k, med[k], min(res[k]), max(res[k]), mem[k])
                                                       for k in runs))
    return {"rounds_ms": dict(res), "median_ms": med, "peak_GiB": mem}


def net_timing(iters, rounds):
    out = {}
    torch.manual_seed(0)
    cfg = testing.make_config(num_layers=152).model.backbone
    cfg.alg_confidences = cfg.vol_confidences = False
    net = pose_resnet.get_pose_net(cfg, device=DEV).to(DEV).train()
    x = torch.randn(20, 3, 384, 384, device=DEV)

    def backbone(norm):
        def step():
            net.zero_grad(set_to_none=True)
            heat, feats, _, _ = net(x, A.backbone_conv, norm)
            (heat.sum() * 1e-4 + feats.sum() * 1e-6).backward()
        return step
    out["backbone"] = _alternate(iters, rounds, {"norm torch": backbone(None), "norm native": backbone(A.batch_norm)},
                                 "ResNet-152 backbone fwd+bwd (B*V=20, 384^2, native convs)")
    del net, x
    torch.cuda.empty_cache()
    v2v = V2VModel(32, 17).to(DEV).train()
    vx = _cl(torch.randn(5, 32, 64, 64, 64, device=DEV))

    def vstep(norm):
        def step():
            v2v.zero_grad(set_to_none=True)
            (v2v(vx, A.v2v_conv, norm).sum() * 1e-4).backward()
        return step
    out["v2v"] = _alternate(iters, rounds, {"norm torch": vstep(None), "norm native": vstep(A.batch_norm)},
                            "V2V fwd+bwd (B=5, 64^3, native convs)")
    del v2v, vx
    torch.cuda.empty_cache()
    return out


def volumetric_step_timing(steps, rounds):
    B, V, S = 5, 4, 384
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    loss_fn = ce.VolumetricCELoss(backend="native")
    torch.manual_seed(0)
    runs, sd = {}, None
    for nb in ("torch", "native"):
        m = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=152, volume_size=64), device=DEV, backend="hybrid",
                                               backbone_backend="native", v2v_backend="native", norm_backend=nb)
        if sd is None:
            sd = m.state_dict()
        m.load_state_dict(sd)
        m = m.to(DEV).train()
        opt = torch.optim.Adam(m.parameters(), lr=1e-4)

        def step(m=m, opt=opt):
            opt.zero_grad(set_to_none=True)
            kp, _, vols, _, _, coord, _ = m(images, None, batch)
            mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
            (0.1 * mae + 0.01 * loss_fn(coord, vols, kp_gt, valid)).backward()
            opt.step()
        runs["native convs, norm " + nb] = step
    return _alternate(steps, rounds, runs, "volumetric training step (ResNet-152, B=5, V=4, 384^2, 64^3, Adam)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bn_train_timing.py needs a CUDA device")
    name, q = card()
    print("device: %s, power limit, max SM clock: %s" % (name, q))
    out = {"device": name, "power_limit_max_sm_clock": q, "classes": class_timing(a.iters, a.rounds)}
    out["nets"] = net_timing(a.iters, a.rounds)
    if not a.no_step:
        out["volumetric_step"] = volumetric_step_timing(a.steps, a.rounds)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
