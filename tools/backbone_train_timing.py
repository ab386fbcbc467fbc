#!/usr/bin/env python
"""Time the 2-D backbone's training passes with the native convolutions (backbone_backend="native": autograd_ops.backbone_conv)
against cuDNN.

    python tools/backbone_train_timing.py [--iters N] [--steps N] [--rounds N] [--batches 20,32] [--no-step] [--json OUT]

Prints the card name, power limit and max SM clock, then:
  1. ResNet-152 backbone forward + backward (PoseResNet, 384^2, train-mode BatchNorm) at B*V = 20 and 32: CUDA-event medians of
     native, cuDNN fp32 (TF32 off) and cuDNN with torch's default TF32, alternated --rounds times, each with its
     torch.cuda.max_memory_allocated;
  2. a per-class kernel table of one native forward + backward at B*V = 20 from a separate torch.profiler run, with the
     algorithmic FLOP/s of the convolution classes (counted from the layer shapes) against the 989 TFLOP/s dense fp16 figure of the
     H100 SXM data sheet;
  3. a config-#5-shaped algebraic training step (ResNet-152 with confidences, B = 5, V = 4, 384^2, MAE, Adam) with
     backbone_backend torch / native, and the recipe volumetric step (B = 5, V = 4, 384^2, 64^3, 0.1 MAE + 0.01 CE, Adam) with
     backbone_backend x v2v_backend in {torch, native}, alternated --rounds times, with peak memory of each.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import lt_b200  # noqa: E402
from lt_b200 import autograd_ops as A, loss as ce, pose_resnet, testing  # noqa: E402
from v2v_train_timing import DEV, FP16_DENSE_PEAK, _Tf32, card, event_median  # noqa: E402

CONFIGS = {"native": (A.backbone_conv, False), "cudnn_fp32": (None, False), "cudnn_tf32": (None, True)}


def backbone_problem(BV, S=384):
    torch.manual_seed(0)
    cfg = testing.make_config(num_layers=152).model.backbone
    cfg.alg_confidences = cfg.vol_confidences = False
    net = pose_resnet.get_pose_net(cfg, device=DEV).to(DEV).train()
    x = torch.randn(BV, 3, S, S, device=DEV)
    return net, x


def backbone_step(net, x, conv):
    net.zero_grad(set_to_none=True)
    heat, feats, _, _ = net(x, conv)
    (heat.sum() * 1e-4 + feats.sum() * 1e-6).backward()


def backbone_timing(iters, rounds, batches):
    out = {}
    for BV in batches:
        net, x = backbone_problem(BV)
        res, mem = defaultdict(list), {}
        for r in range(rounds):
            for name, (conv, tf32) in CONFIGS.items():
                with _Tf32(tf32):
                    torch.cuda.empty_cache()
                    torch.cuda.reset_peak_memory_stats()
                    try:
                        res[name].append(event_median(lambda: backbone_step(net, x, conv), iters))
                    except torch.cuda.OutOfMemoryError:
                        res[name].append(float("nan"))
                    mem[name] = torch.cuda.max_memory_allocated() / 2 ** 30
                print("backbone fwd+bwd B*V=%d round %d %-10s %.2f ms" % (BV, r, name, res[name][-1]))
        med = {k: statistics.median(v) for k, v in res.items()}
        print("ResNet-152 backbone fwd+bwd (B*V=%d, 384^2, train BN), median of rounds: " % BV +
              ", ".join("%s %.2f ms (peak %.2f GiB)" % (k, med[k], mem[k]) for k in CONFIGS))
        out[BV] = {"rounds": dict(res), "median_ms": med, "peak_GiB": mem}
        del net, x
        torch.cuda.empty_cache()
    return out


def conv_flops(net, x):
    """Algorithmic FLOPs of every Conv2d / ConvTranspose2d forward at this input (2 x MACs); wgrad and dgrad count the same (the stem's
    data gradient is not computed)."""
    total = [0.0]

    def hook(m, inp, out):
        w = m.weight
        if isinstance(m, torch.nn.ConvTranspose2d):
            total[0] += 2.0 * inp[0].numel() / inp[0].shape[1] * w.numel()
        else:
            total[0] += 2.0 * out.numel() / out.shape[1] * w.numel()
    hs = [m.register_forward_hook(hook) for m in net.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.ConvTranspose2d))]
    with torch.no_grad():
        net(x)
    for h in hs:
        h.remove()
    return total[0]


def kernel_class(name):
    n = name.lower()
    if "conv_wgrad" in n or "wgrad_reduce" in n:
        return "wgrad (conv_wgrad_kernel + reduce)"
    if "conv_tc_kernel" in n or "splitk_reduce" in n:
        return "forward + dgrad on conv_tc_kernel"
    if any(k in n for k in ("f32_to_s32", "s32_to_f32", "absmax", "gather_weights", "pack_weights", "fold_bn", "stem_s2d")):
        return "conversions + filter packing"
    if "batch_norm" in n or "bn_" in n or "welford" in n:
        return "torch BatchNorm"
    if "pool" in n:
        return "torch max-pool"
    return "torch other (ReLU, adds, sums, copies, index)"


def profile_table(out_dir, BV=20):
    net, x = backbone_problem(BV)
    flops = conv_flops(net, x)
    for _ in range(2):
        backbone_step(net, x, A.backbone_conv)
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        backbone_step(net, x, A.backbone_conv)
        torch.cuda.synchronize()
    times = defaultdict(float)
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0:
            times[kernel_class(e.key)] += t / 1e3
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        prof.export_chrome_trace(os.path.join(out_dir, "backbone_train_native_trace.json"))
    rows = []
    print("per-class device time of one native ResNet-152 backbone forward + backward (B*V=%d, 384^2, torch.profiler), "
          "algorithmic conv FLOPs %.1f GFLOP per pass:" % (BV, flops / 1e9))
    for k, t in sorted(times.items(), key=lambda kv: -kv[1]):
        rate = ""
        if k.startswith("wgrad") and t > 0:
            rate = "%.1f TFLOP/s = %.1f %% of 989" % (flops / t / 1e9, 100 * flops / t * 1e3 / FP16_DENSE_PEAK)
        elif k.startswith("forward") and t > 0:
            rate = "%.1f TFLOP/s = %.1f %% of 989 (forward + dgrad: 2 x %.1f GFLOP)" % (
                2 * flops / t / 1e9, 100 * 2 * flops / t * 1e3 / FP16_DENSE_PEAK, flops / 1e9)
        print("  %-46s %8.2f ms  %s" % (k, t, rate))
        rows.append({"class": k, "ms": t})
    del net, x
    torch.cuda.empty_cache()
    return {"conv_gflop_per_pass": flops / 1e9, "classes": rows}


def _alternate(steps, rounds, runs, label):
    res, mem = defaultdict(list), {}
    for r in range(rounds):
        for key, step in runs.items():
            torch.cuda.reset_peak_memory_stats()
            t = event_median(step, steps, warmup=2)
            mem[key] = torch.cuda.max_memory_allocated() / 2 ** 30
            res[key].append(t)
            print("%s round %d, %s: median %.2f ms over %d steps" % (label, r, key, t, steps))
    med = {k: statistics.median(v) for k, v in res.items()}
    print("%s (TF32 default), median of rounds: " % label + ", ".join("%s %.2f ms (peak %.2f GiB)" % (k, med[k], mem[k]) for k in runs))
    return {"rounds": dict(res), "median_ms": med, "peak_GiB": mem}


def algebraic_step_timing(steps, rounds):
    """Config #5 shape: ResNet-152 algebraic model with confidences at 384^2, B*V = 20 as in the recipe."""
    B, V, S = 5, 4, 384
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    target = torch.from_numpy(np.stack([k[:, :3] for k in batch["keypoints_3d"]])).float().to(DEV)
    torch.manual_seed(0)
    runs, sd = {}, None
    for bb in ("torch", "native"):
        m = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=152), device=DEV, backend="hybrid", backbone_backend=bb)
        if sd is None:
            sd = m.state_dict()
        m.load_state_dict(sd)
        m = m.to(DEV).train()
        opt = torch.optim.Adam(m.parameters(), lr=1e-4)

        def step(m=m, opt=opt):
            opt.zero_grad(set_to_none=True)
            kp3d = m(images, proj, batch)[0]
            torch.abs(kp3d - target).mean().backward()
            opt.step()
        runs["backbone " + bb] = step
    return _alternate(steps, rounds, runs, "algebraic training step (ResNet-152, B=5, V=4, 384^2, conf, Adam)")


def volumetric_step_timing(steps, rounds):
    B, V, S = 5, 4, 384
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    loss_fn = ce.VolumetricCELoss(backend="native")
    torch.manual_seed(0)
    runs, sd = {}, None
    for bb in ("torch", "native"):
        for v2v in ("torch", "native"):
            m = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=152, volume_size=64), device=DEV, backend="hybrid",
                                                   backbone_backend=bb, v2v_backend=v2v)
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
            runs["backbone %s / v2v %s" % (bb, v2v)] = step
    return _alternate(steps, rounds, runs, "volumetric training step (ResNet-152, B=5, V=4, 384^2, 64^3, Adam)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", default="20,32")
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("backbone_train_timing.py needs a CUDA device")
    name, q = card()
    print("device: %s, power limit, max SM clock: %s" % (name, q))
    out = {"device": name, "power_limit_max_sm_clock": q,
           "backbone": backbone_timing(a.iters, a.rounds, [int(b) for b in a.batches.split(",")])}
    out["profile"] = profile_table(os.path.dirname(os.path.abspath(a.json)) if a.json else None)
    if not a.no_step:
        out["algebraic_step"] = algebraic_step_timing(a.steps, a.rounds)
        torch.cuda.empty_cache()
        out["volumetric_step"] = volumetric_step_timing(a.steps, a.rounds)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
