#!/usr/bin/env python
"""Time the V2V network's training passes with the native convolutions (v2v_backend="native": autograd_ops.ConvNdFn /
ConvTranspose3dFn) against cuDNN.

    python tools/v2v_train_timing.py [--iters N] [--steps N] [--rounds N] [--no-step] [--json OUT]

Prints the card name, power limit and max SM clock, then:
  1. V2V forward + backward at the recipe shape (human36m_vol_softmax.yaml: B = 5, 64^3, 32 input channels, 17 joints, train-mode
     BatchNorm), CUDA-event medians of three configurations alternated --rounds times: native; cuDNN fp32 (TF32 off); cuDNN with
     torch's default TF32 -- with torch.cuda.max_memory_allocated of each;
  2. a per-class kernel table of one native forward + backward from a separate torch.profiler run, with the algorithmic FLOP/s of
     the convolution classes (counted from the layer shapes) against the 989 TFLOP/s dense fp16 figure of the H100 SXM data sheet;
  3. one recipe-shaped training step (ResNet-152 volumetric model, backend="hybrid", B = 5, V = 4, 384^2, train mode,
     0.1 MAE + 0.01 CE, Adam) with v2v_backend "torch" and "native" alternated --rounds times, with peak memory of each, and the
     V2V forward + backward time (cuDNN, TF32) as a share of the torch step.
Needs a CUDA device; it does not fall back to anything.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import autograd_ops as A, loss as ce, testing  # noqa: E402
from lt_b200.v2v import V2VModel  # noqa: E402

DEV = "cuda:0"
FP16_DENSE_PEAK = 989e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def event_median(fn, iters, warmup=2):
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


class _Tf32:
    def __init__(self, on):
        self.on = on

    def __enter__(self):
        self.saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = self.on

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.saved


def v2v_problem(B=5, n=64):
    torch.manual_seed(0)
    net = V2VModel(32, 17).to(DEV).train()
    x = torch.randn(B, 32, n, n, n, device=DEV).contiguous(memory_format=torch.channels_last_3d)
    g = torch.randn(B, 17, n, n, n, device=DEV) * 1e-4
    return net, x, g


def v2v_step(net, x, g, conv):
    net.zero_grad(set_to_none=True)
    xi = x.detach().requires_grad_(True)
    net(xi, conv).backward(g)


CONFIGS = {"native": (A.v2v_conv, False), "cudnn_fp32": (None, False), "cudnn_tf32": (None, True)}


def v2v_timing(iters, rounds):
    net, x, g = v2v_problem()
    res = defaultdict(list)
    mem = {}
    for r in range(rounds):
        for name, (conv, tf32) in CONFIGS.items():
            with _Tf32(tf32):
                torch.cuda.reset_peak_memory_stats()
                res[name].append(event_median(lambda: v2v_step(net, x, g, conv), iters))
                mem[name] = torch.cuda.max_memory_allocated() / 2 ** 30
            print("V2V fwd+bwd round %d %-10s %.2f ms" % (r, name, res[name][-1]))
    med = {k: statistics.median(v) for k, v in res.items()}
    print("V2V fwd+bwd (B=5, 64^3, 32 -> 17, train BN), median of rounds: " +
          ", ".join("%s %.2f ms (peak %.2f GiB)" % (k, med[k], mem[k]) for k in CONFIGS))
    return {"rounds": dict(res), "median_ms": med, "peak_GiB": mem}


def conv_flops(net, x):
    """Algorithmic FLOPs of every Conv3d / ConvTranspose3d forward at this input (2 x MACs); wgrad and dgrad count the same."""
    total = [0.0]

    def hook(m, inp, out):
        w = m.weight
        if isinstance(m, torch.nn.ConvTranspose3d):
            total[0] += 2.0 * inp[0].numel() / inp[0].shape[1] * w.numel()
        else:
            total[0] += 2.0 * out.numel() / out.shape[1] * w.numel()
    hs = [m.register_forward_hook(hook) for m in net.modules() if isinstance(m, (torch.nn.Conv3d, torch.nn.ConvTranspose3d))]
    with torch.no_grad():
        net(x)
    for h in hs:
        h.remove()
    return total[0]


def kernel_class(name):
    n = name.lower()
    if "conv_wgrad" in n or "wgrad_reduce" in n:
        return "wgrad (conv_wgrad_kernel + reduce)"
    if "conv_fold" in n:
        return "forward + dgrad on conv_fold_kernel"
    if "conv_tc_kernel" in n or "splitk_reduce" in n:
        return "forward + dgrad on conv_tc_kernel"
    if any(k in n for k in ("f32_to_s32", "s32_to_f32", "absmax", "gather_weights", "pack_weights", "fold_bn")):
        return "conversions + filter packing"
    if "batch_norm" in n or "bn_" in n or "welford" in n:
        return "torch BatchNorm"
    if "max_pool" in n or "pool" in n:
        return "torch max-pool"
    return "torch other (ReLU, adds, sums, copies)"


def profile_table(out_dir):
    net, x, g = v2v_problem()
    flops = conv_flops(net, x)
    for _ in range(2):
        v2v_step(net, x, g, A.v2v_conv)
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        v2v_step(net, x, g, A.v2v_conv)
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
        prof.export_chrome_trace(os.path.join(out_dir, "v2v_train_native_trace.json"))
    conv_t = times["forward + dgrad on conv_fold_kernel"] + times["forward + dgrad on conv_tc_kernel"]
    rows = []
    print("per-class device time of one native V2V forward + backward (torch.profiler), algorithmic conv FLOPs %.1f GFLOP per pass:"
          % (flops / 1e9))
    for k, t in sorted(times.items(), key=lambda kv: -kv[1]):
        rate = ""
        if k.startswith("wgrad") and t > 0:
            rate = "%.1f TFLOP/s = %.1f %% of 989" % (flops / t / 1e9, 100 * flops / t / 1e9 / 989)
        print("  %-42s %8.2f ms  %s" % (k, t, rate))
        rows.append({"class": k, "ms": t})
    if conv_t > 0:
        print("  forward + dgrad classes together: %.1f TFLOP/s = %.1f %% of 989 (2 x %.1f GFLOP)"
              % (2 * flops / conv_t / 1e9, 100 * 2 * flops / conv_t / 1e9 / 989, flops / 1e9))
    return {"conv_gflop_per_pass": flops / 1e9, "classes": rows}


def training_step_timing(steps, rounds, v2v_share_ms):
    B, V, S = 5, 4, 384
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    loss_fn = ce.VolumetricCELoss(backend="native")
    torch.manual_seed(0)
    models = {}
    for v2v in ("torch", "native"):
        m = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=152, volume_size=64), device=DEV, backend="hybrid",
                                               v2v_backend=v2v)
        if models:
            m.load_state_dict(models["torch"][0].state_dict())
        m = m.to(DEV).train()
        models[v2v] = (m, torch.optim.Adam(m.parameters(), lr=1e-4))

    def step(which):
        m, opt = models[which]
        opt.zero_grad(set_to_none=True)
        kp, _, vols, _, _, coord, _ = m(images, None, batch)
        mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
        (0.1 * mae + 0.01 * loss_fn(coord, vols, kp_gt, valid)).backward()
        opt.step()

    res, mem = {"torch": [], "native": []}, {}
    for r in range(rounds):
        for which in ("torch", "native"):
            torch.cuda.reset_peak_memory_stats()
            t = event_median(lambda: step(which), steps, warmup=2)
            mem[which] = torch.cuda.max_memory_allocated() / 2 ** 30
            res[which].append(t)
            print("training step round %d, v2v_backend=%s: median %.2f ms over %d steps" % (r, which, t, steps))
    med = {k: statistics.median(v) for k, v in res.items()}
    print("training step (ResNet-152, B=5, V=4, 384^2, hybrid, Adam, TF32 default): v2v torch %.2f ms (peak %.2f GiB), "
          "v2v native %.2f ms (peak %.2f GiB)" % (med["torch"], mem["torch"], med["native"], mem["native"]))
    print("V2V forward + backward alone (cuDNN, TF32) = %.1f %% of the v2v_backend='torch' step" % (100 * v2v_share_ms / med["torch"]))
    return {"rounds": res, "median_ms": med, "peak_GiB": mem, "v2v_share_of_torch_step": v2v_share_ms / med["torch"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-step", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("v2v_train_timing.py needs a CUDA device")
    name, q = card()
    print("device: %s, power limit, max SM clock: %s" % (name, q))
    out = {"device": name, "power_limit_max_sm_clock": q, "v2v": v2v_timing(a.iters, a.rounds)}
    out["profile"] = profile_table(os.path.dirname(os.path.abspath(a.json)) if a.json else None)
    if not a.no_step:
        out["training_step"] = training_step_timing(a.steps, a.rounds, out["v2v"]["median_ms"]["cudnn_tf32"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
