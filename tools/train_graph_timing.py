#!/usr/bin/env python
"""Time hybrid training steps eager against CUDA-graphed (train_graph=True).

    python tools/train_graph_timing.py [--steps N] [--rounds N] [--profile-steps N] [--json OUT]

Prints the card name, power limit and max SM clock, then for
  1. the recipe volumetric step (ResNet-152, B = 5, V = 4, 384^2, 64^3, 0.1 MAE + 0.01 CE, Adam) and
  2. the algebraic step (ResNet-152 with confidences, B = 5, V = 4, 384^2, MAE, Adam),
each with all native switches (backbone, V2V, norm) and with all torch switches, torch's default TF32 settings:
  - per variant alone: the first step's loss from the same state and seed (eager and graphed must agree), the first step's time
    (for the graphed variant it includes the warm-up and the two captures; the capture cost is that minus the steady step time)
    and the peak memory of the model, its optimizer and its steps;
  - eager and graphed alternated --rounds times, CUDA-event medians of --steps steps per round;
  - from a separate torch.profiler run of --profile-steps graphed steps: the device-busy share of the step's wall time and the
    launches per step that stay eager (kernels, copies and memsets outside the graphs: the loss, AccumulateGrad and Adam).
Needs a CUDA device; it does not fall back to anything.
"""
import argparse
import gc
import json
import os
import statistics
import sys
import time
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import lt_b200  # noqa: E402
from lt_b200 import loss as ce, testing  # noqa: E402
from v2v_train_timing import DEV, card, event_median  # noqa: E402

B, V, S = 5, 4, 384
SWITCHES = {"native": dict(backbone_backend="native", norm_backend="native"), "torch": {}}


def volumetric_workload():
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    loss_fn = ce.VolumetricCELoss(backend="native")
    torch.manual_seed(0)
    state = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=152, volume_size=64), device="cpu",
                                               backend="hybrid").state_dict()

    def make(switches, graph):
        sw = dict(SWITCHES[switches], **({"v2v_backend": "native"} if switches == "native" else {}))
        m = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=152, volume_size=64), device="cpu", backend="hybrid",
                                               train_graph=graph, **sw)
        m.load_state_dict(state)
        return m.to(DEV).train()

    def loss(m):
        kp, _, vols, _, _, coord, _ = m(images, None, batch)
        mae = (torch.abs(kp_gt - kp) * valid).sum() / (3 * valid.sum())
        return 0.1 * mae + 0.01 * loss_fn(coord, vols, kp_gt, valid)
    return make, loss


def algebraic_workload():
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    images = images.to(DEV)
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)
    gt = torch.from_numpy(np.stack(batch["keypoints_3d"])).float().to(DEV)
    kp_gt, valid = gt[..., :3], gt[..., 3:]
    torch.manual_seed(0)
    state = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=152), device="cpu", backend="hybrid").state_dict()

    def make(switches, graph):
        m = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=152), device="cpu", backend="hybrid",
                                              train_graph=graph, **SWITCHES[switches])
        m.load_state_dict(state)
        return m.to(DEV).train()

    def loss(m):
        kp3d = m(images, proj, batch)[0]
        return (torch.abs(kp_gt - kp3d) * valid).sum() / (3 * valid.sum())
    return make, loss


def stepper(m, loss):
    opt = torch.optim.Adam(m.parameters(), lr=1e-4)
    seed = [0]

    def step():
        np.random.seed(seed[0])
        seed[0] += 1
        opt.zero_grad(set_to_none=True)
        out = loss(m)
        out.backward()
        opt.step()
        return out
    return step


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def alone(make, loss, switches, graph, steps):
    """First-step loss and time, steady median and peak memory of one variant on an otherwise empty device."""
    _free()
    torch.cuda.reset_peak_memory_stats()
    m = make(switches, graph)
    step = stepper(m, loss)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first_loss = float(step())
    torch.cuda.synchronize()
    first_ms = (time.perf_counter() - t0) * 1e3
    steady = event_median(step, steps, warmup=1)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del m, step
    return {"first_loss": first_loss, "first_step_ms": first_ms, "steady_ms": steady, "peak_GiB": peak}


def alternated(make, loss, switches, steps, rounds, label):
    runs = {"eager": stepper(make(switches, False), loss), "graphed": stepper(make(switches, True), loss)}
    res = defaultdict(list)
    for r in range(rounds):
        for key, step in runs.items():
            res[key].append(event_median(step, steps, warmup=1))
            print("%s round %d, %s: %.2f ms" % (label, r, key, res[key][-1]), flush=True)
    med = {k: statistics.median(v) for k, v in res.items()}
    print("%s, median of rounds: %s" % (label, ", ".join("%s %.2f ms [%.2f-%.2f]" % (k, med[k], min(res[k]), max(res[k])) for k in runs)))
    del runs
    return {"rounds_ms": dict(res), "median_ms": med}


def _union_us(intervals):
    total, end = 0.0, -1e30
    for a, b in sorted(intervals):
        if b > end:
            total += b - max(a, end)
            end = b
    return total


def profile(make, loss, switches, steps):
    """Device-busy share of the graphed step's wall time and the eager launches per step, from one torch.profiler run."""
    from torch.profiler import ProfilerActivity, profile as tprofile
    _free()
    step = stepper(make(switches, True), loss)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
        wall_us = (time.perf_counter() - t0) * 1e6
    events = prof.events()
    device = [(e.time_range.start, e.time_range.end) for e in events if e.device_type == torch.autograd.DeviceType.CUDA]
    calls = defaultdict(int)
    for e in events:
        if e.name in ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx", "cudaMemcpyAsync",
                      "cudaMemsetAsync", "cudaGraphLaunch"):
            calls[e.name] += 1
    busy = _union_us(device)
    eager = sum(n for k, n in calls.items() if k != "cudaGraphLaunch")
    out = {"wall_ms_per_step": wall_us / steps / 1e3, "device_busy_ms_per_step": busy / steps / 1e3, "device_share": busy / wall_us,
           "eager_launches_per_step": eager / steps, "calls_per_step": {k: v / steps for k, v in calls.items()}}
    del step
    return out


def workload(name, factory, steps, rounds, profile_steps):
    make, loss = factory()
    out = {}
    for switches in ("native", "torch"):
        label = "%s step, %s switches" % (name, switches)
        res = {v: alone(make, loss, switches, v == "graphed", steps) for v in ("eager", "graphed")}
        for v, r in res.items():
            print("%s, %s alone: first-step loss %.9g, first step %.1f ms, steady %.2f ms, peak %.2f GiB"
                  % (label, v, r["first_loss"], r["first_step_ms"], r["steady_ms"], r["peak_GiB"]), flush=True)
        cap = res["graphed"]["first_step_ms"] - res["graphed"]["steady_ms"]
        rel = abs(res["graphed"]["first_loss"] - res["eager"]["first_loss"]) / abs(res["eager"]["first_loss"])
        print("%s: capture cost %.0f ms; first-step loss graphed vs eager: relative difference %.2e" % (label, cap, rel))
        res["capture_ms"], res["first_loss_rel_diff"] = cap, rel
        _free()
        res["alternated"] = alternated(make, loss, switches, steps, rounds, label)
        _free()
        res["profile"] = profile(make, loss, switches, profile_steps)
        p = res["profile"]
        print("%s, graphed under torch.profiler: wall %.2f ms/step, device busy %.2f ms/step (%.1f %%), eager launches per step %.0f %s"
              % (label, p["wall_ms_per_step"], p["device_busy_ms_per_step"], 100 * p["device_share"], p["eager_launches_per_step"],
                 p["calls_per_step"]), flush=True)
        out[switches] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--only", choices=["volumetric", "algebraic"])
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_graph_timing.py needs a CUDA device")
    name, q = card()
    print("device: %s, power limit, max SM clock: %s" % (name, q), flush=True)
    out = {"device": name, "power_limit_max_sm_clock": q}
    for wl, factory in (("volumetric", volumetric_workload), ("algebraic", algebraic_workload)):
        if a.only in (None, wl):
            out[wl] = workload(wl, factory, a.steps, a.rounds, a.profile_steps)
            _free()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
