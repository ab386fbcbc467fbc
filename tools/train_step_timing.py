#!/usr/bin/env python
"""Time the train.py loop body against lt_b200.TrainStep on the two recipe workloads.

    python tools/train_step_timing.py [--steps N] [--rounds N] [--profile-steps N] [--only volumetric|algebraic] [--json OUT]

Workloads (all native switches, torch's default TF32 settings):
  volumetric  ResNet-152, B = 5, V = 4, 384^2, 64^3, MAE + 0.01 CE, scale 0.1, the per-module lrs of human36m_vol_softmax.yaml
  algebraic   ResNet-152 with confidences, B = 8, V = 4, 384^2, MSESmooth 400, scale 0.1 (native backbone and norm)
Two ways of running a step, alternated --rounds times:
  (a) "loop"   the train.py loop body restated (testing.reference_train_step) on a model with train_graph=True: the reference
               criterion formula, the CE loss, every .item() of the loop, the per-parameter .item() gradient norm, clip and Adam;
  (b) "step"   lt_b200.TrainStep: everything after the host geometry in one CUDA graph, nothing read back.
Per round and way: the median of --steps step times, each a host clock around one step that ends in torch.cuda.synchronize().
Per way alone: the first call (for (b) the warm-up and the capture; the capture cost is that minus the steady step time) and the
peak memory.  From a separate torch.profiler run of each: the launches per step outside CUDA graphs and the share of the step's
wall time the device is busy.  Prints the card name and power limit first; needs a CUDA device and does not fall back.
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

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import testing  # noqa: E402
from train_graph_timing import _union_us  # noqa: E402
from v2v_train_timing import DEV, card  # noqa: E402

V, S = 4, 384


def volumetric_workload():
    cfg = lambda: testing.make_train_config(testing.make_config(num_layers=152, volume_size=64), criterion="MAE", lr=1e-4,
                                            use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01, scale_keypoints_3d=0.1,
                                            process_features_lr=1e-3, volume_net_lr=1e-3)
    torch.manual_seed(0)
    state = lt_b200.VolumetricTriangulationNet(cfg(), device="cpu", backend="hybrid").state_dict()

    def make(graph):
        c = cfg()
        m = lt_b200.VolumetricTriangulationNet(c, device="cpu", backend="hybrid", train_graph=graph, backbone_backend="native",
                                               v2v_backend="native", norm_backend="native")
        m.load_state_dict(state)
        return m.to(DEV).train(), c
    return make, 5


def algebraic_workload():
    cfg = lambda: testing.make_train_config(testing.make_alg_config(num_layers=152, use_confidences=True), criterion="MSESmooth",
                                            lr=1e-5, mse_smooth_threshold=400, scale_keypoints_3d=0.1)
    torch.manual_seed(0)
    state = lt_b200.AlgebraicTriangulationNet(cfg(), device="cpu", backend="hybrid").state_dict()

    def make(graph):
        c = cfg()
        m = lt_b200.AlgebraicTriangulationNet(c, device="cpu", backend="hybrid", train_graph=graph, backbone_backend="native",
                                              norm_backend="native")
        m.load_state_dict(state)
        return m.to(DEV).train(), c
    return make, 8


def stepper(make, way, B):
    """-> a function that runs one step of `way` ("loop" or "step") on a fresh model and returns a Python float (the loss)."""
    m, cfg = make(way == "loop")
    opt = testing.recipe_optimizer(m, cfg, capturable=way == "step")      # train.py's plain Adam for the loop
    images, batch = testing.make_batch(B, V, image_size=S, seed=1)
    data = testing.prepare_batch(batch, images, DEV) + (batch,)
    seed = [0]
    train_step = lt_b200.TrainStep(m, opt, cfg) if way == "step" else None

    def step():
        np.random.seed(seed[0])
        seed[0] += 1
        if way == "loop":
            return testing.reference_train_step(m, opt, cfg, *data)[1]["total_loss"]
        return train_step(*data)[1]["total_loss"]
    return step


def timed(step, n):
    """Median and all of n host-clock step times (ms), each ending in a synchronise."""
    times = []
    for _ in range(n):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times), times


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def alone(make, way, B, steps):
    _free()
    torch.cuda.reset_peak_memory_stats()
    step = stepper(make, way, B)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first_loss = float(step())
    torch.cuda.synchronize()
    first_ms = (time.perf_counter() - t0) * 1e3
    steady = timed(step, steps)[0]
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del step
    return {"first_loss": first_loss, "first_call_ms": first_ms, "steady_ms": steady, "peak_GiB": peak}


def alternated(make, B, steps, rounds, label):
    runs = {w: stepper(make, w, B) for w in ("loop", "step")}
    for s in runs.values():
        for _ in range(2):
            s()
    res = defaultdict(list)
    for r in range(rounds):
        for w, s in runs.items():
            res[w].append(timed(s, steps)[0])
            print("%s round %d, %s: %.2f ms" % (label, r, w, res[w][-1]), flush=True)
    med = {w: statistics.median(v) for w, v in res.items()}
    print("%s, median of rounds: %s; loop / step %.3f" % (label, ", ".join("%s %.2f ms [%.2f-%.2f]" % (w, med[w], min(res[w]),
                                                                          max(res[w])) for w in runs), med["loop"] / med["step"]))
    del runs
    return {"rounds_ms": dict(res), "median_ms": med}


def profile(make, way, B, steps):
    from torch.profiler import ProfilerActivity, profile as tprofile
    _free()
    step = stepper(make, way, B)
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
    busy = _union_us([(e.time_range.start, e.time_range.end) for e in events if e.device_type == torch.autograd.DeviceType.CUDA])
    calls = defaultdict(int)
    for e in events:
        if e.name in ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx", "cudaMemcpyAsync",
                      "cudaMemsetAsync", "cudaGraphLaunch", "cudaStreamSynchronize", "cudaMemcpy"):
            calls[e.name] += 1
    eager = sum(n for k, n in calls.items() if k not in ("cudaGraphLaunch", "cudaStreamSynchronize"))
    del step
    return {"wall_ms_per_step": wall_us / steps / 1e3, "device_share": busy / wall_us, "eager_launches_per_step": eager / steps,
            "calls_per_step": {k: v / steps for k, v in calls.items()}}


def workload(name, factory, steps, rounds, profile_steps):
    make, B = factory()
    out = {}
    for way in ("loop", "step"):
        r = out[way] = alone(make, way, B, steps)
        print("%s, %s alone: first-call loss %.9g, first call %.1f ms, steady %.2f ms, peak %.2f GiB"
              % (name, way, r["first_loss"], r["first_call_ms"], r["steady_ms"], r["peak_GiB"]), flush=True)
    out["capture_ms"] = out["step"]["first_call_ms"] - out["step"]["steady_ms"]
    out["first_loss_rel_diff"] = abs(out["step"]["first_loss"] - out["loop"]["first_loss"]) / abs(out["loop"]["first_loss"])
    print("%s: TrainStep capture %.0f ms; first-step total loss, step vs loop: relative difference %.2e"
          % (name, out["capture_ms"], out["first_loss_rel_diff"]), flush=True)
    _free()
    out["alternated"] = alternated(make, B, steps, rounds, name)
    for way in ("loop", "step"):
        _free()
        p = out[way]["profile"] = profile(make, way, B, profile_steps)
        print("%s, %s under torch.profiler: wall %.2f ms/step, device busy %.1f %%, eager launches per step %.0f %s"
              % (name, way, p["wall_ms_per_step"], 100 * p["device_share"], p["eager_launches_per_step"], p["calls_per_step"]),
              flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--only", choices=["volumetric", "algebraic"])
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_step_timing.py needs a CUDA device")
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
