#!/usr/bin/env python
"""Time what torch.use_deterministic_algorithms(True) changes in a volumetric training step.

    python tools/deterministic_timing.py [--rounds N] [--reps N] [--steps N] [--skip-step] [--json OUT]

1. The unprojection backward, atomic (lt_unproject_aggregate_bwd) against fixed-order (lt_unproject_aggregate_bwd_det), per
   aggregation, at the recipe's shapes: B = 5, V = 4, 96^2 maps, C = 32, 64^3 voxels, ring cameras around a 2.8 m cuboid.  The
   fixed-order time includes its workspace allocation and fill (under the flag torch fills every torch.empty).
2. V2V's first pool backward, (5, 32, 64^3) channels_last_3d: native lt_maxpool3d_bwd (flag on) against torch's (flag off).
3. The recipe volumetric lt_b200.TrainStep (ResNet-152, 384^2, all native switches), flag off, on, and off again.
1 and 2: CUDA-event medians of --reps calls per round, the two sides alternated over --rounds rounds.  3: host-clock medians of
--steps replays ending in a synchronise, after the capture.  Peak memory for each.  Prints the card name and power limit first;
needs a CUDA device and does not fall back.
"""
import os

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")     # torch's requirement for deterministic cuBLAS

import argparse  # noqa: E402
import gc  # noqa: E402
import json  # noqa: E402
import statistics  # noqa: E402
import sys  # noqa: E402
import time  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import capi, testing  # noqa: E402
from oracle import vol_oracle as O  # noqa: E402
from v2v_train_timing import DEV, card  # noqa: E402

B, V, C, H, W, N = 5, 4, 32, 96, 96, 64


def _free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def event_median(fn, reps):
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def peak_of(fn):
    _free()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def alternate(sides, rounds, reps, label):
    for fn in sides.values():
        fn()
    res = {k: [] for k in sides}
    for r in range(rounds):
        for k, fn in sides.items():
            res[k].append(event_median(fn, reps))
    med = {k: statistics.median(v) for k, v in res.items()}
    peak = {k: peak_of(fn) for k, fn in sides.items()}
    print("%s: %s" % (label, ", ".join("%s %.3f ms [%.3f-%.3f], peak +%.0f MiB" % (k, med[k], min(res[k]), max(res[k]), peak[k])
                                      for k in sides)), flush=True)
    return {"rounds_ms": res, "median_ms": med, "peak_extra_MiB": peak}


def unprojection_inputs(seed=0):
    rng = np.random.RandomState(seed)
    cams = testing.make_cameras(V, image_size=384, radius=3000.0)
    proj = np.stack([np.stack([O.projection_after_resize(c.K, c.R, c.t, (384, 384), (H, W)) for c in cams])] * B)
    coord = np.stack([O.coord_volume(rng.randn(3) * 100 + [0, 0, 900], 2800.0, N).reshape(-1, 3) for _ in range(B)])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(DEV)
    feats = torch.randn(B, V, H, W, C, device=DEV)
    conf = torch.rand(B, V, C, device=DEV)
    g = torch.randn(B, N ** 3, C, device=DEV)
    return feats, t(proj).reshape(B, V, 12).contiguous(), t(coord), conf, g


def unprojection(rounds, reps):
    feats, proj, coord, conf, g = unprojection_inputs()
    nvox = coord.shape[1]
    out = {}
    for agg in ("sum", "max", "softmax", "conf"):
        a = capi.AGG[agg]
        cf = conf if agg == "conf" else None
        gf = torch.zeros_like(feats)
        gc = torch.zeros(B, V, C, device=DEV) if agg == "conf" else None

        def atomic():
            gf.zero_()
            if gc is not None:
                gc.zero_()
            capi.unproject_aggregate_bwd(feats, proj, coord, cf, g, gf, gc, a)

        def fixed():
            torch.use_deterministic_algorithms(True)
            try:
                gf.zero_()
                if gc is not None:
                    gc.zero_()
                ws = torch.empty(capi.unproject_aggregate_bwd_det_workspace_bytes(B, V, C, H, W, nvox, a, False), dtype=torch.uint8,
                                 device=DEV)
                capi.unproject_aggregate_bwd_det(feats, proj, coord, cf, g, gf, gc, None, None, a, ws)
            finally:
                torch.use_deterministic_algorithms(False)
        out[agg] = alternate({"atomic": atomic, "fixed-order": fixed}, rounds, reps, "unprojection backward %s" % agg)
    return out


def pool(rounds, reps):
    x = torch.randn(B, 32, N, N, N, device=DEV).contiguous(memory_format=torch.channels_last_3d).requires_grad_(True)
    gy = torch.randn(B, 32, N // 2, N // 2, N // 2, device=DEV).contiguous(memory_format=torch.channels_last_3d)
    y_torch = F.max_pool3d(x, 2, 2)
    torch.use_deterministic_algorithms(True)
    y_native = lt_b200.v2v.Pool3DBlock(2)(x)
    torch.use_deterministic_algorithms(False)

    def torch_bwd():
        torch.autograd.grad(y_torch, x, gy, retain_graph=True)

    def native_bwd():
        torch.autograd.grad(y_native, x, gy, retain_graph=True)
    return alternate({"torch (flag off)": torch_bwd, "native (flag on)": native_bwd}, rounds, reps, "V2V pool backward")


def train_step(steps):
    from train_step_timing import volumetric_workload, stepper
    make, b = volumetric_workload()
    out = {}
    for label, flag in (("off", False), ("on", True), ("off again", False)):
        _free()
        torch.use_deterministic_algorithms(flag)
        try:
            torch.cuda.reset_peak_memory_stats()
            step = stepper(make, "step", b)
            step()
            times = []
            for _ in range(steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                step()
                torch.cuda.synchronize()
                times.append((time.perf_counter() - t0) * 1e3)
            out[label] = {"median_ms": statistics.median(times), "min_ms": min(times), "max_ms": max(times),
                          "peak_GiB": torch.cuda.max_memory_allocated() / 2 ** 30}
            del step
        finally:
            torch.use_deterministic_algorithms(False)
        print("TrainStep, flag %s: %.2f ms [%.2f-%.2f], peak %.2f GiB" % (label, out[label]["median_ms"], out[label]["min_ms"],
                                                                      out[label]["max_ms"], out[label]["peak_GiB"]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("deterministic_timing needs a CUDA device")
    res = {"card": card()}
    print(res["card"], flush=True)
    torch.backends.cudnn.benchmark = False
    res["unprojection"] = unprojection(args.rounds, args.reps)
    res["pool"] = pool(args.rounds, args.reps)
    if not args.skip_step:
        res["train_step"] = train_step(args.steps)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
