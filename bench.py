#!/usr/bin/env python
"""Benchmark of the volumetric-triangulation hot path (BASELINE.json metric: volumetric samples/sec).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl native|reference] [--mode tc|tc1|simt]

One "step" = one eval forward of a batch of synthetic multi-view samples (4 views of 3x384x384 -> 17 joints,
ResNet-152 backbone, 64^3 grid, softmax aggregation: BASELINE config #2, batch 8 per GPU) through the native
sm_90a path.  Prints ONE JSON line (rank 0).  See the module docstrings / DESIGN.md for the field definitions.

  value     device-timed throughput, inputs resident in HBM (CUDA events around K graph replays, max over ranks)
  e2e       same metric through the public nn.Module call with pinned-host images copied H2D and the keypoints
            read back D2H inside the timed region
  roofline  dominant kernel (tensor-core conv): algorithmic conv FLOPs / summed per-launch CUDA-event time, vs the
            measured dense bf16 peak (MEASURED_PEAKS.json); unprojection / soft-argmax HBM rooflines alongside
  cpu_baseline  the CPU oracle port of the reference path timed on this box's host cores (rank 0, bounded sample)

--impl reference times the reference's CPU implementation of the path (the oracle port: the reference is pure
Python and is not present on the GPU box) with all host threads, same metric/config.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "volumetric samples/sec (4-view 384x384, 64^3 grid)"


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="native", choices=["native", "reference", "torch_gpu"],
                    help="native: this repo's kernels; reference: the CPU oracle port of the reference path (contract arm); torch_gpu: the "
                         "same torch formulation as the reference on cuda:0 through ATen/cuDNN (secondary bar of SURVEY 8d, not a contract arm)")
    ap.add_argument("--tf32", action="store_true", help="torch_gpu only: allow TF32 in cuDNN / matmul (default: true fp32)")
    ap.add_argument("--mode", default=os.environ.get("LT_B200_CONV", "tc"), choices=["tc", "tc1", "simt"])
    ap.add_argument("--batch", type=int, default=8, help="samples per GPU per step")
    ap.add_argument("--views", type=int, default=4)
    ap.add_argument("--image", type=int, default=384)
    ap.add_argument("--volume", type=int, default=64)
    ap.add_argument("--layers", type=int, default=152)
    ap.add_argument("--collective", default="both", choices=["both", "all_reduce", "reduce_scatter", "p2p", "features"],
                    help="view-group exchange(s) to measure at N > 1: both = the NCCL all-reduce contract path AND the feature-map exchange "
                         "(value = the faster one, both reported under `exchanges`)")
    ap.add_argument("--no-config4", action="store_true", help="N = 8 only: skip the extra 8-view / one-view-per-GPU measurement")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-config5", action="store_true", help="N = 1 only: skip the extra line for BASELINE config #5 (algebraic model)")
    ap.add_argument("--no-torch-gpu", action="store_true", help="skip the ATen/cuDNN secondary bars (fp32 and TF32) of the native arm")
    ap.add_argument("--no-calibrate", action="store_true", help="keep PyTorch default init (faster start, degenerate signal)")
    ap.add_argument("--dump-outputs", metavar="DIR", help="single-GPU native arm: write the outputs of the last timed step as DIR/<name>.npy")
    return ap.parse_args()


def peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        p = json.load(open(path))
        return {"hbm_gbs": p["hbm_gbs"], "bf16_tflops": p.get("bf16_tflops_sustained", p["bf16_tflops"]), "src": "measured"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "src": "H100 SXM data sheet (700 W)"}


class ClockSampler(threading.Thread):
    """nvidia-smi clock / throttle-reason samples during the timed region."""

    def __init__(self, index):
        super().__init__(daemon=True)
        self.index, self.stop_flag, self.rows = index, threading.Event(), []

    def run(self):
        q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        while not self.stop_flag.is_set():
            try:
                out = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits"],
                                     capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:
                pass
            self.stop_flag.wait(0.2)

    def summary(self):
        self.stop_flag.set()
        self.join(timeout=6)
        if not self.rows:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["unavailable"]}
        sm = sorted(float(r[0]) for r in self.rows if r[0].replace(".", "").isdigit())
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for i, n in enumerate(names) if any(len(r) > 2 + i and r[2 + i].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": float(self.rows[0][1]) if self.rows[0][1].isdigit() else None,
                "reasons": reasons, "samples": len(self.rows)}


def cpu_oracle_rate(args, steps, sd=None, images=None, batch=None):
    """samples/sec of the CPU oracle port of the reference path on this box's host cores.

    Bounded sample of the SAME workload: one untimed warm-up forward of one sample, then `steps` timed forwards of a
    whole batch (args.batch samples, ~20 s each for config #2 on 32 threads).  With `sd/images/batch` given (the
    native arm's own weights and inputs) the last forward's outputs are returned as well, for the parity object.
    """
    from oracle import parity
    import lt_b200
    from lt_b200 import testing
    # all host threads the reference can use productively: intra-op scaling of fp32 convs flattens (and on shared,
    # oversubscribed hosts reverses) beyond ~32 threads; LT_BENCH_CPU_THREADS overrides
    torch.set_num_threads(int(os.environ.get("LT_BENCH_CPU_THREADS", min(os.cpu_count(), 32))))
    if sd is None:
        cfg = testing.make_config(num_layers=args.layers, volume_size=args.volume)
        sd = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend="torch").state_dict()   # parameter holder only
    if images is None:
        images, batch = testing.make_batch(args.batch, args.views, image_size=args.image, seed=0)
    B = images.shape[0]
    one = {k: ([c[:1] for c in v] if k == "cameras" else v[:1]) for k, v in batch.items()}
    parity.oracle_forward(sd, images[:1], one, args.volume)       # warm-up (thread pool, allocator)
    total, out = 0.0, None
    for _ in range(steps):
        out, secs = parity.oracle_forward(sd, images, batch, args.volume)
        total += secs
    dt = total / steps
    return B / dt, dt, torch.get_num_threads(), out


def main_reference(args, rank):
    if rank != 0:
        return
    steps, warmup = max(1, min(args.steps, 2)), 1
    rate, dt, threads, _ = cpu_oracle_rate(args, steps)
    line = {
        "impl": "reference", "metric": METRIC, "value": rate, "unit": "samples/s", "n_gpus": args.gpus, "steps": steps,
        "warmup": warmup, "ms_per_step": dt * 1e3, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": "Volumetric(softmax) ResNet-%d, %d views %dx%d, %d^3 grid, batch %d per GPU"
                   % (args.layers, args.views, args.image, args.image, args.volume, args.batch),
                   "note": "CPU arm: %d timed forward(s) of one batch (bounded sample of the same workload), warm-up = one sample" % steps},
        "cpu_baseline": {"value": rate, "unit": "samples/s", "cores": threads, "kind": "port",
                         "sample": "%d timed forward(s) of a %d-sample batch of %d-view inputs, CPU oracle port (torch fp32 + numpy), %d of %d host threads"
                                   % (steps, args.batch, args.views, threads, os.cpu_count())},
        "e2e": {"value": rate, "unit": "samples/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def torch_gpu_rate(args, dev, sd, images_dev, batch, tf32, steps=None):
    """The reference formulation (torch ops through ATen/cuDNN, eval, no autograd) on `dev`: samples/s, CUDA-event timed."""
    import lt_b200
    from lt_b200 import testing
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark)
    torch.backends.cudnn.allow_tf32 = bool(tf32)
    torch.backends.cuda.matmul.allow_tf32 = bool(tf32)
    torch.backends.cudnn.benchmark = True
    try:
        cfg = testing.make_config(num_layers=args.layers, volume_size=args.volume)
        model = lt_b200.VolumetricTriangulationNet(cfg, device=dev, backend="torch")
        model.load_state_dict(sd)
        model = model.to(dev).eval()
        steps = steps or max(2, min(args.steps, 5))
        with torch.no_grad():
            for _ in range(3):
                model(images_dev, None, batch)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                model(images_dev, None, batch)
            e1.record()
            torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        del model
        torch.cuda.empty_cache()
        return {"value": images_dev.shape[0] / (ms / 1e3), "unit": "samples/s", "ms_per_step": ms, "steps": steps,
                "dtype": "tf32" if tf32 else "f32", "what": "same module with backend='torch' (ATen/cuDNN, cudnn.benchmark) on the same GPU, weights and inputs"}
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.benchmark = old


def algebraic_rate(args, dev, vol_model, images_dev, batch, flush):
    """BASELINE config #5: AlgebraicTriangulationNet (ResNet-152 heat-maps + confidence head + 2-D soft-argmax + weighted DLT,
    reference triangulation.py:131-200) on the native kernels, same images / cameras / backbone weights as the volumetric arm."""
    import lt_b200
    from lt_b200 import testing
    alg = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=args.layers), device=dev, backend="native", conv_mode=args.mode)
    alg.backbone.load_state_dict(vol_model.backbone.state_dict(), strict=False)     # shared trunk / deconvs / heat-map head
    alg = alg.to(dev).eval()
    proj = torch.as_tensor(np.ascontiguousarray(testing.image_projections(batch), dtype=np.float32)).to(dev)
    B = images_dev.shape[0]
    steps = max(3, min(args.steps, 10))
    with torch.no_grad():
        for _ in range(3):
            out = alg(images_dev, proj, batch)
        torch.cuda.synchronize()
        launches = alg.engine().launches
        evs = []
        for _ in range(steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = alg(images_dev, proj, batch)
            e1.record()
            evs.append((e0, e1))
        torch.cuda.synchronize()
    ms = sum(a.elapsed_time(b) for a, b in evs) / steps
    finite = bool(torch.isfinite(out[0]).all())
    del alg
    torch.cuda.empty_cache()
    return {"workload": "Algebraic model: ResNet-%d heat-maps + confidences + 2-D soft-argmax + weighted DLT, %d views %dx%d, batch %d, 1 GPU"
                        % (args.layers, images_dev.shape[1], args.image, args.image, B),
            "metric": "algebraic samples/sec", "value": B / (ms / 1e3), "unit": "samples/s", "ms_per_step": ms, "steps": steps,
            "gpu_launches_per_step": launches, "keypoints_finite": finite,
            "timing": "CUDA events around eager (graph-free) module calls, inputs resident, L2 flushed between steps"}


def main_torch_gpu(args, rank):
    """Secondary bar (SURVEY 8d): the reference's own formulation -- torch ops through ATen/cuDNN -- on one GPU, eval mode."""
    if rank != 0:
        return
    import lt_b200
    from lt_b200 import testing
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.allow_tf32 = bool(args.tf32)
    torch.backends.cuda.matmul.allow_tf32 = bool(args.tf32)
    torch.backends.cudnn.benchmark = True
    B, V, S, n = args.batch, args.views, args.image, args.volume
    cfg = testing.make_config(num_layers=args.layers, volume_size=n)
    torch.manual_seed(0)
    model = lt_b200.VolumetricTriangulationNet(cfg, device=dev, backend="torch")
    if not args.no_calibrate:
        testing.randomize_weights(model, seed=0, calib_size=S, calib_views=1)
    model = model.to(dev).eval()
    images, batch = testing.make_batch(B, V, image_size=S, seed=0)
    images_dev = images.to(dev)
    with torch.no_grad():
        for _ in range(max(args.warmup, 3)):
            model(images_dev, None, batch)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            model(images_dev, None, batch)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    print(json.dumps({"impl": "torch_gpu", "metric": METRIC, "value": B * args.steps / (ms / 1e3), "unit": "samples/s", "n_gpus": 1,
                      "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms / args.steps, "higher_is_better": True,
                      "dtype": "tf32" if args.tf32 else "f32", "data": "synthetic",
                      "config": {"workload": "Volumetric(softmax) ResNet-%d, %d views %dx%d, %d^3 grid, batch %d, torch ops (ATen/cuDNN) on cuda:0"
                                 % (args.layers, V, S, S, n, B)}}), flush=True)


EXCHANGE_TEXT = {
    "all_reduce": "packed (sum s*e^s, sum e^s) voxel partials completed by ONE NCCL all-reduce over the view group (north-star contract)",
    "reduce_scatter": "packed voxel partials completed by one NCCL reduce-scatter (each rank receives only its samples)",
    "p2p": "voxel partials stored into the owner rank by the unprojection kernel over NVLink peer memory",
    "features": "32-channel feature maps stored into the owner rank over NVLink peer memory (14x fewer bytes); the owner unprojects all views",
}


class ShardedArm:
    """One view-sharded configuration of the multi-GPU bench: `views` views per sample split over the ranks of a view group."""

    def __init__(self, args, model, world, rank, dev, views):
        from lt_b200 import dist as lt_dist, testing
        self.args, self.model, self.eng, self.dev, self.rank, self.world = args, model, model.engine(), dev, rank, world
        B, S = args.batch, args.image
        self.plan = plan = lt_dist.make_plan(world, rank, views)
        self.pg = lt_dist.new_view_groups(plan)
        self.Bg = Bg = B * plan.group_size
        self.images_g, self.batch = testing.make_batch(Bg, views, image_size=S, seed=100 + plan.group_index)
        self.images = self.images_g[:, plan.views].contiguous()
        self.pinned = self.images.pin_memory()
        self.images_dev = self.images.to(dev)
        from lt_b200.triangulation import backbone_map_size
        hm = (backbone_map_size(S), backbone_map_size(S))
        proj, base, position, stepv, rots, _ = model._host_geometry(self.batch, Bg, (S, S), hm)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(dev)
        self.geo = (up(proj[:, plan.views]), up(position), up(base), up(stepv), up(rots.reshape(Bg, 9)), up(proj))
        self.h2d = self.images.numel() * 4
        self.views = views

    def step(self, img, collective, graph=True):
        g = self.geo
        return self.eng.forward_view_sharded(img, g[0], g[1], g[2], g[3], g[4], self.plan, self.pg, collective, proj_all=g[5],
                                             use_graph=graph)[0]

    def _e2e_pipelined(self, collective, steps):
        """steps x (H2D of this rank's images -> view-sharded forward -> D2H of the key points), upload i+1 overlapping forward i."""
        main = torch.cuda.current_stream()
        if not hasattr(self, "_e2e_state"):
            self._e2e_state = (torch.cuda.Stream(device=self.dev), [torch.empty_like(self.images_dev) for _ in range(2)], [None, None])
        copy_stream, bufs, kp_host = self._e2e_state
        ready = [torch.cuda.Event() for _ in range(2)]
        consumed = [torch.cuda.Event() for _ in range(2)]
        done = [torch.cuda.Event() for _ in range(2)]
        copy_stream.wait_stream(main)

        def upload(i):
            s = i & 1
            with torch.cuda.stream(copy_stream):
                copy_stream.wait_event(consumed[s])          # the step that read bufs[s] (two steps ago) has finished with it
                bufs[s].copy_(self.pinned, non_blocking=True)
                ready[s].record(copy_stream)

        upload(0)
        out = None
        for i in range(steps):
            s = i & 1
            if i + 1 < steps:
                upload(i + 1)
            main.wait_event(ready[s])
            kp = self.step(bufs[s], collective)
            consumed[s].record(main)
            if kp_host[s] is None or kp_host[s].shape != kp.shape:
                kp_host[s] = torch.empty(kp.shape, dtype=kp.dtype).pin_memory()
            kp_host[s].copy_(kp, non_blocking=True)
            done[s].record(main)
            if i >= 1:
                done[1 - s].synchronize()
                out = kp_host[1 - s]
        done[(steps - 1) & 1].synchronize()
        out = kp_host[(steps - 1) & 1]
        main.wait_stream(copy_stream)
        return out

    def describe(self, collective):
        p = self.plan
        return "view-sharded: %d group(s) x %d ranks, %d of %d view(s) per rank, group batch %d; exchange = %s; V2V + soft-argmax batch-sharded; " \
               "stages 1 and 3 replayed as CUDA graphs" % (p.n_groups, p.group_size, len(p.views), self.views, self.Bg, EXCHANGE_TEXT[collective])

    def check_against_single_gpu(self, collective):
        """Key points of the samples this rank owns vs a plain single-GPU forward (all views) of the same samples."""
        own = self.plan.owned_samples(self.Bg)
        lo, hi = own[0], own[-1] + 1
        sub = {"cameras": [c[lo:hi] for c in self.batch["cameras"]], "keypoints_3d": self.batch["keypoints_3d"][lo:hi],
               "pred_keypoints_3d": self.batch["pred_keypoints_3d"][lo:hi]}
        kp_all = self.step(self.images_dev, collective).clone()
        kp_eager = self.step(self.images_dev, collective, graph=False).clone()      # same step without the CUDA graphs (diagnostic)
        saved = (self.model.use_cuda_graph, self.eng.use_graph)
        self.model.use_cuda_graph = self.eng.use_graph = False
        kp_single = self.model(self.images_g[lo:hi].to(self.dev), None, sub)[0]
        kp_single2 = self.model(self.images_g[lo:hi].to(self.dev), None, sub)[0]     # run-to-run repeatability of the reference itself
        self.model.use_cuda_graph, self.eng.use_graph = saved
        torch.cuda.synchronize()
        self.err_eager = float((kp_eager[lo:hi] - kp_single).abs().max())
        self.err_reference_repeat = float((kp_single2 - kp_single).abs().max())
        return float((kp_all[lo:hi] - kp_single).abs().max())

    def measure(self, collective, steps, warmup, flush, barrier):
        """-> dict(dev_ms, e2e_s, launches, kp_err_mm) for this exchange (device-resident arm, then end-to-end arm)."""
        err = self.check_against_single_gpu(collective)
        for _ in range(max(warmup, 3)):
            self.step(self.images_dev, collective)
        barrier()
        launches = self.eng.launches
        evs = []
        for _ in range(steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            self.step(self.images_dev, collective)
            e1.record()
            evs.append((e0, e1))
        barrier()
        dev_ms = sum(a.elapsed_time(b) for a, b in evs)
        # end-to-end arm: every step uploads its own images from pinned host memory and reads its own key points back; the upload of
        # step i+1 runs on a copy stream while step i computes (double-buffered device inputs, key points through pinned memory).
        e2e_mode = "pipelined"
        try:
            self._e2e_pipelined(collective, 2)
            barrier()
            t0 = time.perf_counter()
            kp = self._e2e_pipelined(collective, steps)
            barrier()
        except Exception as exc:   # noqa: BLE001 - fall back to the plain synchronous loop rather than lose the line
            print("rank %d: pipelined e2e arm failed (%s: %s); synchronous loop instead" % (self.rank, type(exc).__name__, exc), file=sys.stderr, flush=True)
            e2e_mode = "synchronous"
            for _ in range(2):
                kp = self.step(self.pinned.to(self.dev, non_blocking=True), collective).cpu()
            barrier()
            t0 = time.perf_counter()
            for _ in range(steps):
                kp = self.step(self.pinned.to(self.dev, non_blocking=True), collective).cpu()
            barrier()
        self.e2e_mode = e2e_mode
        return {"dev_ms": dev_ms, "e2e_s": time.perf_counter() - t0, "launches": launches, "kp_err_mm": err, "d2h": kp.numel() * 4,
                "kp_err_eager_mm": self.err_eager, "kp_ref_repeat_mm": self.err_reference_repeat}


def reduce_max(vals, dev, dist):
    t = torch.tensor(vals, dtype=torch.float64, device=dev)
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return [float(v) for v in t]


DUMP_SAMPLE = 1 << 20   # elements kept of an output larger than that (a fixed, seeded sample)


def output_arrays(out):
    """Host copies of what model(images, None, batch) returns (volumetric path), float32; outputs larger than DUMP_SAMPLE
    elements are reduced to the same seeded sample of flat indices in every run (the indices go along as <name>_index)."""
    kp, feats, vols, _, _, coords, base = out
    arrays = {}
    for name, t in (("keypoints_3d", kp), ("features", feats), ("volumes", vols), ("coord_volumes", coords), ("base_points", base)):
        a = t.detach().float().cpu().numpy()
        if a.size > DUMP_SAMPLE:
            idx = np.sort(np.random.RandomState(0).choice(a.size, DUMP_SAMPLE, replace=False))
            arrays[name + "_index"] = idx.astype(np.float64)
            a = a.ravel()[idx]
        arrays[name] = a.astype(np.float32)
    return arrays


def main_native(args, rank, world, local_rank):
    import lt_b200
    from lt_b200 import testing
    if not torch.cuda.is_available():
        raise SystemExit("bench.py --impl native needs a CUDA device (the native path has no CPU fallback)")
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    dist = None
    if world > 1 and args.dump_outputs:
        raise SystemExit("bench.py --dump-outputs covers the single-GPU arm (--gpus 1)")
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)

    B, V, S, n = args.batch, args.views, args.image, args.volume
    cfg = testing.make_config(num_layers=args.layers, volume_size=n)
    torch.manual_seed(0)
    np.random.seed(0)
    sharded = world > 1
    model = lt_b200.VolumetricTriangulationNet(cfg, device=dev, backend="native", conv_mode=args.mode, use_cuda_graph=True)
    if not args.no_calibrate:
        testing.randomize_weights(model, seed=0, calib_size=S, calib_views=1)
    model = model.to(dev).eval()
    eng = model.engine()
    model.clone_outputs = False
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)   # > 50 MB L2 of the H100

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
            torch.cuda.synchronize()

    exchanges, config4 = None, None
    with torch.no_grad():
        if not sharded:
            images, batch = testing.make_batch(B, V, image_size=S, seed=rank)
            pinned = images.pin_memory()
            images_dev = images.to(dev)
            parallelism = "dp1"
            h2d = images.numel() * 4

            def step(img):
                return model(img, None, batch)[0]

            # ---- device-resident arm: CUDA events around graph replays, L2 flushed between iterations ----
            for _ in range(max(args.warmup, 3)):
                step(images_dev)
            barrier()
            launches = eng.launches
            sampler = ClockSampler(local_rank)
            sampler.start()
            evs = []
            for _ in range(args.steps):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                timed_out = model(images_dev, None, batch)
                e1.record()
                evs.append((e0, e1))
            barrier()
            dev_ms = sum(a.elapsed_time(b) for a, b in evs)
            clocks = sampler.summary()
            dumped = output_arrays(timed_out) if args.dump_outputs else None   # the model's output buffers are reused by later steps

            # ---- end-to-end arm, synchronous: pinned host images -> device, forward, keypoints -> host ----
            for _ in range(2):
                kp = step(pinned.to(dev, non_blocking=True)).cpu()
            barrier()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                kp = step(pinned.to(dev, non_blocking=True)).cpu()
            barrier()
            e2e_sync_s = time.perf_counter() - t0
            d2h = kp.numel() * 4

            # ---- end-to-end, pipelined: the collated HWC batch in pinned memory goes through lt_b200.pipeline.InferenceStream --
            # every step still uploads its own images and reads its own keypoints back, but the upload of batch i+1 overlaps
            # the forward of batch i ----
            from lt_b200 import pipeline
            hwc = pipeline.pinned_empty((B, V, S, S, 3), np.float32)
            hwc[...] = images.permute(0, 1, 3, 4, 2).numpy()
            stream = pipeline.InferenceStream(model)

            def feed(k):
                for _ in range(k):
                    b = dict(batch)
                    b["images"] = hwc
                    yield b
            for _ in stream.run(feed(3)):
                pass
            barrier()
            stream.h2d_bytes = stream.d2h_bytes = 0
            t0 = time.perf_counter()
            for kp_host in stream.run(feed(args.steps)):
                pass
            barrier()
            e2e_s = time.perf_counter() - t0
            assert stream.h2d_bytes == h2d * args.steps and stream.d2h_bytes == d2h * args.steps
            eager_step = lambda: step(images_dev)
        else:
            # ---- view-sharded: G ranks share a group batch of B*G samples and split its views; W/G groups are replicas ----
            arm = ShardedArm(args, model, world, rank, dev, V)
            # `features` first: if the contract all-reduce misbehaves at some size (DESIGN.md section 6) it cannot disturb the other measurement
            names = ["features", "all_reduce"] if args.collective == "both" else [args.collective]
            results = {}
            sampler = ClockSampler(local_rank)
            sampler.start()
            for name in names:
                failed = 0
                try:
                    results[name] = arm.measure(name, args.steps, args.warmup, flush, barrier)
                except Exception as exc:   # noqa: BLE001 - an exchange that cannot be set up on this box is reported, not fatal
                    failed = 1
                    print("rank %d: exchange %r unavailable (%s: %s)" % (rank, name, type(exc).__name__, exc), file=sys.stderr, flush=True)
                if int(reduce_max([failed], dev, dist)[0]):
                    results.pop(name, None)
            clocks = sampler.summary()
            if not results:
                raise SystemExit("no view-group exchange could be set up")
            exchanges = {}
            for name, r in results.items():
                dms, es, err, err_eager, err_rep = reduce_max([r["dev_ms"], r["e2e_s"], r["kp_err_mm"], r["kp_err_eager_mm"], r["kp_ref_repeat_mm"]], dev, dist)
                exchanges[name] = {"value": B * world * args.steps / (dms / 1e3), "unit": "samples/s", "ms_per_step": dms / args.steps,
                                   "e2e": B * world * args.steps / es, "keypoints_vs_single_gpu_mm": err,
                                   "keypoints_vs_single_gpu_mm_without_graphs": err_eager, "single_gpu_reference_repeatability_mm": err_rep,
                                   "gpu_launches_per_step": r["launches"], "exchange": EXCHANGE_TEXT[name]}
                # same inputs, two arithmetic orders (packed exp-sum partials reduced by NCCL vs one fused kernel): measured 0.02-0.07 mm at
                # config #2; the contract against the reference is 1e-3 relative of a 2500 mm cuboid = 2.5 mm.  An exchange whose key points
                # disagree with the single-GPU forward of the same samples is reported but never selected as the line's value.
                exchanges[name]["keypoints_ok"] = bool(err < 0.5)
            if not any(e["keypoints_ok"] for e in exchanges.values()) and rank == 0:
                # reported in the line (`keypoints_ok: false` on every exchange), never a crash: the throughput is still a measurement
                print("WARNING: view-sharded key points differ from the single-GPU forward for every exchange: %s"
                      % {k: v["keypoints_vs_single_gpu_mm"] for k, v in exchanges.items()}, file=sys.stderr, flush=True)
            passing = [k for k in exchanges if exchanges[k]["keypoints_ok"]]
            best = max(passing or list(exchanges), key=lambda k: exchanges[k]["value"])
            r = results[best]
            dev_ms, e2e_s, e2e_sync_s, launches, d2h, h2d = r["dev_ms"], r["e2e_s"], r["e2e_s"], r["launches"], r["d2h"], arm.h2d
            parallelism = arm.describe(best)
            eager_step = lambda: arm.step(arm.images_dev, best, graph=False)
            if world == 8 and V == 4 and not args.no_config4:
                # BASELINE config #4: 8 views, one view per GPU (one view group of 8 ranks)
                failed8, r8, arm8 = 0, None, None
                try:
                    arm8 = ShardedArm(args, model, world, rank, dev, 8)
                    r8 = arm8.measure(best, max(2, args.steps // 2), args.warmup, flush, barrier)
                except Exception as exc:   # noqa: BLE001 - the extra configuration must never cost the headline line
                    failed8 = 1
                    print("rank %d: config #4 arm failed (%s: %s)" % (rank, type(exc).__name__, exc), file=sys.stderr, flush=True)
                if int(reduce_max([failed8], dev, dist)[0]):
                    config4 = {"unavailable": "the 8-view / one-view-per-GPU arm raised on at least one rank (see stderr)"}
                else:
                    dms, es, err = reduce_max([r8["dev_ms"], r8["e2e_s"], r8["kp_err_mm"]], dev, dist)
                    k8 = max(2, args.steps // 2)
                    config4 = {"workload": "Volumetric(softmax) ResNet-%d, 8 views %dx%d, %d^3 grid, one view per GPU, group batch %d" % (args.layers, S, S, n, arm8.Bg),
                               "value": arm8.Bg * k8 / (dms / 1e3), "unit": "samples/s", "ms_per_step": dms / k8, "e2e": arm8.Bg * k8 / es,
                               "exchange": best, "keypoints_vs_single_gpu_mm": err, "keypoints_ok": bool(err < 0.5), "parallelism": arm8.describe(best)}

        # ---- per-kernel timing for the roofline: one eager (non-graph) step with a CUDA-event pair per launch ----
        eng.use_graph = False
        model.use_cuda_graph = False
        eager_step()
        eng.timeline = []
        eager_step()
        torch.cuda.synchronize()
        agg = {}
        per_launch = []
        for label, flops, nbytes, a, b, desc in eng.timeline:
            r = agg.setdefault(label, [0.0, 0.0, 0.0, 0])
            ms = a.elapsed_time(b)
            r[0] += ms; r[1] += flops; r[2] += nbytes; r[3] += 1
            per_launch.append({"kernel": label, "desc": desc, "ms": round(ms, 4), "gflop": round(flops / 1e9, 3), "mb": round(nbytes / 1e6, 3)})
        if os.environ.get("LT_BENCH_TIMELINE") and rank == 0:
            with open(os.environ["LT_BENCH_TIMELINE"], "w") as f:
                json.dump(per_launch, f)
        eng.timeline = None

    # max over ranks
    dev_ms, e2e_s, e2e_sync_s = reduce_max([dev_ms, e2e_s, e2e_sync_s], dev, dist)
    total_samples = B * world * args.steps
    value = total_samples / (dev_ms / 1e3)
    e2e = total_samples / e2e_s

    pk = peaks()
    roof = None
    extra = {}
    kernel_names = {"conv_tc": "conv_tc_kernel", "conv_pair": "conv_tc_kernel", "conv_fold": "conv_tc_kernel", "conv_tail": "v2v_tail_kernel",
                    "conv_ffma": "conv_simt_kernel"}
    tensor_kernels = [k for k in kernel_names if k in agg]
    conv_key = max(tensor_kernels, key=lambda k: agg[k][0]) if tensor_kernels else None

    def tensor_roof(key):
        ms, fl, _, cnt = agg[key]
        ach = fl / (ms / 1e3) / 1e12
        tc = key != "conv_ffma"
        peak = pk["bf16_tflops"] if tc else 75.0
        r = {"kernel": kernel_names[key],
             "bound": "tensor", "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak,
             "launches": cnt, "ms_per_step": ms,
             "peak_source": pk["src"] + (" sustained dense bf16/fp16 (cuBLAS)" if tc else " nominal fp32 FFMA"),
             "timing": "per-launch CUDA-event pairs in one eager (graph-free) step; graph replay is up to ~6 % faster"}
        if tc and args.mode == "tc":
            # fp32-grade results cost three fp16 products per term (hi*hi, hi*lo, lo*hi): tensor-pipe work actually issued
            r["issued_mma_tflops"] = 3.0 * ach
            r["issued_frac"] = 3.0 * ach / peak
        return r

    if conv_key:
        roof = tensor_roof(conv_key)
    for key in tensor_kernels:
        if key != conv_key:
            extra["roofline_" + key] = tensor_roof(key)
    if tensor_kernels:
        # all tensor-core conv kernels together (the V2V + backbone conv path of the north star)
        ms = sum(agg[k][0] for k in tensor_kernels if k != "conv_ffma")
        fl = sum(agg[k][1] for k in tensor_kernels if k != "conv_ffma")
        if ms > 0:
            extra["roofline_conv_all"] = {"bound": "tensor", "achieved": fl / (ms / 1e3) / 1e12, "peak": pk["bf16_tflops"], "unit": "TFLOP/s",
                                          "frac": fl / (ms / 1e3) / 1e12 / pk["bf16_tflops"], "ms_per_step": ms,
                                          "issued_frac": 3.0 * fl / (ms / 1e3) / 1e12 / pk["bf16_tflops"] if args.mode == "tc" else None}
    for key in ("unproject", "softargmax"):
        if key in agg:
            ms, fl, nb, cnt = agg[key]
            ach = nb / (ms / 1e3) / 1e9
            extra["roofline_" + key] = {"bound": "hbm", "achieved": ach, "peak": pk["hbm_gbs"], "unit": "GB/s",
                                        "frac": ach / pk["hbm_gbs"], "ms_per_step": ms, "launches": cnt,
                                        "peak_source": pk["src"] + " copy bandwidth"}
    extra["step_breakdown_ms"] = {k: round(v[0], 3) for k, v in agg.items()}

    cpu = None
    parity_obj = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        # the CPU arm runs the bench's own weights and inputs, so its outputs double as the parity check of this very run:
        # full-size config #2 batch through the native path (graph-free replay of the timed step) vs the oracle
        from oracle import parity
        sd_cpu = {k: v.detach().cpu() for k, v in model.state_dict().items()}
        with torch.no_grad():
            native_out = model(images_dev, None, batch)
        torch.cuda.synchronize()
        rate, dt, threads, oracle_out = cpu_oracle_rate(args, 1, sd_cpu, images, batch)
        cpu = {"value": rate, "unit": "samples/s", "cores": threads, "kind": "port",
               "sample": "1 warm-up forward of one sample + 1 timed forward of the bench's %d-sample batch (same config, same weights and "
                         "inputs as the GPU arm), CPU oracle port, %d of %d host threads" % (B, threads, os.cpu_count())}
        parity_obj = parity.compare_outputs(native_out, oracle_out)
        parity_obj["against"] = "oracle/vol_oracle.volumetric_forward (CPU restatement of reference triangulation.py:245-355) on the bench batch"
        del native_out, oracle_out

    config5 = None
    if rank == 0 and world == 1 and not args.no_config5:
        try:
            config5 = algebraic_rate(args, dev, model, images_dev, batch, flush)
        except Exception as exc:   # noqa: BLE001 - reported in the line, never fatal for the headline measurement
            config5 = {"unavailable": "%s: %s" % (type(exc).__name__, exc)}

    torch_bars = {}
    if rank == 0 and world == 1 and not args.no_torch_gpu:
        # secondary bar (SURVEY 8d): the reference's own torch formulation through ATen/cuDNN on the same GPU, same weights/inputs
        sd_dev = model.state_dict()
        for key, tf32 in (("torch_gpu", False), ("torch_gpu_tf32", True)):
            try:
                torch_bars[key] = torch_gpu_rate(args, dev, sd_dev, images_dev, batch, tf32)
                torch_bars[key]["native_over_this"] = value / torch_bars[key]["value"]
            except Exception as exc:   # noqa: BLE001 - reported in the line
                torch_bars[key] = {"unavailable": "%s: %s" % (type(exc).__name__, exc)}

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": "samples/s", "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": dev_ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": {"tc": "fp16x3 (split-fp16 operands, 3 wgmma products per term, fp32 accumulate)", "tc1": "fp16", "simt": "f32"}[args.mode],
            "data": "synthetic",
            "config": {"workload": "Volumetric(softmax) ResNet-%d, %d views %dx%d, %d^3 grid, batch %d per GPU"
                                   % (args.layers, V, S, S, n, B),
                       "global_batch": B * world, "parallelism": parallelism,
                       "conv_mode": args.mode, "l2": "256 MB buffer written between timed iterations (L2 flush)",
                       "weights": "random (seeded recipe, BN calibrated)" if not args.no_calibrate else "random (default init)"},
            "e2e": {"value": e2e, "unit": "samples/s", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                    "api": ("lt_b200.pipeline.InferenceStream(model).run(batches): pinned HWC batch -> H2D on a copy stream -> layout kernel "
                            "-> forward -> keypoints D2H, upload of batch i+1 overlapping forward i") if not sharded
                           else "engine.forward_view_sharded(..., use_graph=True) per step: pinned images -> H2D on a copy stream (upload of step i+1 overlapping step i) -> forward -> key points D2H through pinned memory",
                    "sync_value": total_samples / e2e_sync_s,
                    "sync_api": "model(images_pinned.to(device, non_blocking=True), None, batch)[0].cpu() per step, no overlap"},
            "gpu_launches": launches * args.steps,
            "clocks": clocks,
            "roofline": roof,
            "cpu_baseline": cpu,
            "parity": parity_obj,
        }
        if exchanges is not None:
            line["exchanges"] = exchanges
        if config4 is not None:
            line["config4"] = config4
        if config5 is not None:
            line["config5"] = config5
        line.update(torch_bars)
        line.update(extra)
        print(json.dumps(line), flush=True)
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, a in dumped.items():
            np.save(os.path.join(args.dump_outputs, name + ".npy"), a)
    if dist is not None:
        dist.destroy_process_group()


def main():
    args = parse()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        main_reference(args, rank)
    elif args.impl == "torch_gpu":
        main_torch_gpu(args, rank)
    else:
        main_native(args, rank, world, local_rank)


if __name__ == "__main__":
    main()
