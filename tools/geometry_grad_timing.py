"""CUDA-event timing of the geometry gradients (csrc/backward.cu, csrc/algebraic.cu) at the volumetric recipe's sizes: B = 5,
V = 4 views of 64 x 64 x 32 feature maps unprojected onto 64^3 voxels, 17 joints; DLT at B = 8, J = 17, V = 4.

Reports medians over rounds that alternate the variants being compared, so drift of the shared machine hits both alike:
- the unprojection backward without (lt_unproject_aggregate_bwd) and with (lt_unproject_aggregate_bwd_geom) the d proj / d coord
  outputs, every aggregation;
- the soft-argmax coordinate backward (lt_softargmax3d_coord_bwd) against the HBM bound of its one read of B J nvox probabilities;
- the DLT projection gradient (lt_triangulate_dlt_proj_bwd) next to the existing DLT backward.
Usage: python tools/geometry_grad_timing.py [--rounds R] [--out DIR]   (needs a GPU; prints one JSON object)"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lt_b200 import capi, testing  # noqa: E402

HBM_PEAK = 3.35e12      # H100 SXM data sheet, bytes / s


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the timing itself does not depend on it
        q = "unknown (%s)" % e
    return q


def time_ms(fn, reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / reps


def alternate(fns, rounds, reps):
    """{name: median ms} over `rounds` rounds, each timing every fn in turn."""
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    samples = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            samples[k].append(time_ms(fn, reps))
    return {k: sorted(v)[len(v) // 2] for k, v in samples.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=11)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("geometry_grad_timing needs a GPU")
    dev = "cuda:0"
    torch.manual_seed(0)
    B, V, C, h, w, n, J = 5, 4, 32, 64, 64, 64, 17
    nvox = n ** 3
    cams = testing.make_cameras(V, image_size=256)
    from oracle import vol_oracle as O
    import numpy as np
    proj = torch.from_numpy(np.stack([np.stack([O.projection_after_resize(c.K, c.R, c.t, (256, 256), (h, w)) for c in cams])] * B)
                            .astype(np.float32)).to(dev).reshape(B, V, 12).contiguous()
    coord = torch.from_numpy(np.stack([O.coord_volume(np.array([0.0, 0.0, 900.0]), 2500.0, n).reshape(-1, 3)] * B)
                             .astype(np.float32)).to(dev)
    feats = torch.randn(B, V, h, w, C, device=dev)
    conf = torch.rand(B, V, C, device=dev) + 0.25
    g = torch.randn(B, nvox, C, device=dev)
    gf = torch.zeros_like(feats)
    gc = torch.zeros(B, V, C, device=dev)
    gp = torch.empty(B, V, 12, device=dev)
    gx = torch.empty(B, nvox, 3, device=dev)
    ws = torch.empty(capi.unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox), dtype=torch.uint8, device=dev)
    res = {"gpu": gpu_info(), "sizes": dict(B=B, V=V, C=C, h=h, w=w, nvox=nvox, J=J), "unproject_bwd_ms": {}}
    for agg_name, agg in (("sum", 0), ("max", 1), ("softmax", 2), ("conf", 3)):
        cf = conf if agg == 3 else None
        gcf = gc if agg == 3 else None
        t = alternate({
            "plain": lambda: capi.unproject_aggregate_bwd(feats, proj, coord, cf, g, gf, gcf, agg),
            "geom": lambda: capi.unproject_aggregate_bwd_geom(feats, proj, coord, cf, g, gf, gcf, gp, gx, agg, ws),
        }, args.rounds, args.reps)
        t["overhead"] = t["geom"] / t["plain"] - 1.0
        res["unproject_bwd_ms"][agg_name] = t

    probs = torch.softmax(torch.randn(B, J, nvox, device=dev), -1)
    gk = torch.randn(B, J, 3, device=dev)
    gcoord = torch.empty(B, nvox, 3, device=dev)
    t = alternate({"coord_bwd": lambda: capi.softargmax3d_coord_bwd(probs, gk, gcoord, B, J, nvox, 1)}, args.rounds, args.reps)["coord_bwd"]
    nbytes = (B * J * nvox + B * nvox * 3) * 4
    res["softargmax_coord_bwd"] = {"ms": t, "bytes": nbytes, "bytes_per_s": nbytes / (t * 1e-3), "share_of_hbm_peak": nbytes / (t * 1e-3) / HBM_PEAK}

    Bd, Jd = 8, 17
    P = proj[:1].reshape(1, V, 3, 4).expand(Bd, V, 3, 4).contiguous()
    X = torch.randn(Bd, Jd, 4, device=dev) * 300
    X[..., 2] += 900
    X[..., 3] = 1
    uvw = torch.einsum("bvij,bkj->bvki", P, X)
    kp = (uvw[..., :2] / uvw[..., 2:3]).contiguous()
    dconf = torch.rand(Bd, V, Jd, device=dev) + 0.1
    gout = torch.randn(Bd, Jd, 3, device=dev)
    gkp, gcf2, gP = torch.empty_like(kp), torch.empty_like(dconf), torch.empty_like(P)
    wsd = torch.empty(capi.triangulate_dlt_proj_bwd_workspace_bytes(Bd, V, Jd), dtype=torch.uint8, device=dev)
    res["dlt_ms"] = alternate({
        "kp_conf_bwd": lambda: capi.triangulate_dlt_bwd(P, kp, dconf, gout, gkp, gcf2),
        "proj_bwd": lambda: capi.triangulate_dlt_proj_bwd(P, kp, dconf, gout, gP, wsd),
    }, args.rounds, args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "geometry_grad_timing.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
