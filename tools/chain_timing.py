#!/usr/bin/env python
"""Time a run of ResNet bottleneck blocks as one chained launch (lt_conv_tc_chain_fwd) against its per-layer launches.

    python tools/chain_timing.py [--rounds N] [--reps N] [--json OUT]

Config #2 shapes (4 views x batch 8 at 384^2 = 32 images): layer 3 of ResNet-152 after its first block (35 blocks at 24^2, 1024 -> 256
-> 256 -> 1024) and layer 2 after its first block (7 blocks at 48^2, 512 -> 128 -> 128 -> 512).  Per-layer: three lt_conv_nd_fwd
launches per block with the engine's split-K workspace.  CUDA-event medians of --reps runs per round, the two sides alternated over
--rounds rounds; the outputs of both sides are compared bit for bit.  Prints the card name and power limit; needs a CUDA device.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

from lt_b200 import capi, engine as eng  # noqa: E402
from v2v_train_timing import DEV, card, event_median  # noqa: E402

RUNS = {"layer3 x35 24^2": (35, 32, 24, 24, 256), "layer2 x7 48^2": (7, 32, 48, 48, 128)}


def setup(blocks, N, H, W, planes, impl):
    g = torch.Generator().manual_seed(0)
    P, C = N * H * W, 4 * planes
    descs = [eng.conv_desc(N, (1, H, W), cin, cout, (1, k, k), (1, 1, 1), (0, k // 2, k // 2), (1, H, W), (1, H, W), cout, capi.FMT_S32,
                           capi.FMT_S32, relu=True, res_mode=res)
             for cin, cout, k, res in ((C, planes, 1, capi.RES_NONE), (planes, planes, 3, capi.RES_NONE), (planes, C, 1, capi.RES_BEFORE_RELU))]
    layers = []
    for _ in range(blocks):
        for d in descs:
            taps = d.KH * d.KW
            w = (torch.randn(taps, d.Cin, d.Cout, generator=g) * (0.7 / (taps * d.Cin) ** 0.5)).to(DEV)
            packed = torch.empty(capi.conv_tc_weight_bytes(taps, d.Cin, d.Cout) // 2, dtype=torch.float16, device=DEV)
            capi.conv_tc_pack_weights(w, packed, taps, d.Cin, d.Cout)
            layers.append((packed, (0.5 + torch.rand(d.Cout, generator=g)).to(DEV), (0.1 * torch.randn(d.Cout, generator=g)).to(DEV)))
    x0 = torch.empty(P * 2 * C, dtype=torch.float16, device=DEV)
    capi.f32_to_s32(torch.rand(P, C, generator=g).to(DEV), x0, P, C)
    ws = eng.splitk_workspace(torch.device(DEV))
    for d in descs:
        d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    plans = [capi.conv_tc_plan(d, torch.cuda.get_device_properties(0).multi_processor_count) for d in descs]
    assert all(p["splits"] == 1 for p in plans), plans
    y1, y2 = (torch.empty(P * 2 * planes, dtype=torch.float16, device=DEV) for _ in range(2))
    outs = [torch.empty_like(x0) for _ in range(2)]
    x = torch.empty_like(x0)

    def per_layer():
        src = x0
        for k in range(blocks):
            (w0, s0, h0), (w1, s1, h1), (w2, s2, h2) = layers[3 * k:3 * k + 3]
            out = outs[k % 2]
            capi.conv_nd(descs[0], src, w0, s0, h0, None, y1, impl)
            capi.conv_nd(descs[1], y1, w1, s1, h1, None, y2, impl)
            capi.conv_nd(descs[2], y2, w2, s2, h2, src, out, impl)
            src = out
        return src

    cdescs = [eng.conv_desc(N, (1, H, W), d.Cin, d.Cout, (1, d.KH, d.KW), (1, 1, 1), (0, d.ph, d.pw), (1, H, W), (1, H, W), d.Cout,
                            capi.FMT_S32, capi.FMT_S32, relu=True, res_mode=d.residual) for d in descs]
    bufs = [torch.empty(P * 2 * planes, dtype=torch.float16, device=DEV) for _ in range(4)]
    counters = torch.empty(capi.conv_tc_chain_plan(cdescs, blocks, 132)["counters"], dtype=torch.int32, device=DEV)

    def chain():
        x.copy_(x0)
        capi.conv_tc_chain(cdescs, blocks, x, bufs, [l[0] for l in layers], [l[1] for l in layers], [l[2] for l in layers], counters, impl)
        return x

    def copy_only():
        x.copy_(x0)

    return per_layer, chain, copy_only, 2.0 * P * sum(d.Cin * d.Cout * d.KH * d.KW for d in descs) * blocks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json")
    a = ap.parse_args()
    name, q = card()
    print("card: %s, power limit / max SM clock: %s" % (name, q), flush=True)
    res = {"card": name, "power_limit_max_sm_clock": q, "runs": {}}
    for label, shape in RUNS.items():
        per_layer, chain, copy_only, flops = setup(*shape, capi.CONV_TC)
        same = torch.equal(per_layer().view(torch.int16), chain().view(torch.int16))
        ms = {"per_layer": [], "chain": [], "copy": []}
        for _ in range(a.rounds):
            ms["per_layer"].append(event_median(per_layer, a.reps))
            ms["chain"].append(event_median(chain, a.reps))
            ms["copy"].append(event_median(copy_only, a.reps))
        med = {k: statistics.median(v) for k, v in ms.items()}
        chain_ms = med["chain"] - med["copy"]   # the chain runs in place: its timed call restores the input first
        r = {"bit_identical": same, "rounds_ms": ms, "per_layer_ms": med["per_layer"], "chain_ms": chain_ms,
             "speedup": med["per_layer"] / chain_ms, "chain_tflops": flops / (chain_ms / 1e3) / 1e12,
             "per_layer_tflops": flops / (med["per_layer"] / 1e3) / 1e12}
        res["runs"][label] = r
        print("%s: per-layer %.3f ms [%.3f-%.3f], chain %.3f ms (copy %.3f subtracted) [%.3f-%.3f], x%.3f, bit-identical %s"
              % (label, med["per_layer"], min(ms["per_layer"]), max(ms["per_layer"]), chain_ms, med["copy"], min(ms["chain"]),
                 max(ms["chain"]), r["speedup"], same), flush=True)
        del per_layer, chain, copy_only
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
