"""Forward rate of TwoStageTriangulationNet against the two-pass protocol it replaces, on the GPU.

    python tools/two_stage_timing.py [--rounds R] [--iters K] [--out DIR]

Shape: ResNet-152 for both stages, B = 8, V = 4, 384 x 384 images, a 64^3 volume, softmax aggregation, seeded weights from
lt_b200.testing.  (a) two-pass: the native algebraic forward, its key points copied to the host (.cpu().numpy()) as
batch['pred_keypoints_3d'], the native volumetric forward (CUDA graph); (b) the composite: both stages and the hand-off from one
CUDA graph.  After a warm-up of each, R alternated rounds of K back-to-back forwards, each round bracketed by CUDA events; the median
round gives ms per forward.  Prints the card name and power limit, both rates, and whether (a) and (b) agree bit for bit."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import testing  # noqa: E402

DEV = "cuda:0"


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def models(layers):
    alg = lt_b200.AlgebraicTriangulationNet(testing.make_alg_config(num_layers=layers), device="cpu")
    testing.randomize_backbone_weights(alg, seed=0)
    vol = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=layers, volume_size=64, use_gt_pelvis=False), device="cpu")
    testing.randomize_weights(vol, seed=1)
    return alg.to(DEV).eval(), vol.to(DEV).eval()


def bits(t):
    return np.ascontiguousarray(t.cpu().numpy()).view(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--layers", type=int, default=152)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "two_stage_timing measures on a GPU"
    B, V, S = 8, 4, 384
    res = {"card": card(), "B": B, "V": V, "image": S, "volume": 64, "layers": args.layers}
    print("card, power limit:", res["card"])
    alg, vol = models(args.layers)
    model = lt_b200.TwoStageTriangulationNet(alg, vol)
    images, batch = testing.make_batch(B, V, image_size=S, seed=2, device=DEV)
    del batch["pred_keypoints_3d"]
    proj = torch.from_numpy(testing.image_projections(batch)).to(DEV)

    def two_pass():
        kp = alg(images, proj, batch)[0]
        return vol(images, None, dict(batch, pred_keypoints_3d=kp.cpu().numpy()))

    def composite():
        return model(images, proj, batch)

    with torch.no_grad():
        a, b = two_pass(), composite()
        torch.cuda.synchronize()
        same = all(np.array_equal(bits(x), bits(y)) for i, (x, y) in enumerate(zip(a, b)) if i not in (3, 4))
        same = same and all(np.array_equal(p.position, q.position) for p, q in zip(a[4], b[4]))
        res["bit_identical"] = bool(same)
        times = {"two_pass": [], "composite": []}
        for r in range(args.rounds):
            for name, fn in (("two_pass", two_pass), ("composite", composite))[::1 if r % 2 == 0 else -1]:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.iters)
    for name, ts in times.items():
        ms = float(np.median(ts))
        res[name] = {"ms_per_forward": ms, "samples_per_s": B * 1e3 / ms, "rounds_ms": [round(t, 3) for t in ts]}
        print("%-9s %8.3f ms / forward  %7.1f samples/s  (rounds: %s)" % (name, ms, B * 1e3 / ms, ", ".join("%.3f" % t for t in ts)))
    res["speedup"] = res["two_pass"]["ms_per_forward"] / res["composite"]["ms_per_forward"]
    print("composite / two-pass rate: %.3fx; outputs bit-identical: %s" % (res["speedup"], res["bit_identical"]))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "two_stage_timing.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
