#!/usr/bin/env python
"""Time the confidence heads' native training tail (head_backend="native") against the torch head.

    python tools/conf_head_timing.py [--rounds N] [--reps N] [--steps N] [--skip-step] [--json OUT]

1. The head tail forward + backward, from the second BatchNorm's output (N, 256, 12, 12) to the sigmoid: native ConfHeadTailFn
   (lt_conf_head_tail_fwd / _bwd) against torch (MaxPool2d, ReLU, mean, three nn.Linear on cuBLAS, Sigmoid), at N = B V = 20 and
   400 (a training batch and val_batch_size 100), channels_last as the native convolutions leave it.
2. The view normalisation forward + backward, (B, 4, 17) with eps 1e-5: native ViewNormalizeFn against torch's formula.
3. The recipe algebraic lt_b200.TrainStep (ResNet-152 with confidences, B = 8, V = 4, 384^2, native conv and norm switches) with
   head_backend "torch" and "native".
1 and 2: CUDA-event medians of --reps calls per round, the sides alternated over --rounds rounds.  3: host-clock medians of --steps
replays ending in a synchronise, after the capture.  Prints the card name and power limit first; needs a CUDA device.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import autograd_ops as A  # noqa: E402
from lt_b200 import pose_resnet, testing  # noqa: E402
from deterministic_timing import _free, alternate  # noqa: E402
from train_step_timing import stepper, timed  # noqa: E402
from v2v_train_timing import DEV, card  # noqa: E402


def head_tail(rounds, reps):
    out = {}
    for N in (20, 400):
        head = pose_resnet.ConfidenceHead(2048, 17).to(DEV).train()
        x = torch.randn(N, 256, 12, 12, device=DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        g = torch.rand(N, 17, device=DEV)
        tail = torch.nn.Sequential(head.features[6], head.features[7])

        def torch_side():
            y = head.head(tail(x).flatten(2).mean(dim=-1))
            y.backward(g)

        def native_side():
            A.conf_head_tail(head, x).backward(g)
        out[N] = alternate({"torch": torch_side, "native": native_side}, rounds, reps, "head tail fwd+bwd N=%d" % N)
    return out


def view_normalize(rounds, reps):
    out = {}
    for B in (5, 100):
        c = (torch.rand(B, 4, 17, device=DEV) + 0.01).requires_grad_(True)
        g = torch.randn(B, 4, 17, device=DEV)

        def torch_side():
            (c / c.sum(dim=1, keepdim=True) + 1e-5).backward(g)

        def native_side():
            A.view_normalize(c, 1e-5).backward(g)
        out[B] = alternate({"torch": torch_side, "native": native_side}, rounds, reps, "view normalisation fwd+bwd B=%d V=4" % B)
    return out


def train_step(steps):
    cfg = lambda: testing.make_train_config(testing.make_alg_config(num_layers=152, use_confidences=True), criterion="MSESmooth",  # noqa: E731
                                            lr=1e-5, mse_smooth_threshold=400, scale_keypoints_3d=0.1)
    torch.manual_seed(0)
    state = lt_b200.AlgebraicTriangulationNet(cfg(), device="cpu", backend="hybrid").state_dict()
    out = {}
    for head in ("torch", "native", "torch again"):
        def make(graph, head=head.split()[0]):
            c = cfg()
            m = lt_b200.AlgebraicTriangulationNet(c, device="cpu", backend="hybrid", train_graph=graph, backbone_backend="native",
                                                  norm_backend="native", head_backend=head)
            m.load_state_dict(state)
            return m.to(DEV).train(), c
        _free()
        step = stepper(make, "step", 8)
        step()
        med, times = timed(step, steps)
        out[head] = {"median_ms": med, "min_ms": min(times), "max_ms": max(times)}
        print("algebraic TrainStep, head_backend %s: %.2f ms [%.2f-%.2f]" % (head, med, min(times), max(times)), flush=True)
        del step
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("conf_head_timing needs a CUDA device")
    res = {"card": card()}
    print(res["card"], flush=True)
    res["head_tail"] = head_tail(args.rounds, args.reps)
    res["view_normalize"] = view_normalize(args.rounds, args.reps)
    if not args.skip_step:
        res["train_step"] = train_step(args.steps)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
