#!/usr/bin/env python
"""Time the validation forward of hybrid-trained models: eager on the torch switches, eager on the native switches, and
eval_backend="native" (the native engine from CUDA graphs).

    python tools/eval_timing.py [--steps N] [--rounds N] [--refreshes N] [--only volumetric|algebraic] [--json OUT]

Workloads (the recipes' models; seeded, calibrated weights):
  volumetric  ResNet-152, V = 4, 384^2, 64^3, softmax aggregation, eval B = 10 and B = 75, TrainStep at B = 5
  algebraic   ResNet-152 with confidences, V = 4, 384^2, eval B = 16 and B = 100, TrainStep at B = 8
Three ways of running model.eval() + torch.no_grad() + model(images, proj, batch), alternated --rounds times per batch size:
  "torch"   backend="hybrid" on the torch switches (cuDNN, torch's default TF32 settings: convolutions in TF32);
  "native"  backend="hybrid" on all native switches (conv, norm, head), eager;
  "engine"  the native-switch model with eval_backend="native".
Per round and way: the median of --steps forwards, each a host clock around one forward (host geometry and upload included) that
ends in torch.cuda.synchronize().  Per batch size, --refreshes times: one TrainStep call, then the first eval forward (re-pack and
capture after the step invalidated the engine) and a second one; then the memory allocated and reserved after one more TrainStep
call (with the cache emptied) and the peaks of both during the two evals after it, with the training graphs resident.  At B = 1
of the same seeded data, every way's outputs against the fp32 CPU oracle (oracle/vol_oracle.py).  Prints the card name and power
limit first; needs a CUDA device and does not fall back.
"""
import argparse
import json
import os
import statistics
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)

import lt_b200  # noqa: E402
from lt_b200 import testing  # noqa: E402
from oracle import vol_oracle as O  # noqa: E402
from train_step_timing import _free, timed  # noqa: E402
from v2v_train_timing import DEV, card  # noqa: E402

V, S = 4, 384
WAYS = ("torch", "native", "engine")


def volumetric_workload():
    cfg = lambda: testing.make_train_config(testing.make_config(num_layers=152, volume_size=64), criterion="MAE", lr=1e-4,
                                            use_volumetric_ce_loss=True, volumetric_ce_loss_weight=0.01, scale_keypoints_3d=0.1,
                                            process_features_lr=1e-3, volume_net_lr=1e-3)
    holder = lt_b200.VolumetricTriangulationNet(cfg(), device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=0, calib_size=128, calib_views=1)
    switches = dict(backbone_backend="native", v2v_backend="native", norm_backend="native", head_backend="native")
    return lt_b200.VolumetricTriangulationNet, cfg, holder.state_dict(), switches, (10, 75), 5


def algebraic_workload():
    cfg = lambda: testing.make_train_config(testing.make_alg_config(num_layers=152, use_confidences=True), criterion="MSESmooth",
                                            lr=1e-5, mse_smooth_threshold=400, scale_keypoints_3d=0.1)
    holder = lt_b200.AlgebraicTriangulationNet(cfg(), device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=0, calib_size=128)
    switches = dict(backbone_backend="native", norm_backend="native", head_backend="native")
    return lt_b200.AlgebraicTriangulationNet, cfg, holder.state_dict(), switches, (16, 100), 8


def make_model(wl, way):
    make, cfg, state, switches = wl[:4]
    c = cfg()
    m = make(c, device="cpu", backend="hybrid", eval_backend="native" if way == "engine" else None,
             **({} if way == "torch" else switches))
    m.load_state_dict(state)
    return m.to(DEV).eval(), c


def data(B, seed=1):
    images, batch = testing.make_batch(B, V, image_size=S, seed=seed)
    return testing.prepare_batch(batch, images, DEV) + (batch,)


def evaluator(m, d):
    def run():
        was = m.training
        m.eval()
        with torch.no_grad():
            out = m(d[0], d[3], d[4])
        m.train(was)
        return out
    return run


def alternated(wl, B, steps, rounds, label):
    d = data(B)
    runs = {w: evaluator(make_model(wl, w)[0], d) for w in WAYS}
    for r in runs.values():
        for _ in range(2):
            r()
    res = defaultdict(list)
    for i in range(rounds):
        for w, r in runs.items():
            res[w].append(timed(r, steps)[0])
            print("%s B=%d round %d, %s: %.2f ms" % (label, B, i, w, res[w][-1]), flush=True)
    med = {w: statistics.median(v) for w, v in res.items()}
    print("%s B=%d, median of rounds: %s; torch / engine %.3f, native / engine %.3f"
          % (label, B, ", ".join("%s %.2f ms [%.2f-%.2f]" % (w, med[w], min(res[w]), max(res[w])) for w in WAYS),
             med["torch"] / med["engine"], med["native"] / med["engine"]), flush=True)
    del runs
    return {"rounds_ms": dict(res), "median_ms": med, "samples_per_s": {w: B / med[w] * 1e3 for w in WAYS}}


def refresh(wl, B, refreshes, label):
    """TrainStep call -> first eval (re-pack + capture) -> second eval, `refreshes` times.  Then once more for memory: after the
    TrainStep call and torch.cuda.empty_cache(), the memory allocated and reserved (the training graphs' pools are reserved memory,
    held while their intermediates are free), and the peaks of both during the two evals that follow, with the training graphs
    resident and the engine invalidated."""
    _free()
    m, cfg = make_model(wl, "engine")
    m.train()
    step = lt_b200.TrainStep(m, testing.recipe_optimizer(m, cfg, capturable=True), cfg)
    train = data(wl[5], seed=2)
    ev = evaluator(m, data(B))
    first, second = [], []
    for i in range(refreshes + 1):
        np.random.seed(i)
        step(*train)
        torch.cuda.synchronize()
        first.append(timed(ev, 1)[0])
        second.append(timed(ev, 1)[0])
    first, second = first[1:], second[1:]          # the first pass also loads modules and sets function attributes
    step(*train)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    gib = 2.0 ** 30
    mem = {"allocated_after_step_GiB": torch.cuda.memory_allocated() / gib, "reserved_after_step_GiB": torch.cuda.memory_reserved() / gib}
    torch.cuda.reset_peak_memory_stats()
    ev()
    ev()
    torch.cuda.synchronize()
    mem.update(peak_allocated_during_evals_GiB=torch.cuda.max_memory_allocated() / gib,
               peak_reserved_during_evals_GiB=torch.cuda.max_memory_reserved() / gib)
    out = dict(first_eval_ms=first, second_eval_ms=second, refresh_ms=statistics.median(first) - statistics.median(second),
               captures=m.engine().captures, **mem)
    print("%s B=%d after a TrainStep call: first eval %s ms, second %s ms, re-pack + capture %.0f ms; after the step %.2f GiB "
          "allocated, %.2f GiB reserved; peak during the evals %.2f GiB allocated, %.2f GiB reserved"
          % (label, B, ["%.1f" % t for t in first], ["%.1f" % t for t in second], out["refresh_ms"], mem["allocated_after_step_GiB"],
             mem["reserved_after_step_GiB"], mem["peak_allocated_during_evals_GiB"], mem["peak_reserved_during_evals_GiB"]), flush=True)
    del step, m
    return out


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max()) / max(float(np.abs(b).max()), float(b.std()), 1e-30)


def against_oracle(wl, label):
    """Every way's outputs at B = 1 against the CPU oracle: relative errors of the maps, key points in mm (3-D) and pixels (2-D)."""
    make, _, state = wl[:3]
    d = data(1, seed=3)
    images, _, _, proj, batch = d
    if make is lt_b200.VolumetricTriangulationNet:
        base = np.stack([k[6, :3] for k in batch["keypoints_3d"]])
        kp_o, feats_o, vols_o, _ = O.volumetric_forward(state, images.cpu(), batch["cameras"], base, volume_size=64)
    else:
        kp_o, kp2d_o, heat_o, conf_o = O.algebraic_forward(state, images.cpu(), proj.cpu().numpy())
    out = {}
    for w in WAYS:
        m = make_model(wl, w)[0]
        o = [t.cpu().numpy() if torch.is_tensor(t) else t for t in evaluator(m, d)()]
        if make is lt_b200.VolumetricTriangulationNet:
            out[w] = {"kp_mm": float(np.abs(o[0] - np.asarray(kp_o)).max()), "features_rel": _rel(o[1], feats_o),
                      "volumes_rel": _rel(o[2], vols_o)}
        else:
            out[w] = {"kp3d_mm": float(np.abs(o[0] - kp_o).max()), "kp2d_px": float(np.abs(o[1] - kp2d_o).max()),
                      "heatmaps_rel": _rel(o[2], heat_o), "conf_abs": float(np.abs(o[3] - conf_o).max())}
        print("%s B=1 vs the fp32 CPU oracle, %s: %s" % (label, w, ", ".join("%s %.3g" % kv for kv in out[w].items())), flush=True)
        del m
        _free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--refreshes", type=int, default=3)
    ap.add_argument("--only", choices=["volumetric", "algebraic"])
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_timing.py needs a CUDA device")
    name, q = card()
    print("device: %s, power limit, max SM clock: %s" % (name, q), flush=True)
    out = {"device": name, "power_limit_max_sm_clock": q}
    for label, factory in (("volumetric", volumetric_workload), ("algebraic", algebraic_workload)):
        if a.only not in (None, label):
            continue
        wl = factory()
        r = out[label] = {"oracle": against_oracle(wl, label)}
        for B in wl[4]:
            _free()
            r["B%d" % B] = {"alternated": alternated(wl, B, a.steps, a.rounds, label)}
            _free()
            r["B%d" % B]["refresh"] = refresh(wl, B, a.refreshes, label)
        _free()
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
