#!/usr/bin/env python
"""Per-class time of the tensor-core convolutions (conv_tc_kernel, conv_fold_kernel) in one eager bench.py step.

    python tools/conv_timeline.py [--timeline FILE] [--bench PATH] [--json OUT] [-- <bench.py arguments>]

Runs `bench.py` with LT_BENCH_TIMELINE pointing at a temporary file (bench.py records one CUDA-event pair per launch
of one eager, graph-free step: label, desc, ms, GFLOP, MB), or reads such a file with --timeline.  The `conv_tc` and
`conv_fold` launches are grouped by kernel and layer description (batch, output grid, Cin, Cout, kernel, stride), so every
class below is one set of layers of identical shape run by one kernel.  Printed per class: launches, ms per step, useful GFLOP and the issued
tensor rate (3 fp16 products per term in the default `tc` mode, 1 in `tc1`).  The other kernels are summed per label.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run_bench(bench, bench_args):
    fd, path = tempfile.mkstemp(suffix=".json", prefix="conv_timeline_")
    os.close(fd)
    env = dict(os.environ, LT_BENCH_TIMELINE=path)
    cmd = [sys.executable, bench] + bench_args
    res = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, text=True)
    if res.returncode != 0:
        raise SystemExit("bench.py exited with %d" % res.returncode)
    with open(path) as f:
        launches = json.load(f)
    os.unlink(path)
    lines = [l for l in res.stdout.splitlines() if l.startswith("{")]
    return launches, (json.loads(lines[-1]) if lines else None)


CONV_KERNELS = ("conv_tc", "conv_fold")


def classify(launches, products):
    classes, others = {}, {}
    for r in launches:
        if r["kernel"] in CONV_KERNELS:
            c = classes.setdefault((r["kernel"], r["desc"]), {"kernel": r["kernel"], "desc": r["desc"], "launches": 0, "ms": 0.0,
                                                              "gflop": 0.0})
            c["launches"] += 1
            c["ms"] += r["ms"]
            c["gflop"] += r["gflop"]
        else:
            o = others.setdefault(r["kernel"], {"kernel": r["kernel"], "launches": 0, "ms": 0.0})
            o["launches"] += 1
            o["ms"] += r["ms"]
    rows = sorted(classes.values(), key=lambda c: -c["ms"])
    for c in rows:
        c["issued_tflops"] = products * c["gflop"] / c["ms"] if c["ms"] > 0 else 0.0
    return rows, sorted(others.values(), key=lambda o: -o["ms"])


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--timeline", help="read this LT_BENCH_TIMELINE file instead of running bench.py")
    ap.add_argument("--bench", default=os.path.join(ROOT, "bench.py"), help="bench.py to run (e.g. of another checkout)")
    ap.add_argument("--json", help="also write the class table as JSON to this file")
    ap.add_argument("--products", type=int, default=None, help="fp16 products per term (default: 1 for --mode tc1, else 3)")
    ap.add_argument("bench_args", nargs=argparse.REMAINDER, help="arguments for bench.py, after --")
    args = ap.parse_args()
    bench_args = [a for a in args.bench_args if a != "--"]
    line = None
    if args.timeline:
        with open(args.timeline) as f:
            launches = json.load(f)
    else:
        launches, line = run_bench(args.bench, bench_args)
    products = args.products or (1 if "tc1" in bench_args else 3)
    rows, others = classify(launches, products)
    total_ms = sum(c["ms"] for c in rows)
    total_gf = sum(c["gflop"] for c in rows)
    print("| kernel | class (desc) | launches | ms | GFLOP | issued TFLOP/s |")
    print("|---|---|---|---|---|---|")
    for c in rows:
        print("| %s | %s | %d | %.3f | %.1f | %.0f |" % (c["kernel"], c["desc"], c["launches"], c["ms"], c["gflop"], c["issued_tflops"]))
    for k in CONV_KERNELS:
        sel = [c for c in rows if c["kernel"] == k]
        ms, gf = sum(c["ms"] for c in sel), sum(c["gflop"] for c in sel)
        print("| **all %s** | | %d | %.3f | %.1f | %.0f |" % (k, sum(c["launches"] for c in sel), ms, gf, products * gf / ms if ms > 0 else 0.0))
    print("| **all** | | %d | %.3f | %.1f | %.0f |" % (sum(c["launches"] for c in rows), total_ms, total_gf,
                                                     products * total_gf / total_ms if total_ms > 0 else 0.0))
    print()
    print("| other kernel | launches | ms |")
    print("|---|---|---|")
    for o in others:
        print("| %s | %d | %.3f |" % (o["kernel"], o["launches"], o["ms"]))
    if line is not None:
        print()
        print("bench.py: %.1f %s, gpu_launches %s" % (line.get("value", 0.0), line.get("unit", ""), line.get("gpu_launches")))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"conv": rows, "other": others, "products": products}, f, indent=1)


if __name__ == "__main__":
    main()
