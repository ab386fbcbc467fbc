"""The training BatchNorm kernels (csrc/norm.cu: bn_reduce_kernel<0, false> / <1, true> / <1, false>, bn_finalize_fwd_kernel,
bn_apply_fwd_kernel<RES, RELU> x 4, bn_finalize_bwd_kernel, bn_apply_bwd_kernel<RELU, DRES> x 4) against the float64 reference of
tests/test_norm_ref_cpu.py, per element, from the exact operands each call received.

Every output (y, save_mean, save_invstd, running_mean, running_var, dx, dr, dgamma, dbeta) is held to the bars derived in
test_norm_ref_cpu's docstring, in train and eval mode, for every case of its table `CASES` (launch plans checked host-side there):
C = 4 ... 2048 with tc < 32 and partial channel blocks, M = 2 ... 10^6, row tails, splits limited by rows and by the CTA cap, and
|mean| = 10^3 std.  The ReLU mask of the reference comes from the native y, as torch autograd uses its own output.  Inputs sit
between guard bands of a NaN sentinel (a read outside them poisons the sums); outputs start as the sentinel between guard bands and
the workspace is exactly lt_batch_norm_workspace_bytes, filled with 0xFF and guarded: guards intact, every output element written.

Also: the table reaches all 13 kernels under torch.profiler; null dgamma / dbeta / dr leave dx bit-identical; a second workspace
fill and a CUDA-graph replay are bit-identical; inputs scaled by 2^+-40, gamma = 0 and < 0, a constant channel with eps > 0 and
eps = 0; one NaN or +Inf in x, a NaN in dY or in the residual, with and without ReLU: the non-finite outputs are the reference's,
dbeta is finite where torch's is and the untouched channels stay within their bars; argument errors at the C ABI leave the outputs
untouched.

Measured on an H100 80GB HBM3 (700 W power limit, 132 SMs), worst err/bar per output (dr is exact everywhere; in eval mode the
running buffers are bit-identical and save_mean is the running mean):
- the table, train: y 0.985, save_mean 0.994, save_invstd 0.986, running_mean 0.620, running_var 0.693, dx 0.865, dgamma 0.844,
  dbeta 0.981; eval: y 0.978, save_invstd 0.976, dx 0.571, dgamma 0.886, dbeta 0.972;
- through autograd_ops.batch_norm: y 0.973, dx 0.769, dgamma 0.749, dbeta 0.959, running_mean 0.484, running_var 0.556;
- edges: y 0.970, save_mean 0.720, save_invstd 0.825, dx 0.653, dgamma 0.739, dbeta 0.962;
- untouched channels of the non-finite cases: y 0.727, dx 0.523, dgamma 0.828, dbeta 0.949.
With the ReLU as fmaxf(y, 0) and the mask y > 0, the non-finite cases whose output holds a NaN fail (a NaN or Inf in x in train mode,
a NaN in x or in the residual in eval mode, a NaN residual in train mode: the ReLU turned the NaN into 0 and the mask dropped its
gradient); every finite case passes with either rule.
"""
import json
import os
import re
import subprocess
import sys

import pytest
import torch
from torch import nn

from lt_b200 import autograd_ops as A
from lt_b200 import capi
from test_gpu_unproject import Guarded
from test_norm_ref_cpu import (CASES, OUTPUTS, _nonfinite_problem, bars, err_over_bar, plan, plan_e64, problem, reference,
                               torch_autograd)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EPS, MOMENTUM = 1e-5, 0.1
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    for (fam, q), v in sorted(WORST.items()):
        print("worst err/bar %-6s %-12s %.3f" % (fam, q, v))


def _sms():
    return capi.device_info()[0]


def _dev(t):
    return {k: None if v is None else v.to(DEV) for k, v in t.items()}


def run_native(t, eps, momentum, training, relu, backward=True, ws_fill=-1, grad_params=True, grad_res=True):
    """One lt_batch_norm_fwd (+ _bwd) on guarded buffers -> (outputs as float32 device tensors, guarded buffers)."""
    M, C = t["x"].shape
    B = {k: None if v is None else Guarded(v.shape, fill=v.to(DEV)) for k, v in t.items()}
    for k in ("save_mean", "save_invstd"):
        B[k] = Guarded((C,))
    B["y"] = Guarded((M, C))
    nbytes = capi.batch_norm_workspace_bytes(M, C)
    assert nbytes % 4 == 0
    B["ws"] = Guarded((nbytes // 4,))
    B["ws"].t.view(torch.int32).fill_(ws_fill)
    r = None if B["r"] is None else B["r"].t
    capi.batch_norm(B["x"].t, r, B["gamma"].t, B["beta"].t, B["rm"].t, B["rv"].t, B["save_mean"].t, B["save_invstd"].t, B["y"].t,
                    M, C, eps, momentum, training, relu, B["ws"].t)
    outs = ["y", "save_mean", "save_invstd"]
    if backward:
        B["dx"] = Guarded((M, C))
        B["dr"] = Guarded((M, C)) if (r is not None and grad_res) else None
        B["dgamma"], B["dbeta"] = (Guarded((C,)), Guarded((C,))) if grad_params else (None, None)
        T = lambda k: None if B[k] is None else B[k].t        # noqa: E731
        capi.batch_norm_bwd(B["x"].t, B["y"].t if relu else None, B["g"].t, B["gamma"].t, B["save_mean"].t, B["save_invstd"].t,
                            B["dx"].t, T("dr"), T("dgamma"), T("dbeta"), M, C, training, relu, B["ws"].t)
        outs += [k for k in ("dx", "dr", "dgamma", "dbeta") if B[k] is not None]
    torch.cuda.synchronize()
    for k, b in B.items():
        assert b is None or b.guards_intact(), k
    for k in outs:
        assert B[k].unwritten() == 0, k
    got = {k: B[k].t.clone() for k in outs}
    got["rm"], got["rv"] = B["rm"].t.clone(), B["rv"].t.clone()
    return got


def check(got, t, eps, training, relu, fam, cols=None):
    """Every output against the reference with the native y as ReLU mask; returns {output: err/bar}.  cols: the channels held to
    their bars (all by default); the non-finite pattern is compared over all channels."""
    M, C = t["x"].shape
    ref = reference(_dev(t), eps, MOMENTUM, training, relu, y_mask=got["y"])
    b = bars(ref, plan_e64(plan(M, C, _sms())))
    w = {}
    for q in OUTPUTS:
        if q not in got:
            continue
        _, same = err_over_bar(got[q], ref[q], b[q])
        assert same, (fam, q, "non-finite pattern differs", torch.isfinite(got[q]).logical_xor(torch.isfinite(ref[q])).nonzero()[:8])
        e, _ = err_over_bar(got[q], ref[q], b[q], cols)
        w[q] = e
        WORST[(fam, q)] = max(WORST.get((fam, q), 0.0), e)
    assert max(w.values()) <= 1.0, (fam, w)
    if not training:
        assert torch.equal(got["rm"], t["rm"].to(DEV)) and torch.equal(got["rv"], t["rv"].to(DEV))
    return w


# ------------------------------------------------------------------------------------------ the table
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("name", list(CASES))
def test_case_vs_float64(name, training):
    c = CASES[name]
    t = problem(c.M, c.C, c.res, seed=c.M % 1000 + c.C, mean=c.mean)
    got = run_native(t, EPS, MOMENTUM, training, c.relu)
    w = check(got, t, EPS, training, c.relu, "train" if training else "eval")
    print("%-28s %-5s %s" % (name, "train" if training else "eval", " ".join("%s %.3f" % kv for kv in w.items())))


AUTOGRAD_CASES = {"C12 M1001 relu res": (7, 11, 13), "C64 M286": (2, 11, 13), "C132 M1537 relu res": (1, 29, 53),
                  "C36 M4099 relu": (4099, 1, 1)}


@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("name", list(AUTOGRAD_CASES))
def test_autograd_batch_norm_vs_float64(name, training):
    """The same cases through autograd_ops.batch_norm on an nn.BatchNorm2d and channels-last (N, C, H, W) views of the rows."""
    c = CASES[name]
    N, H, W = AUTOGRAD_CASES[name]
    t = problem(c.M, c.C, c.res, seed=c.M % 1000 + c.C, mean=c.mean)
    bn = nn.BatchNorm2d(c.C, eps=EPS, momentum=MOMENTUM).to(DEV).train(training)
    with torch.no_grad():
        bn.weight.copy_(t["gamma"])
        bn.bias.copy_(t["beta"])
        bn.running_mean.copy_(t["rm"])
        bn.running_var.copy_(t["rv"])

    def nchw(v):
        return v.to(DEV).view(N, H, W, c.C).permute(0, 3, 1, 2).detach().requires_grad_(True)

    def rows(v):
        return v.permute(0, 2, 3, 1).reshape(c.M, c.C)
    x = nchw(t["x"])
    r = None if t["r"] is None else nchw(t["r"])
    y = A.batch_norm(bn, x, relu=c.relu, residual=r)
    y.backward(t["g"].to(DEV).view(N, H, W, c.C).permute(0, 3, 1, 2))
    got = {"y": rows(y.detach()), "dx": rows(x.grad), "dgamma": bn.weight.grad, "dbeta": bn.bias.grad,
           "rm": bn.running_mean, "rv": bn.running_var}
    if r is not None:
        got["dr"] = rows(r.grad)
    check(got, t, EPS, training, c.relu, "autograd")
    assert int(bn.num_batches_tracked) == (1 if training else 0)


# ------------------------------------------------------------------------------------------ dispatch
_PAT = re.compile(r"(bn_reduce_kernel|bn_apply_fwd_kernel|bn_apply_bwd_kernel|bn_finalize_fwd_kernel|bn_finalize_bwd_kernel)(<[^>]*>)?")
KERNELS = {"bn_reduce_kernel<0, false>", "bn_reduce_kernel<1, true>", "bn_reduce_kernel<1, false>", "bn_finalize_fwd_kernel",
           "bn_finalize_bwd_kernel"} | {"bn_apply_%s_kernel<%s, %s>" % (d, a, b) for d in ("fwd", "bwd") for a in ("true", "false")
                                        for b in ("true", "false")}


def profiled_kernels():
    """Every case of the table (but the 10^6-row one) in train and eval mode under the profiler -> the kernel names launched."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, c in CASES.items():
            if c.M > 100000:
                continue
            t = problem(c.M, c.C, c.res, seed=1)
            for training in (True, False):
                run_native(t, EPS, MOMENTUM, training, c.relu)
        torch.cuda.synchronize()
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    return sorted({m.group(0) for m in (_PAT.search(e.name()) for e in evs) if m})


def test_dispatch_reaches_all_13_kernels():
    """Profiled in a child process (a second profiler session in one process misses its first kernel records)."""
    code = ("import json, sys; sys.path[:0] = %r; import test_gpu_norm_ref as t; print('KERNELS ' + json.dumps(t.profiled_kernels()))"
            % [HERE, ROOT])
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    names = set(json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][len("KERNELS "):]))
    print("kernels launched: %s" % sorted(names))
    assert len(KERNELS) == 13 and names == KERNELS, (KERNELS - names, names - KERNELS)


# ------------------------------------------------------------------------------------------ optional outputs, repeats, graphs
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
def test_optional_outputs_leave_dx_bit_identical(training):
    c = CASES["C132 M1537 relu res"]
    t = problem(c.M, c.C, c.res, seed=5)
    full = run_native(t, EPS, MOMENTUM, training, c.relu)
    for kw in (dict(grad_params=False), dict(grad_res=False), dict(grad_params=False, grad_res=False)):
        part = run_native(t, EPS, MOMENTUM, training, c.relu, **kw)
        assert torch.equal(part["dx"], full["dx"]), kw
        assert "dr" not in part or torch.equal(part["dr"], full["dr"])


@pytest.mark.parametrize("name", ["C12 M1001 relu res", "C2048 M8300 relu res", "C8 M1000003 mean1e3 relu"])
def test_bitwise_repeats_and_graph_replay(name):
    c = CASES[name]
    M, C = c.M, c.C
    t = problem(M, C, c.res, seed=9, mean=c.mean)
    a = run_native(t, EPS, MOMENTUM, True, c.relu, ws_fill=-1)
    b = run_native(t, EPS, MOMENTUM, True, c.relu, ws_fill=0)
    for q in a:
        assert torch.equal(a[q], b[q]), q
    # one forward + backward captured into a graph, replayed from restored running buffers
    d = _dev(t)
    rm0, rv0 = d["rm"].clone(), d["rv"].clone()
    o = {k: torch.empty(M, C, device=DEV) for k in ("y", "dx", "dr")}
    o.update({k: torch.empty(C, device=DEV) for k in ("save_mean", "save_invstd", "dgamma", "dbeta")})
    ws = torch.full((capi.batch_norm_workspace_bytes(M, C) // 4,), -1, dtype=torch.int32, device=DEV).view(torch.float32)
    dr = o["dr"] if c.res else None

    def step():
        capi.batch_norm(d["x"], d["r"], d["gamma"], d["beta"], d["rm"], d["rv"], o["save_mean"], o["save_invstd"], o["y"], M, C, EPS,
                        MOMENTUM, True, c.relu, ws)
        capi.batch_norm_bwd(d["x"], o["y"] if c.relu else None, d["g"], d["gamma"], o["save_mean"], o["save_invstd"], o["dx"], dr,
                            o["dgamma"], o["dbeta"], M, C, True, c.relu, ws)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for k in o:
        o[k].fill_(float("nan"))
    d["rm"].copy_(rm0)
    d["rv"].copy_(rv0)
    graph.replay()
    torch.cuda.synchronize()
    o["rm"], o["rv"] = d["rm"], d["rv"]
    for q in a:
        assert torch.equal(o[q], a[q]), q


# ------------------------------------------------------------------------------------------ edges
def _edge(kind):
    t = problem(1537, 16, True, seed=11)
    eps = EPS
    if kind.startswith("scale"):
        s = 2.0 ** (40 if kind == "scale 2^40" else -40)
        for k in ("x", "r", "rm", "g"):
            t[k] = t[k] * s
        t["rv"] = t["rv"] * s * s
        eps = EPS * s * s
    elif kind == "gamma 0 and < 0":
        t["gamma"][:4] = 0.0
        t["gamma"][4:8] = -t["gamma"][4:8].abs() - 0.5
    elif kind.startswith("constant"):
        t["x"][:, 3] = 0.625
        t["x"][:, 9] = -3.0
        eps = 0.0 if kind == "constant eps 0" else EPS
    return t, eps


@pytest.mark.parametrize("relu", [True, False], ids=["relu", "plain"])
@pytest.mark.parametrize("kind", ["scale 2^40", "scale 2^-40", "gamma 0 and < 0", "constant eps>0", "constant eps 0"])
def test_edges(kind, relu):
    t, eps = _edge(kind)
    for training in (True, False):
        if kind == "constant eps 0" and not training:
            continue            # eval normalises with the running variance
        got = run_native(t, eps, MOMENTUM, training, relu)
        check(got, t, eps, training, relu, "edges")
        if kind == "constant eps 0":
            assert bool((got["save_invstd"][[3, 9]] == 0).all()) and bool(torch.isfinite(got["y"]).all())


# ------------------------------------------------------------------------------------------ non-finite inputs
@pytest.mark.parametrize("training", [True, False], ids=["train", "eval"])
@pytest.mark.parametrize("relu", [True, False], ids=["relu", "plain"])
@pytest.mark.parametrize("kind", ["nan x", "inf x", "nan g", "nan r"])
def test_nonfinite(kind, relu, training):
    """Channels 1 and 2 receive the non-finite value: the set of non-finite outputs equals the reference's (whose pattern equals
    torch's, tests/test_norm_ref_cpu.py), dbeta is finite where torch's is, the other channels stay within their bars."""
    t, eps = _nonfinite_problem(kind, relu, training)
    got = run_native(t, eps, MOMENTUM, training, relu)
    untouched = [c for c in range(t["x"].shape[1]) if c not in (1, 2)]
    check(got, t, eps, training, relu, "nonfin", cols=untouched)
    tor = torch_autograd(t, eps, MOMENTUM, training, relu)
    assert torch.equal(torch.isfinite(got["dbeta"]).cpu(), torch.isfinite(tor["dbeta"]))
    assert torch.equal(torch.isfinite(got["y"]).cpu(), torch.isfinite(tor["y"]))


# ------------------------------------------------------------------------------------------ argument errors
def test_argument_errors_leave_outputs_untouched():
    M, C = 64, 16
    t = problem(M, C, True, seed=2)
    B = {k: Guarded(v.shape, fill=v.to(DEV)) for k, v in t.items()}
    outs = {k: Guarded(s) for k, s in (("save_mean", (C,)), ("save_invstd", (C,)), ("y", (M, C)), ("dx", (M, C)), ("dr", (M, C)),
                                           ("dgamma", (C,)), ("dbeta", (C,)))}
    nbytes = capi.batch_norm_workspace_bytes(M, C)
    ws = Guarded((nbytes // 4 + 4,))
    P = {k: b.t.data_ptr() for k, b in B.items()}
    O = {k: b.t.data_ptr() for k, b in outs.items()}
    lib, st = capi.lib(), capi._stream()
    w = ws.t.data_ptr()

    def fwd(x=P["x"], y=O["y"], Mx=M, Cx=C, training=1, nb=nbytes):
        return lib.lt_batch_norm_fwd(x, P["r"], P["gamma"], P["beta"], P["rm"], P["rv"], O["save_mean"], O["save_invstd"], y, Mx, Cx,
                                     EPS, MOMENTUM, training, 1, w, nb, st)

    def bwd(y=O["y"], gx=O["dx"], Mx=M, Cx=C, training=1, relu=1, nb=nbytes):
        return lib.lt_batch_norm_bwd(P["x"], y if relu else None, P["g"], P["gamma"], O["save_mean"], O["save_invstd"], gx, O["dr"],
                                     O["dgamma"], O["dbeta"], Mx, Cx, training, relu, w, nb, st)
    calls = {"fwd misaligned x": lambda: fwd(x=P["x"] + 4), "fwd misaligned y": lambda: fwd(y=O["y"] + 4),
             "fwd C % 4": lambda: fwd(Cx=C - 2), "fwd M < 2 train": lambda: fwd(Mx=1), "fwd workspace short": lambda: fwd(nb=nbytes - 1),
             "bwd misaligned dx": lambda: bwd(gx=O["dx"] + 4), "bwd C % 4": lambda: bwd(Cx=C - 2), "bwd M < 2 train": lambda: bwd(Mx=1),
             "bwd workspace short": lambda: bwd(nb=nbytes - 1), "bwd null y with relu": lambda: lib.lt_batch_norm_bwd(
                 P["x"], None, P["g"], P["gamma"], O["save_mean"], O["save_invstd"], O["dx"], O["dr"], O["dgamma"], O["dbeta"], M, C, 1, 1,
                 w, nbytes, st)}
    for name, call in calls.items():
        assert call() == -1, name
        torch.cuda.synchronize()
        for k, b in outs.items():
            assert b.unwritten() == b.n and b.guards_intact(), (name, k)
        assert torch.equal(B["rm"].t, t["rm"].to(DEV)) and torch.equal(B["rv"].t, t["rv"].to(DEV)), name
        assert ws.unwritten() == ws.n, name
    assert fwd() == 0 and bwd() == 0            # the same buffers with valid arguments
    torch.cuda.synchronize()
    assert all(b.unwritten() == 0 and b.guards_intact() for b in outs.values())
