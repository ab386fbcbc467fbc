"""The float64 reference, the per-element bars and the launch plan of the training BatchNorm (csrc/norm.cu), no GPU needed.
tests/test_gpu_norm_ref.py holds the kernels to what is defined here.

Reference (`reference`): float64 BatchNorm (+ residual) (+ ReLU) and its backward from the operands the kernels receive, with the true
float64 statistics; the backward's ReLU mask comes from a given output (the native y on the device, as torch autograd uses its own
output), g' = g [!(y <= 0)].  It equals float64 `torch.native_batch_norm` autograd in train and eval mode, and its NaN pattern
equals torch's for a NaN or Inf in x, a NaN in dY or in the residual; a constant channel with eps = 0 normalises with invstd = 0 in
training, as torch's batch statistics do.

Bars (`bars`), u = 2^-24, per element, first order in u, then scaled by (1 + 2^-10) for the second-order terms:
- fp64 sums (both reduces): recursive sums of exact terms (x - x0 and its square, g' and g' (x - mean_f), fp32 products fit 53
  bits) along a chain of at most n = ceil(rows_per_split / ry) + ry + ceil(splits / 8) + 8 additions (a thread's rows, the CTA's row
  groups, a finalize lane, the lanes), so each is within e64 sum|terms|, e64 = (n + 1) 2^-53 (`plan_e64`).
- statistics (train): with dm = mean - x0 and S2 = var + dm^2 = sum (x - x0)^2 / M, the fp64 variance is within dv = (3 e64 +
  2^-51) S2 (its sums, dm^2 and three fp64 roundings); save_mean within dmu = u|mean| + e64 sqrt(S2) + 2^-52 |mean| (the fp32
  rounding and the sum of x - x0); save_invstd within rho invstd, rho = u + dv / (2 (var + eps)) + 2^-51 (the dv term 0 when
  var + eps = 0, where invstd is exactly 0).  Eval: dmu = 0,
  rho = u + 2^-51.
- y: a = gamma invstd; a_f is within (rho + u)|a|, x - mean_f within dmu + u|x - mean|, the fma rounds once, the residual add once:
  |y - ref| <= |a| ((rho + 2u)|x - mean| + dmu) + u|a (x - mean) + beta| [+ u|y_pre|]; the ReLU is 1-Lipschitz.
- running_mean: m mean_f + fl(fl(1 - m) rm) (with or without fma): m dmu + u (m|mean| + 2 (1 - m)|rm| + |ref|); running_var the
  same with M / (M - 1) var, whose fp32 value is within u|v| + dv M / (M - 1) + 2^-52 |v|.  Eval: both bit-identical.
- dbeta = fl(sum g'): u|ref| + e64 sum|g'|.
- dgamma = fl(sum g' (x - mean_f) invstd_f): the sum is about mean_f, so it is off by dmu |sum g'|; (rho + u)|ref| + invstd (dmu
  |sum g'| + e64 (sum|g'||x - mean| + dmu sum|g'|)).
- dx = fl(a_f fl(fl(g' - k1_f) - fl(xhat_f k2_f))), k1 = sum g' / M, k2 = dgamma / M (0 in eval, where dx = a g'): with
  dk1 = u|k1| + e64 sum|g'| / M, dk2 = u|k2| + bar(dgamma) / M and xhat_f within (rho + 2u)|xhat| + invstd dmu,
  |dx - ref| <= |a| (dk1 + u(|g'| + |k1|) + |xhat| dk2 + (rho + 3u)|xhat||k2| + |k2| invstd dmu) + (rho + 3u)|ref|.
- dr = g': exact.

The bars accept a Python restatement of the kernels' arithmetic (`emulate`: fp64 shifted sums, fp32 finalize and apply) and reject
each of eight plausible slips in it (`MUTATIONS`).

Launch plan (`lt_batch_norm_plan`): the GPU table `CASES` reaches every geometry class, checked at 132 and 114 SMs.
"""
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

from lt_b200 import capi

U = 2.0 ** -24
SECOND_ORDER = 1.0 + 2.0 ** -10
MAX_CTAS = 1024        # kBnMaxCtas
MIN_STEPS = 16         # kBnMinSteps
UNROLL = 4             # kBnUnroll
LANES = 8              # kBnLanes
OUTPUTS = ("y", "save_mean", "save_invstd", "rm", "rv", "dx", "dr", "dgamma", "dbeta")

Case = namedtuple("Case", "M C relu res mean")
# the GPU table: name -> (rows M, channels C, ReLU, residual, |mean| / std)
CASES = {
    "C4 M2 relu": Case(2, 4, True, False, 0.0),
    "C4 M3 res": Case(3, 4, False, True, 0.0),
    "C12 M1001 relu res": Case(1001, 12, True, True, 0.0),        # tc 3: 255-thread block, splits limited by rows, row tail
    "C36 M4099 relu": Case(4099, 36, True, False, 0.0),           # tc 9: 252-thread block
    "C64 M286": Case(286, 64, False, False, 0.0),
    "C128 M70000 relu res": Case(70000, 128, True, True, 0.0),    # ceil(M / rows_per_split) below the wanted splits
    "C132 M1537 relu res": Case(1537, 132, True, True, 0.0),      # a channel block with one of 32 columns
    "C160 M1458 res": Case(1458, 160, False, True, 0.0),          # a channel block with 8 of 32 columns
    "C2048 M8300 relu res": Case(8300, 2048, True, True, 0.0),    # workspace bound by kBnMaxCtas / cblocks
    "C8 M1000003 mean1e3 relu": Case(1000003, 8, True, False, 1e3),
}


def plan(M, C, sms):
    return capi.batch_norm_plan(M, C, sms)


def plan_e64(p):
    """Relative bound of the fp64 sums: (longest chain of additions + 1) 2^-53."""
    n = -(-p["rows_per_split"] // p["ry"]) + p["ry"] + -(-p["splits"] // LANES) + LANES
    return (n + 1) * 2.0 ** -53


# ------------------------------------------------------------------------------------------ problems
def problem(M, C, res, seed, mean=0.0, dev="cpu"):
    """fp32 operands of one call: x [M][C] with per-channel scale and offset (offset `mean` x scale when mean > 0), residual, dY,
    gamma (some negative), beta and running buffers."""
    g = torch.Generator().manual_seed(seed)
    scale = torch.rand(C, generator=g) * 2 + 0.1
    off = (mean if mean else 0.5) * scale * torch.where(torch.rand(C, generator=g) < 0.5, -1.0, 1.0)
    x = torch.randn(M, C, generator=g) * scale + off
    r = torch.randn(M, C, generator=g) if res else None
    dy = torch.randn(M, C, generator=g)
    gamma = 1.0 + 0.5 * torch.randn(C, generator=g)
    beta = 0.3 * torch.randn(C, generator=g)
    rm = 0.1 * torch.randn(C, generator=g)
    rv = torch.rand(C, generator=g) + 0.5
    t = dict(x=x, r=r, g=dy, gamma=gamma, beta=beta, rm=rm, rv=rv)
    return {k: None if v is None else v.float().to(dev) for k, v in t.items()}


# ------------------------------------------------------------------------------------------ the float64 reference
def reference(t, eps, momentum, training, relu, y_mask=None):
    """Float64 forward and backward of one call on the fp32 operands `t` (see `problem`); eps and momentum as the fp32 values the
    kernels receive.  y_mask: the output whose sign gives the ReLU mask (default: the reference's own y).  Returns the outputs and
    the intermediates the bars use."""
    d = {k: None if v is None else v.double() for k, v in t.items()}
    x, r, g = d["x"], d["r"], d["g"]
    M = x.shape[0]
    eps, m = float(np.float32(eps)), float(np.float32(momentum))
    if training:
        mu = x.mean(0)
        xc = x - mu
        var = (xc * xc).mean(0)
    else:
        mu, var = d["rm"], d["rv"]
        xc = x - mu
    invstd = 1.0 / torch.sqrt(var + eps)
    if training and eps == 0:
        invstd = torch.where(var == 0, torch.zeros_like(invstd), invstd)      # torch's InvStd: a constant channel gets 0
    a = d["gamma"] * invstd
    p = a * xc + d["beta"]
    ypre = p if r is None else p + r
    y = torch.where(ypre < 0, torch.zeros_like(ypre), ypre) if relu else ypre
    o = dict(y=y, save_mean=mu, save_invstd=invstd, a=a, xc=xc, p=p, ypre=ypre, var=var, M=M, eps=eps, m=m, training=training,
             rm0=d["rm"], rv0=d["rv"])
    if training:
        o["rm"] = (1 - m) * d["rm"] + m * mu
        o["v_unb"] = var * (M / (M - 1))
        o["rv"] = (1 - m) * d["rv"] + m * o["v_unb"]
        o["dm"] = mu - x[0]
    else:
        o["rm"], o["rv"] = d["rm"].clone(), d["rv"].clone()
    if g is not None:
        ym = y if y_mask is None else y_mask.double()
        gp = torch.where(ym <= 0, torch.zeros_like(g), g) if relu else g
        xhat = xc * invstd
        G1 = gp.sum(0)
        Gxh = (gp * xhat).sum(0)
        if training:
            k1, k2 = G1 / M, Gxh / M
            dx = a * (gp - k1 - xhat * k2)
        else:
            k1 = k2 = torch.zeros_like(G1)
            dx = a * gp
        o.update(dx=dx, dr=gp, dgamma=Gxh, dbeta=G1, gp=gp, xhat=xhat, G1=G1, k1=k1, k2=k2)
    return o


def torch_autograd(t, eps, momentum, training, relu):
    """The same call through float64 torch.native_batch_norm (+ add) (+ relu) autograd."""
    d = {k: None if v is None else v.double() for k, v in t.items()}
    eps, m = float(np.float32(eps)), float(np.float32(momentum))
    x = d["x"].t().unsqueeze(0).clone().requires_grad_(True)              # (1, C, M)
    w = d["gamma"].clone().requires_grad_(True)
    b = d["beta"].clone().requires_grad_(True)
    r = None if d["r"] is None else d["r"].t().unsqueeze(0).clone().requires_grad_(True)
    rm, rv = d["rm"].clone(), d["rv"].clone()
    y, sm, si = torch.native_batch_norm(x, w, b, rm, rv, training, m, eps)
    if r is not None:
        y = y + r
    if relu:
        y = torch.relu(y)
    y.backward(d["g"].t().unsqueeze(0))
    o = dict(y=y.detach()[0].t(), rm=rm, rv=rv, dx=x.grad[0].t(), dgamma=w.grad, dbeta=b.grad, dr=None if r is None else r.grad[0].t())
    if training:
        o.update(save_mean=sm, save_invstd=si)
    return o


# ------------------------------------------------------------------------------------------ bars
def bars(ref, e64):
    """Per-element bars of every output (module docstring); e64 from plan_e64 of the launch."""
    M, m, eps = ref["M"], ref["m"], ref["eps"]
    mu, var, invstd, a = ref["save_mean"], ref["var"], ref["save_invstd"], ref["a"]
    if ref["training"]:
        S2 = var + ref["dm"] ** 2
        dv = (3 * e64 + 2.0 ** -51) * S2
        dmu = U * mu.abs() + e64 * S2.sqrt() + 2.0 ** -52 * mu.abs()
        rho = U + torch.where(var + eps > 0, dv / (2 * (var + eps)), torch.zeros_like(dv)) + 2.0 ** -51
    else:
        dv = dmu = torch.zeros_like(mu)
        rho = torch.full_like(mu, U + 2.0 ** -51)
    xc = ref["xc"]
    b = {"save_mean": dmu, "save_invstd": rho * invstd}
    b["y"] = a.abs() * ((rho + 2 * U) * xc.abs() + dmu) + U * ref["p"].abs()
    if ref["ypre"] is not ref["p"]:
        b["y"] = b["y"] + U * ref["ypre"].abs()
    if ref["training"]:
        b["rm"] = m * dmu + U * (m * mu.abs() + 2 * (1 - m) * ref["rm0"].abs() + ref["rm"].abs())
        v = ref["v_unb"]
        dvu = U * v.abs() + dv * (M / (M - 1)) + 2.0 ** -52 * v.abs()
        b["rv"] = m * dvu + U * (m * v.abs() + 2 * (1 - m) * ref["rv0"].abs() + ref["rv"].abs())
    else:
        b["rm"] = b["rv"] = torch.zeros_like(mu)
    if "dx" in ref:
        gp, xhat, G1, k1, k2 = ref["gp"], ref["xhat"], ref["G1"], ref["k1"], ref["k2"]
        gabs = gp.abs().sum(0)
        b["dbeta"] = U * ref["dbeta"].abs() + e64 * gabs
        b["dgamma"] = (rho + U) * ref["dgamma"].abs() + invstd * (dmu * G1.abs() + e64 * ((gp * xc).abs().sum(0) + dmu * gabs))
        if ref["training"]:
            dk1 = U * k1.abs() + e64 * gabs / M
            dk2 = U * k2.abs() + b["dgamma"] / M
        else:
            dk1 = dk2 = torch.zeros_like(k1)
        b["dx"] = (a.abs() * (dk1 + U * (gp.abs() + k1.abs()) + xhat.abs() * dk2 + (rho + 3 * U) * xhat.abs() * k2.abs()
                              + k2.abs() * invstd * dmu) + (rho + 3 * U) * ref["dx"].abs())
        b["dr"] = torch.zeros_like(gp)
    return {k: v * SECOND_ORDER for k, v in b.items()}


def err_over_bar(got, ref, bar, cols=None):
    """(worst |got - ref| / bar over the elements finite in both, non-finite patterns equal).  A zero bar needs equality."""
    got, ref, bar = got.double(), ref.double(), bar.double().expand_as(ref)
    if cols is not None:
        got, ref, bar = got[..., cols], ref[..., cols], bar[..., cols]
    same_pattern = bool(torch.equal(torch.isfinite(got), torch.isfinite(ref)))
    fin = torch.isfinite(got) & torch.isfinite(ref)
    e, b = (got - ref).abs()[fin], bar[fin]
    if e.numel() == 0:
        return 0.0, same_pattern
    over = torch.where(b > 0, e / torch.where(b > 0, b, torch.ones_like(b)), torch.where(e > 0, torch.full_like(e, math.inf), e))
    return float(over.max()), same_pattern


# ------------------------------------------------------------------------------------------ a restatement of the kernels' arithmetic
MUTATIONS = ("unbiased variance normalises", "eps outside the square root", "running_var from the biased variance", "momentum swapped",
             "fp32 E[x^2] - mean^2 variance", "mask y >= 0", "dr without the mask", "k2 from sum g'")


def emulate(t, eps, momentum, training, relu, mutation=None):
    """The kernels' arithmetic in numpy: fp64 sums of x - x[0] and its square, the fp32 finalize (mean, invstd, running buffers,
    coefficients), fp32 apply passes, fp64 backward sums about mean_f; `mutation` (one of MUTATIONS) plants one slip."""
    f32, f64 = np.float32, np.float64
    n = {k: None if v is None else v.numpy() for k, v in t.items()}
    x, r, g = n["x"], n["r"], n["g"]
    M = x.shape[0]
    eps32, m = f32(eps), f32(momentum)
    rm, rv = n["rm"].copy(), n["rv"].copy()
    if training:
        if mutation == "fp32 E[x^2] - mean^2 variance":
            mean_f = (x.sum(0, dtype=f32) / f32(M)).astype(f32)
            var = np.maximum((x * x).sum(0, dtype=f32) / f32(M) - mean_f * mean_f, 0).astype(f64)
        else:
            dx0 = x.astype(f64) - x[0].astype(f64)
            dm = dx0.sum(0) / M
            var = np.maximum((dx0 * dx0).sum(0) / M - dm * dm, 0.0)
            mean_f = (x[0].astype(f64) + dm).astype(f32)
        vn = var * M / (M - 1) if mutation == "unbiased variance normalises" else var
        if mutation == "eps outside the square root":
            is_f = (1.0 / (np.sqrt(vn) + f64(eps32))).astype(f32)
        else:
            is_f = (1.0 / np.sqrt(vn + f64(eps32))).astype(f32)
        vu = (var if mutation == "running_var from the biased variance" else var * (M / (M - 1))).astype(f32)
        one_m = f32(1) - m
        if mutation == "momentum swapped":
            m, one_m = one_m, m
        rm = (m * mean_f + one_m * rm).astype(f32)
        rv = (m * vu + one_m * rv).astype(f32)
    else:
        mean_f = rm.copy()
        is_f = (1.0 / np.sqrt(rv.astype(f64) + f64(eps32))).astype(f32)
    a = (n["gamma"] * is_f).astype(f32)
    d = (x - mean_f).astype(f32)
    o = (a.astype(f64) * d.astype(f64) + n["beta"].astype(f64)).astype(f32)       # fmaf: one rounding (a d is exact in fp64)
    if r is not None:
        o = (o + r).astype(f32)
    y = np.where(o < 0, f32(0), o) if relu else o
    out = dict(y=y, save_mean=mean_f, save_invstd=is_f, rm=rm, rv=rv)
    if relu:
        mask = (y >= 0) if mutation == "mask y >= 0" else ~(y <= 0)
        gp = np.where(mask, g, f32(0)).astype(f32)
    else:
        gp = g
    s1 = gp.astype(f64).sum(0)
    s2 = (gp.astype(f64) * (x.astype(f64) - mean_f.astype(f64))).sum(0)
    dg = s2 * is_f.astype(f64)
    k1 = (s1 / M).astype(f32) if training else np.zeros_like(mean_f)
    k2 = ((s1 if mutation == "k2 from sum g'" else dg) / M).astype(f32) if training else np.zeros_like(mean_f)
    xhat = (d * is_f).astype(f32)
    tt = ((gp - k1).astype(f32) - (xhat * k2).astype(f32)).astype(f32)
    out.update(dbeta=s1.astype(f32), dgamma=dg.astype(f32), dx=(a * tt).astype(f32) if training else (a * gp).astype(f32),
               dr=g if mutation == "dr without the mask" else gp)
    return {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in out.items()}


def worst(got, ref, b):
    """Largest err/bar over OUTPUTS (inf when a non-finite pattern differs)."""
    w = {}
    for q in OUTPUTS:
        if q == "dr" and ref.get("dr") is None:
            continue
        e, same = err_over_bar(got[q], ref[q], b[q])
        w[q] = e if same else math.inf
    return w


# ------------------------------------------------------------------------------------------ tests: the launch plan
@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("name", list(CASES))
def test_plan_covers_the_rows_within_the_workspace(name, sms):
    c = CASES[name]
    p = plan(c.M, c.C, sms)
    C4 = c.C // 4
    assert p["tc"] == min(C4, 32) and p["ry"] == 256 // p["tc"] and p["cblocks"] == -(-C4 // p["tc"])
    rps, s = p["rows_per_split"], p["splits"]
    assert s * rps >= c.M > (s - 1) * rps
    assert 1 <= s <= min(p["want_splits"], p["max_splits"])
    assert p["want_splits"] == -(-4 * sms // p["cblocks"])
    assert p["max_splits"] == min(-(-c.M // (MIN_STEPS * p["ry"])), -(-MAX_CTAS // p["cblocks"]))
    assert 1 <= p["row_blocks"] <= -(-c.M // (UNROLL * p["ry"]))
    assert capi.batch_norm_workspace_bytes(c.M, c.C) == p["max_splits"] * 2 * c.C * 8 + 5 * c.C * 4
    assert plan(c.M, c.C, 78)["max_splits"] == p["max_splits"]          # the workspace does not depend on the device


def test_case_table_reaches_every_geometry_class():
    P = {n: (c, plan(c.M, c.C, 132)) for n, c in CASES.items()}
    got = set()
    for n, (c, p) in P.items():
        C4, by_rows, by_ctas = c.C // 4, -(-c.M // (MIN_STEPS * p["ry"])), -(-MAX_CTAS // p["cblocks"])
        if p["tc"] < 32:
            got.add("tc < 32")
            if p["tc"] * p["ry"] != 256:
                got.add("block of %d threads" % (p["tc"] * p["ry"]))
        if C4 % p["tc"]:
            got.add("partial channel block C%d" % c.C)
        if p["splits"] == by_rows < p["want_splits"]:
            got.add("splits limited by rows")
        if p["max_splits"] == by_ctas < by_rows:
            got.add("workspace limited by kBnMaxCtas / cblocks")
        if p["splits"] < min(p["want_splits"], p["max_splits"]):
            got.add("final splits below the wanted")
        if c.M in (2, 3):
            got.add("M = %d" % c.M)
        if c.M % (UNROLL * p["ry"]):
            got.add("row tail")
    want = {"tc < 32", "block of 255 threads", "block of 252 threads", "partial channel block C132", "partial channel block C160",
            "splits limited by rows", "workspace limited by kBnMaxCtas / cblocks", "final splits below the wanted", "M = 2", "M = 3",
            "row tail"}
    assert want <= got, want - got
    assert CASES["C2048 M8300 relu res"].C == 2048 and P["C2048 M8300 relu res"][1]["max_splits"] == MAX_CTAS // 16
    assert {c.C for c in CASES.values()} >= {4, 12, 36}


def test_plan_rejects_bad_arguments():
    for M, C, sms in ((100, 6, 132), (0, 8, 132), (100, 8, 0)):
        with pytest.raises(RuntimeError):
            plan(M, C, sms)


# ------------------------------------------------------------------------------------------ tests: the reference
REF_CASES = [(97, 8, False, False), (97, 8, True, False), (64, 12, False, True), (130, 16, True, True), (2, 4, True, True)]


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("M,C,relu,res", REF_CASES)
def test_reference_equals_float64_autograd(M, C, relu, res, training):
    t = problem(M, C, res, seed=M + C)
    ref = reference(t, 1e-5, 0.1, training, relu)
    tor = torch_autograd(t, 1e-5, 0.1, training, relu)
    for q, v in tor.items():
        if v is None:
            assert not res and q == "dr"
            continue
        scale = max(float(v.abs().max()), 1e-300)
        if training and M == 2 and q == "dx":       # exactly zero; both sides are rounding noise of x - mean
            assert float((ref[q] - v).abs().max()) <= 1e-12 * float(ref["a"].abs().max() * t["g"].abs().max())
            continue
        assert float((ref[q] - v).abs().max()) <= 1e-12 * scale, q


def _nonfinite_problem(kind, relu, training, seed=3):
    t = problem(64, 8, kind == "nan r", seed)
    if kind == "nan x":
        t["x"][5, 1] = float("nan")
        t["x"][0, 2] = float("nan")                  # the row the forward's shift reads
    elif kind == "inf x":
        t["x"][7, 1] = float("inf")
        t["x"][0, 2] = float("-inf")
    elif kind == "nan g":
        t["g"][9, 1] = float("nan")
        t["g"][11, 2] = float("nan")
    elif kind == "nan r":
        t["r"][3, 1] = float("nan")
        t["r"][13, 2] = float("nan")
    elif kind == "constant eps 0":
        t["x"][:, 1] = 0.75
    return t, (0.0 if kind == "constant eps 0" else 1e-5)


NONFINITE = ("nan x", "inf x", "nan g", "nan r", "constant eps 0")


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("kind", NONFINITE)
def test_reference_nan_pattern_equals_torch(kind, relu, training):
    if kind == "constant eps 0" and not training:
        pytest.skip("eval mode reads the running variance")
    t, eps = _nonfinite_problem(kind, relu, training)
    ref = reference(t, eps, 0.1, training, relu)
    tor = torch_autograd(t, eps, 0.1, training, relu)
    for q, v in tor.items():
        if v is not None:
            assert torch.equal(torch.isfinite(ref[q]), torch.isfinite(v)), (q, torch.isfinite(ref[q]), torch.isfinite(v))
            fin = torch.isfinite(v)
            assert torch.allclose(ref[q][fin], v[fin], rtol=1e-10, atol=1e-12), q
    # torch's own rule, which the kernels now follow: a NaN output passes its gradient, so dbeta stays finite in a NaN channel
    if relu and training and kind in ("nan x", "inf x"):
        assert not bool(torch.isfinite(tor["y"][:, 1]).any()) and bool(torch.isfinite(tor["dbeta"][1]))
        assert float(tor["dbeta"][1]) == pytest.approx(float(t["g"][:, 1].double().sum()), rel=1e-12)


# ------------------------------------------------------------------------------------------ tests: the bars
BAR_CASES = {"C8 M1000 relu res": (1000, 8, True, True, 0.0), "C12 M777": (777, 12, False, False, 0.0),
             "C8 M4096 mean1e3 relu": (4096, 8, True, False, 1e3)}


@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("name", list(BAR_CASES))
def test_bars_accept_the_kernel_arithmetic(name, training):
    M, C, relu, res, mean = BAR_CASES[name]
    t = problem(M, C, res, seed=M, mean=mean)
    em = emulate(t, 1e-5, 0.1, training, relu)
    ref = reference(t, 1e-5, 0.1, training, relu, y_mask=em["y"])
    w = worst(em, ref, bars(ref, plan_e64(plan(M, C, 132))))
    print(name, "train" if training else "eval", " ".join("%s %.3f" % kv for kv in w.items()))
    assert max(w.values()) <= 1.0, w


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_bars_reject_each_mutation(mutation):
    name = "C8 M4096 mean1e3 relu" if mutation == "fp32 E[x^2] - mean^2 variance" else "C8 M1000 relu res"
    M, C, relu, res, mean = BAR_CASES[name]
    t = problem(M, C, res, seed=M, mean=mean)
    em = emulate(t, 1e-5, 0.1, True, relu, mutation)
    ref = reference(t, 1e-5, 0.1, True, relu, y_mask=em["y"] if mutation != "mask y >= 0" else None)
    w = worst(em, ref, bars(ref, plan_e64(plan(M, C, 132))))
    print(mutation, " ".join("%s %.3g" % kv for kv in w.items()))
    assert max(w.values()) > 1.0, w
