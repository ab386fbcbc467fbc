"""Every backward convolution kernel against a float64 reference built from the exact operands it received.

Weight gradient (lt_conv_wgrad_fwd: conv_wgrad_kernel<1 / 2 / 4> + wgrad_reduce_kernel), one case table (WCASES) whose plans are
checked host-side at 132 SMs by tests/test_conv_bwd_cpu.py.  Each case checks, per element of dW:
- |native - ref| <= 2 (8 + ceil(m_tiles / splits) + 3 + splits) 2^-24 sum|x||g| / S + 2^-24 |ref|  (test_conv_bwd_cpu.wgrad_bar:
  8 truncating k16 steps per fresh tile accumulator, one round-to-nearest add per tile of a split, three quadrant adds, the split
  reduce, an exact power-of-two multiply), against test_conv_bwd_cpu.wgrad_reference of the dequantized split-fp16 input and
  scaled output gradient;
- against the original float32 operands, with the split representation term (max(2^-22 |v|, 2^-25) per operand, the low half's
  subnormal floor of common.cuh) added: native error <= max(bar + representation, 2 x the error of float32 torch, TF32 off);
- grad_w between NaN guard bands, starting as a NaN sentinel, and a workspace of exactly lt_conv_wgrad_workspace_bytes pre-filled
  with NaN: guards intact, every element written;
- a second run and a CUDA-graph replay of absmax -> scaled conversion -> wgrad -> reduce are bit-identical to the first run.

Data gradients run on the forward kernels: ConvNdFn, ConvTranspose3dFn and ConvTranspose2dK4Fn backwards with capi.conv_nd recorded,
each data-gradient launch checked per element with the forward suite's reference and bar (tests/test_gpu_conv.py), and its float32
scale checked to equal (1 / filter pre-scale) (1 / S) accum_gain(steps of the kernel that ran).

Output-gradient scale edges (all zero, a power of two and one ulp below, 2^-100 / 2^-101 / 2^100 / 2^101, one NaN, one +Inf) on a
conv, a deconv and the stem, and one NaN in a forward input: every element that is non-finite in the float64 reference is
non-finite in the native result, every finite native element is within an fp32-grade bar.  Input magnitudes 2^-8 and 2^8 stay
within the weight-gradient bar; at 2^-16 the representation floor 2^-25 of the split input is what bounds the error.

Measured on an H100 80GB HBM3 (700 W power limit), largest err/bar per family: conv_wgrad_kernel<1> 0.082, <2> 0.128, <4> 0.159,
k4s2 phases 0.130, k2s2 0.112, stem 0.058, the 44-split large-K layer < 0.001; against float32 operands err/limit <= 0.174.  Data
gradients: conv_lines_kernel 0.022, conv_tc_kernel 0.048, conv_fold_kernel<7, 32> 0.025, split-K 0.008.  Systematic gain of dW on the
large-K layer -1.55e-7 (model -1.34e-7).  Before the fixes in common.cuh, the NaN / Inf and 2^-101 / 2^101 edges failed: NaN came out
as finite values, and 2^-101 gave dX = dW = 0.
"""
import json
import os
import re
import subprocess
import sys
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lt_b200 import autograd_ops as A
from lt_b200 import capi
from test_conv_bwd_cpu import (EPS, _geometry, pow2_scale, s2d, wgrad_bar, wgrad_reference, wgrad_reference_sig, wgrad_steps)
from test_conv_cpu import (F32, RES_NONE, Launch, accum_gain, accum_steps_launched, dequant_fold, dequant_tc, effective_steps,
                           launched_kernels, s32_value)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FOLD = capi.CONV_TC_FOLD
WS_BYTES = 32 << 20


def _ru(v, m):
    return (v + m - 1) // m * m


# ------------------------------------------------------------------------------------------ the weight-gradient case table
# expect: (instantiation, K splits, stages) of every launch at 132 SMs.  kind: conv (3-D form: a 2-D conv has D = 1; padding k // 2)
# | deconv3d (k2 s2, one grouped launch) | deconv2d (k4 s2 p1, four phase launches) | stem (I = (1, H, W) of the images)
WCase = namedtuple("WCase", "expect kind N I cin cout k s")


def wcase(expect, kind="conv", N=2, I=(1, 8, 8), cin=32, cout=32, k=(1, 3, 3), s=(1, 1, 1)):
    return WCase(tuple(expect), kind, N, I, cin, cout, k, s)


W1, W2, W4 = "conv_wgrad_kernel<1>", "conv_wgrad_kernel<2>", "conv_wgrad_kernel<4>"
K3, K7 = (3, 3, 3), (7, 7, 7)
LARGE_K = "large K: 3^3 32->32 at 64^3, N 2"
WCASES = {
    # conv_wgrad_kernel<1>: Cout 32 (6 stages)
    "nwg1 3^3 32->32 partial boxes": wcase((W1, 1, 6), N=2, I=(3, 5, 7), k=K3),
    "nwg1 3^3 16->32 (Cin 16 of 32)": wcase((W1, 1, 6), N=2, I=(4, 5, 6), cin=16, k=K3),
    "nwg1 final_layer 1x1 32->17": wcase((W1, 1, 6), N=2, I=(1, 9, 7), cout=17, k=(1, 1, 1)),
    "nwg1 V2V output_layer 1^3 32->17": wcase((W1, 1, 6), N=2, I=(6, 5, 7), cout=17, k=(1, 1, 1)),
    "nwg1 tiny maps N8 (boxes span samples)": wcase((W1, 1, 6), N=8, I=(2, 2, 2), k=K3),
    "nwg1 7^3 32->16": wcase((W1, 1, 6), N=1, I=(5, 6, 16), cout=16, k=K7),
    # conv_wgrad_kernel<2>: Cout 64 (4 stages)
    "nwg2 3x3 64->64": wcase((W2, 1, 4), N=2, I=(1, 9, 7), cin=64, cout=64),
    "nwg2 stem 12/32 -> 64": wcase((W2, 1, 4), kind="stem", N=2, I=(1, 22, 18), cout=64),
    "nwg2 s2k3 32->64 even": wcase((W2, 1, 4), N=3, I=(1, 8, 10), cin=32, cout=64, s=(1, 2, 2)),
    # conv_wgrad_kernel<4> (2 stages): 4 active, 3 active (the backbone test's head 3x3 -> 96), several groups along N
    "nwg4 3^3 128->128": wcase((W4, 1, 2), N=2, I=(4, 4, 5), cin=128, cout=128, k=K3),
    "nwg4 3 active: head 3x3 32->96": wcase((W4, 1, 2), N=2, I=(1, 8, 6), cin=32, cout=96),
    "nwg4 2 groups, 1 of 4 in the last: 1x1 64->160": wcase((W4, 1, 2), N=2, I=(1, 7, 9), cin=64, cout=160, k=(1, 1, 1)),
    "nwg4 2 groups, 3 of 4 in the last: 1x1 32->224": wcase((W4, 1, 2), N=2, I=(1, 6, 5), cin=32, cout=224, k=(1, 1, 1)),
    "nwg4 s2k3 64->128 odd": wcase((W4, 1, 2), N=2, I=(1, 13, 11), cin=64, cout=128, s=(1, 2, 2)),
    "nwg4 s2k1 64->128 odd": wcase((W4, 1, 2), N=2, I=(1, 13, 11), cin=64, cout=128, k=(1, 1, 1), s=(1, 2, 2)),
    # K split over M tiles
    "split 1x1 32->32 at 64x64, N 2": wcase((W1, 4, 6), N=2, I=(1, 64, 64), k=(1, 1, 1)),
    "split 3x3 64->64 at 64x80, N 2": wcase((W2, 5, 4), N=2, I=(1, 64, 80), cin=64, cout=64),
    LARGE_K: wcase((W1, 44, 6), N=2, I=(64, 64, 64), k=K3),      # 44 splits of 4096 tiles: uneven (93 or 94 tiles)
    # transposed convs
    "deconv3d k2s2 64->32": wcase((W4, 1, 2), kind="deconv3d", N=2, I=(3, 2, 5), cin=64, cout=32),
    "deconv3d k2s2 32->64": wcase((W4, 1, 2), kind="deconv3d", N=2, I=(2, 3, 2), cin=32, cout=64),
    "deconv3d k2s2 64->128": wcase((W4, 1, 2), kind="deconv3d", N=2, I=(1, 2, 3), cin=64, cout=128),
    "deconv2d k4s2 64->32 odd": wcase((W1, 1, 6), kind="deconv2d", N=2, I=(1, 5, 7), cin=64, cout=32),
    "deconv2d k4s2 32->64 even": wcase((W2, 1, 4), kind="deconv2d", N=1, I=(1, 6, 4), cin=32, cout=64),
}

LW = namedtuple("LW", "desc taps cin cout G")


def wgrad_launches(c):
    """The lt_conv_wgrad_fwd launches of a case, as the training functions issue them (autograd_ops)."""
    if c.kind == "conv":
        p = tuple(v // 2 for v in c.k)
        return [LW(A.conv3d_wgrad_desc(c.N, c.I, c.cin, c.cout, c.k, p, c.s), int(np.prod(c.k)), c.cin, c.cout, 1)]
    if c.kind == "deconv3d":
        return [LW(A.conv_transpose3d_desc(c.N, c.I, c.cin, c.cout), 1, c.cin, c.cout, 8)]
    if c.kind == "deconv2d":
        return [LW(A.conv_transpose2d_k4s2_desc(c.N, c.I, c.cin, c.cout, py, px), 4, c.cin, c.cout, 1) for py in (0, 1) for px in (0, 1)]
    return [LW(A.stem_wgrad_desc(c.N, c.I[1], c.I[2], c.cout), 16, 12, c.cout, 1)]


def _dims(c):
    """(input (D, H, W), input channels as stored, output gradient (D, H, W), its channels as stored)."""
    d = wgrad_launches(c)[0].desc
    return (d.ID, d.IH, d.IW), d.Cin, (d.FD, d.FH, d.FW), d.FC


def host_operands(c, seed):
    """float64 CPU operands of a case as the kernel reads them: input [N][ID][IH][IW][Cin stored], output gradient
    [N][FD][FH][FW][FC], real channels random, padding channels zero."""
    g = torch.Generator().manual_seed(seed)
    I, cin_s, Fd, fc = _dims(c)
    if c.kind == "stem":
        x = s2d(torch.randn(c.N, 3, c.I[1], c.I[2], generator=g, dtype=torch.float64))
    else:
        x = torch.zeros(c.N, *I, cin_s, dtype=torch.float64)
        x[..., :c.cin] = torch.randn(c.N, *I, c.cin, generator=g, dtype=torch.float64)
    gy = torch.zeros(c.N, *Fd, fc, dtype=torch.float64)
    gy[..., :c.cout] = torch.randn(c.N, *Fd, c.cout, generator=g, dtype=torch.float64)
    return x, gy


# ------------------------------------------------------------------------------------------ device helpers
@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def _guarded(shape, dtype, fill=None):
    from test_gpu_unproject import Guarded
    return Guarded(shape, dtype, guard=256, fill=fill)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Built:
    """Guarded split-fp16 input and scaled output gradient of one case, the float32 originals, amax bits and 1 / S."""


def build(c, seed=0, x_scale=1.0, dy=None):
    torch.manual_seed(seed)
    b = Built()
    I, cin_s, Fd, fc = _dims(c)
    if c.kind == "stem":
        img = torch.randn(c.N, 3, c.I[1], c.I[2], device=DEV) * x_scale
        b.x = _guarded((c.N, *I, 2 * cin_s), torch.float16)
        capi.stem_s2d(img, b.x.t, c.N, 3, c.I[1], c.I[2])
        b.x_orig = s2d(img.double())
    else:
        x32 = (torch.randn(c.N, *I, c.cin, device=DEV) * x_scale).contiguous()
        b.x = _guarded((c.N, *I, 2 * cin_s), torch.float16)
        capi.f32_to_s32_scaled(x32, b.x.t, x32[..., 0].numel(), c.cin, cin_s)
        b.x_orig = F.pad(x32.double(), (0, cin_s - c.cin))
    b.dy = (torch.randn(c.N, *Fd, c.cout, device=DEV) * 1e-3 if dy is None else dy).contiguous()
    b.amax = torch.empty(1, dtype=torch.int32, device=DEV)
    b.inv = torch.empty(1, dtype=torch.float32, device=DEV)
    b.g = _guarded((c.N, *Fd, 2 * fc), torch.float16)
    capi.absmax(b.dy, b.amax)
    capi.f32_to_s32_scaled(b.dy, b.g.t, b.dy[..., 0].numel(), c.cout, fc, b.amax, b.inv)
    b.dy_orig = F.pad(b.dy.double(), (0, fc - c.cout))
    torch.cuda.synchronize()
    b.S = 1.0 / float(b.inv)
    return b


def run_wgrad(b, lw, g=None, amax=None):
    """One lt_conv_wgrad_fwd into a NaN-sentinel grad_w between guard bands, with a NaN-filled workspace of exactly the bytes
    lt_conv_wgrad_workspace_bytes asks for (also between guard bands) -> (grad_w, workspace)."""
    nbytes = capi.conv_wgrad_workspace_bytes(lw.desc)
    assert nbytes > 0 and nbytes % 4 == 0
    ws = _guarded((nbytes // 4,), torch.float32)
    gw = _guarded((lw.taps, lw.cin, lw.G * lw.cout), torch.float32)
    capi.conv_wgrad(lw.desc, b.x.t, b.g.t if g is None else g, b.amax if amax is None else amax, lw.cin, lw.cout, gw.t, ws.t)
    return gw, ws


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32).clone()


def rep_term(x, g, d, S, cin, cout):
    """The split representation term against float32 operands: each operand v is stored within 2^-22 |v| + 2^-25 (the scaled output
    gradient in its scaled units), so dW moves by at most W(|x|(1 + 2^-22) + 2^-25, |g|(1 + 2^-22) + 2^-25) - W(|x|, |g|)."""
    xa, ga = x.abs(), g.abs()
    return (wgrad_reference(xa * (1 + 2.0 ** -22) + 2.0 ** -25, ga * (1 + 2.0 ** -22) + 2.0 ** -25, d, S, cin, cout)
            - wgrad_reference(xa, ga, d, S, cin, cout))


def f32_operand_check(b, lw, got, plan, label, floor=True):
    """-> largest err / limit against the original float32 operands; limit = max(bar + representation, 2 x float32 torch error)."""
    go = b.dy_orig * b.S                       # exact: S is a power of two
    ref_o, sig_o = wgrad_reference_sig(b.x_orig, go, lw.desc, b.S, lw.cin, lw.cout)
    rep = rep_term(b.x_orig, go, lw.desc, b.S, lw.cin, lw.cout) if floor else 2.0 ** -21 * sig_o
    t32 = wgrad_reference(b.x_orig.float(), go.float(), lw.desc, b.S, lw.cin, lw.cout).double()
    e_o = (got - ref_o).abs()
    lim = torch.maximum(wgrad_bar(ref_o, sig_o, plan) + rep, 2.0 * (t32 - ref_o).abs())
    r = float((e_o / lim.clamp(min=1e-300)).max())
    print("%-48s vs float32 operands: max err %.2e, float32 torch %.2e, largest err/limit %.3f"
          % (label, float(e_o.max()), float((t32 - ref_o).abs().max()), r))
    return r


RATIOS = {}


def _ratio_family(name, c, ratio):
    fam = c.kind if c.kind != "conv" else c.expect[0]
    RATIOS[fam] = max(RATIOS.get(fam, 0.0), ratio)
    print("worst err/bar so far per family: %s" % ", ".join("%s %.3f" % kv for kv in sorted(RATIOS.items())))


@pytest.mark.parametrize("name", list(WCASES))
def test_wgrad_vs_float64(name):
    c = WCASES[name]
    b = build(c, seed=sum(map(ord, name)) % 1000)
    assert b.S == pow2_scale(float(b.dy.abs().max()))
    x_eff, g_eff = s32_value(b.x.t), s32_value(b.g.t)
    sms = _sms()
    lws = wgrad_launches(c)
    outs = []
    worst = 0.0
    for lw in lws:
        gw, ws = run_wgrad(b, lw)
        torch.cuda.synchronize()
        assert gw.guards_intact() and ws.guards_intact(), "a write landed outside grad_w or the workspace"
        assert gw.unwritten() == 0, "%d grad_w elements were never written" % gw.unwritten()
        assert ws.unwritten() == 0, "%d workspace elements (partial tiles) were never written" % ws.unwritten()
        assert b.x.guards_intact() and b.g.guards_intact()
        plan = capi.conv_wgrad_plan(lw.desc, sms)
        ref, sig = wgrad_reference_sig(x_eff, g_eff, lw.desc, b.S, lw.cin, lw.cout)
        got = gw.t.double()
        err = (got - ref).abs()
        ratio = float((err / wgrad_bar(ref, sig, plan).clamp(min=1e-300)).max())
        worst = max(worst, ratio)
        print("%-48s %s splits %d stages %d: largest err/bar %.3f (max err %.2e, max |ref| %.2e)"
              % (name, "conv_wgrad_kernel<%d>" % plan["nwg"], plan["splits"], plan["stages"], ratio, float(err.max()),
                 float(ref.abs().max())))
        assert ratio <= 1.0, (name, ratio)
        assert f32_operand_check(b, lw, got, plan, "") <= 1.0
        gw2, _ = run_wgrad(b, lw)
        torch.cuda.synchronize()
        assert torch.equal(bits(gw2.t), bits(gw.t)), "a second run differs"
        outs.append(gw)
    _ratio_family(name, c, worst)
    # CUDA-graph replay of the whole backward chain: absmax -> scaled conversion -> wgrad -> reduce (warmed up by the eager runs)
    amax2 = torch.empty_like(b.amax)
    inv2 = torch.empty_like(b.inv)
    g2 = torch.empty_like(b.g.t)
    bufs = [(_guarded(o.t.shape, torch.float32), _guarded((capi.conv_wgrad_workspace_bytes(lw.desc) // 4,), torch.float32))
            for lw, o in zip(lws, outs)]
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        capi.absmax(b.dy, amax2)
        capi.f32_to_s32_scaled(b.dy, g2, b.dy[..., 0].numel(), c.cout, b.g.t.shape[-1] // 2, amax2, inv2)
        for lw, (o, w) in zip(lws, bufs):
            capi.conv_wgrad(lw.desc, b.x.t, g2, amax2, lw.cin, lw.cout, o.t, w.t)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(bits(g2), bits(b.g.t)) and float(inv2) == float(b.inv)
    for o, (og, _) in zip(outs, bufs):
        assert og.guards_intact() and torch.equal(bits(og.t), bits(o.t)), "the CUDA-graph replay differs"


@pytest.mark.parametrize("x_scale", [2.0 ** -8, 2.0 ** 8, 2.0 ** -16])
def test_wgrad_input_magnitude(x_scale):
    """The forward input x is split unscaled: at 2^-8 and 2^8 the weight gradient stays within the bar plus the representation term;
    at 2^-16 the high half is an fp16 subnormal and the low half mostly 0, so the representation floor max(2^-22 |x|, 2^-25) of
    common.cuh bounds the error -- 2^-21 sum|x||g| alone (the term for normal halves) is exceeded there."""
    c = wcase((W1, 1, 6), N=2, I=(4, 6, 10), k=K3)
    b = build(c, seed=11, x_scale=x_scale)
    lw = wgrad_launches(c)[0]
    gw, _ = run_wgrad(b, lw)
    torch.cuda.synchronize()
    plan = capi.conv_wgrad_plan(lw.desc, _sms())
    ref, sig = wgrad_reference_sig(s32_value(b.x.t), s32_value(b.g.t), lw.desc, b.S, lw.cin, lw.cout)
    got = gw.t.double()
    assert float(((got - ref).abs() / wgrad_bar(ref, sig, plan)).max()) <= 1.0
    assert f32_operand_check(b, lw, got, plan, "x scaled by 2^%d" % round(np.log2(x_scale))) <= 1.0
    if x_scale == 2.0 ** -16:
        assert f32_operand_check(b, lw, got, plan, "  without the 2^-25 floor", floor=False) > 1.0


# ------------------------------------------------------------------------------------------ data gradients, recorded
# (kind, x shape, weight shape, stride, padding, kernels the data-gradient launch must run)
T128, T64, T32, T16, RED = "conv_tc_kernel<128>", "conv_tc_kernel<64>", "conv_tc_kernel<32>", "conv_tc_kernel<16>", "splitk_reduce_kernel"
DCase = namedtuple("DCase", "kind x w stride pad expect")
DCASES = {
    "lines 3^3 32->32 W16": DCase("conv", (2, 32, 3, 4, 16), (32, 32, 3, 3, 3), 1, 1, ["conv_lines_kernel<32>"]),
    "lines 3^3 32->32 W40": DCase("conv", (1, 32, 2, 3, 40), (32, 32, 3, 3, 3), 1, 1, ["conv_lines_kernel<32>"]),
    "lines 3^3 32->32 W64": DCase("conv", (1, 32, 2, 2, 64), (32, 32, 3, 3, 3), 1, 1, ["conv_lines_kernel<32>"]),
    "conv_tc 3^3 32->32 W12 (scale, not scale_fold)": DCase("conv", (2, 32, 3, 4, 12), (32, 32, 3, 3, 3), 1, 1, [T32, RED]),
    "conv_tc 3^3 32->32 W80 (scale, not scale_fold)": DCase("conv", (1, 32, 2, 3, 80), (32, 32, 3, 3, 3), 1, 1, [T32, RED]),
    "fold7 dgrad 16->32 of 7^3 32->16": DCase("conv", (1, 32, 3, 5, 16), (16, 32, 7, 7, 7), 1, 3, ["conv_fold_kernel<7, 32>"]),
    "split-K V2V 4^3 128->128 N 8": DCase("conv", (8, 128, 4, 4, 4), (128, 128, 3, 3, 3), 1, 1, [T128, RED]),
    "split-K 1x1 dgrad 2048->512": DCase("conv2d", (2, 512, 8, 8), (2048, 512, 1, 1), 1, 0, None),
    "s2k1 1x1 64->128 odd": DCase("conv2d", (2, 64, 13, 11), (128, 64, 1, 1), 2, 0, None),
    "s2k3 grouped 64->128 odd": DCase("conv2d", (2, 64, 13, 11), (128, 64, 3, 3), 2, 1, None),
    "s2k3 grouped 32->64 even": DCase("conv2d", (2, 32, 8, 10), (64, 32, 3, 3), 2, 1, None),
    "deconv3d k2s2 dgrad 2^3 s2": DCase("deconv3d", (2, 64, 3, 2, 5), (64, 32, 2, 2, 2), 2, 0, None),
    "deconv2d k4s2 dgrad 4x4 s2": DCase("deconv2d", (2, 64, 5, 7), (64, 32, 4, 4), 2, 1, None),
}


def _fn(dc):
    if dc.kind == "conv":
        return lambda x, w, b: A.conv3d(x, w, b, (dc.pad,) * 3), lambda x, w, b: F.conv3d(x, w, b, 1, dc.pad)
    if dc.kind == "conv2d":
        return (lambda x, w, b: A.conv2d(x, w, b, (dc.stride,) * 2, (dc.pad,) * 2),
                lambda x, w, b: F.conv2d(x, w, b, dc.stride, dc.pad))
    if dc.kind == "deconv3d":
        return A.conv_transpose3d, lambda x, w, b: F.conv_transpose3d(x, w, b, 2)
    return A.conv_transpose2d_k4s2, lambda x, w, b: F.conv_transpose2d(x, w, b, 2, 1)


def _problem(dc, seed):
    """x, a Kaiming-sized filter and a bias of the case (nn.Conv filters are (Cout, Cin, k...), nn.ConvTranspose (Cin, Cout, k...))."""
    conv = dc.kind.startswith("conv")
    fan = int(np.prod(dc.w[1:])) if conv else dc.w[0]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*dc.x, generator=g)
    w = torch.randn(*dc.w, generator=g) * (1.0 / fan) ** 0.5
    b = torch.randn(dc.w[0] if conv else dc.w[1], generator=g) * 0.1
    return x.to(DEV), w.to(DEV), b.to(DEV)


def run_recorded(fn, x, w, b, gy, record_forward=False):
    """Forward and backward of a training function with every capi.conv_nd call recorded (descriptor, operands, scale, impl and the
    output after the call) -> (backward launches [, forward launches], native (y, dX, dW))."""
    recs = []
    orig = capi.conv_nd

    def rec(d, inp, weight, scale, shift, residual, out, impl):
        r = dict(desc=capi.ConvDesc.from_buffer_copy(d), inp=inp.clone(), weight=weight.clone(), scale=scale.clone(),
                 shift=shift.clone(), impl=impl)
        orig(d, inp, weight, scale, shift, residual, out, impl)
        r["out"] = out.clone()
        recs.append(r)
    capi.conv_nd = rec
    try:
        xn = x.clone().requires_grad_(x.dim() != 4 or fn is not A.stem_conv)
        wn, bn = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
        y = fn(xn, wn, bn)
        fwd = list(recs)
        recs.clear()
        y.backward(gy)
        torch.cuda.synchronize()
    finally:
        capi.conv_nd = orig
    return recs, fwd, (y.detach(), xn.grad, wn.grad)


def check_recorded_launch(r, w_src, S, label):
    """One recorded lt_conv_nd_fwd per element against the forward suite's float64 reference and bar, and its scale."""
    import test_gpu_conv as G
    d, impl = r["desc"], r["impl"]
    k, s, p, O, Fd, os_, oo, og = _geometry(d)
    CW = 32 if impl == FOLD else d.Cout
    L = Launch(d.N, (d.ID, d.IH, d.IW), O, k, s, p, Fd, os_, oo, og, CW, d.FC)
    taps = k[0] * k[1] * k[2]
    if impl == FOLD:
        w_eff = dequant_fold(r["weight"], k[0], _ru(d.Cout, 16))
        folded = accum_steps_launched(impl, L, d.Cin, d.Cout, WS_BYTES)
    else:
        w_eff = dequant_tc(r["weight"], taps, d.Cin, d.Cout)
        folded = taps * d.Cin // 16
    assert effective_steps(impl, L, d.Cin, d.Cout, folded, WS_BYTES) == accum_steps_launched(impl, L, d.Cin, d.Cout, WS_BYTES)
    # the scale: (1 / filter pre-scale) x accum_gain(folded steps), rounded once, times 1 / S of the output gradient
    n_real = (og[0] * og[1] * og[2]) * (w_src.shape[1] if w_src.dim() in (4, 5) and label.startswith("conv") else w_src.shape[0])
    want = float(np.float32(np.float32(accum_gain(folded) / pow2_scale(float(w_src.abs().max()))) * np.float32(1.0 / S)))
    sc = r["scale"]
    assert bool((sc[:n_real] == want).all()) and bool((sc[n_real:] == 0).all()), (label, float(sc[0]), want)
    b = G.Built()
    b.parts = [G.Part(impl, L, d.Cin, d.Cout, folded, None, WS_BYTES)]
    b.x_eff = s32_value(r["inp"])
    b.w_eff = [F.pad(w_eff, (0, CW - w_eff.shape[2]))]
    b.s_eff = [F.pad(sc.double(), (0, CW - sc.numel())) / accum_gain(folded)]
    b.sh_eff = [F.pad(r["shift"].double(), (0, CW - r["shift"].numel()))]
    b.out_shape, b.res_eff = (d.N, *Fd, d.FC), None
    c = G.case("-", mode="tc", fmt=F32, res=RES_NONE, relu=False)
    ref, bar, _ = G.reference(c, b)
    got = r["out"].double().reshape(-1)
    written = ~torch.isnan(ref)
    ratio = float(((got - ref).abs()[written] / bar[written]).max())
    return launched_kernels(impl, L, d.Cin, d.Cout, WS_BYTES), ratio, written


@pytest.mark.parametrize("name", list(DCASES))
def test_dgrad_launches_vs_float64(name):
    dc = DCASES[name]
    x, w, b = _problem(dc, sum(map(ord, name)) % 997)
    fn, ref_fn = _fn(dc)
    with torch.no_grad():
        y0 = ref_fn(x.double(), w.double(), b.double())
    gy = (torch.randn(y0.shape, device=DEV) * 1e-3).float()
    recs, _, (y, gx, gw) = run_recorded(fn, x, w, b, gy)
    assert len(recs) == 1, len(recs)
    S = pow2_scale(float(gy.abs().max()))
    kernels, ratio, written = check_recorded_launch(recs[0], w, S, dc.kind)
    print("%-48s %s: largest err/bar %.3f" % (name, "+".join(kernels), ratio))
    RATIOS["dgrad " + kernels[0]] = max(RATIOS.get("dgrad " + kernels[0], 0.0), ratio)
    if dc.expect is not None:
        assert kernels == dc.expect, (name, kernels)
    if name.startswith("split-K"):
        assert kernels[-1] == RED, kernels
    assert ratio <= 1.0, (name, ratio)
    if name.startswith("s2k1"):
        odd = torch.ones(gx.shape[2:], dtype=torch.bool, device=DEV)
        odd[::2, ::2] = False
        assert bool((gx[:, :, odd] == 0).all()), "s2k1: dX off the even phase must be exactly 0"
    if name.startswith("s2k3") and dc.x[2] % 2:
        d = recs[0]["desc"]
        assert (d.FH, d.FW) == tuple(dc.x[2:]) and int(written.sum()) == int(np.prod(dc.x)) // dc.x[1] * _ru(dc.x[1], 4)


# ------------------------------------------------------------------------------------------ output-gradient scale edges
EDGE_FNS = {
    # (x shape, weight shape, native function, float64 function)
    "conv": ((2, 32, 3, 4, 16), (32, 32, 3, 3, 3), lambda x, w, b: A.conv3d(x, w, b, (1, 1, 1)),
             lambda x, w, b: F.conv3d(x, w, b, 1, 1)),
    "deconv": ((2, 64, 3, 2, 4), (64, 32, 2, 2, 2), A.conv_transpose3d, lambda x, w, b: F.conv_transpose3d(x, w, b, 2)),
    "stem": ((2, 3, 16, 12), (64, 3, 7, 7), A.stem_conv, lambda x, w, b: F.conv2d(x, w, b, 2, 3)),
}
EDGES = ["zero", "pow2", "pow2 - ulp", "2^-100", "2^-101", "2^100", "2^101", "nan", "inf"]


def _edge_dy(shape, edge, seed):
    g = torch.Generator().manual_seed(seed)
    dy = torch.randn(*shape, generator=g)
    i0 = dy.numel() // 3
    if edge == "zero":
        return torch.zeros(shape)
    if edge in ("nan", "inf"):
        dy = dy * 1e-3
        dy.view(-1)[i0] = float(edge)
        return dy
    if edge.startswith("pow2"):
        top = np.float32(2.0 ** -3) if edge == "pow2" else np.nextafter(np.float32(2.0 ** -3), np.float32(0))
    else:
        top = np.float32(2.0 ** int(edge[2:]))
    dy = dy / dy.abs().max() * float(top) * 0.5
    dy.view(-1)[i0] = float(top)
    assert float(dy.abs().max()) == float(top)
    return dy


def _rule(nat, ref, bar, label):
    """Non-finite in the reference -> non-finite in the native result; finite native elements within the bar."""
    nat, ref = nat.double(), ref.double()
    bad = ~torch.isfinite(ref)
    assert bool((~torch.isfinite(nat[bad])).all()), "%s: %d elements non-finite in float64 came out finite" % (
        label, int(torch.isfinite(nat[bad]).sum()))
    fin = torch.isfinite(nat) & ~bad
    r = float(((nat - ref).abs()[fin] / bar[fin]).max()) if bool(fin.any()) else 0.0
    print("%-40s non-finite %d / %d, largest err/bar over the finite %.3f" % (label, int(bad.sum()), ref.numel(), r))
    assert r <= 1.0, (label, r)


def _edge_bars(ref_fn, x, w, b, gy, S, steps):
    """float64 autograd of ref_fn -> (y, dX, dW) with per-element fp32-grade bars: 2 steps 2^-24 sig + 2^-23 |ref| + the split
    representation term of x, w (pre-scaled by its power of two) and the scaled gy."""
    def grads(xx, ww, bb, gg, need_x):
        xx = xx.double().requires_grad_(need_x)
        ww = ww.double().requires_grad_(True)
        y = ref_fn(xx, ww, bb.double())
        y.backward(gg.double())
        return y.detach(), (xx.grad if need_x else None), ww.grad
    need_x = x.shape[1] != 3
    ref = grads(x, w, b, gy, need_x)
    zb = torch.zeros_like(b)
    sig = grads(x.abs(), w.abs(), zb, gy.abs(), need_x)
    Sw = pow2_scale(float(w.abs().max()))
    up = lambda v, s: v.abs().double() * (1 + 2.0 ** -22) + 2.0 ** -25 / s
    sig2 = grads(up(x, 1.0), up(w, Sw), zb, up(gy, S), need_x)
    bars = []
    for r, s1, s2 in zip(ref, sig, sig2):
        bars.append(None if r is None else 2.0 * steps * EPS * s1 + 2.0 ** -23 * r.abs() + (s2 - s1) + 1e-300)
    return ref, bars


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("which", list(EDGE_FNS))
def test_output_gradient_scale_edges(which, edge):
    """dY all zero gives exactly zero dX and dW; a power-of-two max and one ulp below it, max|dY| at 2^-100 / 2^-101 / 2^100 /
    2^101 stay fp32-grade (the scale's exponent is clamped, not reset to 1, so 2^-101 is not flushed to fp16 zeros and 2^101 does not
    saturate); one NaN or +Inf in dY makes every element it reaches non-finite (split_s32 keeps it non-finite)."""
    xs, ws_, fn, ref_fn = EDGE_FNS[which]
    g = torch.Generator().manual_seed(7)
    x = torch.randn(*xs, generator=g).to(DEV)
    fan = int(np.prod(ws_[1:])) if which != "deconv" else ws_[0]
    w = (torch.randn(*ws_, generator=g) * (1.0 / fan) ** 0.5).to(DEV)
    b = (torch.randn(ws_[0] if which != "deconv" else ws_[1], generator=g) * 0.1).to(DEV)
    with torch.no_grad():
        yshape = ref_fn(x.double(), w.double(), b.double()).shape
    gy = _edge_dy(yshape, edge, 3).to(DEV)
    finite = gy[torch.isfinite(gy)]
    S = pow2_scale(float(finite.abs().max()))
    recs, _, (y, gx, gw) = run_recorded(fn, x, w, b, gy)
    taps = int(np.prod(ws_[2:]))
    steps = taps * max(ws_[0], ws_[1], 32) // 16 + 64
    ref, bars = _edge_bars(ref_fn, x, w, b, gy, S, steps)
    if edge == "zero":
        assert bool((gw == 0).all()) and (gx is None or bool((gx == 0).all()))
    for nat, r, bar, lab in zip((gx, gw), ref[1:], bars[1:], ("dX", "dW")):
        if r is None:
            continue
        _rule(nat, r, bar, "%s dY %s %s" % (which, edge, lab))


def test_forward_input_nan():
    """One NaN in the forward input x: the output elements and the dW elements it reaches are non-finite, the rest within the bar."""
    xs, ws_, fn, ref_fn = EDGE_FNS["conv"]
    g = torch.Generator().manual_seed(8)
    x = torch.randn(*xs, generator=g)
    x.view(-1)[x.numel() // 2 + 5] = float("nan")
    x = x.to(DEV)
    w = (torch.randn(*ws_, generator=g) * (1.0 / np.prod(ws_[1:])) ** 0.5).to(DEV)
    b = (torch.randn(ws_[0], generator=g) * 0.1).to(DEV)
    gy = (torch.randn(xs[0], ws_[0], *xs[2:], generator=g) * 1e-3).to(DEV)
    _, _, (y, gx, gw) = run_recorded(fn, x, w, b, gy)
    ref, bars = _edge_bars(ref_fn, x, w, b, gy, pow2_scale(float(gy.abs().max())), 27 * 32 // 16 + 64)
    _rule(y, ref[0], bars[0], "x NaN: output")
    _rule(gw, ref[2], bars[2], "x NaN: dW")


def test_split_conversions_keep_non_finite_values():
    """lt_f32_to_s32_scaled and lt_f32_to_s32 follow split_s32's rule: NaN -> NaN halves, +-Inf -> +-Inf high half and a NaN low
    half, beyond-fp16 finite values saturate at +-65504; padding channels are zero, never NaN."""
    v = torch.tensor([float("nan"), float("inf"), -float("inf"), 7e4, -1e9, 1.5, 0.0, -3.25] * 4, device=DEV).reshape(1, 32)
    out = torch.empty(1, 128, dtype=torch.float16, device=DEV)
    capi.f32_to_s32_scaled(v, out, 1, 32, 64)
    hi, lo = out[0, :32].float().cpu(), out[0, 32:64].float().cpu()
    assert bool((out[0, 64:] == 0).all())
    assert bool(torch.isnan(hi[0::8]).all()) and bool(torch.isnan(lo[0::8]).all())
    assert bool((hi[1::8] == float("inf")).all()) and bool((hi[2::8] == -float("inf")).all()) and bool(torch.isnan(lo[1::8]).all())
    assert bool((hi[3::8] + lo[3::8] == 65504).all()) and bool((hi[4::8] + lo[4::8] == -65504).all())
    assert bool((hi[5::8] == 1.5).all()) and bool((hi[7::8] == -3.25).all())
    out2 = torch.empty(1, 64, dtype=torch.float16, device=DEV)
    capi.f32_to_s32(v.contiguous(), out2, 1, 32)
    assert torch.equal(out2.view(torch.int16)[:, :64][~torch.isnan(out2)], out.view(torch.int16)[:, :64][~torch.isnan(out[:, :64])])
    assert torch.equal(torch.isnan(out2), torch.isnan(out[:, :64]))


@pytest.mark.parametrize("name", ["tc 3^3 s2 odd cout64 S32", "lines W31 H5 D2 cout32 F32", "tc128 3x3 res-before S32"])
def test_split_fp16_epilogues_keep_nan(name):
    """A NaN in a split-fp16 input stays NaN through the conv_tc and conv_lines epilogues' split_s32x2 (split-fp16 output) and
    their float32 stores: every output element the float64 reference makes NaN is NaN, the rest within the forward suite's bar.
    ReLU is off: the kernels' fmaxf(v, 0) maps NaN to 0 where torch keeps it."""
    import test_gpu_conv as G
    c = G.CASES[name]._replace(relu=False, res=RES_NONE, fmt=G.S32)
    b = G.build(c, seed=4)
    rows = b.x.t.reshape(-1, b.x.t.shape[-1])
    r0 = rows.shape[0] // 2
    rows[r0, 3] = float("nan")                     # channel 3 (hi) of one pixel; its lo stays as it was
    b.x_eff = s32_value(b.x.t)
    out = G.new_out(c, b)
    G.run(c, b, out.t)
    torch.cuda.synchronize()
    ref, bar, _ = G.reference(c, b)
    got = s32_value(out.t).reshape(-1)
    written = ~torch.isnan(ref) | torch.isnan(bar)
    assert bool(torch.isnan(ref).any())
    _rule(got[written], ref[written], bar[written], "%s, one NaN input" % name)


# ------------------------------------------------------------------------------------------ dispatch and gain
_PAT = re.compile(r"(conv_wgrad_kernel|wgrad_reduce_kernel|absmax_kernel|f32_to_s32_scaled_kernel)(<[^>]*>)?")


def profiled_wgrad_launches():
    """Every weight-gradient case (but the large-K one) built and launched once under the profiler -> (kernel names in launch
    order, the conv_wgrad_kernel instantiations expected)."""
    from torch.profiler import ProfilerActivity, profile
    expected = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, c in WCASES.items():
            if name == LARGE_K:
                continue
            b = build(c, seed=1)
            for lw in wgrad_launches(c):
                run_wgrad(b, lw)
                expected.append(c.expect[0])
        torch.cuda.synchronize()
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    names = []
    for e in sorted(evs, key=lambda e: e.start_ns()):
        m = _PAT.search(e.name())
        if m:
            names.append(m.group(0))
    return names, expected


def test_dispatch_reaches_every_wgrad_instantiation():
    """The case table launches conv_wgrad_kernel<1>, <2> and <4> in the order its cases name them, each followed by
    wgrad_reduce_kernel, and the conversion kernels absmax_kernel and f32_to_s32_scaled_kernel.  Profiled in a child process (a
    second profiler session in one process misses its first kernel records)."""
    code = ("import json, sys; sys.path[:0] = %r; import test_gpu_conv_bwd as t; print('LAUNCHES ' + json.dumps(t.profiled_wgrad_launches()))"
            % [HERE, ROOT])
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    names, expected = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")][-1][len("LAUNCHES "):])
    wg = [n for n in names if n.startswith("conv_wgrad_kernel")]
    assert wg == expected, [(i, a, b) for i, (a, b) in enumerate(zip(wg, expected)) if a != b][:5] or (len(wg), len(expected))
    after = [names[i + 1] if i + 1 < len(names) else None for i, n in enumerate(names) if n.startswith("conv_wgrad_kernel")]
    assert all(a == "wgrad_reduce_kernel" for a in after)
    want = {W1, W2, W4, "wgrad_reduce_kernel", "absmax_kernel", "f32_to_s32_scaled_kernel"}
    print("instantiations launched: %s" % sorted(set(names)))
    assert want <= set(names), want - set(names)


def test_wgrad_accumulation_gain():
    """g = sum (n - r) r / sum r^2 over dW of the large-K layer (4096 M tiles): the systematic relative gain of the native weight
    gradient against float64 from its exact operands.  The 8 truncating k16 steps per fresh tile accumulator predict about
    -0.28 x 8 x 2^-24 = -1.3e-7; the tile sums and the reduce round to nearest.  Not compensated: |g| must stay within the
    systematic share of the bar, the 8 truncating steps at 2^-24 each (4.8e-7)."""
    c = WCASES[LARGE_K]
    num = den = 0.0
    for seed in (21, 22):
        b = build(c, seed=seed)
        lw = wgrad_launches(c)[0]
        gw, _ = run_wgrad(b, lw)
        torch.cuda.synchronize()
        ref = wgrad_reference(s32_value(b.x.t), s32_value(b.g.t), lw.desc, b.S, lw.cin, lw.cout)
        n = gw.t.double()
        num += float(((n - ref) * ref).sum())
        den += float((ref * ref).sum())
        del b
    g = num / den
    plan = capi.conv_wgrad_plan(wgrad_launches(c)[0].desc, _sms())
    print("dW gain of %s (%d M tiles, %d splits, bar steps %d): g %+.2e (model -0.28 x 8 x 2^-24 = %+.2e)"
          % (LARGE_K, plan["m_tiles"], plan["splits"], wgrad_steps(plan), g, -0.28 * 8 * EPS))
    assert abs(g) <= 8 * EPS, g
