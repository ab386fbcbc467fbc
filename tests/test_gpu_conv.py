"""Every forward convolution kernel against a float64 reference built from the exact operands it received: each branch of
lt_conv_nd_fwd (conv_tc_kernel<128 / 64 / 32 / 16> with and without split-K, conv_lines_kernel<16 / 32>, conv_fold_kernel<7, 16 / 32>,
the six conv_simt_kernel variants) and the plain V2V tail (v2v_tail_kernel<0>), with guarded buffers, bitwise repeats and the
accumulation gain folded into the tensor-core scales.

Reference (tests/test_conv_cpu.py): float64 on the device from the dequantized split-fp16 input, the dequantized packed filter and the
folded scale divided by the gain it carries.  The bar is per element:
    |native - ref| <= 2 (eps_prod + steps 2^-24) |scale| sum|x||w| + eps_out |ref| + 2^-23 (|shift| + |residual| + |ref|)
c = 2 because a truncating addition loses up to 2^-23 of the running sum where round-to-nearest loses 2^-24; sum|x||w| bounds every
partial sum.  eps_prod: 2^-22 for three-term products (the dropped lo x lo), 2^-11 for LT_CONV_TC1 (hi x hi only), 0 for FFMA.  steps:
the k16 steps into the launched kernel's main accumulator (test_conv_cpu.accum_steps_launched; taps x Cin FFMAs for simt) plus its
fp32 additions (split-K reduce, the kw sum of conv_lines, the epilogue).  eps_out: 2^-22 |ref| + 2^-25 for split-fp16 output (the
low half's subnormal floor).  A second check uses
the original float32 operands with the 2^-21 split representation term added, under the yardstick rule: native error <= max(bar,
2 x the error of float32 torch, TF32 off).

Inputs and residuals sit between NaN guard bands with their padding channels zero (the contract); outputs start as a NaN sentinel
between guard bands.  Every case asserts that the guards are intact, no sentinel survives and channels [Cout, FC) are zero, that a
second run is bit-identical, that an in-place residual gives the out-of-place bits, and that a CUDA-graph replay gives them too.

Measured on an H100 80GB HBM3 (700 W power limit), largest err/bar per family: conv_tc_kernel 0.16 (LT_CONV_TC1 0.28), split-K 0.12,
conv_lines_kernel 0.045, conv_fold_kernel<7, .> 0.025, conv_simt_kernel 0.03, v2v_tail_kernel<0> 0.011.  Accumulation gain g (as folded;
at accum_steps = 0): 7^3 +1.1e-6; -1.03e-5.  3^3 lines 64^3 -1.7e-8; -3.2e-7.  conv_tc 3x3 256 +8.0e-8; -2.3e-6.  1x1 2048 +8.1e-9;
-2.1e-6.  V2V 4^3 split-K -6.8e-9; -1.6e-7 (+3.45e-6 as folded before the reduce pass rescaled to one split's steps).  3^3 W 80 on
conv_tc_kernel +2.9e-8; -8.7e-7 (-5.7e-7 before it kept its own scale).  simt -1.4e-9 at both.
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
from torch import nn

from lt_b200 import capi, engine as eng_mod
from test_conv_cpu import (F32, RES_AFTER, RES_BEFORE, RES_NONE, S32, Launch, accum_gain, accum_steps_launched, conv_acc, dequant_fold,
                           dequant_tc, effective_steps, epilogue, output_index, reduce_gain, s32_rows, s32_value, tc_plan)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TC, TC1, SIMT, FOLD = capi.CONV_TC, capi.CONV_TC1, capi.CONV_SIMT, capi.CONV_TC_FOLD
WS_BYTES = 32 << 20


def _ru(v, m):
    return (v + m - 1) // m * m


# ------------------------------------------------------------------------------------------ the case table
# kind: conv | deconv2d (k4 s2 p1 as four phase launches) | deconv3d (k2 s2 as one grouped launch) | stem (7x7 s2 via the 2x2
# space-to-depth input) | tail (v2v_tail_kernel<0>).  I: input (D, H, W) (stem: image H, W with D = 1).  out_c: FC of a float32
# output (engine out_c), default the engine's.  inplace: also run with the residual in the output buffer.  ws: pass the split-K
# workspace (the engine always does).
Case = namedtuple("Case", "expect kind mode N I cin cout k s p fmt res relu out_c ws")


def case(expect, kind="conv", mode="tc", N=1, I=(1, 8, 8), cin=32, cout=32, k=(1, 3, 3), s=(1, 1, 1), p=None, fmt=S32, res=RES_NONE,
         relu=True, out_c=None, ws=True):
    if p is None:
        p = tuple(v // 2 for v in k)
    return Case(tuple(expect if isinstance(expect, (list, tuple)) else [expect]), kind, mode, N, I, cin, cout, k, s, p, fmt, res, relu,
                out_c, ws)


T128, T64, T32, T16, RED = "conv_tc_kernel<128>", "conv_tc_kernel<64>", "conv_tc_kernel<32>", "conv_tc_kernel<16>", "splitk_reduce_kernel"
LN16, LN32, FD16, FD32 = "conv_lines_kernel<16>", "conv_lines_kernel<32>", "conv_fold_kernel<7, 16>", "conv_fold_kernel<7, 32>"
K3, K7 = (3, 3, 3), (7, 7, 7)
CASES = {
    # ---- conv_tc_kernel: N tiles, terms, split-K, epilogues, residual modes x formats, boxes
    "tc128 3x3 res-before S32": case(T128, N=2, I=(1, 12, 10), cin=64, cout=128, res=RES_BEFORE, ws=False),
    "tc128 3x3 s2 odd F32": case(T128, N=2, I=(1, 13, 11), cin=32, cout=128, s=(1, 2, 2), fmt=F32, ws=False),
    "tc64 1x1 res-after S32": case(T64, N=3, I=(1, 9, 7), cin=96, cout=64, k=(1, 1, 1), res=RES_AFTER, ws=False),
    "tc64 1x1 res-before F32": case(T64, N=2, I=(1, 11, 13), cin=64, cout=64, k=(1, 1, 1), fmt=F32, res=RES_BEFORE, ws=False),
    "tc32 3^3 cout17 partial boxes S32": case(T32, N=1, I=(3, 5, 6), cin=64, cout=17, k=K3, res=RES_BEFORE, ws=False),
    "tc32 3^3 cout17 res-after F32": case(T32, N=2, I=(3, 5, 7), cin=64, cout=17, k=K3, fmt=F32, res=RES_AFTER, ws=False),
    "tc16 3x3 cout40 FC44 F32": case(T16, N=2, I=(1, 7, 9), cin=32, cout=40, fmt=F32, out_c=44, ws=False),
    "tc16 3x3 cout80 res-before F32": case(T16, N=1, I=(1, 9, 10), cin=64, cout=80, fmt=F32, res=RES_BEFORE, ws=False),
    "tc16 1x1 cout40 res-after F32": case(T16, N=3, I=(1, 5, 5), cin=32, cout=40, k=(1, 1, 1), fmt=F32, res=RES_AFTER, ws=False),
    "tc1 3x3 res-before S32": case(T64, mode="tc1", N=2, I=(1, 10, 9), cin=64, cout=64, res=RES_BEFORE, ws=False),
    "tc1 1x1 cout80 F32": case(T16, mode="tc1", N=2, I=(1, 6, 7), cin=32, cout=80, k=(1, 1, 1), fmt=F32, ws=False),
    "tc 3^3 s2 odd cout64 S32": case(T64, N=1, I=(5, 7, 9), cin=32, cout=64, k=K3, s=(2, 2, 2), ws=False),
    "tc tiny batch-spanning box S32": case(T32, N=8, I=(2, 2, 2), cin=64, cout=32, k=K3, res=RES_BEFORE, ws=False),
    "tc 1x1 partial batch box F32": case(T64, N=5, I=(1, 3, 3), cin=64, cout=64, k=(1, 1, 1), fmt=F32, res=RES_AFTER, ws=False),
    "tc 3^3 W80 fold-packed -> conv_tc": case(T32, N=1, I=(3, 5, 80), cin=32, cout=32, k=K3, res=RES_BEFORE, ws=False),
    "tc 3^3 W12 fold-packed -> conv_tc": case(T32, N=2, I=(4, 6, 12), cin=32, cout=16, k=K3, res=RES_AFTER, ws=False),
    "tc V2V output 1x1 cout17 FC20 F32": case(T32, N=1, I=(6, 6, 6), cin=32, cout=17, k=(1, 1, 1), fmt=F32, out_c=20, relu=False),
    # split-K
    "splitk V2V 4^3 res-before S32": case([T128, RED], N=8, I=(4, 4, 4), cin=128, cout=128, k=K3, res=RES_BEFORE),
    "splitk V2V 2^3 res-after S32": case([T128, RED], N=8, I=(2, 2, 2), cin=128, cout=128, k=K3, res=RES_AFTER),
    "splitk 3x3 cout64 res-after F32": case([T64, RED], N=2, I=(1, 6, 6), cin=256, cout=64, fmt=F32, res=RES_AFTER),
    "splitk 3x3 cout48 F32": case([T16, RED], N=1, I=(1, 5, 7), cin=256, cout=48, fmt=F32, res=RES_BEFORE),
    "single-pass 3x3 cout64 (no workspace) F32": case(T64, N=2, I=(1, 6, 6), cin=256, cout=64, fmt=F32, res=RES_AFTER, ws=False),
    # transposed convs and the stem
    "deconv2d k4s2 odd cout32": case([T32] * 4, kind="deconv2d", N=2, I=(1, 5, 7), cin=64, cout=32),
    "deconv2d k4s2 odd cout64": case([T64] * 4, kind="deconv2d", N=1, I=(1, 3, 5), cin=32, cout=64),
    "deconv3d k2s2 cout32": case(T128, kind="deconv3d", N=2, I=(3, 2, 5), cin=64, cout=32, res=RES_AFTER),
    "deconv3d k2s2 cout64": case(T128, kind="deconv3d", N=1, I=(2, 3, 2), cin=128, cout=64, res=RES_AFTER),
    "deconv3d k2s2 cout128": case(T128, kind="deconv3d", N=2, I=(1, 2, 3), cin=64, cout=128, res=RES_AFTER),
    "stem s2d 7x7 s2 (split-K)": case([T64, RED], kind="stem", N=2, I=(1, 14, 18), cin=3, cout=64),
    # ---- conv_lines_kernel: W, partial / short h blocks, D, planes vs 132 SMs, Cout, formats
    "lines W16 H5 D2 cout8": case(LN16, N=1, I=(2, 5, 16), cout=8, k=K3, res=RES_BEFORE),
    "lines W17 H7 D1 cout16": case(LN16, N=2, I=(1, 7, 17), cout=16, k=K3),
    "lines W21 H9 D2 cout20 F32": case(LN32, N=1, I=(2, 9, 21), cout=20, k=K3, fmt=F32, res=RES_AFTER),
    "lines W22 H4 D1 cout32": case(LN32, N=3, I=(1, 4, 22), cout=32, k=K3, res=RES_BEFORE),
    "lines W31 H5 D2 cout32 F32": case(LN32, N=2, I=(2, 5, 31), cout=32, k=K3, fmt=F32),
    "lines W32 H6 D2 cout16": case(LN16, N=1, I=(2, 6, 32), cout=16, k=K3, res=RES_AFTER),
    "lines W33 H3 D1 cout32": case(LN32, N=1, I=(1, 3, 33), cout=32, k=K3),
    "lines W48 H5 D3 cout20": case(LN32, N=1, I=(3, 5, 48), cout=20, k=K3, res=RES_BEFORE),
    "lines W63 H3 D2 cout8": case(LN16, N=2, I=(2, 3, 63), cout=8, k=K3, res=RES_AFTER),
    "lines W64 H3 D1 cout32 F32": case(LN32, N=1, I=(1, 3, 64), cout=32, k=K3, fmt=F32, res=RES_BEFORE),
    "lines 132 planes (= SMs)": case(LN32, N=2, I=(66, 2, 64), cout=32, k=K3, res=RES_BEFORE),
    "lines 133 planes (SMs + 1)": case(LN16, N=1, I=(133, 2, 64), cout=16, k=K3),
    "lines 264 planes (2 x SMs)": case(LN32, N=2, I=(66, 8, 32), cout=32, k=K3, fmt=F32, res=RES_AFTER),
    "lines 265 planes (2 x SMs + 1)": case(LN32, N=1, I=(53, 20, 32), cout=20, k=K3, res=RES_BEFORE),
    # ---- conv_fold_kernel<7, NC>
    "fold7 W16 H9 D3 cout16": case(FD16, N=1, I=(3, 9, 16), cout=16, k=K7, res=RES_BEFORE),
    "fold7 W17 H13 D5 cout32 F32": case(FD32, N=2, I=(5, 13, 17), cout=32, k=K7, fmt=F32),
    "fold7 W27 H18 D3 cout20": case(FD32, N=1, I=(3, 18, 27), cout=20, k=K7, res=RES_AFTER),
    "fold7 W64 H7 D1 cout16 F32": case(FD16, N=1, I=(1, 7, 64), cout=16, k=K7, fmt=F32, out_c=32, res=RES_AFTER),
    "fold7 W71 H5 D3 cout32": case(FD32, N=1, I=(3, 5, 71), cout=32, k=K7, res=RES_BEFORE),
    # ---- conv_simt_kernel: three tiles x vectorised / scalar A
    "simt 256x16 scalar (stem-like)": case("conv_simt_kernel<256, 16, 4, 4, false>", mode="simt", N=2, I=(1, 9, 11), cin=3, cout=4,
                                           k=(1, 7, 7), s=(1, 2, 2), fmt=F32),
    "simt 256x16 vec": case("conv_simt_kernel<256, 16, 4, 4, true>", mode="simt", N=1, I=(3, 5, 6), cin=32, cout=16, k=K3, fmt=F32,
                            res=RES_BEFORE),
    "simt 128x32 scalar": case("conv_simt_kernel<128, 32, 4, 4, false>", mode="simt", N=2, I=(1, 7, 5), cin=5, cout=24, fmt=F32,
                               res=RES_AFTER),
    "simt 128x32 vec": case("conv_simt_kernel<128, 32, 4, 4, true>", mode="simt", N=1, I=(2, 9, 7), cin=16, cout=32, k=K3, fmt=F32),
    "simt 128x64 scalar": case("conv_simt_kernel<128, 64, 8, 4, false>", mode="simt", N=1, I=(1, 8, 9), cin=7, cout=40, fmt=F32),
    "simt 128x64 vec s2": case("conv_simt_kernel<128, 64, 8, 4, true>", mode="simt", N=2, I=(1, 11, 9), cin=48, cout=64, s=(1, 2, 2),
                               fmt=F32, res=RES_BEFORE),
    # ---- the plain V2V tail at row counts that are not multiples of 128
    "tail rows 200": case("v2v_tail_kernel<0>", kind="tail", N=1, I=(2, 10, 10), cout=17, fmt=F32, out_c=20),
    "tail rows 1331": case("v2v_tail_kernel<0>", kind="tail", N=1, I=(11, 11, 11), cout=17, fmt=F32, out_c=20),
}
CONV_KERNELS = [T128, T64, T32, T16, RED, LN16, LN32, FD16, FD32] + [
    "conv_simt_kernel<%s, %s>" % (t, v) for t in ("256, 16, 4, 4", "128, 32, 4, 4", "128, 64, 8, 4") for v in ("true", "false")] + [
    "v2v_tail_kernel<0>"]
AUX_KERNELS = ["absmax_kernel", "gather_weights_kernel", "pack_weights_kernel", "fold_pack_weights_kernel", "fold_bn_kernel",
               "stem_s2d_kernel", "f32_to_s32_kernel"]

# one launch of a case: impl, the Launch geometry (CW = channels it computes), Cin and desc->Cout as passed, the steps its scale folds
Part = namedtuple("Part", "impl L cin desc_cout folded_steps phase ws")


def case_launches(c):
    """The lt_conv_nd_fwd launches of a case, host-only: as the engine would issue them (engine.launch_conv, deconv2d_k4s2, deconv3d_k2s2)."""
    tc = c.mode != "simt"
    impl0 = {"tc": TC, "tc1": TC1, "simt": SIMT}[c.mode]
    ws = WS_BYTES if c.ws else 0
    if c.kind == "tail":
        return [Part(None, None, 32, 32, None, None, 0)]
    if c.kind == "deconv2d":
        cin_p, cout_p = _ru(c.cin, 32), _ru(c.cout, 32)
        F_ = (1, 2 * c.I[1], 2 * c.I[2])
        return [Part(TC, Launch(c.N, c.I, c.I, (1, 2, 2), (1, 1, 1), (0, 1 - py, 1 - px), F_, (1, 2, 2), (0, py, px), (1, 1, 1), cout_p,
                                cout_p), cin_p, cout_p, 4 * cin_p // 16, (py, px), ws) for py in (0, 1) for px in (0, 1)]
    if c.kind == "deconv3d":
        cin_p = _ru(c.cin, 32)
        F_ = tuple(2 * v for v in c.I)
        return [Part(TC, Launch(c.N, c.I, c.I, (1, 1, 1), (1, 1, 1), (0, 0, 0), F_, (2, 2, 2), (0, 0, 0), (2, 2, 2), 8 * c.cout, c.cout),
                     cin_p, 8 * c.cout, cin_p // 16, None, ws)]
    if c.kind == "stem":
        I = (1, c.I[1] // 2, c.I[2] // 2)
        cout_p = _ru(c.cout, 32)
        return [Part(TC, Launch(c.N, I, I, (1, 4, 4), (1, 1, 1), (0, 2, 2), I, (1, 1, 1), (0, 0, 0), (1, 1, 1), cout_p, cout_p), 32,
                     cout_p, 16 * 32 // 16, None, ws)]
    taps = c.k[0] * c.k[1] * c.k[2]
    cin_p = _ru(c.cin, 32) if tc else c.cin
    cout_p = (_ru(c.cout, 32 if c.fmt == S32 else 16)) if tc else _ru(c.cout, 4)
    O = tuple((c.I[a] + 2 * c.p[a] - c.k[a]) // c.s[a] + 1 for a in range(3))
    FC = c.out_c if c.out_c else (_ru(c.cout, 32) if c.fmt == S32 and tc else cout_p)
    fold_packed = (c.mode == "tc" and cin_p == 32 and c.cout <= 32 and c.k[0] == c.k[1] == c.k[2] and c.k[0] in (3, 7)
                   and c.p == (c.k[0] // 2,) * 3 and c.s == (1, 1, 1))
    steps = taps * cin_p // 16 if tc else 0          # pk.scale; pk.scale_fold: 9 Cin / 16 for 3^3
    if fold_packed and eng_mod.fold_width_ok(c.k[2], c.I[2]) and FC == 32 and O == c.I:
        steps = (9 if c.k[0] == 3 else taps) * cin_p // 16
        return [Part(FOLD, Launch(c.N, c.I, O, c.k, c.s, c.p, O, (1, 1, 1), (0, 0, 0), (1, 1, 1), 32, FC), 32, c.cout, steps, None, ws)]
    return [Part(impl0, Launch(c.N, c.I, O, c.k, c.s, c.p, O, (1, 1, 1), (0, 0, 0), (1, 1, 1), cout_p, FC), cin_p, cout_p, steps, None, ws)]


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


def _bn(c, seed):
    g = torch.Generator().manual_seed(seed)
    bn = nn.BatchNorm3d(c)
    bn.weight.data = torch.rand(c, generator=g) + 0.5
    bn.bias.data = torch.randn(c, generator=g) * 0.3
    bn.running_mean = torch.randn(c, generator=g) * 0.2
    bn.running_var = torch.rand(c, generator=g) + 0.5
    return bn.eval().to(DEV)


def _split_rows(x32):
    """float32 [..., C] on the device -> split-fp16 rows through lt_f32_to_s32, checked bitwise against numpy split_s32."""
    s = torch.empty(*x32.shape[:-1], 2 * x32.shape[-1], dtype=torch.float16, device=DEV)
    capi.f32_to_s32(x32.contiguous(), s, x32[..., 0].numel(), x32.shape[-1])
    want = torch.from_numpy(s32_rows(x32.cpu().numpy()))
    assert torch.equal(s.cpu().view(torch.int16), want.view(torch.int16))
    return s


class Built:
    """Packed filters, guarded input / residual, the exact operands and the original float32 operands of one case."""


def build(c, seed=0):
    torch.manual_seed(seed)
    b = Built()
    b.parts = case_launches(c)
    tc = c.mode != "simt"
    b.in_fmt = S32 if tc else F32
    if c.kind == "tail":
        return _build_tail(c, b)
    # ---- modules and packs (engine packing: absmax, gather, pack, fold pack, fold_bn)
    if c.kind == "conv":
        mod = nn.Conv3d(c.cin, c.cout, c.k, c.s, c.p, bias=True).to(DEV)
        b.mod, b.bn = mod, _bn(c.cout, seed + 1)
        pk = eng_mod.pack_conv(mod, b.bn, mode=c.mode, out_fmt=c.fmt)
        b.packs = [pk]
        b.w_orig = mod.weight.detach().double().permute(2, 3, 4, 1, 0).reshape(-1, c.cin, c.cout)
    elif c.kind == "deconv2d":
        mod = nn.ConvTranspose2d(c.cin, c.cout, 4, 2, 1).to(DEV)
        bn = _bn(c.cout, seed + 1)
        ph = eng_mod.pack_deconv2d_k4s2(mod, bn, mode=c.mode)
        b.packs = [ph[p.phase] for p in b.parts]
        b.w_orig = None
    elif c.kind == "deconv3d":
        mod = nn.ConvTranspose3d(c.cin, c.cout, 2, 2).to(DEV)
        pk = eng_mod.pack_deconv3d_k2s2(mod, _bn(c.cout, seed + 1), mode=c.mode)
        assert isinstance(pk, eng_mod.ConvPack)
        b.packs = [pk]
        b.w_orig = None
    else:   # stem
        mod = nn.Conv2d(3, c.cout, 7, 2, 3).to(DEV)
        b.packs = [eng_mod.pack_stem_s2d(mod, _bn(c.cout, seed + 1), mode=c.mode)]
        b.w_orig = None
    b.scales, b.shifts = [], []
    for part, pk in zip(b.parts, b.packs):
        sc, sh = (pk.scale_fold, pk.shift) if part.impl == FOLD else (pk.scale, pk.shift)
        if part.impl == FOLD:
            assert pk.w_fold is not None and (pk.scale_fold is pk.scale) == (pk.k[0] == 7)
            sc, sh = F.pad(sc, (0, 32 - sc.numel())), F.pad(sh, (0, 32 - sh.numel()))   # the fold kernels read all 32 channels they write
        b.scales.append(sc)
        b.shifts.append(sh)
    # ---- input
    L0 = b.parts[0].L
    if c.kind == "stem":
        img = torch.randn(c.N, 3, c.I[1], c.I[2], device=DEV)
        b.x = _guarded((c.N, *L0.I, 64), torch.float16)
        capi.stem_s2d(img, b.x.t, c.N, 3, c.I[1], c.I[2])
        b.x_orig = None
    else:
        cin_p = b.parts[0].cin
        x32 = torch.zeros(c.N, *L0.I, cin_p, device=DEV)
        x32[..., :c.cin] = torch.randn(c.N, *L0.I, c.cin, device=DEV)
        b.x = _guarded((c.N, *L0.I, 2 * cin_p), torch.float16, fill=_split_rows(x32)) if tc else _guarded(x32.shape, torch.float32, x32)
        b.x_orig = x32.double()
    b.x_eff = s32_value(b.x.t) if tc else b.x.t.double()
    # ---- residual and output
    b.out_shape = (c.N, *L0.F, L0.FC)
    b.res, b.res_eff = None, None
    if c.res != RES_NONE:
        r32 = torch.zeros(b.out_shape, device=DEV)
        r32[..., :c.cout] = 0.7 * torch.randn(*b.out_shape[:-1], c.cout, device=DEV)
        b.res = _guarded((*b.out_shape[:-1], 2 * L0.FC), torch.float16, _split_rows(r32)) if c.fmt == S32 else _guarded(b.out_shape, torch.float32, r32)
        b.res_eff = s32_value(b.res.t) if c.fmt == S32 else b.res.t.double()
    b.ws = torch.full((WS_BYTES // 4,), float("nan"), device=DEV) if c.ws else None
    # ---- exact weights, scales
    b.weights, b.w_eff, b.s_eff, b.sh_eff = [], [], [], []
    for part, pk in zip(b.parts, b.packs):
        L = part.L
        taps = L.k[0] * L.k[1] * L.k[2]
        if part.impl == FOLD:
            nc = _ru(part.desc_cout, 16)
            w = dequant_fold(pk.w_fold, L.k[0], nc)
            b.weights.append(pk.w_fold)
        elif part.impl == SIMT:
            w = pk.w.double()
            b.weights.append(pk.w)
        else:
            w = dequant_tc(pk.w, taps, pk.cin, pk.cout_p)
            b.weights.append(pk.w)
        cw = L.CW
        w = F.pad(w, (0, cw - w.shape[2]))
        sc0, sh0 = b.scales[len(b.w_eff)], b.shifts[len(b.w_eff)]
        sc = F.pad(sc0.double(), (0, cw - sc0.numel())) / accum_gain(part.folded_steps)
        sh = F.pad(sh0.double(), (0, cw - sh0.numel()))
        b.w_eff.append(w)
        b.s_eff.append(sc)
        b.sh_eff.append(sh)
    return b


def _build_tail(c, b):
    J, FC = c.cout, c.out_c
    c1, c2, c3 = nn.Conv3d(32, 32, 1).to(DEV), nn.Conv3d(32, 32, 1).to(DEV), nn.Conv3d(32, J, 1).to(DEV)
    with torch.no_grad():
        c3.weight.mul_(6.0)
    b.packs = [eng_mod.pack_conv(c1, _bn(32, 5), mode="tc"), eng_mod.pack_conv(c2, _bn(32, 6), mode="tc"),
               eng_mod.pack_conv(c3, None, mode="tc", out_fmt=F32)]
    assert b.packs[2].cout_p == _ru(FC, 16)
    rows = c.N * int(np.prod(c.I))
    x32 = torch.randn(rows, 32, device=DEV)
    b.x = _guarded((rows, 64), torch.float16, fill=_split_rows(x32))
    b.x_eff = s32_value(b.x.t)
    b.rows, b.out_shape, b.res, b.ws = rows, (rows, FC), None, None
    b.w_eff = [dequant_tc(pk.w, 1, 32, pk.cout_p)[0] for pk in b.packs]
    b.s_eff = [pk.scale.double() / accum_gain(2) for pk in b.packs]
    b.sh_eff = [pk.shift.double() for pk in b.packs]
    return b


def _desc(c, part, in_fmt, ws):
    L = part.L
    d = capi.ConvDesc(N=L.N, ID=L.I[0], IH=L.I[1], IW=L.I[2], Cin=part.cin, OD=L.O[0], OH=L.O[1], OW=L.O[2], Cout=part.desc_cout,
                      KD=L.k[0], KH=L.k[1], KW=L.k[2], sd=L.s[0], sh=L.s[1], sw=L.s[2], pd=L.p[0], ph=L.p[1], pw=L.p[2],
                      FD=L.F[0], FH=L.F[1], FW=L.F[2], FC=L.FC, osd=L.os[0], osh=L.os[1], osw=L.os[2], ood=L.oo[0], ooh=L.oo[1],
                      oow=L.oo[2], relu=int(c.relu), residual=c.res, in_format=in_fmt, out_format=c.fmt, ogd=L.og[0], ogh=L.og[1],
                      ogw=L.og[2])
    if ws is not None:
        d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel() * 4
    return d


def run(c, b, out, res=None):
    """Every launch of the case into `out` (a tensor); res: the residual tensor (default the built one)."""
    if c.kind == "tail":
        p1, p2, p3 = b.packs
        capi.v2v_tail(b.x.t, p1.w, p2.w, p3.w, p1.scale, p1.shift, p2.scale, p2.shift, p3.scale, p3.shift, out, b.rows, c.out_c)
        return
    if res is None and b.res is not None:
        res = b.res.t
    for part, w, sc, sh in zip(b.parts, b.weights, b.scales, b.shifts):
        capi.conv_nd(_desc(c, part, b.in_fmt, b.ws), b.x.t, w, sc, sh, res, out, part.impl)


def new_out(c, b):
    L0 = b.out_shape
    return _guarded((*L0[:-1], 2 * L0[-1]), torch.float16) if c.fmt == S32 else _guarded(L0, torch.float32)


def out_value(c, t):
    return s32_value(t) if c.fmt == S32 else t.double()


def eps_prod(mode):
    return {"tc": 2.0 ** -22, "tc1": 2.0 ** -11, "simt": 0.0}[mode]


def bound_steps(c, part):
    """Steps of the per-element bar: the main accumulator's k16 steps (FFMA chain for simt) plus the kernel's fp32 additions."""
    L = part.L
    if part.impl == SIMT:
        return L.k[0] * L.k[1] * L.k[2] * part.cin + 3
    steps = int(np.ceil(accum_steps_launched(part.impl, L, part.cin, part.desc_cout, part.ws))) + 4
    if part.impl == FOLD and L.k[0] == 3:
        steps += 2
    if part.impl in (TC, TC1):
        steps += tc_plan(L, part.cin, part.desc_cout, part.ws)["splits"]
    return steps


def reference(c, b, x_eff=None, w_effs=None):
    """(ref, bar, sig) float64 over the flat output; NaN where no launch writes.  sig = |scale| sum|x||w| per element."""
    n = int(np.prod(b.out_shape))
    ref = torch.full((n,), float("nan"), dtype=torch.float64, device=DEV)
    bar, sig = torch.zeros_like(ref), torch.zeros_like(ref)
    x = b.x_eff if x_eff is None else x_eff
    for i, part in enumerate(b.parts):
        L, w, sc, sh = part.L, (b.w_eff if w_effs is None else w_effs)[i], b.s_eff[i], b.sh_eff[i]
        acc = conv_acc(x, w, L).reshape(-1)
        sg = conv_acc(x.abs(), w.abs(), L).reshape(-1)
        oi, si = output_index(L, DEV)
        ch = si % L.CW
        r = b.res_eff.reshape(-1)[oi] if c.res != RES_NONE else torch.zeros(len(oi), dtype=torch.float64, device=DEV)
        v = epilogue(acc[si], sc[ch], sh[ch], r, c.relu, c.res)
        s = sc[ch].abs() * sg[si]
        assert bool(torch.isnan(ref[oi]).all()), "launches of a case overlap"
        ref[oi] = v
        sig[oi] = s
        bar[oi] = (2.0 * (eps_prod(c.mode) + bound_steps(c, part) * 2.0 ** -24) * s + (2.0 ** -22 * v.abs() + 2.0 ** -25 if c.fmt == S32 else 0.0)
                   + 2.0 ** -23 * (sh[ch].abs() + r.abs() + v.abs()))
    return ref, bar, sig


def tail_reference(c, b):
    """The three chained 1x1 GEMMs in float64 with the error bars propagated through the split-fp16 hidden layers."""
    x = b.x_eff
    e = torch.zeros_like(x)
    steps = 6 + 4
    for i in range(3):
        w, sc, sh = b.w_eff[i], b.s_eff[i], b.sh_eff[i]
        a = x @ w
        sg = x.abs() @ w.abs() * sc.abs()
        v = a * sc + sh
        own = 2.0 * (2.0 ** -22 + steps * 2.0 ** -24) * sg + 2.0 ** -23 * (sh.abs() + v.abs())
        prop = (e @ w.abs()) * sc.abs()
        if i < 2:
            v = torch.clamp(v, min=0.0)
            own = own + 2.0 ** -22 * v.abs() + 2.0 ** -25    # the hidden activation is stored split-fp16
        x, e = v, own + prop
    FC = c.out_c
    return x[:, :FC].reshape(-1), e[:, :FC].reshape(-1), None


def check_buffers(c, b, out):
    assert out.guards_intact(), "a write landed outside the output"
    assert out.unwritten() == 0, "%d output elements were never written" % out.unwritten()
    assert b.x.guards_intact() and (b.res is None or b.res.guards_intact())
    v = out_value(c, out.t).reshape(*b.out_shape)
    assert bool((v[..., c.cout:] == 0).all()), "padding channels [Cout, FC) are not zero"
    return v.reshape(-1)


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == torch.float16 else torch.int32).clone()


RATIOS = {}


@pytest.mark.parametrize("name", list(CASES))
def test_conv_kernels_vs_float64(name):
    c = CASES[name]
    b = build(c, seed=sum(map(ord, name)) % 1000)
    out = new_out(c, b)
    run(c, b, out.t)
    torch.cuda.synchronize()
    got = check_buffers(c, b, out)
    ref, bar, _ = tail_reference(c, b) if c.kind == "tail" else reference(c, b)
    assert not bool(torch.isnan(ref).any())
    err = (got - ref).abs()
    ratio = float((err / bar.clamp(min=1e-300)).max())
    fam = c.expect[0]
    RATIOS[fam] = max(RATIOS.get(fam, 0.0), ratio)
    print("%-44s largest err/bar %.3f  (max err %.2e, max |ref| %.2e)" % (name, ratio, float(err.max()), float(ref.abs().max())))
    assert ratio <= 1.0, (name, ratio)
    # ---- against the original float32 operands (plain convs): the yardstick rule with the split representation term
    if c.kind == "conv" and b.x_orig is not None:
        L = b.parts[0].L
        w32 = b.w_orig.float().double()
        S = 2.0 ** round(float(np.log2(float(b.w_eff[0].abs().max()) / float(w32.abs().max())))) if c.mode != "simt" else 1.0
        w_o = F.pad(w32, (0, 0, 0, b.parts[0].cin - c.cin)) * S
        w_o = F.pad(w_o, (0, L.CW - c.cout))
        ref_o, bar_o, sig_o = reference(c, b, x_eff=b.x_orig, w_effs=[w_o])
        acc32 = conv_acc(b.x_orig.float(), w_o.float(), L).reshape(-1)
        oi, si = output_index(L, DEV)
        ch = si % L.CW
        r32 = None if c.res == RES_NONE else b.res_eff.float().reshape(-1)[oi]
        t32 = torch.full_like(ref_o, float("nan"))
        t32[oi] = epilogue(acc32[si], b.s_eff[0].float()[ch], b.sh_eff[0].float()[ch], r32, c.relu, c.res).double()
        e_o = (got - ref_o).abs()
        lim = torch.maximum(bar_o + 2.0 ** -21 * sig_o, 2.0 * (t32 - ref_o).abs())
        print("%-44s vs float32 operands: max err %.2e, float32 torch %.2e, largest err/limit %.3f"
              % ("", float(e_o.max()), float((t32 - ref_o).abs().max()), float((e_o / lim.clamp(min=1e-300)).max())))
        assert bool((e_o <= lim).all())
    # ---- repeatability: a second run, the in-place residual, a CUDA-graph replay
    out2 = new_out(c, b)
    run(c, b, out2.t)
    torch.cuda.synchronize()
    assert torch.equal(bits(out2.t), bits(out.t)), "a second run differs"
    if c.res != RES_NONE:
        io = new_out(c, b)
        io.t.copy_(b.res.t)
        run(c, b, io.t, res=io.t)
        torch.cuda.synchronize()
        assert io.guards_intact() and torch.equal(bits(io.t), bits(out.t)), "the in-place residual differs from out-of-place"
    og = new_out(c, b)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run(c, b, og.t)
    g.replay()
    torch.cuda.synchronize()
    assert og.guards_intact() and torch.equal(bits(og.t), bits(out.t)), "the CUDA-graph replay differs"


def test_packed_operands_match_numpy():
    """lt_conv_tc_pack_weights and lt_conv_fold_pack_weights (both 3^3 and 7^3 layouts) against the numpy packers, bit for bit."""
    from test_conv_cpu import pack_fold_np, pack_tc_np
    rng = np.random.RandomState(3)
    w = rng.randn(9, 64, 40).astype(np.float32)
    packed = torch.empty(capi.conv_tc_weight_bytes(9, 64, 40) // 2, dtype=torch.float16, device=DEV)
    capi.conv_tc_pack_weights(torch.from_numpy(w).to(DEV), packed, 9, 64, 40)
    assert torch.equal(packed.cpu().view(torch.int16).reshape(-1), torch.from_numpy(pack_tc_np(w, 48)).view(torch.int16).reshape(-1))
    for k, cout in ((3, 32), (3, 16), (7, 16), (7, 20)):
        w = (rng.randn(k ** 3, 32, cout) * 0.1).astype(np.float32)
        packed = torch.empty(capi.conv_fold_weight_bytes(k, cout) // 2, dtype=torch.float16, device=DEV)
        capi.conv_fold_pack_weights(torch.from_numpy(w).to(DEV), packed, k, cout)
        assert torch.equal(packed.cpu().view(torch.int16).reshape(-1), torch.from_numpy(pack_fold_np(w, k)).view(torch.int16).reshape(-1)), (k, cout)


# ------------------------------------------------------------------------------------------ dispatch reaches every instantiation
_PAT = re.compile(r"(conv_tc_kernel|splitk_reduce_kernel|conv_lines_kernel|conv_fold_kernel|conv_simt_kernel|v2v_tail_kernel|"
                  r"fold_pack_weights_kernel|pack_weights_kernel|gather_weights_kernel|absmax_kernel|fold_bn_kernel|stem_s2d_kernel|"
                  r"f32_to_s32_kernel)(<[^>]*>)?")


def profiled_launches():
    """Every case packed and launched once under the profiler -> (kernel names in launch order, the conv kernels expected)."""
    from torch.profiler import ProfilerActivity, profile
    expected = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for name, c in CASES.items():
            b = build(c, seed=1)
            out = new_out(c, b)
            run(c, b, out.t)
            expected += list(c.expect)
        torch.cuda.synchronize()
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    names = []
    for e in sorted(evs, key=lambda e: e.start_ns()):
        m = _PAT.search(e.name())
        if m:
            names.append(m.group(0))
    return names, expected


def test_dispatch_reaches_every_instantiation():
    """Each case launches the kernels it names, in order; together they cover every conv kernel instantiation of conv_tc.cu,
    conv_fold.cu, conv_simt.cu and the plain tail of conv_tail.cu, and the packing kernels.  Profiled in a child process (a second
    profiler session in one process misses its first kernel records)."""
    code = ("import json, sys; sys.path[:0] = %r; import test_gpu_conv as t; print('LAUNCHES ' + json.dumps(t.profiled_launches()))"
            % [HERE, ROOT])
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    names, expected = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")][-1][len("LAUNCHES "):])
    conv = [n for n in names if n.split("<")[0] in {k.split("<")[0] for k in CONV_KERNELS}]
    assert conv == expected, [(i, a, b) for i, (a, b) in enumerate(zip(conv, expected)) if a != b][:5] or (len(conv), len(expected))
    print("instantiations launched: %s" % sorted(set(names)))
    assert set(CONV_KERNELS) <= set(names) and set(AUX_KERNELS) <= set(names), sorted((set(CONV_KERNELS) | set(AUX_KERNELS)) - set(names))


# ------------------------------------------------------------------------------------------ the accumulation gain
# (name, case, repeats): F32 output, no ReLU, no residual, about 10^6 outputs per layer
GAIN_LAYERS = [
    ("7^3 conv_fold", case(FD16, N=1, I=(40, 40, 40), cout=16, k=K7, fmt=F32, out_c=32, relu=False), 1),
    ("3^3 conv_lines 64^3", case(LN32, N=1, I=(64, 64, 64), cout=32, k=K3, fmt=F32, relu=False), 1),
    ("conv_tc 3x3 256", case(T128, N=4, I=(1, 32, 32), cin=256, cout=256, fmt=F32, relu=False, ws=False), 1),
    ("conv_tc 1x1 2048", case(T128, N=8, I=(1, 16, 16), cin=2048, cout=512, k=(1, 1, 1), fmt=F32, relu=False, ws=False), 1),
    ("V2V 4^3 split-K", case([T128, RED], N=8, I=(4, 4, 4), cin=128, cout=128, k=K3, fmt=F32, relu=False), 16),
    ("3^3 fold-packed W80 -> conv_tc", case(T32, N=1, I=(20, 20, 80), cout=32, k=K3, fmt=F32, relu=False), 1),
    ("simt (control)", case("conv_simt_kernel<128, 32, 4, 4, true>", mode="simt", N=1, I=(32, 32, 32), cout=32, k=K3, fmt=F32,
                            relu=False), 1),
]


def _gain_sums(c, b, scale, s_ref):
    """sum (n - r)(r - shift), sum (r - shift)^2 over the real channels, native run with `scale`, reference with s_ref (float64)."""
    part = b.parts[0]
    out = torch.empty(b.out_shape, device=DEV)
    capi.conv_nd(_desc(c, part, b.in_fmt, b.ws), b.x.t, b.weights[0], scale, b.shifts[0], None, out, part.impl)
    L = part.L
    acc = conv_acc(b.x_eff, b.w_eff[0], L)[..., :c.cout]
    r_sh = acc * s_ref[:c.cout]
    n_sh = out.double()[..., :c.cout] - b.sh_eff[0][:c.cout]
    return float(((n_sh - r_sh) * r_sh).sum()), float((r_sh * r_sh).sum())


@pytest.mark.parametrize("name,c,reps", GAIN_LAYERS, ids=[g[0] for g in GAIN_LAYERS])
def test_accumulation_gain(name, c, reps):
    """g = sum (n - r)(r - shift) / sum (r - shift)^2: the systematic gain of the native layer against float64 from its exact operands,
    with the scale as folded (r from scale / gain) and re-folded at accum_steps = 0 (r from that scale).  As shipped |g| must stay within
    a quarter of the gain the scale applies (or 5e-8)."""
    from test_conv_cpu import launched_kernels
    part = case_launches(c)[0]
    assert launched_kernels(part.impl, part.L, part.cin, part.desc_cout, part.ws) == list(c.expect)
    num_f = den_f = num_0 = den_0 = 0.0
    for rep in range(reps):
        b = build(c, seed=100 + rep)
        mod, bn = b.mod, b.bn
        # the scale re-folded at accum_steps = 0, with the same filter pre-scale
        amax = None
        if c.mode != "simt":
            amax = torch.empty(1, dtype=torch.int32, device=DEV)
            capi.absmax(mod.weight.detach().float().contiguous(), amax)
        sc0, sh0 = torch.zeros_like(b.scales[0]), torch.zeros_like(b.shifts[0])
        capi.fold_bn(bn.weight.detach(), bn.bias.detach(), bn.running_mean, bn.running_var, mod.bias.detach(), bn.eps, c.cout, c.cout,
                     sc0[:c.cout], sh0[:c.cout], amax, accum_steps=0)
        assert torch.equal(sh0, b.shifts[0])
        a, d = _gain_sums(c, b, b.scales[0], b.s_eff[0])
        num_f, den_f = num_f + a, den_f + d
        # at accum_steps = 0 the split-K reduce still applies its factor: the reference carries it, so g is the shrinkage alone
        rg = reduce_gain(part.L, part.cin, part.desc_cout, part.ws) if part.impl in (TC, TC1) else 1.0
        a, d = _gain_sums(c, b, sc0, sc0.double() * rg)
        num_0, den_0 = num_0 + a, den_0 + d
    steps = accum_steps_launched(part.impl, part.L, part.cin, part.desc_cout, part.ws)
    applied = accum_gain(effective_steps(part.impl, part.L, part.cin, part.desc_cout, part.folded_steps, part.ws)) - 1.0
    g_f, g_0 = num_f / den_f, num_0 / den_0
    print("%-32s gain applied %.2e (%d steps folded, %.1f launched): g as folded %+.2e, g at accum_steps 0 %+.2e, rate %.3f"
          % (name, applied, part.folded_steps, steps, g_f, g_0, -g_0 / (steps * 2.0 ** -24) if steps else 0.0))
    assert abs(g_f) <= max(0.25 * applied, 5e-8), (name, g_f, g_0, applied)
