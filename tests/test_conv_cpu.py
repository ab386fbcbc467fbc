"""Float64 semantics of lt_conv_nd_fwd, exact operand helpers and the host-side dispatch of the forward convolutions, without a GPU.

- `conv_reference` is lt_conv_nd_fwd in float64 (include/lt_b200.h): taps, stride and front padding, the output mapping (os* / oo*,
  stride-phase transposed convs), grouped outputs (og*: Cout / G channels per phase, the odd phase that group_extent shortens), the
  channels a launch writes (FC may be wider than the filter's real channel count), the three residual modes, ReLU, and F32 or
  split-fp16 output.  It works on torch tensors of any device: tests/test_gpu_conv.py runs it on the GPU in float64.  Here it is
  checked against torch float64 conv2d / conv3d / conv_transpose2d / conv_transpose3d.
- numpy split-fp16 (`split_np`) and the dequantizers of the three packed weight layouts: conv_tc [tap][Cin/32][CoutP][32 hi | 32 lo],
  3^3 fold [kd][kh][kw][NC][...], 7^3 fold [kw][kd][kh][NC][...].
- Dispatch mirrors: lt_conv_tc_plan at 132 SMs with the engine's split-K workspace, conv_fold_supported / engine.fold_width_ok, the
  conv_simt tile choice.  Every GPU case of tests/test_gpu_conv.py names the kernel it must reach and is checked against these here.
- The accumulation-step model: the tensor-core steps per main accumulator of the kernel that launches, which is what the folded
  scale's gain must assume.
"""
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lt_b200 import capi, engine as eng_mod

SMS = 132
WS_BYTES = 32 << 20            # engine.SPLITK_WS_BYTES: the split-K scratch of every conv launch
RES_NONE, RES_BEFORE, RES_AFTER = capi.RES_NONE, capi.RES_BEFORE_RELU, capi.RES_AFTER_RELU
F32, S32 = capi.FMT_F32, capi.FMT_S32
ACCUM_RATE = 0.28              # lt_fold_bn_fwd: scale x (1 + ACCUM_RATE x steps x 2^-24)


# ------------------------------------------------------------------------------------------ split-fp16 and packed layouts
def split_np(x):
    """float32 -> (hi, lo) float16 as split_s32 (common.cuh): clamp finite values to +-65504, hi = fp16_rn(x), lo = fp16_rn(x - hi).
    NaN stays NaN in both halves, +-Inf gives hi = +-Inf and lo = NaN."""
    x = np.asarray(x, dtype=np.float32)
    x = np.where(np.isfinite(x), np.clip(x, np.float32(-65504.0), np.float32(65504.0)), x)
    with np.errstate(invalid="ignore"):
        hi = x.astype(np.float16)
        lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def join_np(hi, lo):
    return hi.astype(np.float64) + lo.astype(np.float64)


def s32_rows(x):
    """float32 [..., C] (C % 32 == 0) -> the split-fp16 rows [..., C/32, 32 hi | 32 lo] as stored, float16 [..., 2C]."""
    hi, lo = split_np(x)
    sh = x.shape[:-1] + (x.shape[-1] // 32, 32)
    return np.concatenate([hi.reshape(sh), lo.reshape(sh)], -1).reshape(x.shape[:-1] + (2 * x.shape[-1],))


def s32_value(rows):
    """float16 split rows [..., 2C] (torch, any device) -> float64 [..., C] = hi + lo."""
    sh = rows.shape[:-1]
    r = rows.reshape(*sh, rows.shape[-1] // 64, 2, 32).double()
    return (r[..., 0, :] + r[..., 1, :]).reshape(*sh, rows.shape[-1] // 2)


def dequant_tc(packed, taps, cin, coutp, hi_only=False):
    """lt_conv_tc_pack_weights layout [tap][Cin/32][CoutP][32 hi | 32 lo] -> float64 [taps][Cin][CoutP]."""
    r = packed.reshape(taps, cin // 32, coutp, 2, 32).double()
    v = r[..., 0, :] if hi_only else r[..., 0, :] + r[..., 1, :]
    return v.permute(0, 1, 3, 2).reshape(taps, cin, coutp)


def dequant_fold(packed, k, nc):
    """lt_conv_fold_pack_weights -> float64 [k^3 taps (kd, kh, kw)][32][NC]: 3^3 slots in (kd, kh, kw) order, 7^3 in (kw, kd, kh)."""
    r = packed.reshape(k ** 3, nc, 2, 32).double()
    v = (r[:, :, 0, :] + r[:, :, 1, :]).permute(0, 2, 1)        # [slot][ci][co]
    if k == 3:
        return v
    return v.reshape(k, k, k, 32, nc).permute(1, 2, 0, 3, 4).reshape(k ** 3, 32, nc)   # slot (kw, kd, kh) -> tap (kd, kh, kw)


def pack_tc_np(w, coutp):
    """float32 [taps][Cin][Cout] -> the conv_tc packed layout, float16 [taps][Cin/32][CoutP][64] (rows Cout .. CoutP-1 zero)."""
    taps, cin, cout = w.shape
    wp = np.zeros((taps, cin, coutp), np.float32)
    wp[..., :cout] = w
    hi, lo = split_np(wp.reshape(taps, cin // 32, 32, coutp).transpose(0, 1, 3, 2))
    return np.concatenate([hi, lo], -1)


def pack_fold_np(w, k):
    """float32 [k^3 (kd, kh, kw)][32][Cout] -> the fold packed layout, float16 [slots][NC][64]."""
    cout = w.shape[2]
    nc = (cout + 15) // 16 * 16
    wp = np.zeros((k ** 3, 32, nc), np.float32)
    wp[..., :cout] = w
    if k == 7:
        wp = wp.reshape(k, k, k, 32, nc).transpose(2, 0, 1, 3, 4).reshape(k ** 3, 32, nc)
    hi, lo = split_np(wp.transpose(0, 2, 1))
    return np.concatenate([hi, lo], -1)


# ------------------------------------------------------------------------------------------ float64 semantics of lt_conv_nd_fwd
Launch = namedtuple("Launch", "N I O k s p F os oo og CW FC")   # I, O, k, s, p, F, os, oo, og: (d, h, w); CW: channels it computes


def conv_acc(x, w, L):
    """sum_{taps, ci} in[n, o s - p + t, ci] W[t, ci, co] over the launch's O grid: x float64 [N][ID][IH][IW][Cin], w [taps][Cin][CW]
    -> [N][OD][OH][OW][CW].  Zero padding in front (p) and wherever a tap falls past the input."""
    pads = []
    for ax in (2, 1, 0):      # F.pad order: W, H, D
        back = max(0, (L.O[ax] - 1) * L.s[ax] + L.k[ax] - L.p[ax] - L.I[ax])
        pads += [L.p[ax], back]
    xt = F.pad(x.permute(0, 4, 1, 2, 3), pads)
    wt = w.reshape(*L.k, w.shape[1], w.shape[2]).permute(4, 3, 0, 1, 2)
    y = F.conv3d(xt, wt, stride=L.s)[:, :, :L.O[0], :L.O[1], :L.O[2]]
    return y.permute(0, 2, 3, 4, 1)


def group_extent(n, f, off, ph, os):
    """conv_tc.cu group_extent: positions of a launch axis that output phase ph writes inside an extent f."""
    return min(n, (f - off - ph + os - 1) // os)


def output_index(L, device="cpu"):
    """(flat indices into the [N][FD][FH][FW][FC] output, flat indices into the launch's [N][OD][OH][OW][CW] values) of every element
    the launch writes: channel block g of oc = CW / G channels goes to phase (a, b, c) of the output lattice; positions outside the
    tensor (group_extent) and channels >= FC are not written."""
    G = L.og[0] * L.og[1] * L.og[2]
    oc = L.CW // G if G > 1 else L.CW
    outs, srcs = [], []
    for g in range(G):
        ph = (g // (L.og[1] * L.og[2]), (g // L.og[2]) % L.og[1], g % L.og[2]) if G > 1 else (0, 0, 0)
        ext = [group_extent(L.O[a], L.F[a], L.oo[a], ph[a], L.os[a]) for a in range(3)]
        nch = min(oc, L.FC)
        if min(ext) <= 0 or nch <= 0:
            continue
        n, od, oh, ow, c = torch.meshgrid(*[torch.arange(v, device=device) for v in (L.N, *ext, nch)], indexing="ij")
        fd, fh, fw = (od * L.os[0] + L.oo[0] + ph[0], oh * L.os[1] + L.oo[1] + ph[1], ow * L.os[2] + L.oo[2] + ph[2])
        outs.append(((((n * L.F[0] + fd) * L.F[1] + fh) * L.F[2] + fw) * L.FC + c).reshape(-1))
        srcs.append(((((n * L.O[0] + od) * L.O[1] + oh) * L.O[2] + ow) * L.CW + g * oc + c).reshape(-1))
    return torch.cat(outs), torch.cat(srcs)


def epilogue(acc, scale, shift, res, relu, mode):
    """act(acc x scale + shift (+ residual)) in float64: res is the residual at the same elements (or None)."""
    v = acc * scale + shift
    if mode == RES_BEFORE:
        v = v + res
    if relu:
        v = torch.clamp(v, min=0.0)
    if mode == RES_AFTER:
        v = v + res
    return v


def conv_reference(x, w, L, scale, shift, res_full=None, mode=RES_NONE, relu=False, out_fmt=F32):
    """lt_conv_nd_fwd of one launch in float64 -> (out_idx, values): the flat output elements it writes and their values.  x, w, scale,
    shift (length CW) float64; res_full: the float64 residual tensor [N][FD][FH][FW][FC] (its values at the written elements are read);
    split-fp16 output rounds each value through split_s32."""
    acc = conv_acc(x, w, L).reshape(-1)
    oi, si = output_index(L, x.device)
    ch = si % L.CW
    r = None if mode == RES_NONE else res_full.reshape(-1)[oi]
    v = epilogue(acc[si], scale[ch], shift[ch], r, relu, mode)
    if out_fmt == S32:
        hi, lo = split_np(v.cpu().numpy().astype(np.float32))
        v = torch.from_numpy(join_np(hi, lo)).to(x.device)
    return oi, v


# ------------------------------------------------------------------------------------------ dispatch mirrors
def fold_supported(L, cin, cout, in_fmt=S32):
    """conv_fold_supported (csrc/conv_fold.cu) for a launch with desc->Cout = cout (the real count)."""
    k = L.k[0]
    return (L.k[0] == L.k[1] == L.k[2] and k in (3, 7) and cin == 32 and cout <= 32 and L.s == (1, 1, 1) and L.p == (k // 2,) * 3
            and L.O == L.I and L.os == (1, 1, 1) and L.oo == (0, 0, 0) and L.F == L.O and L.FC == 32 and in_fmt == S32
            and L.I[2] >= 16 and (k == 7 or L.I[2] <= 64))


def simt_kernel(cout, cin):
    """conv_simt_fwd's tile for CoutW = round_up(Cout, 4) and its A path (vectorised when Cin % 16 == 0)."""
    cw = (cout + 3) // 4 * 4
    tile = (256, 16, 4, 4) if cw <= 16 else (128, 32, 4, 4) if cw <= 32 else (128, 64, 8, 4)
    return "conv_simt_kernel<%d, %d, %d, %d, %s>" % (tile + ("true" if cin % 16 == 0 else "false",))


def tc_desc(L, cin, cout, ws=WS_BYTES):
    d = capi.ConvDesc(N=L.N, ID=L.I[0], IH=L.I[1], IW=L.I[2], Cin=cin, OD=L.O[0], OH=L.O[1], OW=L.O[2], Cout=cout, KD=L.k[0], KH=L.k[1],
                      KW=L.k[2], sd=L.s[0], sh=L.s[1], sw=L.s[2], pd=L.p[0], ph=L.p[1], pw=L.p[2], FD=L.F[0], FH=L.F[1], FW=L.F[2], FC=L.FC,
                      osd=L.os[0], osh=L.os[1], osw=L.os[2], ood=L.oo[0], ooh=L.oo[1], oow=L.oo[2], ogd=L.og[0], ogh=L.og[1], ogw=L.og[2],
                      in_format=S32, out_format=S32)
    d.workspace, d.workspace_bytes = (4096 if ws else None), ws   # the plan never dereferences the workspace
    return d


def tc_plan(L, cin, cout, ws=WS_BYTES):
    return capi.conv_tc_plan(tc_desc(L, cin, cout, ws), SMS)


def launched_kernels(impl, L, cin, cout, ws=WS_BYTES):
    """The kernels one lt_conv_nd_fwd launch runs: cout is desc->Cout (real for LT_CONV_TC_FOLD, padded otherwise); ws: the split-K
    workspace bytes passed (0: none)."""
    if impl == capi.CONV_SIMT:
        return [simt_kernel(cout, cin)]
    if impl == capi.CONV_TC_FOLD:
        assert fold_supported(L, cin, cout)
        nc = 16 if cout <= 16 else 32
        return ["conv_lines_kernel<%d>" % nc if L.k[0] == 3 else "conv_fold_kernel<7, %d>" % nc]
    p = tc_plan(L, cin, cout, ws)
    return ["conv_tc_kernel<%d>" % p["nt"]] + (["splitk_reduce_kernel"] if p["splits"] > 1 else [])


def accum_steps_launched(impl, L, cin, cout, ws=WS_BYTES):
    """Tensor-core k16 steps into the main (hi x hi) accumulator of one output in the launched kernel: conv_tc 2 per K chunk, over a
    split-K launch the mean over its splits; conv_lines 9 Cin / 16 per kw column; conv_fold K^3 Cin / 16; 0 for the FFMA kernel."""
    if impl == capi.CONV_SIMT:
        return 0
    taps = L.k[0] * L.k[1] * L.k[2]
    if impl == capi.CONV_TC_FOLD:
        return (9 if L.k[0] == 3 else taps) * cin // 16
    p = tc_plan(L, cin, cout, ws)
    return 2 * p["chunks"] / p["splits"]


def effective_steps(impl, L, cin, cout, folded_steps, ws=WS_BYTES):
    """The steps the applied gain compensates: the folded scale's, rescaled by splitk_reduce_kernel to one split's share."""
    if impl in (capi.CONV_TC, capi.CONV_TC1):
        return folded_steps / tc_plan(L, cin, cout, ws)["splits"]
    return folded_steps


def reduce_gain(L, cin, cout, ws=WS_BYTES):
    """splitk_reduce_kernel's factor (TcParams.ws_gain): accum_gain of one split's steps over that of the whole K loop, in float32."""
    p = tc_plan(L, cin, cout, ws)
    return float(np.float32(accum_gain(2.0 * p["chunks"] / p["splits"]) / accum_gain(2.0 * p["chunks"])))


def accum_gain(steps):
    return 1.0 + ACCUM_RATE * steps * 2.0 ** -24


# ------------------------------------------------------------------------------------------ tests: the reference
def _rand(*shape, seed):
    return torch.from_numpy(np.random.RandomState(seed).randn(*shape)).double()


def _plain(N, I, k, s, p, cw, FC, O=None):
    O = O or tuple((I[a] + 2 * p[a] - k[a]) // s[a] + 1 for a in range(3))
    return Launch(N, I, O, k, s, p, O, (1, 1, 1), (0, 0, 0), (1, 1, 1), cw, FC)


@pytest.mark.parametrize("k,s,p,I", [((1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 7, 9)), ((1, 3, 3), (1, 2, 2), (0, 1, 1), (1, 13, 11)),
                                     ((3, 3, 3), (1, 1, 1), (1, 1, 1), (5, 4, 6)), ((1, 1, 1), (1, 2, 2), (0, 0, 0), (1, 9, 7)),
                                     ((7, 7, 7), (1, 1, 1), (3, 3, 3), (4, 9, 8)), ((1, 4, 4), (1, 1, 1), (0, 2, 2), (1, 6, 5))])
@pytest.mark.parametrize("mode", [RES_NONE, RES_BEFORE, RES_AFTER])
def test_reference_plain_conv_vs_torch(k, s, p, I, mode):
    """Plain convs with stride and front padding (the stem's 4x4 pad 2 is asymmetric: one padded row in front, none behind is needed
    for the last output), FC wider than the real Cout, the residual modes and ReLU."""
    N, cin, cout, cw, FC = 2, 5, 6, 8, 12
    x, wt = _rand(N, cin, *I, seed=1), _rand(cout, cin, *k, seed=2)
    scale, shift = _rand(cw, seed=3), _rand(cw, seed=4)
    scale[cout:] = 0.0
    shift[cout:] = 0.0
    O = tuple((I[a] + 2 * p[a] - k[a]) // s[a] + 1 for a in range(3))
    if k == (1, 4, 4):
        O = (1, 3, 3)        # stem: H/2 outputs of a pad-2 4x4 conv over an odd side
    L = _plain(N, I, k, s, p, cw, FC, O)
    res = _rand(N, *O, FC, seed=5)
    res[..., cout:] = 0.0
    w = torch.zeros(int(np.prod(k)), cin, cw, dtype=torch.float64)
    w[..., :cout] = wt.permute(2, 3, 4, 1, 0).reshape(-1, cin, cout)
    oi, v = conv_reference(x.permute(0, 2, 3, 4, 1).contiguous(), w, L, scale, shift, res, mode, relu=True)
    want = F.conv3d(F.pad(x, (p[2], p[2], p[1], p[1], p[0], p[0])), wt, stride=s)[:, :, :O[0], :O[1], :O[2]].permute(0, 2, 3, 4, 1)
    want = torch.cat([want, torch.zeros(*want.shape[:-1], FC - cout, dtype=torch.float64)], -1)
    want = epilogue(want, torch.cat([scale[:cout], torch.zeros(FC - cout, dtype=torch.float64)]),
                    torch.cat([shift[:cout], torch.zeros(FC - cout, dtype=torch.float64)]), res if mode else None, True, mode)
    got = torch.full((N * int(np.prod(O)) * FC,), float("nan"), dtype=torch.float64)
    got[oi] = v
    assert len(oi) == got.numel() - N * int(np.prod(O)) * (FC - cw)      # channels cw .. FC-1 are not written
    got = got.reshape(want.shape)
    torch.testing.assert_close(got[..., :cw], want[..., :cw], rtol=1e-12, atol=1e-12)
    assert bool((got[..., :cw][..., cout:] == (res[..., cout:cw] if mode == RES_AFTER else 0.0)).all())


@pytest.mark.parametrize("H,W", [(5, 7), (6, 6), (1, 3)])
def test_reference_k4s2_phases_vs_conv_transpose2d(H, W):
    """ConvTranspose2d(k4, s2, p1) as the four stride-phase 2x2 launches of engine.pack_deconv2d_k4s2 (os 2, oo = phase) on odd sides:
    the union of the phases is the whole output, each element written once."""
    N, cin, cout = 2, 4, 3
    x, wt = _rand(N, cin, H, W, seed=6), _rand(cin, cout, 4, 4, seed=7)
    want = F.conv_transpose2d(x, wt, stride=2, padding=1).permute(0, 2, 3, 1)
    out = torch.full((N * 2 * H * 2 * W * cout,), float("nan"), dtype=torch.float64)
    xs = x.unsqueeze(2).permute(0, 2, 3, 4, 1).contiguous()
    flat = wt.reshape(-1)
    for py in (0, 1):
        for px in (0, 1):
            (base, (_, s_th, s_tw, s_ci, s_co)), pad = eng_mod.deconv2d_k4s2_phase(py, px, cout)
            th, tw, ci, co = torch.meshgrid(*[torch.arange(v) for v in (2, 2, cin, cout)], indexing="ij")
            w = flat[base + th * s_th + tw * s_tw + ci * s_ci + co * s_co].reshape(4, cin, cout)     # lt_conv_gather_weights_fwd
            L = Launch(N, (1, H, W), (1, H, W), (1, 2, 2), (1, 1, 1), pad, (1, 2 * H, 2 * W), (1, 2, 2), (0, py, px), (1, 1, 1), cout, cout)
            oi, v = conv_reference(xs, w, L, torch.ones(cout, dtype=torch.float64), torch.zeros(cout, dtype=torch.float64))
            assert bool(torch.isnan(out[oi]).all())
            out[oi] = v
    torch.testing.assert_close(out.reshape(want.shape), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("D,H,W", [(2, 3, 4), (1, 1, 1), (3, 2, 5)])
def test_reference_grouped_k2s2_vs_conv_transpose3d(D, H, W):
    """ConvTranspose3d(k2, s2) as ONE 1x1x1 launch with N = 8 x Cout and og = (2, 2, 2): block g -> phase (g / 4, g / 2 % 2, g % 2)."""
    N, cin, cout = 2, 5, 3
    x, wt = _rand(N, cin, D, H, W, seed=8), _rand(cin, cout, 2, 2, 2, seed=9)
    want = F.conv_transpose3d(x, wt, stride=2).permute(0, 2, 3, 4, 1)
    w = wt.permute(0, 2, 3, 4, 1).reshape(1, cin, 8 * cout)        # column block g = (a, b, c) phase
    L = Launch(N, (D, H, W), (D, H, W), (1, 1, 1), (1, 1, 1), (0, 0, 0), (2 * D, 2 * H, 2 * W), (2, 2, 2), (0, 0, 0), (2, 2, 2), 8 * cout, cout)
    oi, v = conv_reference(x.permute(0, 2, 3, 4, 1).contiguous(), w, L, torch.ones(8 * cout, dtype=torch.float64),
                           torch.zeros(8 * cout, dtype=torch.float64))
    out = torch.full((want.numel(),), float("nan"), dtype=torch.float64)
    out[oi] = v
    assert len(oi) == want.numel() and len(set(oi.tolist())) == want.numel()
    torch.testing.assert_close(out.reshape(want.shape), want, rtol=1e-12, atol=1e-12)


def test_reference_odd_phase_is_shortened():
    """A grouped launch into an odd-sized tensor (the stride-2 data gradient's layout): phase 1 of an axis of extent 2 n - 1 has n - 1
    positions, so that phase writes fewer; nothing lands outside the tensor."""
    L = Launch(1, (2, 3, 3), (2, 3, 3), (1, 1, 1), (1, 1, 1), (0, 0, 0), (3, 5, 6), (2, 2, 2), (0, 0, 0), (2, 2, 2), 8 * 4, 4)
    oi, si = output_index(L)
    assert len(oi) == len(set(oi.tolist())) == 3 * 5 * 6 * 4         # every element exactly once
    assert group_extent(3, 5, 0, 1, 2) == 2 and group_extent(3, 5, 0, 0, 2) == 3 and group_extent(2, 3, 0, 1, 2) == 1


def test_reference_split_fp16_output():
    """Split-fp16 output rounds each value through split_s32: within 2^-22 relative plus the low half's subnormal floor 2^-25, clamped
    at the fp16 range."""
    L = _plain(1, (1, 3, 4), (1, 1, 1), (1, 1, 1), (0, 0, 0), 4, 4)
    x = _rand(1, 1, 3, 4, 4, seed=10)
    w = _rand(1, 4, 4, seed=11)
    sc = torch.tensor([1.0, 1e-3, 1e5, 1.0], dtype=torch.float64)
    oi, v32 = conv_reference(x, w, L, sc, torch.zeros(4, dtype=torch.float64))
    _, vs = conv_reference(x, w, L, sc, torch.zeros(4, dtype=torch.float64), out_fmt=S32)
    big = v32.abs() > 65504.0
    assert bool(big.any()) and bool((vs[big].abs() <= 65504.0 + 2.0 ** -14 * 65504).all())
    ok = ~big
    assert bool(((vs[ok] - v32[ok]).abs() <= 2.0 ** -22 * v32[ok].abs() + 2.0 ** -25).all())


# ------------------------------------------------------------------------------------------ tests: operand helpers
def test_split_np_is_exact_and_round_to_nearest():
    rng = np.random.RandomState(0)
    x = np.concatenate([rng.randn(4096) * 10.0 ** rng.uniform(-6, 4, 4096), [0.0, -0.0, 65504.0, -7e4, 1e-9, 2.0 ** -24]]).astype(np.float32)
    hi, lo = split_np(x)
    xc = np.clip(x, -65504, 65504).astype(np.float64)
    ulp = np.abs(np.nextafter(hi, np.float16(0)).astype(np.float64) - hi)      # toward zero: no overflow at 65504
    assert np.all(np.abs(hi.astype(np.float64) - xc) <= np.maximum(ulp, 2.0 ** -24) / 2 * 2)
    err = np.abs(join_np(hi, lo) - xc)
    normal = np.abs(xc) > 2.0 ** -3          # lo stays normal: 2^-22 relative
    assert np.all(err[normal] <= 2.0 ** -22 * np.abs(xc[normal]))
    assert np.all(err <= 2.0 ** -22 * np.abs(xc) + 2.0 ** -25)    # fp16 subnormal floor of the low part


def test_dequantizers_invert_the_packers():
    rng = np.random.RandomState(1)
    w = rng.randn(9, 64, 40).astype(np.float32)
    got = dequant_tc(torch.from_numpy(pack_tc_np(w, 48)), 9, 64, 48)
    hi, lo = split_np(w)
    assert torch.equal(got[..., :40], torch.from_numpy(join_np(hi, lo))) and bool((got[..., 40:] == 0).all())
    assert torch.equal(dequant_tc(torch.from_numpy(pack_tc_np(w, 48)), 9, 64, 48, hi_only=True)[..., :40],
                       torch.from_numpy(hi.astype(np.float64)))
    for k, cout in ((3, 32), (3, 16), (7, 16), (7, 20)):
        w = rng.randn(k ** 3, 32, cout).astype(np.float32)
        hi, lo = split_np(w)
        got = dequant_fold(torch.from_numpy(pack_fold_np(w, k)), k, (cout + 15) // 16 * 16)
        assert torch.equal(got[..., :cout], torch.from_numpy(join_np(hi, lo)))
    # the 7^3 layout puts kw outermost: slot 1 is tap (kd 0, kh 1, kw 0)
    w = np.zeros((343, 32, 16), np.float32)
    w[7, 0, 0] = 1.0
    assert pack_fold_np(w, 7)[1, 0, 0] == 1.0


# ------------------------------------------------------------------------------------------ tests: dispatch mirrors and step model
def test_fold_supported_matches_the_engine_width_rule():
    for k in (3, 7):
        for W in (8, 15, 16, 17, 33, 63, 64, 65, 80, 128):
            L = _plain(1, (4, 5, W), (k,) * 3, (1, 1, 1), (k // 2,) * 3, 32, 32)
            assert fold_supported(L, 32, 32) == eng_mod.fold_width_ok(k, W)
    L = _plain(1, (4, 5, 32), (3, 3, 3), (1, 1, 1), (1, 1, 1), 32, 32)
    assert not fold_supported(L._replace(FC=64), 32, 32) and not fold_supported(L, 64, 32) and not fold_supported(L, 32, 48)


def test_simt_tiles():
    assert simt_kernel(4, 4) == "conv_simt_kernel<256, 16, 4, 4, false>"
    assert simt_kernel(17, 32) == "conv_simt_kernel<128, 32, 4, 4, true>"
    assert simt_kernel(33, 48) == "conv_simt_kernel<128, 64, 8, 4, true>"


def test_gpu_case_table_reaches_its_kernels():
    """Every case of tests/test_gpu_conv.py reaches the kernels it names (host-side: the plan at 132 SMs with the engine's workspace,
    the fold predicate and the simt tile), so a table that stops reaching a branch fails here without a GPU."""
    import test_gpu_conv as G
    reached = set()
    for name, c in G.CASES.items():
        got = []
        for part in G.case_launches(c):
            got += ["v2v_tail_kernel<0>"] if c.kind == "tail" else launched_kernels(part.impl, part.L, part.cin, part.desc_cout, part.ws)
        assert got == list(c.expect), (name, got, c.expect)
        reached.update(got)
    missing = set(G.CONV_KERNELS) - reached
    assert not missing, missing


def test_accumulation_steps_match_the_folded_gain():
    """The gain applied to every case assumes the steps of the kernel that launches: split-K layers fold taps x Cin / 16 steps and the
    reduce pass rescales to one split's share; fold-packed 3^3 layers carry the 9 Cin / 16 scale for conv_lines_kernel and the
    27 Cin / 16 one for conv_tc_kernel (engine.pack_filter)."""
    import test_gpu_conv as G
    for name, c in G.CASES.items():
        for part in G.case_launches(c):
            if part.impl in (None, capi.CONV_SIMT):
                continue
            want = accum_steps_launched(part.impl, part.L, part.cin, part.desc_cout, part.ws)
            got = effective_steps(part.impl, part.L, part.cin, part.desc_cout, part.folded_steps, part.ws)
            assert got == want, (name, got, want)
