"""Float64 semantics of lt_conv_wgrad_fwd, its launch plan and accumulation model, and the split-fp16 rule for non-finite values,
without a GPU.

- `wgrad_reference` is the weight gradient of the lt_conv_nd_fwd launch a descriptor describes, in float64, written from the
  descriptor alone (taps, stride, front padding, the output mapping os* / oo* and grouped outputs og*) and not from the kernel's
  index helpers: dW[t][ci][g oc + co] = sum_{n, o} x[n, o s - p + t][ci] dY[n, o os + oo + phase(g)][g oc + co] / S.  It works on
  torch tensors of any device and dtype (tests/test_gpu_conv_bwd.py runs it on the GPU in float64 and float32).  Here it is checked
  against torch float64 autograd for every descriptor family the training convolutions issue, and against the kernel's own index
  mapping (lt_test_conv_wgrad_host) on every case of the GPU table.
- `lt_conv_wgrad_plan` (nwg, ngroups, m_tiles, splits, stages at a given SM count): every GPU case reaches the instantiation, split
  count and ring depth it names at the H100's 132 SMs, and together the cases cover every branch of the plan.
- `wgrad_bar`: the per-element error bar of the native weight gradient, derived from the kernel's accumulation order.
- `pow2_scale`: the power-of-two scale weight_pow2_scale (common.cuh) derives from max|v|.
"""
import math
from collections import namedtuple

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lt_b200 import autograd_ops as A
from lt_b200 import capi
from test_conv_cpu import join_np, split_np

SMS = 132
EPS = 2.0 ** -24


# ------------------------------------------------------------------------------------------ float64 semantics of lt_conv_wgrad_fwd
def _geometry(d):
    k, s, p = (d.KD, d.KH, d.KW), (d.sd, d.sh, d.sw), (d.pd, d.ph, d.pw)
    O, Fd = (d.OD, d.OH, d.OW), (d.FD, d.FH, d.FW)
    os_, oo, og = (d.osd, d.osh, d.osw), (d.ood, d.ooh, d.oow), tuple(max(v, 1) for v in (d.ogd, d.ogh, d.ogw))
    return k, s, p, O, Fd, os_, oo, og


def wgrad_reference(x, g, d, S=1.0, cin=None, cout=None):
    """lt_conv_wgrad_fwd of descriptor d: x [N][ID][IH][IW][d.Cin], g [N][FD][FH][FW][d.FC] (the output gradient as stored, i.e.
    scaled by S) -> dW [taps (kd, kh, kw)][cin][G cout] in x's dtype, divided by S.  cin / cout: the real channel counts (default
    the descriptor's).  Positions a group's phase puts outside the output tensor contribute nothing; taps that fall outside the
    input read zeros."""
    k, s, p, O, Fd, os_, oo, og = _geometry(d)
    G = og[0] * og[1] * og[2]
    oc = d.Cout // G if G > 1 else d.Cout
    cin = d.Cin if cin is None else cin
    cout = oc if cout is None else cout
    I = (d.ID, d.IH, d.IW)
    pads = []
    for ax in (2, 1, 0):          # F.pad order: W, H, D; zeros in front (p) and wherever the last taps fall past the input
        pads += [p[ax], max(0, (O[ax] - 1) * s[ax] + k[ax] - p[ax] - I[ax])]
    xt = F.pad(x.permute(0, 4, 1, 2, 3), pads)[:, :cin]                 # [N][cin][D'][H'][W']
    dw = torch.zeros(k[0] * k[1] * k[2], cin, G * cout, dtype=x.dtype, device=x.device)
    for gi in range(G):
        ph = (gi // (og[1] * og[2]), (gi // og[2]) % og[1], gi % og[2])
        idx = [torch.arange(O[a], device=x.device) * os_[a] + oo[a] + ph[a] for a in range(3)]
        inside = [(i < Fd[a]) for a, i in enumerate(idx)]
        gg = g[:, idx[0].clamp(max=Fd[0] - 1)][:, :, idx[1].clamp(max=Fd[1] - 1)][:, :, :, idx[2].clamp(max=Fd[2] - 1)]
        mask = (inside[0].view(-1, 1, 1) & inside[1].view(1, -1, 1) & inside[2].view(1, 1, -1)).to(x.dtype)
        gg = (gg[..., :cout] * mask[None, :, :, :, None]).reshape(-1, cout)      # [N O][cout]: a group's channels are 0 .. FC - 1
        t = 0
        for kd in range(k[0]):
            for kh in range(k[1]):
                for kw in range(k[2]):
                    xs = xt[:, :, kd:kd + (O[0] - 1) * s[0] + 1:s[0], kh:kh + (O[1] - 1) * s[1] + 1:s[1], kw:kw + (O[2] - 1) * s[2] + 1:s[2]]
                    dw[t, :, gi * cout:(gi + 1) * cout] = xs.permute(1, 0, 2, 3, 4).reshape(cin, -1) @ gg
                    t += 1
    return dw / S


def wgrad_reference_sig(x, g, d, S=1.0, cin=None, cout=None):
    """(dW, sum |x||g| / S) per element: the second bounds every partial sum the kernel forms."""
    return wgrad_reference(x, g, d, S, cin, cout), wgrad_reference(x.abs(), g.abs(), d, S, cin, cout)


def wgrad_steps(plan):
    """Rounding steps one dW element passes through in conv_wgrad_kernel + wgrad_reduce_kernel, weighted as they bound the error:
    - each M tile of 128 positions is 8 k16 wgmma steps into a fresh accumulator, each adding with truncation (<= 2^-23 of the
      running sum, i.e. 2 x 2^-24: the factor 2 of the bar);
    - the tile's result is added into an fp32 register sum with round-to-nearest: one step per tile of the split, at most
      ceil(m_tiles / splits) of them;
    - the epilogue adds the four quadrants hi*hi + ((hi*lo + lo*hi) + lo*lo): 3 steps;
    - wgrad_reduce_kernel adds the `splits` partial tiles in split order: `splits` steps;
    - the division by S is an exact power-of-two multiply.
    Every intermediate is bounded by sum |x||g|, and the products of fp16 halves are exact in fp32."""
    return 8 + -(-plan["m_tiles"] // plan["splits"]) + 3 + plan["splits"]


def wgrad_bar(ref, sig, plan):
    """|native - ref| <= 2 steps 2^-24 sum|x||g| / S + 2^-24 |ref| (the final rounding to float32) per element."""
    return 2.0 * wgrad_steps(plan) * EPS * sig + EPS * ref.abs()


def pow2_scale(amax):
    """weight_pow2_scale (common.cuh) of max|v| (a finite float32 >= 0): 2^(9 - floor(log2 max)), the exponent kept inside
    [-126, 126] so that S and 1 / S are exact normal floats; 1 for an all-zero tensor."""
    if amax == 0.0:
        return 1.0
    bits = int(np.array(amax, np.float32).view(np.int32))
    e = (bits >> 23) - 127
    return 2.0 ** min(max(9 - e, -126), 126)


# ------------------------------------------------------------------------------------------ tests: the reference vs autograd
def _cl(t, cp):
    """(N, C, [D,] H, W) float64 -> channels-last (N, D, H, W, cp), D = 1 for 2-D, channels C .. cp-1 zero."""
    if t.dim() == 4:
        t = t.unsqueeze(2)
    out = torch.zeros(*t.shape[:1], *t.shape[2:], cp, dtype=t.dtype)
    out[..., :t.shape[1]] = t.permute(0, 2, 3, 4, 1)
    return out


def _close(got, want):
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max()), float((got - want).abs().max())


def _problem(x_shape, w_shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*x_shape, generator=g, dtype=torch.float64), torch.randn(*w_shape, generator=g, dtype=torch.float64)


@pytest.mark.parametrize("k,dims,cin,cout", [(1, (3, 4, 5), 40, 17), (3, (4, 3, 5), 32, 48), (7, (3, 5, 4), 16, 32)])
def test_reference_same_conv3d_vs_autograd(k, dims, cin, cout):
    N = 2
    x, w = _problem((N, cin, *dims), (cout, cin, k, k, k), k)
    w.requires_grad_(True)
    y = F.conv3d(x, w, None, 1, k // 2)
    gy = torch.randn_like(y)
    y.backward(gy)
    d = A.conv3d_wgrad_desc(N, dims, cin, cout, (k,) * 3, (k // 2,) * 3)
    S = 2.0 ** 7
    got = wgrad_reference(_cl(x, d.Cin), _cl(gy * S, d.FC), d, S, cin, cout)
    _close(got.reshape(k, k, k, cin, cout).permute(4, 3, 0, 1, 2), w.grad)
    ref, sig = wgrad_reference_sig(_cl(x, d.Cin), _cl(gy, d.FC), d, 1.0, cin, cout)
    assert bool((sig >= ref.abs()).all())
    assert bool((sig[ref != 0] > 0).all())          # 7^3 over a 3-deep map: the outermost kd taps only ever meet the padding


@pytest.mark.parametrize("k,HW", [(1, (9, 7)), (1, (8, 10)), (3, (13, 11)), (3, (8, 10)), (3, (2, 3))])
def test_reference_stride2_conv2d_vs_autograd(k, HW):
    """s2k1 and s2k3 (pad 1) over odd and even sides: the input is traversed at stride 2, the last tap of an even side reads the
    zero padding behind it."""
    N, cin, cout = 2, 36, 20
    x, w = _problem((N, cin, *HW), (cout, cin, k, k), 10 + k)
    w.requires_grad_(True)
    y = F.conv2d(x, w, None, 2, k // 2)
    gy = torch.randn_like(y)
    y.backward(gy)
    d = A.conv3d_wgrad_desc(N, (1, *HW), cin, cout, (1, k, k), (0, k // 2, k // 2), (1, 2, 2))
    assert (d.OH, d.OW) == tuple(y.shape[2:])
    got = wgrad_reference(_cl(x, d.Cin), _cl(gy, d.FC), d, 1.0, cin, cout)
    _close(got.reshape(k, k, cin, cout).permute(3, 2, 0, 1), w.grad)


@pytest.mark.parametrize("HW", [(5, 7), (4, 6), (1, 1)])
def test_reference_k4s2_phases_vs_autograd(HW):
    """ConvTranspose2d(k4, s2, p1): the four phase descriptors, each scattered to its four taps, give autograd's dW."""
    N, cin, cout = 2, 24, 40
    x, w = _problem((N, cin, *HW), (cin, cout, 4, 4), 20)
    w.requires_grad_(True)
    y = F.conv_transpose2d(x, w, None, 2, 1)
    gy = torch.randn_like(y)
    y.backward(gy)
    got = torch.full((cin, cout, 4, 4), float("nan"), dtype=torch.float64)
    for py in (0, 1):
        for px in (0, 1):
            d = A.conv_transpose2d_k4s2_desc(N, (1, *HW), cin, cout, py, px)
            gp = wgrad_reference(_cl(x, d.Cin), _cl(gy, d.FC), d, 1.0, cin, cout)
            got[:, :, 1 - py::2, 1 - px::2] = A.conv_transpose2d_k4s2_wgrad_scatter(gp, py, px)
    assert not bool(torch.isnan(got).any())
    _close(got, w.grad)


@pytest.mark.parametrize("dims,cout", [((2, 3, 4), 32), ((1, 1, 1), 64), ((3, 2, 5), 32)])
def test_reference_grouped_k2s2_vs_autograd(dims, cout):
    """ConvTranspose3d(k2, s2) as the one grouped 1x1x1 GEMM: column block g = a 4 + b 2 + c is output phase (a, b, c)."""
    N, cin = 2, 32
    x, w = _problem((N, cin, *dims), (cin, cout, 2, 2, 2), 30)
    w.requires_grad_(True)
    y = F.conv_transpose3d(x, w, None, 2)
    gy = torch.randn_like(y)
    y.backward(gy)
    d = A.conv_transpose3d_desc(N, dims, cin, cout)
    got = wgrad_reference(_cl(x, d.Cin), _cl(gy, d.FC), d, 1.0, cin, cout)
    _close(got.reshape(cin, 8, cout).permute(0, 2, 1).reshape(cin, cout, 2, 2, 2), w.grad)


def s2d(img):
    """lt_stem_s2d_fwd's layout: (N, 3, H, W) -> (N, 1, H/2, W/2, 32), channel (r 2 + s) 3 + c = img[c][2 y + r][2 x + s], 12 .. 31 zero."""
    N, C, H, W = img.shape
    out = torch.zeros(N, 1, H // 2, W // 2, 32, dtype=img.dtype, device=img.device)
    for r in (0, 1):
        for s in (0, 1):
            out[:, 0, :, :, (r * 2 + s) * C:(r * 2 + s + 1) * C] = img[:, :, r::2, s::2].permute(0, 2, 3, 1)
    return out


@pytest.mark.parametrize("HW", [(16, 12), (10, 14)])
def test_reference_stem_s2d_vs_autograd(HW):
    """The stem's 4x4 stride-1 conv over the space-to-depth input (12 real channels of 32), mapped back by stem_wgrad_index."""
    N, cout = 2, 40
    img, w = _problem((N, 3, *HW), (cout, 3, 7, 7), 40)
    w.requires_grad_(True)
    y = F.conv2d(img, w, None, 2, 3)
    gy = torch.randn_like(y)
    y.backward(gy)
    d = A.stem_wgrad_desc(N, HW[0], HW[1], cout)
    gs = wgrad_reference(s2d(img), _cl(gy, d.FC), d, 1.0, 12, cout)
    got = gs.reshape(16 * 12, cout)[A.stem_wgrad_index("cpu")].t().reshape(cout, 3, 7, 7)
    _close(got, w.grad)


def test_reference_matches_the_kernel_index_mapping_on_the_gpu_cases():
    """lt_test_conv_wgrad_host (the kernel's wgrad_boxes / wgrad_in_row / wgrad_out_row over its M tiles) and the reference agree on
    every case of the GPU table but the large-K one: the helpers the kernel uses map every (tap, position, group) exactly once."""
    import test_gpu_conv_bwd as G
    for name, c in G.WCASES.items():
        if name == G.LARGE_K:
            continue
        x, g = G.host_operands(c, seed=3)
        for lw in G.wgrad_launches(c):
            want = wgrad_reference(x, g, lw.desc, 1.0, lw.cin, lw.cout)
            got = torch.empty(want.shape, dtype=torch.float32)
            capi.conv_wgrad_host(lw.desc, x.float().contiguous(), g.float().contiguous(), lw.cin, lw.cout, got)
            err = float((got.double() - want).abs().max())
            assert err <= 1e-6 * float(want.abs().max()), (name, err)


# ------------------------------------------------------------------------------------------ tests: the launch plan
def test_gpu_case_table_reaches_its_kernels():
    """Every case of tests/test_gpu_conv_bwd.py reaches the instantiation, K split count and ring depth it names at 132 SMs, and
    the table covers every branch: conv_wgrad_kernel<1 / 2 / 4>, a <4> CTA with 3 active warpgroups, several CTA groups along N
    with a partial last one, splits 1 and a split count that does not divide m_tiles, 2, 4 and 6 stages."""
    import test_gpu_conv_bwd as G
    seen = set()
    for name, c in G.WCASES.items():
        for lw in G.wgrad_launches(c):
            p = capi.conv_wgrad_plan(lw.desc, SMS)
            got = ("conv_wgrad_kernel<%d>" % p["nwg"], p["splits"], p["stages"])
            assert got == c.expect, (name, got, c.expect)
            ncb = lw.desc.Cout // 32
            active_last = ncb - (p["ngroups"] - 1) * p["nwg"]
            seen.add(got[0])
            seen.add(("stages", p["stages"]))
            seen.add("splits 1" if p["splits"] == 1 else "splits > 1, uneven" if p["m_tiles"] % p["splits"] else "splits > 1")
            if p["nwg"] == 4 and p["ngroups"] == 1 and active_last == 3:
                seen.add("<4> with 3 active")
            if p["ngroups"] > 1 and active_last < p["nwg"]:
                seen.add("partial last group")
    want = {"conv_wgrad_kernel<1>", "conv_wgrad_kernel<2>", "conv_wgrad_kernel<4>", ("stages", 2), ("stages", 4), ("stages", 6),
            "splits 1", "splits > 1, uneven", "<4> with 3 active", "partial last group"}
    assert want <= seen, want - seen


def test_plan_rules():
    """nwg = min(Cout / 32, 4) with 3 -> 4; stages = 200 KiB / (16 KiB (1 + nwg)) capped at 6; splits <= max(1, m_tiles / 16) and
    the grid stays within 16 CTAs per SM; the split depends on the SM count it is planned for; the workspace holds one fp32 partial
    dW per split."""
    for cout, nwg in ((32, 1), (64, 2), (96, 4), (128, 4), (160, 4), (224, 4)):
        d = A.conv3d_wgrad_desc(2, (8, 8, 8), 32, cout, (3, 3, 3), (1, 1, 1))
        p = capi.conv_wgrad_plan(d, SMS)
        assert p["nwg"] == nwg and p["ngroups"] == -(-(cout // 32) // nwg)
        assert p["stages"] == min(6, 200 * 1024 // (16384 * (1 + nwg)))
        assert p["m_tiles"] >= -(-2 * 512 // 128)
        assert 1 <= p["splits"] <= max(1, p["m_tiles"] // 16)
        assert 27 * p["ngroups"] * p["splits"] <= 16 * SMS
    d = A.conv3d_wgrad_desc(2, (64, 64, 64), 32, 32, (3, 3, 3), (1, 1, 1))
    splits = {sm: capi.conv_wgrad_plan(d, sm)["splits"] for sm in (132, 114, 78)}
    assert len(set(splits.values())) > 1, splits
    assert capi.conv_wgrad_workspace_bytes(d) == capi.conv_wgrad_plan(d, SMS)["splits"] * 27 * 32 * 32 * 4
    with pytest.raises(RuntimeError):
        capi.conv_wgrad_plan(d, 0)


def test_bar_model():
    """The bar's step count for a few plans: one tile (8 + 1 + 3 + 1) and the large-K layer's ceil(m_tiles / splits) tiles."""
    assert wgrad_steps({"m_tiles": 1, "splits": 1}) == 13
    assert wgrad_steps({"m_tiles": 4096, "splits": 44}) == 8 + 94 + 3 + 44
    ref, sig = torch.tensor([1.0, -2.0]), torch.tensor([3.0, 2.0])
    assert torch.equal(wgrad_bar(ref, sig, {"m_tiles": 1, "splits": 1}), 26 * EPS * sig + EPS * ref.abs())


def test_pow2_scale_rule():
    """S puts max|v| S into [512, 1024) while 9 - floor(log2 max) stays inside [-126, 126]; outside, the exponent is clamped (it
    is no longer reset to S = 1), so gradients at 2^-101 or 2^101 keep their bits."""
    for e in (-100, -3, 0, 7, 100):
        for m in (2.0 ** e, np.nextafter(np.float32(2.0 ** (e + 1)), np.float32(0))):
            assert 512 <= float(m) * pow2_scale(float(m)) < 1024
    assert pow2_scale(2.0 ** -101) == 2.0 ** 110 and pow2_scale(2.0 ** 101) == 2.0 ** -92
    assert pow2_scale(2.0 ** -126) == 2.0 ** 126 and pow2_scale(1e-45) == 2.0 ** 126          # subnormal max: clamped
    assert pow2_scale(float(np.finfo(np.float32).max)) == 2.0 ** -118
    assert pow2_scale(0.0) == 1.0


# ------------------------------------------------------------------------------------------ tests: split-fp16 of non-finite values
def test_split_keeps_non_finite_values_non_finite():
    """split_s32 (common.cuh): NaN stays NaN in both halves; +-Inf keeps an infinite high half and a NaN low half, so hi + lo is
    NaN rather than a finite +-65504; finite values beyond the fp16 range saturate at +-65504 as documented."""
    x = np.array([np.nan, np.inf, -np.inf, 7e4, -1e9, 65504.0, 1.5, -0.0], np.float32)
    hi, lo = split_np(x)
    v = join_np(hi, lo)
    assert np.isnan(hi[0]) and np.isnan(lo[0]) and np.isnan(v[0])
    assert hi[1] == np.inf and hi[2] == -np.inf and np.isnan(lo[1]) and np.isnan(lo[2]) and not np.isfinite(v[1:3]).any()
    assert v[3] == 65504.0 and v[4] == -65504.0 and lo[3] == 0 and lo[4] == 0
    assert v[5] == 65504.0 and v[6] == 1.5 and v[7] == 0.0
