"""Every glue kernel of csrc/misc.cu (but feature_scatter_kernel, which tests/test_gpu_unproject.py covers) against the exact
references of tests/test_glue_ref_cpu.py.

Each output sits between guard bands and starts as a NaN sentinel (`Guarded`): after a call the guards are intact and every element
was written; a gather into one column block leaves the other blocks of its rows untouched.  Every kernel also runs past its launch
cap (16 CTAs per SM for the grid-stride helpers, 1024 CTAs for absmax, 4096 for the filter gather), so its loop takes more than one
pass.  "Bit-exact" is equality of bit patterns, except that a NaN only has to meet a NaN: the device writes the canonical fp16 NaN
where numpy keeps the float32 payload.  Two kernels have a bar instead:
- lt_fold_bn_fwd: at most 1 float32 ulp from the float64 reference (the kernel's double `beta - mean sc` may be contracted to an FMA);
- lt_coord_volume_fwd with a rotation: per component u (3 sum_k |R_ik v_k| + |out_i|), u = 2^-24, from the float32 v the kernel forms.

Measured on an H100 80GB HBM3 (700 W power limit): fold, 0 of 13,608 outputs differ from the reference; rotated coordinates, worst
err / bar 0.84 (B = 8, n = 64), 0.70 (B = 3, n = 17).
"""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from lt_b200 import autograd_ops as A
from lt_b200 import capi, engine
from test_conv_bwd_cpu import pow2_scale
from test_conv_cpu import s32_rows, split_np
from test_glue_ref_cpu import (NULLS, POOLS, coord_bar, coord_ref, fold_ref, gather_ref, maxpool_ref, pool_input, s2d_ref, same_bits)
from test_gpu_unproject import Guarded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F32, S32 = capi.FMT_F32, capi.FMT_S32


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def grid_cap():
    """Work items of one pass of grid_for (misc.cu): 16 CTAs of 256 threads per SM."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 16 * 256


def written(g):
    """Guards intact and no sentinel left -> the tensor as numpy."""
    torch.cuda.synchronize()
    assert g.guards_intact(), "a write outside the output"
    assert g.unwritten() == 0, "%d elements not written" % g.unwritten()
    return g.t.cpu().numpy()


def amax_bits(x):
    """Bit pattern of max |finite x| as lt_absmax_fwd leaves it (0 when there is none)."""
    a = np.abs(np.asarray(x, np.float32).reshape(-1))
    a = a[np.isfinite(a)]
    return int(np.float32(a.max() if a.size else 0.0).view(np.int32))


def bits_to_float(b):
    return float(np.array(b, np.int32).view(np.float32))


def specials(shape, seed, scale=1.0):
    """float32 values over many binades with the split-fp16 edge cases: fp16 subnormal and below, beyond 65504, +-Inf, NaN, -0."""
    rng = np.random.RandomState(seed)
    x = (rng.randn(*shape) * np.exp2(rng.randint(-30, 20, size=shape))).astype(np.float32) * np.float32(scale)
    flat = x.reshape(-1)
    ex = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 65504.0, 65519.0, 65520.0, -70000.0, 1e30, 6.1e-5, 5.9e-8, 3e-8, 2.9e-8,
                   1e-9, -4e-6], np.float32) * np.float32(scale)
    pos = rng.randint(0, flat.size, size=8 * ex.size)
    flat[pos] = np.resize(ex, pos.size)
    return x


def scaled_input(P, C, mode):
    """specials, or for mode "tiny" values of at most 2^-140 (float32 subnormals; S hits the +126 clamp) and for "huge" values up
    to 3.3e38, both with NaN and +-Inf among them."""
    x = specials((P, C), seed=P + C)
    fin = np.isfinite(x)
    if mode == "tiny":
        rng = np.random.RandomState(P)
        x[fin] = np.clip((rng.randn(int(fin.sum())) * 2.0 ** -142), -2.0 ** -140, 2.0 ** -140).astype(np.float32)
        x.reshape(-1)[7] = -2.0 ** -140
    elif mode == "huge":
        x[fin] = np.clip(x[fin].astype(np.float64) * 2.0 ** 100, -3.3e38, 3.3e38).astype(np.float32)
        x.reshape(-1)[5] = 3.3e38
    return x


# ------------------------------------------------------------------------------------------ split-fp16 conversions
@pytest.mark.parametrize("P, C", [(1000, 64), (3, 32), ("cap", 32)])
def test_split_fp16_round_trip_is_bit_exact(P, C):
    if P == "cap":
        P = grid_cap() * 4 // C + 37
        assert P * C // 4 > grid_cap()
    x = specials((P, C), seed=C)
    s = Guarded((P, 2 * C), torch.float16)
    capi.f32_to_s32(cu(x), s.t, P, C)
    rows = written(s)
    assert same_bits(rows, s32_rows(x))
    y = Guarded((P, C))
    capi.s32_to_f32(s.t, y.t, P, C)
    hi, lo = split_np(x)
    with np.errstate(invalid="ignore"):
        want = hi.astype(np.float32) + lo.astype(np.float32)          # hi + lo is exact in float32
    assert same_bits(written(y), want)


SCALED = [  # (pixels, C, CP, amax mode): "none" = no absmax_bits, "chain" = lt_absmax_fwd of the input, "tiny" = max at 2^-140,
            # "huge" = max near FLT_MAX (with Inf / NaN present in the data)
    (500, 1, 32, "chain"), (301, 17, 32, "chain"), (300, 31, 32, "none"), (257, 32, 32, "chain"), (255, 33, 64, "chain"),
    (129, 17, 64, "tiny"), (200, 33, 64, "huge"), ("cap", 33, 64, "chain")]


@pytest.mark.parametrize("P, C, CP, mode", SCALED)
def test_scaled_split_is_bit_exact(P, C, CP, mode):
    if P == "cap":
        P = grid_cap() // (CP // 4) + 5
        assert P * CP // 4 > grid_cap()
    x = scaled_input(P, C, mode)
    xd = cu(x)
    bits = None
    if mode != "none":
        bits = torch.empty(1, dtype=torch.int32, device=DEV)
        capi.absmax(xd, bits)
        assert int(bits.item()) == amax_bits(x)
    S = 1.0 if bits is None else pow2_scale(np.float32(bits_to_float(amax_bits(x))))
    if mode == "tiny":
        assert S == 2.0 ** 126
    out = Guarded((P, 2 * CP), torch.float16)
    inv = Guarded((1,))
    capi.f32_to_s32_scaled(xd, out.t, P, C, CP, bits, inv.t)
    want = np.zeros((P, CP), np.float32)
    want[:, :C] = x * np.float32(S)
    assert same_bits(written(out), s32_rows(want))
    assert float(written(inv)[0]) == 1.0 / S


# ------------------------------------------------------------------------------------------ absmax
def _absmax_case(name):
    rng = np.random.RandomState(len(name))
    if name == "zeros":
        return np.zeros(1000, np.float32)
    if name == "one":
        return np.float32([-0.375])
    if name == "subnormal max":
        return (rng.rand(777).astype(np.float32) * np.float32(2.0 ** -130)).astype(np.float32)
    if name == "nan and inf beside the max":
        x = rng.randn(4099).astype(np.float32)
        x[1000] = -9.5                                              # the max, in the same warp as an Inf and a NaN
        x[1001], x[1002], x[3000] = np.inf, np.nan, -np.inf
        return x
    if name == "only non-finite":
        return np.float32([np.nan, np.inf, -np.inf] * 100)
    if name == "n % 256 != 0":
        return rng.randn(1000).astype(np.float32)
    x = rng.randn(1024 * 256 * 3 + 17).astype(np.float32)            # several grid-stride passes
    x[1024 * 256 * 2 + 5] = 11.0
    x[1024 * 256 * 2 + 6] = -np.inf
    return x


@pytest.mark.parametrize("name", ["zeros", "one", "subnormal max", "nan and inf beside the max", "only non-finite", "n % 256 != 0",
                                  "past the cap"])
def test_absmax_is_the_bit_pattern_of_the_finite_max(name):
    x = _absmax_case(name)
    bits = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    capi.absmax(cu(x), bits)
    assert int(bits.item()) == amax_bits(x)


# ------------------------------------------------------------------------------------------ filter gather
def _gather_check(w, srcs, k, cin, cin_p, cout, blk_p, out_ld, scaled):
    """Gathers each source into its column block of one [taps][cin_p][out_ld] buffer, checking after each call that the blocks not
    yet written keep the sentinel; returns nothing, asserts bit equality with gather_ref."""
    wd = cu(w)
    taps = k[0] * k[1] * k[2]
    bits = None
    S = 1.0
    if scaled:
        bits = torch.empty(1, dtype=torch.int32, device=DEV)
        capi.absmax(wd, bits)
        S = pow2_scale(np.float32(bits_to_float(amax_bits(w))))
    out = Guarded((taps, cin_p, out_ld))
    want = np.zeros((taps, cin_p, out_ld), np.float32)
    for g, (base, strides) in enumerate(srcs):
        col0 = g * cout if len(srcs) > 1 else 0
        capi.conv_gather_weights(wd, base, strides, k, cin, cin_p, cout, blk_p, out.t, bits, out_ld=out_ld, out_col0=col0)
        want[:, :, col0:col0 + blk_p] = gather_ref(w, base, strides, k, cin, cin_p, cout, blk_p, S)
        torch.cuda.synchronize()
        assert out.guards_intact()
        got = out.t.cpu().numpy()
        done = col0 + blk_p
        assert same_bits(got[:, :, :done], want[:, :, :done])
        assert (got[:, :, done:].view(np.int32) == np.int32(0x7FC5A5A5)).all(), "a write into another column block"
    assert out.unwritten() == 0


def test_gather_conv2d_with_padding_and_scale():
    w = torch.randn(48, 40, 3, 3, generator=torch.Generator().manual_seed(1)).numpy() * np.float32(0.03)
    T = 9
    _gather_check(w, [(0, (T, 3, 1, T, 40 * T))], (1, 3, 3), 40, 64, 48, 64, 64, True)


def test_gather_conv3d_without_scale():
    w = torch.randn(17, 20, 3, 3, 3, generator=torch.Generator().manual_seed(2)).numpy()
    _gather_check(w, [(0, (9, 3, 1, 27, 20 * 27))], (3, 3, 3), 20, 32, 17, 32, 32, False)


def test_gather_deconv2d_k4s2_phases():
    w = torch.randn(64, 48, 4, 4, generator=torch.Generator().manual_seed(3)).numpy()
    for py in (0, 1):
        for px in (0, 1):
            (base, strides), _ = engine.deconv2d_k4s2_phase(py, px, 48)
            _gather_check(w, [(base, strides)], (1, 2, 2), 64, 64, 48, 64, 64, True)


def test_gather_deconv3d_k2s2_column_blocks():
    """The eight phases side by side along N, one column block each, as engine.pack_deconv3d_k2s2 packs them."""
    w = torch.randn(40, 32, 2, 2, 2, generator=torch.Generator().manual_seed(4)).numpy()
    srcs = [(a * 4 + b * 2 + c, (0, 0, 0, 32 * 8, 8)) for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    _gather_check(w, srcs, (1, 1, 1), 40, 64, 32, 32, 8 * 32, True)


def test_gather_flipped_taps_of_the_data_gradient():
    w = torch.randn(24, 16, 3, 3, 3, generator=torch.Generator().manual_seed(5)).numpy()
    (base, strides), k, _, _, ci, co = A.conv3d_dgrad_filter(w.shape, (1, 1, 1))
    _gather_check(w, [(base, strides)], k, ci, 32, co, 32, 32, True)
    w2 = torch.randn(32, 24, 3, 3, generator=torch.Generator().manual_seed(6))
    srcs, k, _, groups, ci, co = A.conv_s2_dgrad_filter(w2.shape, (2, 2))
    wp = A.pad_s2_filter(w2, (2, 2)).contiguous().numpy()
    _gather_check(wp, srcs, k, ci, 32, co, co, 4 * co, True)


def test_gather_past_its_launch_cap():
    """3x3 2048 -> 512: 9.4 M elements, more than 4096 CTAs x 256 threads."""
    w = (torch.randn(512, 2048, 3, 3, generator=torch.Generator().manual_seed(7)) * 0.01).numpy()
    w[3, 5, 1, 1] = np.inf                                         # ignored by the scale, gathered as Inf x S
    assert 9 * 2048 * 512 > 4096 * 256
    _gather_check(w, [(0, (9, 3, 1, 9, 2048 * 9))], (1, 3, 3), 2048, 2048, 512, 512, 512, True)


# ------------------------------------------------------------------------------------------ BatchNorm folding
def test_fold_bn_within_one_ulp():
    worst, differ, total = 0.0, 0, 0
    for C, CP in ((40, 64), (200, 224), (3, 4)):
        g = torch.Generator().manual_seed(C)
        base = dict(gamma=torch.rand(C, generator=g) + 0.5, beta=torch.randn(C, generator=g), mean=torch.randn(C, generator=g) * 3,
                    var=torch.rand(C, generator=g) * 2 + 1e-3, bias=torch.randn(C, generator=g))
        for nulls in NULLS:
            p = dict(base, **nulls)
            if p["mean"] is None:
                p["var"] = None
            for amax in (None, np.float32(0.0371)):
                for steps in (0, 686):
                    bits = None if amax is None else torch.tensor([int(amax.view(np.int32))], dtype=torch.int32, device=DEV)
                    S = 1.0 if amax is None else pow2_scale(amax)
                    sc, sh = Guarded((CP,)), Guarded((CP,))
                    dev = {k: None if v is None else v.to(DEV) for k, v in p.items()}
                    capi.fold_bn(dev["gamma"], dev["beta"], dev["mean"], dev["var"], dev["bias"], 1e-5, C, CP, sc.t, sh.t, bits,
                                 accum_steps=steps)
                    want = fold_ref(*[None if p[k] is None else p[k].numpy() for k in ("gamma", "beta", "mean", "var", "bias")],
                                    1e-5, C, CP, S=S, steps=steps)
                    for got, w in zip((written(sc), written(sh)), want):
                        assert not got[C:].any() and not np.signbit(got[C:]).any()
                        ulp = np.spacing(np.abs(w[:C])).astype(np.float64)
                        err = np.abs(got[:C].astype(np.float64) - w[:C])
                        worst = max(worst, float((err / ulp).max()))
                        differ += int((err > 0).sum())
                        total += C
    print("\nfold_bn: worst %.2f ulp, %d of %d outputs differ from the float64 reference rounded once" % (worst, differ, total))
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------ coordinate volume
def _rotations(B, rng):
    q = rng.randn(B, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w), 2 * (x * y + z * w), 1 - 2 * (x * x + z * z),
                     2 * (y * z - x * w), 2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).astype(np.float32)


@pytest.mark.parametrize("B, n, rotated, transfer", [(8, 64, False, False), (8, 64, False, True), (8, 64, True, True), (3, 17, True, False),
                                                     (1, 2, True, False)])
def test_coord_volume(B, n, rotated, transfer):
    """Per-sample position, centre and rotation, one step per axis for the batch (include/lt_b200.h)."""
    rng = np.random.RandomState(B * n + rotated * 2 + transfer)
    center = (rng.randn(B, 3) * 300 + [0, 0, 900]).astype(np.float32)
    side = rng.uniform(1500, 3000, size=(B, 1))
    position = (center - side / 2 + rng.randn(B, 3) * 10).astype(np.float32)
    step = (side.mean() / (n - 1) * rng.uniform(0.9, 1.1, size=3)).astype(np.float32)       # step[3]: one for every sample
    rot = _rotations(B, rng) if rotated else np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (B, 1))
    if n == 64:
        assert B * n ** 3 > grid_cap()
    out = Guarded((B, n, n, n, 3))
    capi.coord_volume(cu(position), cu(center), cu(step), cu(rot), out.t, transfer)
    got = written(out)
    want, v, out64 = coord_ref(position, center, step, rot, n, transfer)
    if not rotated:
        assert same_bits(got, want)
    else:
        ratio = float((np.abs(got.astype(np.float64) - out64) / coord_bar(rot, v, out64)).max())
        print("\ncoord_volume B=%d n=%d rotated: worst err / bar %.3f" % (B, n, ratio))
        assert ratio <= 1.0


# ------------------------------------------------------------------------------------------ max pooling
POOL_CASES = [  # (pool, N, D, H, W, C, format)
    ("stem 3x3 s2 p1", 2, 1, 11, 13, 4, F32), ("stem 3x3 s2 p1", 2, 1, 11, 13, 64, S32), ("head 2x2 s2", 1, 1, 9, 7, 2048, F32),
    ("head 2x2 s2", 1, 1, 9, 7, 2048, S32), ("head 2x2 s2", 3, 1, 5, 6, 12, F32), ("v2v 2^3 s2", 2, 7, 9, 5, 32, S32),
    ("v2v 2^3 s2", 1, 8, 8, 8, 128, F32), ("stem 3x3 s2 p1", 20, 1, 192, 192, 64, S32)]


@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: "%s %s %s" % (c[0], "x".join(map(str, c[1:6])), "f32" if c[6] == F32 else "s32"))
def test_maxpool(case):
    name, N, D, H, W, C, fmt = case
    k, s, p = POOLS[name]
    x = pool_input(N, D, H, W, C, seed=H * W + C)
    OD, OH, OW = ((n + 2 * pp - kk) // ss + 1 for n, kk, ss, pp in zip((D, H, W), k, s, p))
    if N == 20:
        assert N * OH * OW * C // 4 > grid_cap()
    if fmt == F32:
        inp = cu(x)
        out = Guarded((N, OD, OH, OW, C))
        capi.maxpool(inp, out.t, F32, N, D, H, W, C, k, s, p, OD, OH, OW)
        got = written(out)
        want = maxpool_ref(x, k, s, p)
        assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN positions differ (NaN count: kernel %d, reference %d)" % (
            int(np.isnan(got).sum()), int(np.isnan(want).sum()))
        assert same_bits(got, want)
    else:
        rows = s32_rows(x)
        hi, lo = rows.reshape(*x.shape[:4], C // 32, 2, 32)[..., 0, :], rows.reshape(*x.shape[:4], C // 32, 2, 32)[..., 1, :]
        with np.errstate(invalid="ignore"):
            joined = (hi.astype(np.float32) + lo.astype(np.float32)).reshape(x.shape)   # what the kernel loads (Inf -> Inf + NaN)
        out = Guarded((N, OD, OH, OW, 2 * C), torch.float16)
        capi.maxpool(cu(rows), out.t, S32, N, D, H, W, C, k, s, p, OD, OH, OW)
        got = written(out)
        want = s32_rows(maxpool_ref(joined, k, s, p))
        assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN positions differ"
        assert same_bits(got, want)


# ------------------------------------------------------------------------------------------ stem space-to-depth
@pytest.mark.parametrize("N, C, H, W", [(2, 1, 10, 14), (3, 3, 14, 22), (1, 5, 6, 6), (2, 8, 18, 10), (20, 3, 384, 384)])
def test_stem_s2d(N, C, H, W):
    x = specials((N, C, H, W), seed=C * H)
    if N == 20:
        assert N * (H // 2) * (W // 2) > grid_cap()
    out = Guarded((N, H // 2, W // 2, 64), torch.float16)
    capi.stem_s2d(cu(x), out.t, N, C, H, W)
    assert same_bits(written(out), s2d_ref(x))


# ------------------------------------------------------------------------------------------ layout conversions
@pytest.mark.parametrize("N, C, H, W, Cp", [(3, 3, 10, 14, 4), (2, 5, 7, 9, 37), (1, 32, 3, 5, 32), (3, 3, 450, 450, 4)])
def test_nchw_to_nhwc(N, C, H, W, Cp):
    x = specials((N, C, H, W), seed=H + Cp)
    out = Guarded((N, H, W, Cp))
    capi.nchw_to_nhwc(cu(x), out.t, N, C, H, W, Cp)
    want = np.zeros((N, H, W, Cp), np.float32)
    want[..., :C] = x.transpose(0, 2, 3, 1)
    assert same_bits(written(out), want)


@pytest.mark.parametrize("N, P, Cs, C", [(2, 1000, 45, 37), (3, 140, 4, 3), (1, 31, 32, 32), (2, 70001, 64, 33)])
def test_cl_to_cf(N, P, Cs, C):
    x = specials((N, P, Cs), seed=P + C)
    out = Guarded((N, C, P))
    capi.cl_to_cf(cu(x), out.t, N, P, Cs, C)
    assert same_bits(written(out), np.ascontiguousarray(x[..., :C].transpose(0, 2, 1)))


IMAGE_CASES = [("u8 table", 2, 1, 9, 13), ("u8 table", 2, 2, 9, 13), ("u8 table", 3, 4, 8, 8), ("u8", 2, 3, 7, 5), ("f32", 2, 3, 7, 5),
               ("f64", 2, 4, 9, 6), ("u8 table", 4, 3, 400, 400), ("f64", 4, 1, 400, 400)]


@pytest.mark.parametrize("kind, N, C, H, W", IMAGE_CASES)
def test_images_hwc_to_nchw(kind, N, C, H, W):
    rng = np.random.RandomState(N * C * H)
    lut = None
    if kind.startswith("u8"):
        x = rng.randint(0, 256, size=(N, H, W, C)).astype(np.uint8)
        x.reshape(-1)[:2] = (0, 255)
        if kind == "u8 table":
            lut = (rng.randn(C, 256) * 3).astype(np.float32)
            lut[0, 7] = np.nan
            want = lut[np.arange(C), x].transpose(0, 3, 1, 2)
        else:
            want = x.astype(np.float32).transpose(0, 3, 1, 2)
    elif kind == "f32":
        x = specials((N, H, W, C), seed=C)
        want = x.transpose(0, 3, 1, 2)
    else:
        x = rng.randn(N, H, W, C) * 10.0 ** rng.randint(-50, 50, size=(N, H, W, C))
        x.reshape(-1)[:8] = (1e39, -1e39, 3.5e38, 1e-40, -1e-45, 1e-46, np.nan, 2.0 ** -149 * 1.5)
        with np.errstate(over="ignore"):
            want = x.astype(np.float32).transpose(0, 3, 1, 2)
    if H == 400:
        assert N * H * W > grid_cap()
    out = Guarded((N, C, H, W))
    capi.images_hwc_to_nchw(cu(x), None if lut is None else cu(lut), out.t, N, C, H, W)
    assert same_bits(written(out), np.ascontiguousarray(want))


# ------------------------------------------------------------------------------------------ the training backward's chain in a graph
def test_absmax_and_scaled_split_replay_bit_identically_from_a_cuda_graph():
    P, C, CP = 4096, 40, 64
    x = cu(specials((P, C), seed=3))
    bits = torch.empty(1, dtype=torch.int32, device=DEV)
    out = torch.empty((P, 2 * CP), dtype=torch.float16, device=DEV)
    inv = torch.empty(1, device=DEV)

    def chain():
        capi.absmax(x, bits)
        capi.f32_to_s32_scaled(x, out, P, C, CP, bits, inv)

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        chain()
    for seed in (4, 5):
        x.copy_(cu(specials((P, C), seed=seed, scale=2.0 ** (seed * 7))))
        chain()
        want = (out.clone(), bits.clone(), inv.clone())
        out.zero_()
        bits.zero_()
        inv.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int16), want[0].view(torch.int16))
        assert torch.equal(bits, want[1]) and torch.equal(inv, want[2])


# ------------------------------------------------------------------------------------------ dispatch
MISC_KERNELS = ["coord_volume_kernel", "maxpool_kernel", "images_hwc_to_nchw_kernel<unsigned char>", "images_hwc_to_nchw_kernel<float>",
                "images_hwc_to_nchw_kernel<double>", "nchw_to_nhwc_kernel", "stem_s2d_kernel", "f32_to_s32_kernel",
                "f32_to_s32_scaled_kernel", "s32_to_f32_kernel", "cl_to_cf_kernel", "absmax_kernel", "gather_weights_kernel",
                "fold_bn_kernel"]


def _kernel_names(prof):
    pat = re.compile(r"(coord_volume|maxpool|images_hwc_to_nchw|nchw_to_nhwc|stem_s2d|f32_to_s32_scaled|f32_to_s32|s32_to_f32|cl_to_cf|"
                     r"absmax|gather_weights|fold_bn)_kernel(<[^>]*>)?")
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    names = []
    for e in sorted(evs, key=lambda e: e.start_ns()):
        m = pat.search(e.name())
        if m:
            names.append(m.group(0))
    return names


def run_in_fresh_process(module, fn):
    """`module`.`fn`() (a function of a test module that returns JSON-able data) in a Python process of its own: a profiler session
    there is the process's first, so no earlier session in the test run can change which kernels it records."""
    tests = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import %s as m; print('RESULT=' + json.dumps(m.%s()))"
            % (tests, os.path.dirname(tests), module, fn))
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], capture_output=True, text=True, timeout=600)
    lines = [l for l in res.stdout.splitlines() if l.startswith("RESULT=")]
    assert res.returncode == 0 and lines, res.stdout[-2000:] + res.stderr[-4000:]
    return json.loads(lines[-1][len("RESULT="):])


def profiled_misc_launches():
    """One call of each entry point, in the order of MISC_KERNELS, under torch.profiler -> the misc.cu kernels launched."""
    from torch.profiler import ProfilerActivity, profile
    f = torch.randn(2, 8, 8, 32, device=DEV)
    s = torch.empty((2, 8, 8, 64), dtype=torch.float16, device=DEV)
    img = torch.randn(2, 3, 8, 8, device=DEV)
    bits = torch.empty(1, dtype=torch.int32, device=DEV)
    one = torch.ones(32, device=DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        capi.coord_volume(one[:3], one[:3], one[:3], one[:9], torch.empty((1, 4, 4, 4, 3), device=DEV))
        capi.maxpool(f, torch.empty((2, 4, 4, 32), device=DEV), F32, 2, 1, 8, 8, 32, (1, 2, 2), (1, 2, 2), (0, 0, 0), 1, 4, 4)
        capi.images_hwc_to_nchw(torch.zeros((1, 4, 4, 3), dtype=torch.uint8, device=DEV), None, torch.empty((1, 3, 4, 4), device=DEV), 1, 3, 4, 4)
        capi.images_hwc_to_nchw(torch.zeros((1, 4, 4, 3), device=DEV), None, torch.empty((1, 3, 4, 4), device=DEV), 1, 3, 4, 4)
        capi.images_hwc_to_nchw(torch.zeros((1, 4, 4, 3), dtype=torch.float64, device=DEV), None, torch.empty((1, 3, 4, 4), device=DEV),
                                1, 3, 4, 4)
        capi.nchw_to_nhwc(img, torch.empty((2, 8, 8, 4), device=DEV), 2, 3, 8, 8, 4)
        capi.stem_s2d(img, torch.empty((2, 4, 4, 64), dtype=torch.float16, device=DEV), 2, 3, 8, 8)
        capi.f32_to_s32(f, s, 128, 32)
        capi.f32_to_s32_scaled(f, s, 128, 32, 32)
        capi.s32_to_f32(s, f, 128, 32)
        capi.cl_to_cf(f.view(2, 64, 32), torch.empty((2, 32, 64), device=DEV), 2, 64, 32, 32)
        capi.absmax(f, bits)
        capi.conv_gather_weights(f, 0, (0, 0, 0, 32, 1), (1, 1, 1), 32, 32, 32, 32, torch.empty((1, 32, 32), device=DEV), bits)
        capi.fold_bn(None, None, None, None, None, 0.0, 32, 32, torch.empty(32, device=DEV), torch.empty(32, device=DEV))
        torch.cuda.synchronize()
    return _kernel_names(prof)


def test_the_table_reaches_every_misc_kernel():
    """One call of each entry point launches the kernel MISC_KERNELS names; with feature_scatter_kernel (tests/test_gpu_unproject.py)
    these are all fifteen kernel instantiations of misc.cu."""
    names = run_in_fresh_process("test_gpu_glue_ref", "profiled_misc_launches")
    assert names == MISC_KERNELS, names
