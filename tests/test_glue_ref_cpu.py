"""Exact references of the glue kernels of csrc/misc.cu, checked here without a GPU; tests/test_gpu_glue_ref.py holds the kernels to them.

- split-fp16 rows: `split_np` / `join_np` / `s32_rows` of tests/test_conv_cpu.py, the power-of-two scale `pow2_scale` of
  tests/test_conv_bwd_cpu.py (weight_pow2_scale, clamped to 2^+-126).
- `maxpool_ref`: a window max with torch's rule (a NaN wins, a value replaces the running maximum only if strictly greater, taps in
  the padding count as -inf), against F.max_pool2d / F.max_pool3d for the engine's three pools.
- `s2d_ref`: the stem's 2x2 space-to-depth, against the inverse of engine.stem_s2d_filter (the 7x7 stride-2 conv equals the 4x4
  stride-1 conv of the rearranged filter over the rearranged input).
- `gather_ref`: lt_conv_gather_weights_fwd's affine map as numpy indexing, against torch.permute of Conv2d / Conv3d /
  ConvTranspose2d (k4 s2 phases) / ConvTranspose3d (k2 s2) weights and the flipped / phase maps of the data gradients.
- `fold_ref`: lt_fold_bn_fwd in float64, against torch's eval-mode BatchNorm for every null combination.
- `coord_ref`: lt_coord_volume_fwd (float32 grid, float64 rotation), bit-equal to the oracle's coordinate volume at theta = 0.
- Every argument check of misc.cu's C entry points returns its error before it touches a pointer.
"""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from lt_b200 import autograd_ops as A
from lt_b200 import capi, engine
from oracle import vol_oracle as O
from test_conv_bwd_cpu import pow2_scale
from test_conv_cpu import join_np, s32_rows, split_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ACCUM_RATE = 0.28                         # kAccumTruncRate of csrc/common.cuh


def accum_gain(steps):
    """accum_gain (common.cuh): 1 + kAccumTruncRate x steps x 2^-24, in float64."""
    return 1.0 + ACCUM_RATE * steps * 5.9604644775390625e-08


# ------------------------------------------------------------------------------------------ references
def maxpool_ref(x, k, s, p):
    """Channels-last float32 (N, D, H, W, C) -> (N, OD, OH, OW, C), floor output size: per window, taps in (d, h, w) order, m starts
    at -inf and takes v if v > m or v is NaN (torch's max_pool rule).  Padding is -inf, which never replaces m."""
    x = np.asarray(x, np.float32)
    N, D, H, W, C = x.shape
    dims = (D, H, W)
    out = [(n + 2 * pp - kk) // ss + 1 for n, kk, ss, pp in zip(dims, k, s, p)]
    xp = np.pad(x, [(0, 0)] + [(pp, pp) for pp in p] + [(0, 0)], constant_values=-np.inf)
    m = np.full((N, *out, C), -np.inf, np.float32)
    for a in range(k[0]):
        for b in range(k[1]):
            for e in range(k[2]):
                v = xp[:, a:a + s[0] * (out[0] - 1) + 1:s[0], b:b + s[1] * (out[1] - 1) + 1:s[1], e:e + s[2] * (out[2] - 1) + 1:s[2]]
                with np.errstate(invalid="ignore"):
                    m = np.where((v > m) | np.isnan(v), v, m)
    return m


def s2d_float(x):
    """Images (N, C, H, W) float32, C <= 8, H and W even -> (N, H/2, W/2, 32) float32 with channel (r*2 + s)*C + c =
    x[c][2y + r][2x + s] and channels 4C..31 zero (stem_s2d_kernel)."""
    N, C, H, W = x.shape
    out = np.zeros((N, H // 2, W // 2, 32), np.float32)
    for r in (0, 1):
        for s in (0, 1):
            out[..., (r * 2 + s) * C:(r * 2 + s + 1) * C] = x[:, :, r::2, s::2].transpose(0, 2, 3, 1)
    return out


def s2d_ref(x):
    """lt_stem_s2d_fwd: the split-fp16 rows [N][H/2][W/2][64] of s2d_float."""
    return s32_rows(s2d_float(x))


def gather_ref(w, base, strides, k, cin, cin_p, cout, cout_p, S=1.0):
    """lt_conv_gather_weights_fwd as numpy indexing -> float32 [taps][cin_p][cout_p]: element (td, th, tw, ci, co) =
    w.flat[base + td s_td + th s_th + tw s_tw + ci s_ci + co s_co] x S for ci < cin and co < cout, else 0."""
    flat = np.asarray(w, np.float32).reshape(-1)
    s_td, s_th, s_tw, s_ci, s_co = strides
    ax = [np.arange(n).reshape([-1 if i == d else 1 for i in range(5)]) for d, n in enumerate((k[0], k[1], k[2], cin, cout))]
    idx = base + ax[0] * s_td + ax[1] * s_th + ax[2] * s_tw + ax[3] * s_ci + ax[4] * s_co
    out = np.zeros((k[0] * k[1] * k[2], cin_p, cout_p), np.float32)
    out[:, :cin, :cout] = (flat[idx] * np.float32(S)).reshape(-1, cin, cout)
    return out


def fold_ref(gamma, beta, mean, var, bias, eps, C, CP, S=1.0, steps=0):
    """lt_fold_bn_fwd in float64, each output rounded once to float32: sc = gamma / sqrt(var + float32(eps)), sh = beta - mean sc
    (+ bias sc), scale = sc / S x accum_gain(steps); mean None -> no BatchNorm (sc = 1, sh = bias); gamma / beta / bias None -> 1 / 0 / 0;
    channels C..CP-1 zero."""
    d = lambda v, dflt: np.full(C, dflt) if v is None else np.asarray(v, np.float32)[:C].astype(np.float64)
    if mean is not None:
        sc = d(gamma, 1.0) / np.sqrt(d(var, 0.0) + float(np.float32(eps)))
        sh = d(beta, 0.0) - d(mean, 0.0) * sc
        if bias is not None:
            sh = sh + d(bias, 0.0) * sc
    else:
        sc, sh = np.ones(C), d(bias, 0.0)
    scale, shift = np.zeros(CP, np.float32), np.zeros(CP, np.float32)
    scale[:C] = (sc * (1.0 / S) * accum_gain(steps)).astype(np.float32)
    shift[:C] = sh.astype(np.float32)
    return scale, shift


def coord_grid(position, center, step, n, transfer=False):
    """The float32 voxel vectors v = position + step x index - centre (one rounding per operation, as the kernel's __fmul_rn /
    __fadd_rn) -> (B, n, n, n, 3); transfer: out[a][b][c] = base[a][c][n-1-b] (CMU -> H36M)."""
    position, center, step = (np.asarray(t, np.float32).reshape(-1, 1, 1, 1, 3) for t in (position, center, step))
    idx = np.arange(n, dtype=np.float32)
    grid = np.stack(np.meshgrid(idx, idx, idx, indexing="ij"), -1)[None]
    v = (position + step * grid) - center
    if transfer:
        v = v.transpose(0, 1, 3, 2, 4)[:, :, ::-1]
    return np.ascontiguousarray(v)


def coord_ref(position, center, step, rot, n, transfer=False):
    """lt_coord_volume_fwd: (float32 out, float32 v, float64 R v + c) with R the float32 matrices (B, 9)."""
    v = coord_grid(position, center, step, n, transfer)
    R = np.asarray(rot, np.float32).astype(np.float64).reshape(-1, 1, 1, 1, 3, 3)
    c = np.asarray(center, np.float32).astype(np.float64).reshape(-1, 1, 1, 1, 3)
    out64 = (R @ v.astype(np.float64)[..., None])[..., 0] + c
    return out64.astype(np.float32), v, out64


def coord_bar(rot, v, out):
    """Per component: u (3 sum_k |R_ik v_k| + |out_i|), u = 2^-24 -- three roundings in the fused dot product, one in + c."""
    R = np.abs(np.asarray(rot, np.float32).astype(np.float64).reshape(-1, 1, 1, 1, 3, 3))
    return 2.0 ** -24 * (3 * (R @ np.abs(v.astype(np.float64))[..., None])[..., 0] + np.abs(out))


def same_bits(a, b):
    """Equal bit patterns, except that a NaN only has to meet a NaN (payloads may differ)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    it = {2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize]
    return bool(np.array_equal(na, nb) and np.array_equal(a.view(it)[~na], b.view(it)[~nb]))


# ------------------------------------------------------------------------------------------ references vs torch / the oracle
POOLS = {"stem 3x3 s2 p1": ((1, 3, 3), (1, 2, 2), (0, 1, 1)), "head 2x2 s2": ((1, 2, 2), (1, 2, 2), (0, 0, 0)),
         "v2v 2^3 s2": ((2, 2, 2), (2, 2, 2), (0, 0, 0))}


def pool_input(N, D, H, W, C, seed):
    """Random values with NaN, +-Inf and whole windows of negative values (so a padded window's maximum is negative)."""
    rng = np.random.RandomState(seed)
    x = rng.randn(N, D, H, W, C).astype(np.float32)
    flat = x.reshape(-1)
    pick = rng.randint(0, flat.size, size=max(4, flat.size // 50))
    q = len(pick) // 4
    flat[pick[:q]] = np.nan
    flat[pick[q:2 * q]] = np.inf
    flat[pick[2 * q:3 * q]] = -np.inf
    x[:, :, :2, :2] = -np.abs(x[:, :, :2, :2]) - 1.0       # the corner windows: every tap negative
    return x


@pytest.mark.parametrize("name", list(POOLS))
@pytest.mark.parametrize("shape", [(2, 6, 11, 12, 8), (1, 5, 7, 9, 4)])
def test_maxpool_reference_matches_torch(name, shape):
    k, s, p = POOLS[name]
    x = pool_input(*shape, seed=sum(shape))
    got = maxpool_ref(x, k, s, p)
    t = torch.from_numpy(x).permute(0, 4, 1, 2, 3)
    if k[0] == 1:
        N, D = shape[:2]
        t2 = t.permute(0, 2, 1, 3, 4).reshape(N * D, shape[4], shape[2], shape[3])
        want = F.max_pool2d(t2, k[1:], s[1:], p[1:]).reshape(N, D, shape[4], *got.shape[2:4]).permute(0, 1, 3, 4, 2)
    else:
        want = F.max_pool3d(t, k, s, p).permute(0, 2, 3, 4, 1)
    assert int(np.isnan(got).sum()) > 0
    assert same_bits(got, np.ascontiguousarray(want.numpy()))


def test_maxpool_rule_keeps_nan_where_fmax_drops_it():
    x = np.array([1.0, np.nan, 3.0, 2.0], np.float32).reshape(1, 1, 2, 2, 1)
    assert np.isnan(maxpool_ref(x, (1, 2, 2), (1, 2, 2), (0, 0, 0))).all()
    assert bool(F.max_pool2d(torch.tensor([[[[1.0, float("nan")], [3.0, 2.0]]]]), 2).isnan().all())


@pytest.mark.parametrize("C", [3, 1, 8])
def test_s2d_reference_is_the_inverse_of_the_stem_filter_rearrangement(C):
    """conv2d(x, w, stride 2, pad 3) == conv2d(pad(s2d(x), front 2, back 1), stem_s2d_filter(w)) in float64; the filter rearrangement
    is engine.stem_s2d_filter (3 channels), generalised to C channels with the same rule."""
    g = torch.Generator().manual_seed(C)
    x = torch.randn(2, C, 14, 10, generator=g)
    w = torch.randn(5, C, 7, 7, generator=g)
    if C == 3:
        wt = engine.stem_s2d_filter(w).double()                                  # [4][4][32][Cout]
    else:
        wt = torch.zeros(4, 4, 32, 5, dtype=torch.float64)
        for a in range(4):
            for b in range(4):
                for r in (0, 1):
                    for s in (0, 1):
                        ky, kx = 2 * a + r - 1, 2 * b + s - 1
                        if 0 <= ky < 7 and 0 <= kx < 7:
                            wt[a, b, (r * 2 + s) * C:(r * 2 + s + 1) * C] = w[:, :, ky, kx].t().double()
    s2d = torch.from_numpy(s2d_float(x.numpy())).double().permute(0, 3, 1, 2)
    got = F.conv2d(F.pad(s2d, (2, 1, 2, 1)), wt.permute(3, 2, 0, 1))
    want = F.conv2d(x.double(), w.double(), stride=2, padding=3)
    assert float((got - want).abs().max()) <= 1e-12 * float(want.abs().max())
    rows = s2d_ref(x.numpy())
    assert rows.shape == (2, 7, 5, 64) and rows.dtype == np.float16
    hi, lo = split_np(s2d_float(x.numpy()))
    assert same_bits(rows[..., :32], hi) and same_bits(rows[..., 32:], lo) and not rows[..., 4 * C:32].any()
    assert np.abs(join_np(hi, lo) - s2d_float(x.numpy())).max() <= 2.0 ** -25 + 2.0 ** -21 * np.abs(x.numpy()).max()


def _perm(t, *dims):
    return t.detach().permute(*dims).contiguous().numpy()


def test_gather_reference_matches_the_weight_permutations():
    g = torch.Generator().manual_seed(0)
    # Conv2d (Cout, Cin, KH, KW): the engine's source map; CinP > Cin, CoutP > Cout
    w = torch.randn(6, 5, 3, 3, generator=g)
    got = gather_ref(w.numpy(), 0, (9, 3, 1, 9, 45), (1, 3, 3), 5, 8, 6, 12)
    assert np.array_equal(got[:, :5, :6], _perm(w, 2, 3, 1, 0).reshape(9, 5, 6)) and not got[:, 5:].any() and not got[:, :, 6:].any()
    # Conv3d
    w = torch.randn(4, 3, 3, 3, 3, generator=g)
    got = gather_ref(w.numpy(), 0, (9, 3, 1, 27, 81), (3, 3, 3), 3, 3, 4, 4)
    assert np.array_equal(got, _perm(w, 2, 3, 4, 1, 0).reshape(27, 3, 4))
    # ConvTranspose2d k4 s2 p1 (Cin, Cout, 4, 4): phase (py, px) taps ky = 3 - py - 2 th, kx = 3 - px - 2 tw
    w = torch.randn(5, 6, 4, 4, generator=g)
    for py in (0, 1):
        for px in (0, 1):
            (base, strides), _ = engine.deconv2d_k4s2_phase(py, px, 6)
            want = w[:, :, [3 - py, 1 - py]][:, :, :, [3 - px, 1 - px]]
            assert np.array_equal(gather_ref(w.numpy(), base, strides, (1, 2, 2), 5, 5, 6, 6), _perm(want, 2, 3, 0, 1).reshape(4, 5, 6))
    # ConvTranspose3d k2 s2 (Cin, Cout, 2, 2, 2): the eight 1x1x1 phases, side by side in one row as the engine packs them
    w = torch.randn(5, 4, 2, 2, 2, generator=g)
    for a in (0, 1):
        for b in (0, 1):
            for c in (0, 1):
                got = gather_ref(w.numpy(), a * 4 + b * 2 + c, (0, 0, 0, 4 * 8, 8), (1, 1, 1), 5, 5, 4, 4)
                assert np.array_equal(got[0], w[:, :, a, b, c].numpy())
    # the data gradient's flipped filter (negated tap strides), Cin and Cout swapped
    w = torch.randn(6, 5, 3, 3, 3, generator=g)
    (base, strides), k, _, _, ci, co = A.conv3d_dgrad_filter(w.shape, (1, 1, 1))
    got = gather_ref(w.numpy(), base, strides, k, ci, ci, co, co)
    assert np.array_equal(got, _perm(w.flip(2, 3, 4), 2, 3, 4, 0, 1).reshape(27, 6, 5))
    w2 = torch.randn(6, 5, 3, 3, generator=g)
    (base, strides), k, _, _, ci, co = A.conv3d_dgrad_filter(w2.shape, (1, 1))
    assert np.array_equal(gather_ref(w2.numpy(), base, strides, k, ci, ci, co, co), _perm(w2.flip(2, 3), 2, 3, 0, 1).reshape(9, 6, 5))
    # the stride-2 data gradient's phases of the padded filter: tap u of phase 0 reads index 1 + 2u, of phase 1 index 2 - 2u
    srcs, k, _, groups, ci, co = A.conv_s2_dgrad_filter(w2.shape, (2, 2))
    wp = A.pad_s2_filter(w2, (2, 2))
    taps = {0: [1, 3], 1: [2, 0]}
    for gidx, (base, strides) in enumerate(srcs):
        a, b = divmod(gidx, 2)
        want = wp[:, :, taps[a]][:, :, :, taps[b]]
        assert np.array_equal(gather_ref(wp.numpy(), base, strides, (1,) + k[1:], ci, ci, co, co), _perm(want, 2, 3, 0, 1).reshape(4, 6, 5))


@pytest.mark.parametrize("amax, S", [(0.0, 1.0), (0.75, 2.0 ** 10), (1.0, 2.0 ** 9), (2.0 ** -140, 2.0 ** 126), (3.0e38, 2.0 ** -118),
                                     (1.7e38, 2.0 ** -117)])
def test_pow2_scale_and_its_clamp(amax, S):
    assert pow2_scale(np.float32(amax)) == S
    assert np.float32(S) * np.float32(1.0 / S) == 1.0


NULLS = [dict(), dict(gamma=None), dict(beta=None), dict(bias=None), dict(gamma=None, beta=None, bias=None),
         dict(mean=None), dict(mean=None, bias=None)]


@pytest.mark.parametrize("nulls", NULLS, ids=lambda d: "+".join(sorted(d)) or "all")
def test_fold_reference_matches_batchnorm(nulls):
    """acc x scale + shift (S = 1, no gain) == BatchNorm(acc + bias) of torch in float64 to float32 rounding of scale / shift."""
    g = torch.Generator().manual_seed(len(nulls))
    C, CP, eps = 40, 64, 1e-5
    p = dict(gamma=torch.rand(C, generator=g) + 0.5, beta=torch.randn(C, generator=g), mean=torch.randn(C, generator=g),
             var=torch.rand(C, generator=g) + 0.1, bias=torch.randn(C, generator=g))
    p.update(nulls)
    if p["mean"] is None:
        p["var"] = None
    scale, shift = fold_ref(*[None if p[k] is None else p[k].numpy() for k in ("gamma", "beta", "mean", "var", "bias")], eps, C, CP)
    assert not scale[C:].any() and not shift[C:].any()
    acc = torch.randn(7, C, generator=g, dtype=torch.float64)
    y = acc + (0 if p["bias"] is None else p["bias"].double())
    if p["mean"] is not None:
        f = lambda v: None if v is None else v.double()
        y = F.batch_norm(y, p["mean"].double(), p["var"].double(), f(p["gamma"]), f(p["beta"]), False, 0.0, float(np.float32(eps)))
    got = acc * torch.from_numpy(scale[:C]).double() + torch.from_numpy(shift[:C]).double()
    assert float((got - y).abs().max()) <= 4e-7 * float(y.abs().max())


def test_fold_reference_applies_scale_and_gain():
    s1, _ = fold_ref(None, None, None, None, None, 0.0, 4, 4)
    assert np.array_equal(s1, np.ones(4, np.float32))
    s, _ = fold_ref(None, None, None, None, None, 0.0, 4, 4, S=2.0 ** 10, steps=686)
    assert s[0] == np.float32(2.0 ** -10 * (1 + 0.28 * 686 * 2.0 ** -24))


def test_accum_gain_constant_is_the_one_in_common_cuh():
    src = open(os.path.join(ROOT, "learnable-triangulation-pytorch_b200", "csrc", "common.cuh")).read()
    m = re.search(r"constexpr double kAccumTruncRate = ([0-9.eE+-]+);", src)
    assert m and float(m.group(1)) == ACCUM_RATE
    assert "5.9604644775390625e-08" in src


@pytest.mark.parametrize("transfer", [False, True])
def test_coord_reference_equals_the_oracle_without_rotation(transfer):
    n = 9
    rng = np.random.RandomState(int(transfer))
    for _ in range(3):
        base = rng.randn(3) * 300 + [0, 0, 900]
        side = 2500.0
        want = O.coord_volume(base, side, n, 0.0, (0, 0, 1), transfer)
        got, _, _ = coord_ref(np.float32(base - side / 2), np.float32(base), np.float32([side / (n - 1)] * 3),
                              np.eye(3, dtype=np.float32).reshape(1, 9), n, transfer)
        assert same_bits(got[0], want)


def test_coord_reference_with_rotation_is_inside_its_bar_of_the_oracle():
    n, theta = 8, 1.1
    base = np.array([40.0, -70.0, 950.0])
    R = O.rotation_matrix((0, 0, 1), theta).astype(np.float32)
    got, v, out64 = coord_ref(np.float32(base - 1250.0), np.float32(base), np.float32([2500.0 / (n - 1)] * 3), R.reshape(1, 9), n)
    want = O.coord_volume(base, 2500.0, n, theta, (0, 0, 1))
    assert np.abs(got[0].astype(np.float64) - want).max() <= 2 * coord_bar(R.reshape(1, 9), v, out64).max()


# ------------------------------------------------------------------------------------------ argument checks at the C ABI
def test_misc_entry_points_reject_bad_arguments_before_touching_memory():
    buf = torch.zeros(64)
    p = buf.data_ptr()
    lib = capi.lib()
    F32, S32 = capi.FMT_F32, capi.FMT_S32

    def rejects(rc, text):
        assert rc != 0
        assert text.encode() in lib.lt_last_error_string(), lib.lt_last_error_string()

    rejects(lib.lt_maxpool_fwd(p, p, F32, 1, 1, 4, 4, 6, 1, 2, 2, 1, 2, 2, 0, 0, 0, 1, 2, 2, None), "C % 4 != 0")
    rejects(lib.lt_maxpool_fwd(p, p, S32, 1, 1, 4, 4, 16, 1, 2, 2, 1, 2, 2, 0, 0, 0, 1, 2, 2, None), "split-fp16 needs C % 32 == 0")
    rejects(lib.lt_maxpool_fwd(None, p, F32, 1, 1, 4, 4, 4, 1, 2, 2, 1, 2, 2, 0, 0, 0, 1, 2, 2, None), "maxpool: null pointer")
    rejects(lib.lt_f32_to_s32(p, p, 4, 48, None), "f32_to_s32: C % 32 != 0")
    rejects(lib.lt_s32_to_f32(p, p, 4, 16, None), "s32_to_f32: C % 32 != 0")
    rejects(lib.lt_stem_s2d_fwd(p, p, 1, 3, 7, 8, None), "need C <= 8 and even H, W")
    rejects(lib.lt_stem_s2d_fwd(p, p, 1, 3, 8, 9, None), "need C <= 8 and even H, W")
    rejects(lib.lt_stem_s2d_fwd(p, p, 1, 9, 8, 8, None), "need C <= 8 and even H, W")
    rejects(lib.lt_f32_to_s32_scaled(p, p, 4, 17, 48, None, None, None), "CP % 32 == 0")
    rejects(lib.lt_f32_to_s32_scaled(p, p, 4, 33, 32, None, None, None), "CP % 32 == 0")
    rejects(lib.lt_conv_gather_weights_fwd(p, 0, 9, 3, 1, 9, 45, 1, 3, 3, 5, 8, 6, 8, None, p, 16, 9, None),
            "column block [9, 17) exceeds the row length 16")
    rejects(lib.lt_conv_gather_weights_fwd(p, 0, 9, 3, 1, 9, 45, 1, 3, 3, 5, 4, 6, 8, None, p, 0, 0, None), "conv_gather_weights: bad arguments")
    rejects(lib.lt_fold_bn_fwd(p, p, p, p, None, 1e-5, 40, 32, None, 0, p, p, None), "fold_bn: bad arguments")
    rejects(lib.lt_fold_bn_fwd(p, p, p, None, None, 1e-5, 4, 4, None, 0, p, p, None), "fold_bn: bad arguments")
    rejects(lib.lt_fold_bn_fwd(None, None, None, None, None, 0.0, 4, 4, None, -1, p, p, None), "fold_bn: bad arguments")
    rejects(lib.lt_images_hwc_to_nchw_fwd(p, 0, None, p, 1, 5, 4, 4, None), "images_hwc_to_nchw: bad arguments")
    rejects(lib.lt_images_hwc_to_nchw_fwd(p, 1, p, p, 1, 3, 4, 4, None), "the table applies to uint8 input only")
    rejects(lib.lt_images_hwc_to_nchw_fwd(p, 2, p, p, 1, 3, 4, 4, None), "the table applies to uint8 input only")
    rejects(lib.lt_images_hwc_to_nchw_fwd(p, 3, None, p, 1, 3, 4, 4, None), "unknown input dtype 3")
    rejects(lib.lt_cl_to_cf_f32(p, p, 65536, 4, 4, 4, None), "cl_to_cf: bad arguments")
    rejects(lib.lt_cl_to_cf_f32(p, p, 1, 4, 4, 5, None), "cl_to_cf: bad arguments")
    rejects(lib.lt_nchw_to_nhwc_f32(p, p, 1, 4, 2, 2, 3, None), "nchw_to_nhwc: bad arguments")
    rejects(lib.lt_coord_volume_fwd(p, p, p, p, p, 1, 1, 0, None), "coord_volume: bad size B=1 n=1")
    rejects(lib.lt_coord_volume_fwd(p, p, p, None, p, 1, 4, 0, None), "coord_volume: null pointer")
    rejects(lib.lt_absmax_fwd(p, 0, p, None), "absmax: bad arguments")
