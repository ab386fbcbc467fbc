"""Every soft-argmax kernel against float64 `torch_ops` (pinned to the reference by tests/test_oracle_vs_reference.py): each branch
lt_softargmax3d_fwd dispatches to (classic channels-last, generic strides, streaming), the fused V2V tail's statistics with
lt_softargmax3d_finish_fwd, the backward, and the two models at joint counts other than 17.

Scenes and references come from tests/test_softargmax_cpu.py.  Bars: BAR = 2e-6 of scale (max |ref|, its spread), with the yardstick
rule: the native error against float64 must not exceed max(BAR, 2 x the error of float32 torch against float64).  Key points are
measured against the scale of the reference key points.

Logits sit inside a NaN-filled allocation with one sample of guard on either side; outputs start as a NaN sentinel with guards on
either side, and the workspace is refilled with the sentinel before every call, so a read outside the logits, a partial the merge
reads but the call did not write, a missing write or a stray write each fails the test.  Every forward runs twice (bit-identical) and
once without volumes (bit-identical key points), under torch.cuda.set_sync_debug_mode("error").

Measured on an H100 80GB HBM3 (700 W power limit), largest native error / its float32 yardstick against float64 (key points; volumes):
- classic channels-last: mode 0 5.9e-7 / 6.8e-6; 5.9e-8 / 5.9e-8.  mode 1 1.0e-6 / 4.6e-6; 2.7e-6 / 2.9e-7 (SOFTMAX_VOL_BAR).
  mode 2 1.2e-6 / 7.0e-6; 5.9e-8 / 5.9e-8;
- generic strides: mode 0 1.1e-7 / 1.1e-5; 6.8e-8.  mode 1 2.2e-7 / 6.3e-6; 1.7e-7 / 1.7e-7.  mode 2 3.2e-7 / 1.1e-5; 6.8e-8;
- streaming: mode 0 1.2e-7 / 5.7e-5; 6.1e-8.  mode 1 3.2e-7 / 3.3e-5; 7.1e-7 / 2.2e-7;
- fused tail + finish: mode 0 1.0e-7 / 4.9e-6; 6.9e-8.  mode 1 1.9e-7 / 3.0e-6; 4.1e-7 / 3.0e-7;
- softmax offsets -1024 ... +1024: classic 6.7e-7; 1.0e-6, generic 2.1e-7; 1.8e-7, streaming 2.7e-7; 3.0e-7, tail 1.8e-7; 2.1e-7.
  Before the streaming kernels formed l - max ahead of the scaling by log2(e), the streaming volumes reached 9e-6 - 3.6e-5 and the
  tail's 2.7e-5 at |offset| = 1024, and the 128^2 x 100 heat-map case 2.5e-6 (now 1.6e-7);
- backward: mode 0 1.1e-7 / 9.9e-8, mode 1 1.3e-6 / 2.1e-6, mode 2 2.1e-7 / 1.5e-7 (one voxel: the exact gradient is 0, and both
  float32 paths leave rounding noise of ~1e-8 x |d key point| |x|); recipe 64^3 x B 5 x J 17: 1.6e-7 / 1.4e-7, 1.2e-6 / 1.1e-6,
  1.2e-7 / 1.5e-6;
- models: volumetric J 16 / 17 / 20 / 21 key points 0.04 / 0.09 / 0.13 / 0.20 mm, volumes 8.8e-5 / 8.7e-5 / 1.2e-4 / 1.6e-4; algebraic
  ReLU heat-maps 2.0e-5, 2-D key points 2e-4 px, 3-D 3e-3 mm.
"""
import contextlib
import json
import os
import re
import subprocess
import sys
from collections import namedtuple

import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import capi, testing
from oracle import vol_oracle as O
from test_gpu_ops import _bn_for, _engine, act_from_nchw
from test_gpu_unproject import Guarded
from test_softargmax_cpu import (KINDS, OFFSETS, channels_last, coords_for, err, grad_floor, make_logits, pixel_grid, reference,
                                 reference_grad, upstream)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BAR = 2e-6
# Softmax volumes: the online softmax rescales running sums by exp(m_old - m_new) through ex2.approx, whose argument rounding costs
# about |m_old - m_new| x 2^-24 of relative error per rescale.  The classic kernels' volumes reach 2.7e-6 of scale on one scene (27^3
# voxels, logit spread ~20, 10 chunk partials) where float32 torch, which subtracts one final max, stays at 3e-7.
SOFTMAX_VOL_BAR = 4e-6


@contextlib.contextmanager
def no_sync():
    torch.cuda.set_sync_debug_mode("error")
    try:
        yield
    finally:
        torch.cuda.set_sync_debug_mode("default")


def check(label, got, ref, yard_ref, bar=BAR, floor=1e-30):
    e, y = err(got, ref, floor), err(yard_ref, ref, floor)
    print("%-48s native %.1e  yardstick %.1e" % (label, e, y))
    assert e <= max(bar, 2 * y), (label, e, y)
    return e, y


def bits(t):
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------ forward: the dispatch table
Case = namedtuple("Case", "branch B J nvox vs modes mult grid")   # vs None: NCDHW; grid None: coordinate volume, else (h, w) pixels
M012, M01 = (0, 1, 2), (0, 1)
FWD_CASES = {
    # classic channels-last (chan_stride 1, J <= 32, voxel stride >= J; not streamed)
    "cl J1 vs1 n1": Case("classic", 2, 1, 1, 1, M012, 1.7, None),
    "cl J5 vs5 n7": Case("classic", 3, 5, 7, 5, M012, 1.0, None),
    "cl J1 vs16 n2048": Case("classic", 2, 1, 2048, 16, M012, 1.3, None),
    "cl J5 vs16 n2047": Case("classic", 2, 5, 2047, 16, M012, 1.7, None),
    "cl J17 vs20 n2048": Case("classic", 2, 17, 2048, 20, M012, 1.0, None),
    "cl J17 vs32 n2049": Case("classic", 3, 17, 2049, 32, M012, 1.7, None),
    "cl J32 vs32 n8000": Case("classic", 2, 32, 8000, 32, M012, 1.3, None),
    "cl J17 vs36 n8000": Case("classic", 2, 17, 8000, 36, M012, 1.0, None),
    "cl J17 vs20 27^3 (odd)": Case("classic", 2, 17, 27 ** 3, 20, M012, 1.7, None),
    "cl J16 vs16 64^3": Case("classic", 2, 16, 64 ** 3, 16, M012, 1.0, None),
    "cl 2-D J17 vs32 64x64 x100": Case("classic", 3, 17, 64 * 64, 32, (2,), 100.0, (64, 64)),
    "cl 2-D J17 vs32 128x128 x100": Case("classic", 2, 17, 128 * 128, 32, (2,), 100.0, (128, 128)),
    # generic strides: NCDHW (op.py, autograd_ops.py) and channels-last with J > 32
    "ncdhw J1 n7": Case("generic", 2, 1, 7, None, M012, 1.0, None),
    "ncdhw J17 n2049": Case("generic", 2, 17, 2049, None, M012, 1.7, None),
    "ncdhw J5 20^3": Case("generic", 3, 5, 8000, None, M012, 1.3, None),
    "cl J40 vs40 n3000": Case("generic", 2, 40, 3000, 40, M012, 1.0, None),
    # streaming: vs % 4 == 0, 20 <= vs <= 32, J <= vs, nvox % 8 == 0, nvox >= 16384; tile heights T = 200 / 168 / 144 / 128
    "st vs20 J17 n16384 B1 (82 tiles)": Case("stream", 1, 17, 16384, 20, M01, 1.7, None),
    "st vs20 J20 n16384 B3 (identity partials)": Case("stream", 3, 20, 16384, 20, M01, 1.0, None),
    "st vs24 J21 n16384 B2": Case("stream", 2, 21, 16384, 24, M01, 1.3, None),
    "st vs24 J24 n16392 B5": Case("stream", 5, 24, 16392, 24, M01, 1.0, None),
    "st vs28 J25 n16384 B2": Case("stream", 2, 25, 16384, 28, M01, 1.7, None),
    "st vs28 J28 n20000 B3": Case("stream", 3, 28, 20000, 28, M01, 1.0, None),
    "st vs32 J32 n16392 B2": Case("stream", 2, 32, 16392, 32, M01, 1.3, None),
    "st vs32 J17 n16384 B5": Case("stream", 5, 17, 16384, 32, M01, 1.0, None),
    "st vs20 J17 64^3 B5": Case("stream", 5, 17, 64 ** 3, 20, M01, 1.0, None),
    "st 2-D J17 vs32 128x128 x100": Case("stream", 2, 17, 128 * 128, 32, (1,), 100.0, (128, 128)),
}
FWD_PARAMS = [(name, mode) for name, c in FWD_CASES.items() for mode in c.modes]


def expected_kernels(branch, mode, volumes):
    if branch == "stream":
        t = "true" if mode == 1 else "false"
        return ["stream_stats_kernel<%s>" % t, "softargmax_stream_merge"] + (["stream_normalize_kernel<%s>" % t] if volumes else [])
    k = "cl" if branch == "classic" else "generic"
    return ["softargmax_partial_" + k, "softargmax_finalize"] + (["softargmax_normalize_" + k] if volumes else [])


ALL_KERNELS = ["softargmax_partial_cl", "softargmax_partial_generic", "softargmax_finalize", "softargmax_normalize_cl",
               "softargmax_normalize_generic", "stream_stats_kernel<true>", "stream_stats_kernel<false>", "softargmax_stream_merge",
               "stream_normalize_kernel<true>", "stream_normalize_kernel<false>", "v2v_tail_kernel<1>", "v2v_tail_kernel<2>",
               "softargmax_bwd_dot_kernel", "softargmax_bwd_apply_kernel"]


def case_scene(name, offset=0.0, kind=None):
    """(logits (B, J, nvox) float32, coordinates (B, nvox, 3) float32)."""
    c = FWD_CASES[name]
    seed = sum(map(ord, name)) % 1000
    kind = kind or KINDS[seed % 3]
    coord = pixel_grid(c.B, *c.grid) if c.grid else coords_for(c.B, c.nvox, seed)
    return make_logits(c.B, c.J, c.nvox, kind, seed, offset=offset), coord


def device_logits(x, vs):
    """Guarded device logits: channels-last (B, nvox, vs) with NaN padding, or NCDHW (vs None); with the call's strides."""
    B, J, nvox = x.shape
    host = channels_last(x, vs) if vs else x
    L = Guarded(host.shape, guard=int(np.prod(host.shape[1:])) + 3 & ~3, fill=torch.from_numpy(host))
    strides = (nvox * vs, vs, 1) if vs else (J * nvox, 1, nvox)
    return L, strides


def native_forward(L, strides, coord, B, J, nvox, mult, mode, volumes=True):
    """lt_softargmax3d_fwd on guarded buffers -> (key points, volumes or None)."""
    ws = Guarded((capi.softargmax3d_workspace_bytes(B, J, nvox) // 4 + 1,))
    kp = Guarded((B, J, 3))
    vol = Guarded((B, J, nvox)) if volumes else None
    with no_sync():
        capi.softargmax3d(L.t, *strides, coord, None if vol is None else vol.t, kp.t, ws.t, B, J, nvox, mult, mode)
    torch.cuda.synchronize()
    assert L.guards_intact() and ws.guards_intact() and kp.guards_intact() and kp.unwritten() == 0
    if vol is not None:
        assert vol.guards_intact() and vol.unwritten() == 0
    return kp.t, (None if vol is None else vol.t)


def forward_checked(label, x, coord, vs, mult, mode):
    """Native forward twice with volumes and once without, against float64; returns (kp, volumes)."""
    B, J, nvox = x.shape
    L, strides = device_logits(x, vs)
    c = torch.from_numpy(coord).to(DEV)
    kp, vol = native_forward(L, strides, c, B, J, nvox, mult, mode)
    kp2, vol2 = native_forward(L, strides, c, B, J, nvox, mult, mode)
    kp3, _ = native_forward(L, strides, c, B, J, nvox, mult, mode, volumes=False)
    assert torch.equal(bits(kp), bits(kp2)) and torch.equal(bits(vol), bits(vol2)) and torch.equal(bits(kp), bits(kp3)), label
    assert bool(torch.isfinite(kp).all()) and bool(torch.isfinite(vol).all()), label
    ref_kp, ref_vol = reference(x, coord, mult, mode, device=DEV)
    y_kp, y_vol = reference(x, coord, mult, mode, torch.float32, DEV)
    ek = check(label + " key points", kp, ref_kp, y_kp)
    ev = check(label + " volumes", vol, ref_vol, y_vol, SOFTMAX_VOL_BAR if mode == 1 else BAR)
    return ek, ev


@pytest.mark.parametrize("name,mode", FWD_PARAMS, ids=["%s-mode%d" % p for p in FWD_PARAMS])
def test_forward_vs_float64(name, mode):
    c = FWD_CASES[name]
    x, coord = case_scene(name)
    forward_checked("%s mode %d" % (name, mode), x, coord, c.vs, c.mult, mode)


OFFSET_CASES = ["cl J17 vs32 n2049", "ncdhw J17 n2049", "st vs20 J20 n16384 B3 (identity partials)", "st vs32 J32 n16392 B2",
                "st vs28 J25 n16384 B2"]


@pytest.mark.parametrize("name", OFFSET_CASES)
@pytest.mark.parametrize("kind", KINDS)
def test_softmax_offsets_vs_float64(name, kind):
    """Softmax is shift-invariant and the scenes are exact in float32 at every offset, so one float64 answer holds for all offsets."""
    c = FWD_CASES[name]
    for off in OFFSETS:
        x, coord = case_scene(name, offset=off, kind=kind)
        forward_checked("%s %s offset %+g" % (name, kind, off), x, coord, c.vs, 1.0, 1)


def test_zero_mass_joint_gives_nan_key_point():
    """Mode 2 with one joint of no ReLU mass: that joint's key point is NaN (0 / 0, as in the reference), the others are unaffected."""
    for vs in (20, None):
        x = make_logits(2, 3, 3000, "diffuse", 4, zero_mass_joint=1)
        coord = coords_for(2, 3000, 4)
        L, strides = device_logits(x, vs)
        kp, vol = native_forward(L, strides, torch.from_numpy(coord).to(DEV), 2, 3, 3000, 1.0, 2)
        ref_kp, ref_vol = reference(x, coord, 1.0, 2, device=DEV)
        assert bool(torch.isnan(kp[:, 1]).all()) and bool(torch.isfinite(kp[:, [0, 2]]).all())
        assert err(kp[:, [0, 2]], ref_kp[:, [0, 2]]) <= BAR and err(vol, ref_vol) <= BAR


def _kernel_names(prof):
    pat = re.compile(r"(softargmax_\w+|stream_\w+_kernel|v2v_tail_kernel)(<[^>]*>)?")
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    names = []
    for e in sorted(evs, key=lambda e: e.start_ns()):
        m = pat.search(e.name())
        if m:
            names.append(m.group(0))
    return names


# ------------------------------------------------------------------------------------------ fused V2V tail + finish
def tail_inputs(J, N, spatial, offset=0.0, seed=5):
    """Split-fp16 input rows and packed back1 / back2 / output layers; the output bias carries `offset`."""
    torch.manual_seed(seed)
    c1, c2, c3 = torch.nn.Conv3d(32, 32, 1).eval(), torch.nn.Conv3d(32, 32, 1).eval(), torch.nn.Conv3d(32, J, 1).eval()
    with torch.no_grad():
        c3.weight.mul_(6.0)      # logit spread of a few units: peaked softmax
        c3.bias.add_(offset)
    bn1, bn2 = _bn_for(c1, 5), _bn_for(c2, 6)
    e = _engine("tc")
    b1, b2 = e._pack_conv(c1.to(DEV), bn1.to(DEV)), e._pack_conv(c2.to(DEV), bn2.to(DEV))
    b3 = e._pack_conv(c3.to(DEV), None, out_fmt=capi.FMT_F32)
    xa = act_from_nchw(torch.randn(N, 32, *spatial), capi.FMT_S32)
    return (xa.data, b1.w, b2.w, b3.w, b1.scale, b1.shift, b2.scale, b2.shift, b3.scale, b3.shift)


def native_tail(args, N, J, FC, nvox, coord, mult, mode):
    """lt_v2v_tail_stats_fwd + lt_softargmax3d_finish_fwd on guarded buffers -> (logits (N, J, nvox), key points, volumes)."""
    ws = Guarded((capi.softargmax3d_workspace_bytes(N, J, nvox) // 4 + 1,))
    lg = Guarded((N * nvox, FC))
    kp, vol = Guarded((N, J, 3)), Guarded((N, J, nvox))
    with no_sync():
        G = capi.v2v_tail_stats(*args, lg.t, N, nvox, FC, coord, J, mult, mode, ws.t)
        capi.softargmax3d_finish(lg.t, nvox * FC, FC, coord, vol.t, kp.t, ws.t, N, J, nvox, G, mult, mode)
    torch.cuda.synchronize()
    for g in (ws, lg, kp, vol):
        assert g.guards_intact()
    assert lg.unwritten() == kp.unwritten() == vol.unwritten() == 0
    return lg.t.view(N, nvox, FC)[:, :, :J].permute(0, 2, 1), kp.t, vol.t


@pytest.mark.parametrize("J", [17, 20])
@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("spatial,N", [((32, 32, 16), 3), ((64, 64, 32), 2)])
def test_fused_tail_statistics_vs_float64(J, mode, spatial, N):
    """The float64 input is the tail's own logits, so this checks the statistics and the finish, not the convolutions."""
    nvox, mult = int(np.prod(spatial)), 1.7
    args = tail_inputs(J, N, spatial)
    coord = torch.from_numpy(coords_for(N, nvox, J)).to(DEV)
    lg, kp, vol = native_tail(args, N, J, 20, nvox, coord, mult, mode)
    lg2, kp2, vol2 = native_tail(args, N, J, 20, nvox, coord, mult, mode)
    assert torch.equal(bits(lg), bits(lg2)) and torch.equal(bits(kp), bits(kp2)) and torch.equal(bits(vol), bits(vol2))
    x = lg.contiguous()
    ref_kp, ref_vol = reference(x, coord, mult, mode, device=DEV)
    y_kp, y_vol = reference(x, coord, mult, mode, torch.float32, DEV)
    label = "tail J%d mode %d %s N%d" % (J, mode, spatial, N)
    check(label + " key points", kp, ref_kp, y_kp)
    check(label + " volumes", vol, ref_vol, y_vol, SOFTMAX_VOL_BAR if mode == 1 else BAR)


@pytest.mark.parametrize("offset", OFFSETS)
def test_fused_tail_softmax_offsets_vs_float64(offset):
    N, J, spatial = 3, 17, (32, 32, 16)
    nvox = int(np.prod(spatial))
    coord = torch.from_numpy(coords_for(N, nvox, 3)).to(DEV)
    lg, kp, vol = native_tail(tail_inputs(J, N, spatial, offset=offset), N, J, 20, nvox, coord, 1.0, 1)
    x = lg.contiguous()
    ref_kp, ref_vol = reference(x, coord, 1.0, 1, device=DEV)
    y_kp, y_vol = reference(x, coord, 1.0, 1, torch.float32, DEV)
    check("tail offset %+g key points" % offset, kp, ref_kp, y_kp)
    check("tail offset %+g volumes" % offset, vol, ref_vol, y_vol, SOFTMAX_VOL_BAR)


def test_fused_tail_refuses_a_width_the_finish_cannot_stream():
    """J <= 16 packs the logits 16 (or fewer) floats wide, which the streaming finish does not read: the statistics variant refuses
    such a width, so no partials are produced that nothing can merge."""
    N, J, nvox = 1, 16, 32 * 32 * 16
    args = tail_inputs(J, N, (32, 32, 16))
    coord = torch.from_numpy(coords_for(N, nvox, 1)).to(DEV)
    ws = torch.empty(capi.softargmax3d_workspace_bytes(N, J, nvox) // 4 + 1, device=DEV)
    lg = torch.empty((N * nvox, 16), device=DEV)
    with pytest.raises(RuntimeError, match="v2v_tail_stats"):
        capi.v2v_tail_stats(*args, lg, N, nvox, 16, coord, J, 1.0, 1, ws)


# ------------------------------------------------------------------------------------------ backward
def native_backward(probs, coord, g_kp, g_vol, mult, mode):
    """lt_softargmax3d_bwd on guarded d logits and scratch; asserts every d logit written, only the mode's scratch written."""
    B, J, nvox = probs.shape
    GL = Guarded((B, J, nvox))
    S = Guarded((2 * B * J + 64,))
    with no_sync():
        capi.softargmax3d_bwd(probs, coord, g_kp, g_vol, GL.t, S.t, B, J, nvox, mult, mode)
    torch.cuda.synchronize()
    assert GL.guards_intact() and GL.unwritten() == 0 and S.guards_intact()
    used = {0: 0, 1: B * J, 2: 2 * B * J}[mode]
    sv = S.t.view(S.itype)
    assert bool((sv[:used] != S.bits).all()) and bool((sv[used:] == S.bits).all()), mode
    return GL.t


def backward_checked(label, x, coord, mult, mode, with_gvol, seed=3):
    B, J, nvox = x.shape
    g_kp, g_vol = upstream(B, J, nvox, seed, 1.0 if mode == 0 else float(np.abs(coord).max()) / nvox)
    g_vol = g_vol if with_gvol else None
    want, vol = reference_grad(x, coord, mult, mode, g_kp, g_vol, device=DEV)
    yard, _ = reference_grad(x, coord, mult, mode, g_kp, g_vol, torch.float32, DEV)
    t = lambda a: None if a is None else torch.from_numpy(a).to(DEV)
    got = native_backward(vol.float().contiguous(), t(coord), t(g_kp), t(g_vol), mult, mode)
    got2 = native_backward(vol.float().contiguous(), t(coord), t(g_kp), t(g_vol), mult, mode)
    assert torch.equal(bits(got), bits(got2))
    return check(label, got, want, yard, floor=1e-6 * grad_floor(g_kp, coord, mult))


@pytest.mark.parametrize("nvox", [1, 511, 512, 513])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("with_gvol", [True, False])
def test_backward_vs_float64(nvox, mode, with_gvol):
    B, J = 2, 3
    x = make_logits(B, J, nvox, "peaked", nvox)
    coord = coords_for(B, nvox, nvox)
    backward_checked("bwd n%d mode %d gvol %d" % (nvox, mode, with_gvol), x, coord, 1.7, mode, with_gvol)


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_backward_recipe_shape_vs_float64(mode):
    """64^3 voxels, B 5, J 17: the volumetric training step's soft-argmax."""
    B, J, nvox = 5, 17, 64 ** 3
    x = make_logits(B, J, nvox, "peaked", 17)
    backward_checked("bwd recipe mode %d" % mode, x, coords_for(B, nvox, 17), 1.7, mode, True)


def test_backward_size_limit():
    """One CTA row per (sample, joint): B * J = 65535 is accepted (and correct), 65536 refused."""
    x = make_logits(65535, 1, 3, "diffuse", 1)
    backward_checked("bwd B*J 65535", x, coords_for(65535, 3, 1), 1.0, 1, True)
    p = torch.full((4096, 16, 2), 0.5, device=DEV)
    with pytest.raises(RuntimeError, match="bad sizes"):
        capi.softargmax3d_bwd(p, torch.zeros(4096, 2, 3, device=DEV), torch.zeros(4096, 16, 3, device=DEV), None, torch.empty_like(p),
                              torch.empty(2 * 65536, device=DEV), 4096, 16, 2, 1.0, 1)


# ------------------------------------------------------------------------------------------ launches
def profiled_launches():
    """Every forward case (with and without volumes), the fused tail + finish in both modes and the backward of modes 1 and 0 under
    the CUDA profiler -> (names of the soft-argmax kernels launched, in order; the names expected)."""
    from torch.profiler import ProfilerActivity, profile
    runs, expected = [], []
    for name, c in FWD_CASES.items():
        x, coord = case_scene(name)
        L, strides = device_logits(x, c.vs)
        co = torch.from_numpy(coord).to(DEV)
        ws = torch.empty(capi.softargmax3d_workspace_bytes(c.B, c.J, c.nvox) // 4 + 1, device=DEV)
        kp = torch.empty((c.B, c.J, 3), device=DEV)
        vol = torch.empty((c.B, c.J, c.nvox), device=DEV)
        for mode in c.modes:
            for v in (vol, None):
                runs.append((L.t, *strides, co, v, kp, ws, c.B, c.J, c.nvox, c.mult, mode))
                expected += expected_kernels(c.branch, mode, v is not None)
    N, J, spatial = 2, 17, (32, 32, 16)
    nvox = int(np.prod(spatial))
    args = tail_inputs(J, N, spatial)
    coord = torch.from_numpy(coords_for(N, nvox, 2)).to(DEV)
    lg = torch.empty((N * nvox, 20), device=DEV)
    ws = torch.empty(capi.softargmax3d_workspace_bytes(N, J, nvox) // 4 + 1, device=DEV)
    kp, vol = torch.empty((N, J, 3), device=DEV), torch.empty((N, J, nvox), device=DEV)
    g = torch.randn((N, J, 3), device=DEV)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for r in runs:
            capi.softargmax3d(*r)
        for mode in (1, 0):
            G = capi.v2v_tail_stats(*args, lg, N, nvox, 20, coord, J, 1.0, mode, ws)
            capi.softargmax3d_finish(lg, nvox * 20, 20, coord, vol, kp, ws, N, J, nvox, G, 1.0, mode)
            expected += ["v2v_tail_kernel<%d>" % (1 if mode else 2), "softargmax_stream_merge",
                         "stream_normalize_kernel<%s>" % ("true" if mode else "false")]
        for mode in (1, 0):
            capi.softargmax3d_bwd(vol, coord, g, None, torch.empty_like(vol), ws, N, J, nvox, 1.0, mode)
            expected += (["softargmax_bwd_dot_kernel"] if mode else []) + ["softargmax_bwd_apply_kernel"]
        torch.cuda.synchronize()
    return _kernel_names(prof), expected


def test_dispatch_reaches_every_instantiation():
    """Each forward case launches the kernels of its branch (with and without volumes); with the fused tail in both modes and one
    backward of modes 1 and 0 the launches cover all 14 soft-argmax instantiations.  The profiling runs in a child process: after one
    profiler session, a later session in the same process misses its first few kernel records, and
    tests/test_gpu_unproject.py profiles too."""
    code = ("import json, sys; sys.path[:0] = %r; import test_gpu_softargmax as t; print('LAUNCHES ' + json.dumps(t.profiled_launches()))"
            % [HERE, ROOT])
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    names, expected = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("LAUNCHES ")][-1][len("LAUNCHES "):])
    assert len(names) == len(expected), (len(names), len(expected))
    for i, (got, want) in enumerate(zip(names, expected)):
        assert got == want, (i, got, want)
    print("instantiations launched: %s" % sorted(set(names)))
    assert len(set(ALL_KERNELS)) == len(ALL_KERNELS) == 14 and set(names) == set(ALL_KERNELS), sorted(set(ALL_KERNELS) ^ set(names))


# ------------------------------------------------------------------------------------------ models
CUBOID_MM = 2500.0


@pytest.mark.parametrize("num_joints", [16, 17, 20, 21])
def test_volumetric_model_joint_counts_vs_oracle(num_joints):
    """Native tensor-core model at 32^3: J 17..20 run the fused tail + streaming finish, J 16 and 21 the unfused tail + the classic
    soft-argmax.  DESIGN section 2 contract."""
    B, V, S, n = 1, 2, 128, 32
    cfg = testing.make_config(num_layers=50, volume_size=n, num_joints=num_joints)
    holder = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend="torch")
    testing.randomize_weights(holder, seed=1, calib_size=S)
    sd = holder.state_dict()
    images, batch = testing.make_batch(B, V, image_size=S, seed=3)
    base = np.stack([k[6, :3] for k in batch["keypoints_3d"]])
    kp_o, _, vols_o, _ = O.volumetric_forward(sd, images, batch["cameras"], base, volume_size=n)
    model = lt_b200.VolumetricTriangulationNet(testing.make_config(num_layers=50, volume_size=n, num_joints=num_joints), device="cpu",
                                               backend="native", conv_mode="tc", use_cuda_graph=False)
    model.load_state_dict(sd)
    model = model.to(DEV).eval()
    with torch.no_grad():
        kp, _, vols, _, _, _, _ = model(images.to(DEV), None, batch)
    torch.cuda.synchronize()
    e_kp = float((kp.cpu() - kp_o).abs().max())
    e_v = float((vols.cpu() - vols_o).abs().max()) / max(float(vols_o.abs().max()), float(vols_o.std()))
    print("volumetric J %d: key points %.4f mm, volumes %.1e" % (num_joints, e_kp, e_v))
    assert e_kp < 1e-3 * CUBOID_MM and e_v < 1e-3
    assert torch.equal(vols.cpu().reshape(B, num_joints, -1).argmax(-1), vols_o.reshape(B, num_joints, -1).argmax(-1))


def test_algebraic_model_relu_heatmaps_vs_torch():
    """heatmap_softmax: false (ReLU heat-maps x 100, mass-normalised key points: mode 2 of the classic kernels) against the torch
    backend on the same weights, run on the CPU (cuDNN's default TF32 convolutions would dominate the comparison).  DESIGN section 2
    contract."""
    B, V, S = 2, 3, 128
    cfg = testing.make_alg_config(num_layers=50)
    cfg.model.heatmap_softmax = False
    holder = lt_b200.AlgebraicTriangulationNet(cfg, device="cpu", backend="torch")
    testing.randomize_backbone_weights(holder, seed=5, calib_size=S)
    holder.eval()
    images, batch = testing.make_batch(B, V, image_size=S, seed=9)
    proj = torch.from_numpy(testing.image_projections(batch))
    with torch.no_grad():
        kp3_t, kp2_t, heat_t, _ = holder(images, proj, batch)
    model = lt_b200.AlgebraicTriangulationNet(cfg, device=DEV, backend="native", conv_mode="tc")
    model.load_state_dict(holder.state_dict(), strict=True)
    model = model.to(DEV).eval()
    with torch.no_grad():
        kp3, kp2, heat, _ = (t.cpu() for t in model(images.to(DEV), proj.to(DEV), batch))
    assert bool(torch.isfinite(kp3).all()) and bool(torch.isfinite(kp2).all())
    e_heat = float((heat - heat_t).abs().max()) / max(float(heat_t.abs().max()), float(heat_t.std()))
    e2, e3 = float((kp2 - kp2_t).abs().max()), float((kp3 - kp3_t).abs().max())
    print("algebraic ReLU heat-maps: heat %.1e, 2-D %.4f px, 3-D %.4f mm" % (e_heat, e2, e3))
    assert e_heat < 1e-3 and e2 < 0.02 and e3 < 1e-3 * CUBOID_MM
    assert torch.equal(heat.reshape(B, V, 17, -1).argmax(-1), heat_t.reshape(B, V, 17, -1).argmax(-1))
