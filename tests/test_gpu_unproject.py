"""Every unprojection kernel against float64 `torch_ops` (pinned to the reference by tests/test_oracle_vs_reference.py): each
instantiation `launch_unproject` dispatches to, the view-sharded exchange kernels run on one GPU with ordinary local buffers standing
in for the peers' memory, and the backward.

Scenes come from tests/test_unproject_cpu.py.  On exact-geometry scenes every tap position is exact in float32, so the forward is held
to BAR = 2e-6 of scale (max |ref|, its spread): what remains is at most four fused products per tap, the sums over views and the exp /
reciprocal units.  Split-fp16 output adds the round-trip bound of test_split_fp16_round_trip_precision.  Camera scenes (positions not
exact) and the backward (float atomics reorder its sums) use the yardstick rule: the native error against float64 must not exceed
max(bar, 2 x the error of float32 torch_ops against float64).

Features sit inside a NaN-filled allocation with one map of guard on either side, so a read outside the tensor shows up as NaN;
outputs, partials and push slots start as a NaN sentinel with guards on either side, so a missing write leaves the sentinel and a
stray write changes a guard.  The options that select kernel variants are process-wide: each test that sets them restores them.

Measured on an H100 80GB HBM3 (700 W power limit), largest error over all cases:
- exact-geometry forward: 3.4e-7 in F32 and in split-fp16 (bar 2e-6); partials 3.0e-7; split views + finalize 2.5e-7; softmax
  scores of |s| ~ 60 through the partials 1.5e-7;
- camera-scene forward: at most 0.64 of its yardstick bound (largest native error 2.7e-5, on a 96 x 96 max aggregation);
- exact-geometry backward: 5.6e-7 (bar 2e-6, all cases below the bar itself); V 80 x C 128 with d conf 1.3e-7;
- recipe-shape backward: d features 9.9e-6 (softmax) and 9.5e-6 (conf) against float32 yardsticks of 1.4e-5 and 1.1e-5, d conf
  6.9e-6 against 7.8e-6.
"""
import contextlib
import re
from collections import namedtuple

import numpy as np
import pytest
import torch

from lt_b200 import capi, op
from test_unproject_cpu import (AGGS, camera_scene, err, exact_scene, max_near_ties, reference, reference_grads, reference_partial,
                                scale_of, tensors)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BAR = 2e-6
F32, S32 = capi.FMT_F32, capi.FMT_S32
SENTINEL = {torch.float32: (torch.int32, 0x7FC5A5A5), torch.float16: (torch.int16, 0x7E5A)}   # quiet NaNs with a payload


class Guarded:
    """A tensor of `shape` inside one allocation with `guard` elements of sentinel on either side; the tensor itself starts as the
    sentinel too, or as a copy of `fill`."""

    def __init__(self, shape, dtype=torch.float32, guard=256, fill=None):
        self.n, self.g = int(np.prod(shape)), guard
        self.itype, self.bits = SENTINEL[dtype]
        self.full = torch.empty(self.n + 2 * guard, dtype=dtype, device=DEV)
        self.full.view(self.itype).fill_(self.bits)
        self.t = self.full[guard:guard + self.n].view(shape)
        if fill is not None:
            self.t.copy_(fill)

    def guards_intact(self):
        v = self.full.view(self.itype)
        return bool((v[:self.g] == self.bits).all()) and bool((v[self.g + self.n:] == self.bits).all())

    def unwritten(self):
        return int((self.t.reshape(-1).view(self.itype) == self.bits).sum())


@contextlib.contextmanager
def options(**kw):
    saved = capi.get_options()
    try:
        capi.set_options(**kw)
        yield
    finally:
        capi.set_options(**saved)


def guarded_features(f):
    return Guarded(f.shape, guard=int(np.prod(f.shape[2:])), fill=f)


def to_f32(out, fmt):
    if fmt == F32:
        return out
    B, nvox, C2 = out.shape
    f = torch.empty((B, nvox, C2 // 2), dtype=torch.float32, device=DEV)
    capi.s32_to_f32(out.contiguous(), f, B * nvox, C2 // 2)
    return f


def native_forward(sc, agg, fmt=F32, feats=None):
    """lt_unproject_aggregate_fwd on guarded buffers -> float32 (B, nvox, C); asserts no read outside the features, every output
    written, no write outside it."""
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    F = guarded_features(f) if feats is None else None
    out = Guarded((B, nvox, C)) if fmt == F32 else Guarded((B, nvox, 2 * C), torch.float16)
    capi.unproject_aggregate(F.t if feats is None else feats, p, c, cf if agg == "conf" else None, out.t, fmt, capi.AGG[agg])
    torch.cuda.synchronize()
    assert out.guards_intact() and out.unwritten() == 0 and (F is None or F.guards_intact())
    got = to_f32(out.t, fmt)
    assert bool(torch.isfinite(got).all())
    return got


def fmt_bar(fmt, ref):
    return BAR if fmt == F32 else BAR + 2.0 ** -21 + 2.0 ** -25 / scale_of(ref)


# ------------------------------------------------------------------------------------------ forward: the dispatch table
# Every instantiation launch_unproject can launch, line by line in the order of its branches.
V2_LINES = [                                       # LT_UNPROJ_V2(FMT), FMT = LT_FMT_F32 (0) / LT_FMT_S32 (1)
    "unproject_v2_kernel<4, {fmt}, true, 3, 8>",    # cpl == 8 && V == 4 && lb == 3
    "unproject_v2_kernel<4, {fmt}, true, 2, 8>",    # cpl == 8 && V == 4
    "unproject_v2_kernel<8, {fmt}, true, 1, 8>",    # cpl == 8 && V == 8
    "unproject_v2_kernel<4, {fmt}, false, 2, 8>",   # cpl == 8 && V < 4
    "unproject_v2_kernel<8, {fmt}, false, 1, 8>",   # cpl == 8
    "unproject_v2_kernel<4, {fmt}, true, 5, 4>",    # V == 4 && lb == 5
    "unproject_v2_kernel<4, {fmt}, true, 4, 4>",    # V == 4
    "unproject_v2_kernel<8, {fmt}, true, 3, 4>",    # V == 8
    "unproject_v2_kernel<4, {fmt}, false, 5, 4>",   # V < 4
    "unproject_v2_kernel<8, {fmt}, false, 3, 4>",   # otherwise
]
FAST_LINES = ["unproject_fast_kernel<%d, %d, 4>" % (g, m)   # switch (G) { case GG: LT_UNPROJ_FAST(GG, 4) }, V <= 2 / <= 4 / else
              for g in (1, 2, 4, 8, 16, 32) for m in (2, 4, 8)]
GENERIC_LINES = ["unproject_kernel<4, true>", "unproject_kernel<4, false>", "unproject_kernel<1, true>", "unproject_kernel<1, false>"]
ALL_KERNELS = ([line.format(fmt=f) for f in (F32, S32) for line in V2_LINES] + FAST_LINES + GENERIC_LINES
               + ["unproject_finalize_kernel", "feature_scatter_kernel", "unproject_bwd_kernel"])

Case = namedtuple("Case", "kernel B V C hw nvox aggs opts")
V2 = dict(unproject_v2=1, unproject_cpl=4, unproject_lb=0, unproject_brick=0)
V2_8 = dict(V2, unproject_cpl=8)
NO_V2 = dict(unproject_v2=0)
SM = ("softmax",)
FWD_CASES = {
    # production-shape kernel: C = 32, softmax, full output
    "v2 cpl4 V4 lb5": Case("unproject_v2_kernel<4, {fmt}, true, 5, 4>", 2, 4, 32, (8, 32), 500, SM, dict(V2, unproject_lb=5)),
    "v2 cpl4 V4": Case("unproject_v2_kernel<4, {fmt}, true, 4, 4>", 3, 4, 32, (16, 16), 700, SM, V2),
    "v2 cpl4 V8": Case("unproject_v2_kernel<8, {fmt}, true, 3, 4>", 2, 8, 32, (4, 8), 400, SM, V2),
    "v2 cpl4 V1": Case("unproject_v2_kernel<4, {fmt}, false, 5, 4>", 2, 1, 32, (2, 2), 300, SM, V2),
    "v2 cpl4 V3": Case("unproject_v2_kernel<4, {fmt}, false, 5, 4>", 3, 3, 32, (32, 8), 500, SM, V2),
    "v2 cpl4 V5": Case("unproject_v2_kernel<8, {fmt}, false, 3, 4>", 2, 5, 32, (8, 8), 400, SM, V2),
    "v2 cpl4 V7": Case("unproject_v2_kernel<8, {fmt}, false, 3, 4>", 2, 7, 32, (1, 4), 300, SM, V2),
    "v2 cpl8 V4 lb3": Case("unproject_v2_kernel<4, {fmt}, true, 3, 8>", 2, 4, 32, (16, 16), 500, SM, dict(V2_8, unproject_lb=3)),
    "v2 cpl8 V4": Case("unproject_v2_kernel<4, {fmt}, true, 2, 8>", 3, 4, 32, (8, 32), 400, SM, V2_8),
    "v2 cpl8 V8": Case("unproject_v2_kernel<8, {fmt}, true, 1, 8>", 2, 8, 32, (8, 8), 300, SM, V2_8),
    "v2 cpl8 V2": Case("unproject_v2_kernel<4, {fmt}, false, 2, 8>", 2, 2, 32, (2, 1), 300, SM, V2_8),
    "v2 cpl8 V5": Case("unproject_v2_kernel<8, {fmt}, false, 1, 8>", 2, 5, 32, (32, 8), 400, SM, V2_8),
    "v2 cpl8 V7": Case("unproject_v2_kernel<8, {fmt}, false, 1, 8>", 3, 7, 32, (4, 4), 300, SM, V2_8),
    # brick walk on cubic grids (n^3 voxels, n % brick == 0), each voxel order; n = 6 is not divisible by 4: linear walk
    **{"v2 cpl%d brick%d order%d n%d" % (cpl, bs, order, n): Case("unproject_v2_kernel<4, {fmt}, true, %d, %d>" % (4 if cpl == 4 else 2, cpl),
                                                                  2, 4, 32, (16, 16), n ** 3, SM,
                                                                  dict(V2, unproject_cpl=cpl, unproject_brick=bs, unproject_brick_order=order))
       for cpl in (4, 8) for bs, n in ((4, 8), (8, 16)) for order in (0, 1, 2)},
    "v2 cpl4 brick4 n6 linear": Case("unproject_v2_kernel<4, {fmt}, true, 4, 4>", 2, 4, 32, (8, 8), 216, SM, dict(V2, unproject_brick=4)),
    "v2 cpl8 brick4 n6 linear": Case("unproject_v2_kernel<4, {fmt}, true, 2, 8>", 2, 4, 32, (8, 8), 216, SM, dict(V2_8, unproject_brick=4)),
    "v2 cpl8 brick8 order2 V7": Case("unproject_v2_kernel<8, {fmt}, false, 1, 8>", 2, 7, 32, (8, 8), 512, SM,
                                     dict(V2_8, unproject_brick=8, unproject_brick_order=2)),
    # fast kernel: C = 4 G, V <= 8
    "fast G1 V1": Case(FAST_LINES[0], 2, 1, 4, (1, 4), 300, AGGS, {}),
    "fast G1 V3": Case(FAST_LINES[1], 3, 3, 4, (8, 8), 400, AGGS, {}),
    "fast G1 V5": Case(FAST_LINES[2], 2, 5, 4, (4, 2), 300, AGGS, {}),
    "fast G2 V2": Case(FAST_LINES[3], 2, 2, 8, (2, 2), 300, AGGS, {}),
    "fast G2 V4": Case(FAST_LINES[4], 2, 4, 8, (8, 32), 400, AGGS, {}),
    "fast G2 V7": Case(FAST_LINES[5], 3, 7, 8, (16, 16), 300, AGGS, {}),
    "fast G4 V1": Case(FAST_LINES[6], 2, 1, 16, (32, 8), 400, AGGS, {}),
    "fast G4 V3": Case(FAST_LINES[7], 2, 3, 16, (4, 4), 300, AGGS, {}),
    "fast G4 V8": Case(FAST_LINES[8], 2, 8, 16, (2, 8), 300, AGGS, {}),
    "fast G8 V2": Case(FAST_LINES[9], 2, 2, 32, (8, 8), 400, AGGS, NO_V2),
    "fast G8 V4": Case(FAST_LINES[10], 3, 4, 32, (16, 16), 300, AGGS, NO_V2),
    "fast G8 V5": Case(FAST_LINES[11], 2, 5, 32, (8, 32), 300, AGGS, NO_V2),
    "fast G16 V2": Case(FAST_LINES[12], 2, 2, 64, (4, 4), 300, AGGS, {}),
    "fast G16 V3": Case(FAST_LINES[13], 2, 3, 64, (8, 8), 300, AGGS, {}),
    "fast G16 V8": Case(FAST_LINES[14], 2, 8, 64, (2, 2), 200, AGGS, {}),
    "fast G32 V1": Case(FAST_LINES[15], 2, 1, 128, (8, 8), 300, AGGS, {}),
    "fast G32 V4": Case(FAST_LINES[16], 2, 4, 128, (4, 8), 200, AGGS, {}),
    "fast G32 V7": Case(FAST_LINES[17], 2, 7, 128, (2, 4), 200, AGGS, {}),
    # generic kernel: VEC 4 when C % 4 == 0 (C / 4 not a power of two, or C > 128), VEC 1 otherwise; per-view samples stored for V <= 8
    "generic C12 V3": Case(GENERIC_LINES[0], 2, 3, 12, (8, 8), 400, AGGS, {}),
    "generic C24 V8": Case(GENERIC_LINES[0], 2, 8, 24, (4, 4), 300, AGGS, {}),
    "generic C96 V4": Case(GENERIC_LINES[0], 3, 4, 96, (8, 8), 300, AGGS, {}),
    "generic C256 V2": Case(GENERIC_LINES[0], 2, 2, 256, (4, 4), 200, AGGS, {}),
    "generic C12 V9": Case(GENERIC_LINES[1], 2, 9, 12, (8, 8), 300, AGGS, {}),
    "generic C32 V66": Case(GENERIC_LINES[1], 2, 66, 32, (2, 4), 200, AGGS, {}),
    "generic C256 V9": Case(GENERIC_LINES[1], 2, 9, 256, (2, 2), 200, AGGS, {}),
    "generic C5 V3": Case(GENERIC_LINES[2], 3, 3, 5, (8, 32), 400, AGGS, {}),
    "generic C5 V1": Case(GENERIC_LINES[2], 2, 1, 5, (1, 1), 200, AGGS, {}),
    "generic C5 V9": Case(GENERIC_LINES[3], 2, 9, 5, (4, 4), 300, AGGS, {}),
    "generic C5 V66": Case(GENERIC_LINES[3], 2, 66, 5, (2, 2), 200, AGGS, {}),
}
FWD_PARAMS = [(name, agg) for name, c in FWD_CASES.items() for agg in c.aggs]


def case_scene(name):
    c = FWD_CASES[name]
    return exact_scene(c.B, c.V, c.C, c.hw[0], c.hw[1], c.nvox, seed=sum(map(ord, name)))


def formats(C):
    return (F32, S32) if C % 32 == 0 else (F32,)


@pytest.mark.parametrize("name,agg", FWD_PARAMS, ids=["%s-%s" % p for p in FWD_PARAMS])
def test_forward_exact_geometry_vs_float64(name, agg):
    c = FWD_CASES[name]
    sc = case_scene(name)
    ref = reference(sc, agg, DEV)
    with options(**c.opts):
        for fmt in formats(c.C):
            e = err(native_forward(sc, agg, fmt), ref)
            print("%-34s %-7s %s  %.1e" % (name, agg, "s32" if fmt else "f32", e))
            assert e <= fmt_bar(fmt, ref), (name, agg, fmt, e)


def test_forward_identical_views_and_sample_specific_projections():
    """Two identical views; and the same scene with sample 1's projections swapped for sample 0's must change sample 1's output."""
    for name, opts in (("v2", V2), ("fast", NO_V2)):
        sc = exact_scene(2, 4, 32, 8, 8, 400, seed=3, identical_views=True)
        with options(**opts):
            for agg in (SM if name == "v2" else AGGS):
                ref = reference(sc, agg, DEV)
                assert err(native_forward(sc, agg), ref) <= BAR
                swapped = sc._replace(proj=np.stack([sc.proj[0], sc.proj[0]]))
                assert err(native_forward(swapped, agg)[1], ref[1]) > 1e-2


CAMERA_CASES = {   # name -> (B, V, C, h, w, n, options)
    "v2 9x13": (2, 4, 32, 9, 13, 8, V2), "v2 cpl8 V6 9x13": (2, 6, 32, 9, 13, 8, V2_8), "fast 9x13": (2, 3, 16, 9, 13, 8, {}),
    "generic C5 9x13": (2, 3, 5, 9, 13, 8, {}), "generic C12 V9 9x13": (2, 9, 12, 9, 13, 6, {}), "v2 96x96": (2, 4, 32, 96, 96, 16, V2),
    "fast C32 96x96": (2, 4, 32, 96, 96, 16, NO_V2),
}


@pytest.mark.parametrize("name", list(CAMERA_CASES))
def test_forward_camera_scenes_yardstick(name):
    B, V, C, h, w, n, opts = CAMERA_CASES[name]
    sc = camera_scene(B, V, C, h, w, n, seed=len(name))
    with options(**opts):
        for agg in AGGS:
            ref = reference(sc, agg, DEV)
            yard = err(reference(sc, agg, DEV, torch.float32), ref)
            for fmt in formats(C):
                e = err(native_forward(sc, agg, fmt), ref)
                print("%-22s %-7s %s  native %.1e  yardstick %.1e" % (name, agg, "s32" if fmt else "f32", e, yard))
                assert e <= max(fmt_bar(fmt, ref), 2 * yard), (name, agg, fmt, e, yard)


def _kernel_names(prof):
    pat = re.compile(r"(unproject\w*_kernel|feature_scatter_kernel)(<[^>]*>)?")
    evs = [e for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA]
    names = []
    for e in sorted(evs, key=lambda e: e.start_ns()):
        m = pat.search(e.name())
        if m:
            names.append(m.group(0))
    return names


def test_dispatch_reaches_every_instantiation():
    """Each case of the forward table launches the kernel it names, and together with one finalize, reduce-finalize, feature
    scatter and backward call the launches cover every instantiation of ALL_KERNELS."""
    from torch.profiler import ProfilerActivity, profile
    runs = []
    for name, c in FWD_CASES.items():
        sc = case_scene(name)
        f, p, co, cf = tensors(sc, DEV, torch.float32)
        for agg in c.aggs:
            for fmt in formats(c.C):
                out = torch.empty((c.B, c.nvox, c.C if fmt == F32 else 2 * c.C), dtype=torch.float32 if fmt == F32 else torch.float16,
                                  device=DEV)
                runs.append((c.opts, (f, p, co, cf if agg == "conf" else None, out, fmt, capi.AGG[agg]), c.kernel.format(fmt=fmt)))
    sc = exact_scene(2, 2, 32, 4, 4, 64, seed=1)
    f, p, co, cf = tensors(sc, DEV, torch.float32)
    part = torch.randn((2, 2, 64, 32), device=DEV).abs()
    out = torch.empty((2, 64, 32), device=DEV)
    buf = torch.empty((1, 2, 2, 4, 4, 32), device=DEV)
    g = torch.randn((2, 64, 32), device=DEV)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for opts, args, _ in runs:
            with options(**opts):
                capi.unproject_aggregate(*args)
        capi.unproject_finalize(part, out, F32, 2, 32, 64, capi.AGG["softmax"])
        capi.unproject_reduce_finalize(part, 1, out, F32, 2, 32, 64, capi.AGG["softmax"])
        capi.feature_scatter(f, [buf.data_ptr()], 0, 2)
        capi.unproject_aggregate_bwd(f, p, co, cf, g, torch.zeros_like(f), torch.zeros_like(cf), capi.AGG["conf"])
        torch.cuda.synchronize()
    names = _kernel_names(prof)
    expected = [k for _, _, k in runs] + ["unproject_finalize_kernel"] * 2 + ["feature_scatter_kernel", "unproject_bwd_kernel"]
    assert len(names) == len(expected)
    for i, (got, want) in enumerate(zip(names, expected)):
        assert got == want, (i, got, want)
    assert len(set(ALL_KERNELS)) == len(ALL_KERNELS) == 45 and set(names) == set(ALL_KERNELS), sorted(set(ALL_KERNELS) ^ set(names))


# ------------------------------------------------------------------------------------------ view-sharded exchange kernels
PARTIAL_CASES = {"fast C4 V3": (2, 3, 4, 8, 8, 400), "fast C32 V2": (3, 2, 32, 8, 32, 300), "fast C128 V4": (2, 4, 128, 4, 4, 200),
                 "generic C12 V3": (2, 3, 12, 8, 8, 300), "generic C5 V3": (2, 3, 5, 32, 8, 300), "generic C5 V9": (2, 9, 5, 4, 4, 200),
                 "generic C32 V9": (2, 9, 32, 4, 8, 200)}


def native_partial(sc, agg, views=None):
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    if views is not None:
        f, p, cf = f[:, views].contiguous(), p[:, views].contiguous(), cf[:, views].contiguous()
    B, V, h, w, C = f.shape
    nvox = c.shape[1]
    F = guarded_features(f)
    part = Guarded((B, 2 if agg == "softmax" else 1, nvox, C))
    capi.unproject_partial(F.t, p, c, cf if agg == "conf" else None, part.t, capi.AGG[agg])
    torch.cuda.synchronize()
    assert F.guards_intact() and part.guards_intact() and part.unwritten() == 0
    return part.t


@pytest.mark.parametrize("name", list(PARTIAL_CASES))
@pytest.mark.parametrize("agg", AGGS)
def test_partial_vs_float64(name, agg):
    sc = exact_scene(*PARTIAL_CASES[name], seed=len(name) + 17)
    got, ref = native_partial(sc, agg), reference_partial(sc, agg, DEV)
    for k in range(ref.shape[1]):
        e = err(got[:, k], ref[:, k])
        print("%-16s %-7s plane %d  %.1e" % (name, agg, k, e))
        assert e <= BAR, (name, agg, k, e)


def combine(parts, agg):
    out = parts[0].clone()
    for q in parts[1:]:
        out = torch.maximum(out, q) if agg == "max" else out + q
    return out


@pytest.mark.parametrize("G", [2, 4])
@pytest.mark.parametrize("C", [12, 32])
@pytest.mark.parametrize("agg", AGGS)
def test_split_views_and_finalize_match_single_pass(G, C, agg):
    B, V, nvox = 2, 8, 300
    sc = exact_scene(B, V, C, 8, 32, nvox, seed=G * 10 + C)
    total = combine([native_partial(sc, agg, list(range(r, V, G))) for r in range(G)], agg)
    ref = reference(sc, agg, DEV)
    for fmt in formats(C):
        out = Guarded((B, nvox, C)) if fmt == F32 else Guarded((B, nvox, 2 * C), torch.float16)
        capi.unproject_finalize(total.contiguous(), out.t, fmt, B, C, nvox, capi.AGG[agg])
        torch.cuda.synchronize()
        assert out.guards_intact() and out.unwritten() == 0
        e = err(to_f32(out.t, fmt), ref)
        print("G %d C %d %-7s %s  %.1e" % (G, C, agg, "s32" if fmt else "f32", e))
        assert e <= fmt_bar(fmt, ref), (G, C, agg, fmt, e)


@pytest.mark.parametrize("G", [2, 4])
@pytest.mark.parametrize("C", [4, 32, 128])
@pytest.mark.parametrize("agg", AGGS)
def test_push_into_owner_slots_and_reduce_finalize(G, C, agg):
    """Rank r's push writes slot r of every owner and nothing else; each owner's reduce-finalize over its G slots is the single-pass
    output of its samples."""
    B, V, nvox = 4, 8, 300
    per, P = B // G, 2 if agg == "softmax" else 1
    sc = exact_scene(B, V, C, 4, 8, nvox, seed=G * 100 + C)
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    bufs = [Guarded((G, per, P, nvox, C)) for _ in range(G)]
    ptrs = [b.t.data_ptr() for b in bufs]
    for r in range(G):
        before = [b.full.clone() for b in bufs]
        vs = list(range(r, V, G))
        F = guarded_features(f[:, vs].contiguous())
        capi.unproject_push(F.t, p[:, vs].contiguous(), c, cf[:, vs].contiguous() if agg == "conf" else None, ptrs, r, capi.AGG[agg])
        torch.cuda.synchronize()
        assert F.guards_intact()
        for o, b in enumerate(bufs):
            assert b.guards_intact()
            slots, old = b.t.view(b.itype), before[o][b.g:b.g + b.n].view(b.t.shape).view(b.itype)
            for s in range(G):
                if s == r:
                    assert not bool((slots[s] == b.bits).any()), (r, o)
                else:
                    assert torch.equal(slots[s], old[s]), (r, o, s)
    ref = reference(sc, agg, DEV)
    for o, b in enumerate(bufs):
        for fmt in formats(C):
            out = Guarded((per, nvox, C)) if fmt == F32 else Guarded((per, nvox, 2 * C), torch.float16)
            capi.unproject_reduce_finalize(b.t, G, out.t, fmt, per, C, nvox, capi.AGG[agg])
            torch.cuda.synchronize()
            assert out.guards_intact() and out.unwritten() == 0
            want = ref[o * per:(o + 1) * per]
            e = err(to_f32(out.t, fmt), want)
            assert e <= fmt_bar(fmt, want), (G, C, agg, o, fmt, e)


@pytest.mark.parametrize("G", [2, 4])
@pytest.mark.parametrize("C", [5, 32])
def test_feature_scatter_assembles_global_view_order(G, C):
    """Owner buffers filled by every view rank hold the features bit for bit in global view order, and unprojecting an owner buffer
    gives bit for bit the single-GPU output of the owner's samples."""
    B, V, h, w, nvox = 4, 8, 4, 8, 300
    per = B // G
    sc = exact_scene(B, V, C, h, w, nvox, seed=G + C)
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    bufs = [Guarded((per, V, h, w, C), guard=h * w * C) for _ in range(G)]
    for r in range(G):
        capi.feature_scatter(f[:, r::G].contiguous(), [b.t.data_ptr() for b in bufs], r, V)
    torch.cuda.synchronize()
    for o, b in enumerate(bufs):
        assert b.guards_intact()
        assert torch.equal(b.t.view(torch.int32), f[o * per:(o + 1) * per].contiguous().view(torch.int32)), o
    for agg in AGGS:
        single = native_forward(sc, agg)
        for o, b in enumerate(bufs):
            own = sc._replace(proj=sc.proj[o * per:(o + 1) * per], coord=sc.coord[o * per:(o + 1) * per], conf=sc.conf[o * per:(o + 1) * per],
                              feats=sc.feats[o * per:(o + 1) * per])
            got = native_forward(own, agg, feats=b.t)
            assert torch.equal(got.view(torch.int32), single[o * per:(o + 1) * per].contiguous().view(torch.int32)), (agg, o)


@pytest.mark.parametrize("C", [32, 12])
def test_softmax_partials_at_large_scores(C):
    """Softmax partials are unshifted exponentials: scores up to |s| ~ 60 (e^60 ~ 1e26) still finalize to the bar.  The limit (header
    at lt_unproject_partial_fwd, DESIGN section 6): e^s overflows above s ~ 88."""
    B, V, nvox = 2, 4, 400
    sc = exact_scene(B, V, C, 8, 8, nvox, seed=C)
    sc = sc._replace(feats=np.random.RandomState(C).uniform(-60, 60, sc.feats.shape).astype(np.float32))
    ref = reference(sc, "softmax", DEV)
    assert float(ref.abs().max()) > 55
    total = combine([native_partial(sc, "softmax", [r, r + 2]) for r in range(2)], "softmax")
    assert float(total[:, 1].max()) > 1e24
    out = torch.empty((B, nvox, C), device=DEV)
    capi.unproject_finalize(total.contiguous(), out, F32, B, C, nvox, capi.AGG["softmax"])
    e = err(out, ref)
    print("C %d |s| ~ 60: %.1e" % (C, e))
    assert e <= BAR, e


# ------------------------------------------------------------------------------------------ backward
BWD_BAR = 2e-6
BWD_HW = {1: (8, 32), 3: (32, 8), 8: (16, 16), 9: (2, 1), 66: (1, 4)}


def upstream(sc, agg, seed):
    B, nvox, C = sc.coord.shape[0], sc.coord.shape[1], sc.feats.shape[-1]
    g = torch.from_numpy(np.random.RandomState(seed).randn(B, nvox, C).astype(np.float32)).to(DEV)
    if agg == "max":
        near = max_near_ties(sc, DEV)
        assert float(near.float().mean()) < 0.01
        g = g.masked_fill(near, 0.0)
    return g


def hybrid_grads(sc, agg, g, want_conf=True):
    """op.unproject_heatmaps(backend="hybrid") -> (d features channels-last, d conf or None)."""
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    B, nvox = c.shape[:2]
    heat = f.permute(0, 1, 4, 2, 3).contiguous().requires_grad_(True)
    cf.requires_grad_(want_conf and agg == "conf")
    out = op.unproject_heatmaps(heat, p, c.reshape(B, nvox, 1, 1, 3), agg, cf, backend="hybrid")
    out.backward(g.transpose(1, 2).reshape(out.shape))
    return heat.grad.permute(0, 1, 3, 4, 2), (cf.grad if cf.requires_grad else None)


def direct_grads(sc, agg, g, gf0=None, gc0=None, with_gconf=True):
    """lt_unproject_aggregate_bwd on guarded buffers that start at gf0 / gc0 (zero if None)."""
    f, p, c, cf = tensors(sc, DEV, torch.float32)
    F = guarded_features(f)
    GF = Guarded(f.shape, fill=torch.zeros_like(f) if gf0 is None else gf0)
    GC = Guarded(cf.shape, fill=torch.zeros_like(cf) if gc0 is None else gc0) if (with_gconf and agg == "conf") else None
    capi.unproject_aggregate_bwd(F.t, p, c, cf if agg == "conf" else None, g.contiguous(), GF.t, None if GC is None else GC.t,
                                 capi.AGG[agg])
    torch.cuda.synchronize()
    assert F.guards_intact() and GF.guards_intact() and (GC is None or GC.guards_intact())
    return GF.t, (None if GC is None else GC.t)


def yardstick_check(label, got, ref, yard_ref):
    e, y = err(got, ref), err(yard_ref, ref)
    print("%-36s native %.1e  yardstick %.1e" % (label, e, y))
    assert e <= max(BWD_BAR, 2 * y), (label, e, y)


@pytest.mark.parametrize("V", [1, 3, 8, 9, 66])
@pytest.mark.parametrize("C", [4, 32, 128])
@pytest.mark.parametrize("agg", AGGS)
def test_backward_exact_geometry_vs_float64(V, C, agg):
    """Through op.unproject_heatmaps(backend="hybrid") with d conf requested, and directly with d conf NULL.  max: float64 and the
    float32 yardstick run on the CPU, where torch routes exact ties (out-of-map views at 0, two identical views) to the first view as
    the kernel does."""
    h, w = BWD_HW[V]
    sc = exact_scene(2, V, C, h, w, 300, seed=V * 1000 + C, identical_views=V >= 3)
    g = upstream(sc, agg, V + C)
    dev = "cpu" if agg == "max" else DEV
    ref_f, ref_c = reference_grads(sc, agg, g, dev)
    yard_f, yard_c = reference_grads(sc, agg, g, dev, torch.float32)
    gf, gc = hybrid_grads(sc, agg, g)
    yardstick_check("V %d C %d %s d features" % (V, C, agg), gf, ref_f, yard_f)
    if agg == "conf":
        yardstick_check("V %d C %d %s d conf" % (V, C, agg), gc, ref_c, yard_c)
    gf2, none = direct_grads(sc, agg, g, with_gconf=False)
    assert none is None
    yardstick_check("V %d C %d %s d features, no d conf" % (V, C, agg), gf2, ref_f, yard_f)


@pytest.mark.parametrize("agg", ["softmax", "conf"])
def test_backward_recipe_shape_vs_float64(agg):
    """The hybrid training step's shape: B 2, V 4, C 32, 96 x 96 maps, 64^3 voxels, camera scene; float64 reference on the GPU."""
    sc = camera_scene(2, 4, 32, 96, 96, 64, seed=5)
    g = upstream(sc, agg, 9)
    ref_f, ref_c = reference_grads(sc, agg, g, DEV)
    yard_f, yard_c = reference_grads(sc, agg, g, DEV, torch.float32)
    gf, gc = hybrid_grads(sc, agg, g)
    yardstick_check("recipe %s d features" % agg, gf, ref_f, yard_f)
    if agg == "conf":
        yardstick_check("recipe %s d conf" % agg, gc, ref_c, yard_c)


@pytest.mark.parametrize("agg", AGGS)
def test_backward_accumulates_into_its_outputs(agg):
    sc = exact_scene(2, 3, 32, 8, 8, 512, seed=11)
    g = upstream(sc, agg, 4)
    gen = torch.Generator(device=DEV).manual_seed(2)
    gf0 = torch.randn(sc.feats.shape, device=DEV, generator=gen)
    gc0 = torch.randn(sc.conf.shape, device=DEV, generator=gen)
    gf, gc = direct_grads(sc, agg, g)
    af, ac = direct_grads(sc, agg, g, gf0, gc0)
    assert err(af, gf0 + gf) <= 1e-6
    if agg == "conf":
        assert err(ac, gc0 + gc) <= 1e-6


def test_backward_conf_accumulator_limit_and_channel_check():
    """With d conf, the [V][C] accumulator takes V * C = 10240 (40 KB) and refuses one view more; without d conf it is not needed.
    C % 4 != 0 is refused."""
    sc = exact_scene(1, 80, 128, 2, 2, 64, seed=80)
    g = upstream(sc, "conf", 1)
    ref_f, ref_c = reference_grads(sc, "conf", g, DEV)
    yard_f, yard_c = reference_grads(sc, "conf", g, DEV, torch.float32)
    gf, gc = direct_grads(sc, "conf", g)
    yardstick_check("V 80 C 128 conf d features", gf, ref_f, yard_f)
    yardstick_check("V 80 C 128 conf d conf", gc, ref_c, yard_c)
    sc = exact_scene(1, 81, 128, 2, 2, 64, seed=81)
    g = upstream(sc, "conf", 1)
    with pytest.raises(RuntimeError, match=r"V \* C too large for the confidence-gradient accumulator"):
        direct_grads(sc, "conf", g)
    direct_grads(sc, "conf", g, with_gconf=False)
    sc = exact_scene(1, 2, 6, 4, 4, 64, seed=6)
    with pytest.raises(RuntimeError, match=r"C % 4 != 0"):
        direct_grads(sc, "sum", upstream(sc, "sum", 1))
