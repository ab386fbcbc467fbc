"""conv_tc_kernel's double-buffered staged epilogue: the k-th work unit of a CTA uses tile buffer k & 1, and the next unit's residual
tile loads into the other buffer while this unit's epilogue and store run.  Every case runs at least five units on every CTA, so
each buffer is handed between warp 1 (TMA residual load and store) and the consumer warpgroups at least twice, with each buffer's
own barrier phase.  Launches with more K chunks per unit keep one buffer; one case covers that side.

Covered: all three residual modes, the in-place residual (out aliases the residual, bit-identical to out-of-place), partial M tiles,
a float32 output narrower than its N tile, N tiles 32 / 64 / 128, a stride-2 input, the grouped k2 s2 3-D deconv with its skip and
the four stride-phase launches of the 2-D k4 s2 deconv.  Each output is held per element to tests/test_gpu_conv.py's float64 bar,
and a second run must be bit-identical.  lt_conv_tc_plan confirms the layout every launch took."""
import pytest
import torch

from lt_b200 import capi
from test_gpu_conv import (F32, K3, RES_AFTER, RES_BEFORE, RES_NONE, S32, T128, T32, T64, _desc, bits, build, case, case_launches,
                           check_buffers, new_out, reference, run)

pytestmark = pytest.mark.gpu

MIN_UNITS_PER_CTA = 5

# Every case but the last keeps at most 4 K chunks per unit, where the launch takes two tile buffers; the last has 8 and takes one.
CASES = {
    "tc128 1x1 res-before partial tiles S32": case(T128, N=19, I=(1, 47, 45), cin=64, cout=256, k=(1, 1, 1), res=RES_BEFORE, ws=False),
    "tc128 1x1 res-after S32": case(T128, N=20, I=(1, 24, 24), cin=128, cout=1024, k=(1, 1, 1), res=RES_AFTER, ws=False),
    "tc128 1x1 no residual S32": case(T128, N=20, I=(1, 48, 48), cin=64, cout=256, k=(1, 1, 1), ws=False),
    "tc128 1x1 cout117 FC120 res-before F32": case(T128, N=40, I=(1, 45, 47), cin=32, cout=117, k=(1, 1, 1), fmt=F32, out_c=120,
                                                   res=RES_BEFORE, ws=False),
    "tc64 1x1 res-after partial tiles S32": case(T64, N=45, I=(1, 43, 45), cin=96, cout=64, k=(1, 1, 1), res=RES_AFTER, ws=False),
    "tc32 1x1 cout20 FC20 F32": case(T32, N=90, I=(1, 31, 31), cin=32, cout=20, k=(1, 1, 1), fmt=F32, out_c=20, res=RES_AFTER,
                                     ws=False),
    "tc32 1x1 cout96 res-before S32": case(T32, N=30, I=(1, 50, 46), cin=64, cout=96, k=(1, 1, 1), res=RES_BEFORE, ws=False),
    "tc128 1x1 s2 res-before S32": case(T128, N=68, I=(1, 73, 69), cin=128, cout=128, k=(1, 1, 1), s=(1, 2, 2), res=RES_BEFORE,
                                        ws=False),
    "deconv3d k2s2 cout32 skip": case(T128, kind="deconv3d", N=11, I=(15, 16, 17), cin=64, cout=32, res=RES_AFTER),
    "deconv2d k4s2 cout64": case([T64] * 4, kind="deconv2d", N=40, I=(1, 47, 45), cin=32, cout=64),
    "tc128 1x1 8 chunks res-after S32 (one buffer)": case(T128, N=20, I=(1, 24, 24), cin=256, cout=1024, k=(1, 1, 1), res=RES_AFTER,
                                                          ws=False),
}
SHORT_K = 4     # conv_tc.cu kTcShortK


def _plans(c, b, sms):
    return [capi.conv_tc_plan(_desc(c, part, b.in_fmt, b.ws), sms) for part in b.parts]


@pytest.mark.parametrize("name", list(CASES))
def test_double_buffered_epilogue_vs_float64(name):
    c = CASES[name]
    b = build(c, seed=sum(map(ord, name)) % 1000)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for p in _plans(c, b, sms):
        assert p["splits"] == 1 and p["epi_buffers"] == (2 if p["chunks"] <= SHORT_K else 1), p
        assert "conv_tc_kernel<%d>" % p["nt"] in c.expect, (p, c.expect)
        assert p["m_tiles"] * p["n_tiles"] >= MIN_UNITS_PER_CTA * p["grid"], p
    out = new_out(c, b)
    run(c, b, out.t)
    torch.cuda.synchronize()
    got = check_buffers(c, b, out)
    ref, bar, _ = reference(c, b)
    assert not bool(torch.isnan(ref).any())
    ratio = float(((got - ref).abs() / bar.clamp(min=1e-300)).max())
    print("%-44s largest err/bar %.3f" % (name, ratio))
    assert ratio <= 1.0, (name, ratio)
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


def test_case_table_covers_the_epilogue_variants():
    cs = list(CASES.values())
    assert {c.res for c in cs} == {RES_NONE, RES_BEFORE, RES_AFTER}
    assert {c.fmt for c in cs} == {S32, F32}
    assert {T128, T64, T32} <= {k for c in cs for k in c.expect}
    assert {"deconv2d", "deconv3d"} <= {c.kind for c in cs}
    assert any(max(c.s) == 2 for c in cs)
    assert any(c.fmt == F32 and c.out_c is not None and c.out_c % 32 for c in cs)
    assert K3 not in {c.k for c in cs if c.cin == 32 and c.cout <= 32}    # no case is diverted to the fold kernels
    chunks = [capi.conv_tc_plan(_desc(c, part, S32, None), 132)["chunks"] for c in cs for part in case_launches(c)]
    assert max(chunks) > SHORT_K and sorted(chunks)[-2] <= SHORT_K                 # one case on the single-buffer side
