"""GPU tests of the plane-major tiles of conv_fold_kernel<7, NC> against float64, at test_gpu_conv's per-element bars.

A tile is 8 (w) x 16 (h) x Dt (d) outputs, Dt = 64 / NC (4 at NC = 16, 2 at NC = 32); each input plane of the tile is loaded
once and one wgmma per K slice feeds all Dt output planes, whose taps outside the filter are zero.  The cases cover volumes
shallower than a tile, depths that leave a partial last tile, H not a multiple of 16, W at one, two and several w tiles, two
batch items, both N widths, both output formats and the residual modes, plus the in-place residual."""
import pytest
import torch

import test_gpu_conv as T
from test_gpu_conv import _no_tf32  # noqa: F401  (autouse: float64 references without TF32)
from test_conv_cpu import F32, RES_AFTER, RES_BEFORE, RES_NONE

pytestmark = pytest.mark.gpu

K7 = T.K7
CASES = {
    # NC = 16 (4 planes per tile)
    "nc16 D1 H16 W16": T.case(T.FD16, N=1, I=(1, 16, 16), cout=16, k=K7),
    "nc16 D2 H9 W17 F32 res-after": T.case(T.FD16, N=1, I=(2, 9, 17), cout=16, k=K7, fmt=F32, out_c=32, res=RES_AFTER),
    "nc16 D6 H21 W64 res-before": T.case(T.FD16, N=1, I=(6, 21, 64), cout=16, k=K7, res=RES_BEFORE),
    "nc16 D9 H5 W80 F32": T.case(T.FD16, N=1, I=(9, 5, 80), cout=16, k=K7, fmt=F32, out_c=32),
    "nc16 N2 D5 H18 W17 res-before": T.case(T.FD16, N=2, I=(5, 18, 17), cout=12, k=K7, res=RES_BEFORE),
    "nc16 N2 D8 H16 W16 F32 res-before": T.case(T.FD16, N=2, I=(8, 16, 16), cout=16, k=K7, fmt=F32, out_c=32,
                                                  res=RES_BEFORE),
    # NC = 32 (2 planes per tile)
    "nc32 D1 H7 W16 F32": T.case(T.FD32, N=1, I=(1, 7, 16), cout=32, k=K7, fmt=F32),
    "nc32 D3 H17 W80 res-after": T.case(T.FD32, N=1, I=(3, 17, 80), cout=32, k=K7, res=RES_AFTER),
    "nc32 N2 D4 H9 W64 F32 res-before": T.case(T.FD32, N=2, I=(4, 9, 64), cout=20, k=K7, fmt=F32, res=RES_BEFORE),
    "nc32 N2 D5 H16 W17": T.case(T.FD32, N=2, I=(5, 16, 17), cout=32, k=K7, res=RES_NONE),
}


@pytest.mark.parametrize("name", list(CASES))
def test_fold7_plane_tiles_vs_float64(name):
    c = CASES[name]
    assert [p.impl for p in T.case_launches(c)] == [T.FOLD]
    b = T.build(c, seed=sum(map(ord, name)) % 1000)
    out = T.new_out(c, b)
    T.run(c, b, out.t)
    torch.cuda.synchronize()
    got = T.check_buffers(c, b, out)
    ref, bar, _ = T.reference(c, b)
    assert not bool(torch.isnan(ref).any())
    ratio = float(((got - ref).abs() / bar.clamp(min=1e-300)).max())
    print("%-36s largest err/bar %.3f" % (name, ratio))
    assert ratio <= 1.0, (name, ratio)
    if c.res != RES_NONE:   # the residual read from the output buffer itself
        io = T.new_out(c, b)
        io.t.copy_(b.res.t)
        T.run(c, b, io.t, res=io.t)
        torch.cuda.synchronize()
        assert io.guards_intact() and torch.equal(T.bits(io.t), T.bits(out.t)), "the in-place residual differs from out-of-place"
