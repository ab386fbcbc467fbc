"""Host-side work decomposition of the persistent tensor-core conv (lt_conv_tc_plan) at the config #2 layer shapes, no GPU needed."""
import pytest

from lt_b200 import capi

SMS = 132
WS = 32 << 20           # engine.SPLITK_WS_BYTES: the split-K scratch of every conv launch

# (N, out D, H, W, Cin, Cout, kernel, stride, splits expected at 132 SMs)
CONFIG2 = [
    (32, 1, 24, 24, 256, 256, (1, 3, 3), 1, 1),       # layer 3 3x3, 288 tiles x 72 chunks: the reduce pass costs more than the tail wave
    (32, 1, 24, 24, 1024, 256, (1, 1, 1), 1, 1),      # layer 3 reduce, 288 tiles
    (32, 1, 24, 24, 256, 1024, (1, 1, 1), 1, 1),      # layer 3 expand + residual, 1152 tiles
    (32, 1, 48, 48, 128, 128, (1, 3, 3), 1, 1),       # layer 2 3x3, 576 tiles
    (32, 1, 12, 12, 512, 512, (1, 3, 3), 1, 3),       # layer 4 3x3, 144 tiles x 144 chunks
    (32, 1, 12, 12, 2048, 512, (1, 1, 1), 1, 3),      # layer 4 reduce, 144 tiles
    (32, 1, 12, 12, 2048, 256, (1, 2, 2), 1, 7),      # deconv0 phase, 72 tiles x 256 chunks
    (32, 1, 96, 96, 64, 256, (1, 1, 1), 1, 1),        # layer 1 expand, 4608 tiles x 2 chunks
    (8, 8, 8, 8, 128, 128, (3, 3, 3), 1, 4),          # V2V 8^3 level
    (8, 4, 4, 4, 128, 128, (3, 3, 3), 1, 27),         # V2V 4^3 level
    (8, 2, 2, 2, 128, 128, (3, 3, 3), 1, 27),         # V2V 2^3 level
    (8, 16, 16, 16, 128, 128, (3, 3, 3), 1, 1),       # V2V 16^3 level, 256 tiles
    (8, 2, 2, 2, 128, 1024, (1, 1, 1), 1, 1),         # V2V deconv as one grouped-size GEMM, 4 chunks
]


def _desc(N, od, oh, ow, cin, cout, k, s, ws=WS):
    kd, kh, kw = k
    d = capi.ConvDesc(N=N, ID=od * (s if kd > 1 else 1), IH=oh * s, IW=ow * s, Cin=cin, OD=od, OH=oh, OW=ow, Cout=(cout + 15) // 16 * 16,
                      KD=kd, KH=kh, KW=kw, sd=s if kd > 1 else 1, sh=s, sw=s, pd=kd // 2, ph=kh // 2, pw=kw // 2,
                      FD=od, FH=oh, FW=ow, FC=cout, osd=1, osh=1, osw=1, in_format=capi.FMT_S32, out_format=capi.FMT_S32)
    # the plan never dereferences the workspace; a non-NULL pointer only says that one exists
    d.workspace, d.workspace_bytes = (4096 if ws else None), ws
    return d


def _units(p):
    return p["m_tiles"] * p["n_tiles"] * p["splits"]


@pytest.mark.parametrize("case", CONFIG2)
def test_plan_config2_shapes(case):
    *shape, want_splits = case
    p = capi.conv_tc_plan(_desc(*shape), SMS)
    units = _units(p)
    assert p["splits"] == want_splits, p
    assert 1 <= p["grid"] <= SMS and p["grid"] == min(units, SMS)
    assert p["chunks"] == shape[6][0] * shape[6][1] * shape[6][2] * shape[4] // 32
    if p["splits"] > 1:
        assert p["chunks"] // p["splits"] >= 4                                   # every unit keeps a few chunks of K
        assert p["splits"] * p["m_tiles"] * p["n_tiles"] * 128 * p["nt"] * 4 <= WS
        waves = -(-units // p["grid"])
        assert units / (waves * p["grid"]) >= 0.8, p                             # a split exists to fill the SMs


@pytest.mark.parametrize("case", CONFIG2)
def test_plan_without_split(case):
    """tc_splitk = 0, or no workspace, never splits; the persistent grid is still min(tiles, SMs)."""
    *shape, _ = case
    for p in (capi.conv_tc_plan(_desc(*shape), SMS, splitk=0), capi.conv_tc_plan(_desc(*shape, ws=0), SMS)):
        assert p["splits"] == 1
        assert p["grid"] == min(p["m_tiles"] * p["n_tiles"], SMS)


def test_plan_workspace_bounds_the_split():
    d = _desc(32, 1, 12, 12, 2048, 256, (1, 2, 2), 1, ws=2 * 72 * 128 * 128 * 4)
    assert capi.conv_tc_plan(d, SMS)["splits"] <= 2


@pytest.mark.parametrize("sms", [1, 7, 66, 132, 1000])
def test_plan_grid_never_exceeds_sms_or_units(sms):
    for case in CONFIG2:
        p = capi.conv_tc_plan(_desc(*case[:-1]), sms)
        assert 1 <= p["grid"] <= min(sms, _units(p))
