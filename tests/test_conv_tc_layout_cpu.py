"""Shared-memory layout of the persistent tensor-core conv as lt_conv_tc_plan exports it (operand ring stages, epilogue tile buffers)
at the config #2 layer shapes, no GPU needed.  Launches that stage their epilogue (no K split, N tile of 32 or more) take two tile
buffers when a unit has at most 4 K chunks and one otherwise; the ring gets the rest of the 224 KB budget."""
import pytest

from lt_b200 import capi
from test_conv_tc_plan import CONFIG2, SMS, _desc

BUDGET = 224 * 1024
A_TILE = 128 * 128            # one ring stage holds this A box plus Nt x 128 bytes of B
SLAB = 128 * 128              # one 32-channel slab of an epilogue tile buffer
SHORT_K = 4                   # conv_tc.cu kTcShortK
STAGES = {(128, 2): 3, (64, 2): 6, (32, 2): 8, (128, 1): 5, (64, 1): 8, (32, 1): 8}   # ring stages beside (nt, tile buffers)


def _layout_bytes(p):
    return p["stages"] * (A_TILE + p["nt"] * 128) + p["epi_buffers"] * p["nt"] // 32 * SLAB


@pytest.mark.parametrize("case", CONFIG2)
def test_layout_config2_shapes(case):
    p = capi.conv_tc_plan(_desc(*case[:-1]), SMS)
    if p["splits"] == 1 and p["nt"] >= 32:
        assert p["epi_buffers"] == (2 if p["chunks"] <= SHORT_K else 1), p
        assert p["stages"] == STAGES[p["nt"], p["epi_buffers"]], p
    else:
        assert p["epi_buffers"] == 0, p
        assert p["stages"] == min(8, BUDGET // (A_TILE + p["nt"] * 128)), p
    assert 3 <= p["stages"] <= 8 and _layout_bytes(p) <= BUDGET, p


def test_config2_has_launches_on_both_sides_of_the_threshold():
    """The backbone's 1x1 expansions with 2 and 4 K chunks (layer 1 64 -> 256, layer 2 128 -> 512) stage their epilogue in two
    buffers; layer 3's 256 -> 1024 (8 chunks) and the long 3x3 layers keep one buffer and the deeper ring."""
    two = [(32, 1, 96, 96, 64, 256, (1, 1, 1), 1), (32, 1, 48, 48, 128, 512, (1, 1, 1), 1)]
    one = [(32, 1, 24, 24, 256, 1024, (1, 1, 1), 1), (32, 1, 24, 24, 256, 256, (1, 3, 3), 1), (32, 1, 24, 24, 1024, 256, (1, 1, 1), 1)]
    for shape in two:
        p = capi.conv_tc_plan(_desc(*shape), SMS)
        assert p["nt"] == 128 and p["splits"] == 1 and p["epi_buffers"] == 2 and p["stages"] == 3, p
    for shape in one:
        p = capi.conv_tc_plan(_desc(*shape), SMS)
        assert p["nt"] == 128 and p["splits"] == 1 and p["epi_buffers"] == 1 and p["stages"] == 5, p


@pytest.mark.parametrize("cin,buffers", [(32, 2), (128, 2), (160, 1), (256, 1)])
def test_threshold_on_chunks_per_unit(cin, buffers):
    p = capi.conv_tc_plan(_desc(32, 1, 24, 24, cin, 256, (1, 1, 1), 1), SMS)
    assert p["chunks"] == cin // 32 and p["epi_buffers"] == buffers, p


@pytest.mark.parametrize("case", CONFIG2)
def test_layout_without_split(case):
    """Without a split-K workspace every launch of N tile 32 or more stages its epilogue."""
    p = capi.conv_tc_plan(_desc(*case[:-1], ws=0), SMS)
    assert p["splits"] == 1
    assert p["epi_buffers"] == (0 if p["nt"] < 32 else 2 if p["chunks"] <= SHORT_K else 1), p
    assert _layout_bytes(p) <= BUDGET, p
