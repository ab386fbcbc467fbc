"""Host-side plan of the chained bottleneck launch (lt_conv_tc_chain_plan / lt_conv_tc_chain_deps), no GPU needed.

The dependency lists the kernel waits on are computed by the same function on the host.  Checked here: every unit waits only for
units with smaller numbers; the tiles it waits for are exactly the tiles its receptive field reads (restated from the M-tile box);
every write-after-read hazard of the rotating intermediate buffers is covered by the dependencies, transitively; and any number of
CTAs taking units in order finishes whatever order the units complete in."""
import random
from functools import lru_cache

import pytest

from lt_b200 import capi, engine as eng

# (N, H, W, planes, blocks): config #2 (ResNet-152, 4 views x batch 8 at 384^2) layers 3 and 2, ResNet-50 layers 3 and 2, and grids
# with partial tiles along every axis
SHAPES = {
    "cfg2 layer3": (32, 24, 24, 256, 35),
    "cfg2 layer2": (32, 48, 48, 128, 7),
    "r50 layer3": (32, 24, 24, 256, 5),
    "r50 layer2": (32, 48, 48, 128, 3),
    "20x12 partial": (1, 12, 20, 256, 2),
    "7x13 batch 3": (3, 7, 13, 128, 3),
    "1x1 batch 5": (5, 1, 1, 128, 2),
}


def descs(N, H, W, planes):
    def d(cin, cout, k, p, res):
        return eng.conv_desc(N, (1, H, W), cin, cout, (1, k, k), (1, 1, 1), (0, p, p), (1, H, W), (1, H, W), cout, capi.FMT_S32,
                             capi.FMT_S32, relu=True, res_mode=res)
    return [d(4 * planes, planes, 1, 0, capi.RES_NONE), d(planes, planes, 3, 1, capi.RES_NONE),
            d(planes, 4 * planes, 1, 0, capi.RES_BEFORE_RELU)]


def pick_box(OW, OH, OD, N):
    """conv_tc.cu's pick_box: the power-of-two (bw, bh, bd, bn) box of 128 positions that pads the grid least, wider rows first."""
    p2 = lambda v: 1 << (v - 1).bit_length()
    cdiv = lambda a, b: -(-a // b)
    best, box = None, None
    bw = 1
    while bw <= 128:
        bh = 1
        while bw * bh <= 128:
            bd = 1
            while bw * bh * bd <= 128:
                bn = 128 // (bw * bh * bd)
                if not (bw > p2(OW) or bh > p2(OH) or bd > p2(OD) or bn > p2(N)):
                    score = cdiv(OW, bw) * bw * cdiv(OH, bh) * bh * cdiv(OD, bd) * bd * cdiv(N, bn) * bn * (1.0 + 1e-3 / bw)
                    if best is None or score < best:
                        best, box = score, (bw, bh, bd, bn)
                bd *= 2
            bh *= 2
        bw *= 2
    if box is None:   # no box fits the grid: rows of min(p2(OW), 128) positions
        bw = min(p2(OW), 128)
        box = (bw, 1, 1, 128 // bw)
    return box


class Chain:
    def __init__(self, name):
        N, H, W, planes, self.blocks = SHAPES[name]
        self.N, self.H, self.W = N, H, W
        self.d = descs(N, H, W, planes)
        self.plan = capi.conv_tc_chain_plan(self.d, self.blocks, 132)
        self.box = pick_box(W, H, 1, N)
        bw, bh, _, bn = self.box
        self.tw, self.th, self.tn = -(-W // bw), -(-H // bh), -(-N // bn)
        assert self.plan["m_tiles"] == self.tw * self.th * self.tn
        self.nt = self.plan["n_tiles"]
        self.upb = self.plan["m_tiles"] * sum(self.nt)

    def unit(self, layer, m, n):
        k, c = divmod(layer, 3)
        return k * self.upb + self.plan["m_tiles"] * sum(self.nt[:c]) + m * self.nt[c] + n

    @lru_cache(maxsize=None)
    def deps(self, layer, m):
        """(src layer, need, tiles) of (layer, M tile m), from the planner."""
        u = self.unit(layer, m, 0)
        L, mm, n, src, need, tiles = capi.conv_tc_chain_deps(self.d, self.blocks, u)
        assert (L, mm, n) == (layer, m, 0)
        return src, need, frozenset(tiles)

    def reads(self, layer, m):
        """M tiles of its input that (layer, tile m) reads, from the box: output positions inside the grid, input positions
        inside the grid (the rest is zero padding)."""
        bw, bh, _, bn = self.box
        r = 1 if layer % 3 == 1 else 0
        tw0, th0, tn0 = m % self.tw, (m // self.tw) % self.th, m // (self.tw * self.th)
        out = set()
        for y in range(th0 * bh, min((th0 + 1) * bh, self.H)):
            for x in range(tw0 * bw, min((tw0 + 1) * bw, self.W)):
                for iy in range(max(y - r, 0), min(y + r, self.H - 1) + 1):
                    for ix in range(max(x - r, 0), min(x + r, self.W - 1) + 1):
                        out.add((tn0 * self.th + iy // bh) * self.tw + ix // bw)
        return out


@pytest.mark.parametrize("name", list(SHAPES))
def test_plan_counts(name):
    c = Chain(name)
    p = c.plan
    assert p["n_tiles"] == [c.d[0].Cout // 128, c.d[1].Cout // 128, c.d[2].Cout // 128]
    assert p["units"] == c.blocks * c.upb and p["grid"] == min(p["units"], 132)
    assert p["counters"] == 1 + 3 * c.blocks * p["m_tiles"]
    if name == "cfg2 layer3":
        assert p["m_tiles"] == 144 and p["units"] == 35 * 144 * 12


@pytest.mark.parametrize("name", list(SHAPES))
def test_deps_are_the_receptive_field_and_come_first(name):
    c = Chain(name)
    for layer in range(3 * min(c.blocks, 3)):
        for m in range(c.plan["m_tiles"]):
            src, need, tiles = c.deps(layer, m)
            if layer == 0:
                assert src == -1 and not tiles
                continue
            assert src == layer - 1 and need == c.nt[(layer - 1) % 3]
            assert tiles == c.reads(layer, m), (layer, m)
            first = c.unit(layer, m, 0)
            assert all(c.unit(src, t, n) < first for t in tiles for n in range(need))
    # the last units of a long chain decode to the right layer too
    last = c.plan["units"] - 1
    assert capi.conv_tc_chain_deps(c.d, c.blocks, last)[:3] == (3 * c.blocks - 1, c.plan["m_tiles"] - 1, c.nt[2] - 1)


def _ancestors_reach(c, start, targets, floor):
    """Every (layer, tile) of `targets` completes before `start` may begin: reachable through the dependency lists (layers >= floor)."""
    seen, stack, left = set(), [start], set(targets)
    while stack and left:
        layer, m = stack.pop()
        src, _, tiles = c.deps(layer, m)
        if src < floor:
            continue
        for t in tiles:
            if (src, t) not in seen:
                seen.add((src, t))
                left.discard((src, t))
                stack.append((src, t))
    return not left


@pytest.mark.parametrize("name", list(SHAPES))
def test_buffer_hazards_are_covered(name):
    """Layer (k, 0) writes Y1[k % 2], (k, 1) Y2[k % 2], (k, 2) the block input X in place.  Before a unit overwrites a tile, every unit
    that reads the tile's previous contents has finished: (k - 2, 1) halo readers of Y1, (k - 2, 2) of Y2, (k, 0) of X."""
    c = Chain(name)
    blocks = min(c.blocks, 5)
    for k in range(blocks):
        for m in range(c.plan["m_tiles"]):
            if k >= 2:
                readers = {(3 * (k - 2) + 1, t) for t in range(c.plan["m_tiles"]) if m in c.reads(3 * (k - 2) + 1, t)}
                assert _ancestors_reach(c, (3 * k, m), readers, 3 * (k - 2) + 1), ("Y1", k, m)
                assert _ancestors_reach(c, (3 * k + 1, m), {(3 * (k - 2) + 2, m)}, 3 * (k - 2) + 2), ("Y2", k, m)
            assert _ancestors_reach(c, (3 * k + 2, m), {(3 * k, m)}, 3 * k), ("X", k, m)


@pytest.mark.parametrize("name,blocks,ctas", [("cfg2 layer3", 3, 132), ("cfg2 layer3", 3, 5), ("20x12 partial", 2, 3),
                                              ("7x13 batch 3", 3, 1), ("1x1 batch 5", 2, 2)])
def test_random_completion_orders_never_stall(name, blocks, ctas):
    """`ctas` workers take units in order from one counter; a taken unit starts once its dependencies are complete and completes at a
    random time after that.  Every run finishes."""
    c = Chain(name)
    units = c.upb * blocks
    done = {}   # (layer, tile) -> N tiles stored
    decode = {}
    for layer in range(3 * blocks):
        for m in range(c.plan["m_tiles"]):
            for n in range(c.nt[layer % 3]):
                decode[c.unit(layer, m, n)] = (layer, m)
    rng = random.Random(7)
    for trial in range(3):
        done.clear()
        nxt, busy = 0, []
        while nxt < units and len(busy) < ctas:
            busy.append(nxt)
            nxt += 1
        finished = 0
        while busy:
            ready = []
            for u in busy:
                layer, m = decode[u]
                src, need, tiles = c.deps(layer, m)
                if src < 0 or all(done.get((src, t), 0) >= need for t in tiles):
                    ready.append(u)
            assert ready, "stall with units %s in flight" % busy
            u = rng.choice(ready)
            busy.remove(u)
            done[decode[u]] = done.get(decode[u], 0) + 1
            finished += 1
            if nxt < units:
                busy.append(nxt)
                nxt += 1
        assert finished == units


def test_rejects_what_it_cannot_chain():
    d = descs(4, 12, 12, 128)
    with pytest.raises(RuntimeError):
        capi.conv_tc_chain_plan(d, 37, 132)        # more blocks than one launch's parameter block holds
    bad = descs(4, 12, 12, 128)
    bad[1].sh = bad[1].sw = 2
    with pytest.raises(RuntimeError):
        capi.conv_tc_chain_plan(bad, 2, 132)
    bad = descs(4, 12, 12, 64)                     # N tile 64
    with pytest.raises(RuntimeError):
        capi.conv_tc_chain_plan(bad, 2, 132)
    bad = descs(4, 12, 12, 128)
    bad[0].residual = capi.RES_BEFORE_RELU
    with pytest.raises(RuntimeError):
        capi.conv_tc_chain_plan(bad, 2, 132)
