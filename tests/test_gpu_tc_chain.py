"""The chained bottleneck launch (lt_conv_tc_chain_fwd) against the per-layer launches it replaces, bit for bit.

Each block is 1x1 reduce + ReLU, 3x3 + ReLU, 1x1 expansion + residual before ReLU, all split-fp16.  The per-layer path runs the three
lt_conv_nd_fwd launches per block without split-K (the chain is only used where the per-layer plan does not split).  Every output
and intermediate buffer sits between NaN-filled guard bands that must survive, and both paths read the same packed filters."""
import numpy as np
import pytest
import torch

from lt_b200 import capi, engine as eng

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 4096   # fp16 elements of NaN before and after every tensor the chain writes


def guarded(n):
    """(whole NaN-filled buffer, its middle n fp16 elements)."""
    big = torch.full((n + 2 * GUARD,), float("nan"), dtype=torch.float16, device=DEV)
    return big, big[GUARD:GUARD + n]


def s32(x32, pixels, C):
    out = torch.empty(pixels * 2 * C, dtype=torch.float16, device=DEV)
    capi.f32_to_s32(x32, out, pixels, C)
    return out


def make_layers(blocks, planes, seed):
    g = torch.Generator().manual_seed(seed)
    shapes = [(1, 4 * planes, planes), (9, planes, planes), (1, planes, 4 * planes)]
    layers = []
    for _ in range(blocks):
        for taps, cin, cout in shapes:
            w = (torch.randn(taps, cin, cout, generator=g) * (0.7 / np.sqrt(taps * cin))).to(DEV)
            packed = torch.empty(capi.conv_tc_weight_bytes(taps, cin, cout) // 2, dtype=torch.float16, device=DEV)
            capi.conv_tc_pack_weights(w.contiguous(), packed, taps, cin, cout)
            scale = (0.5 + torch.rand(cout, generator=g)).to(DEV)
            shift = (0.1 * torch.randn(cout, generator=g)).to(DEV)
            layers.append((packed, scale, shift))
    return layers


def descs(N, H, W, planes):
    def d(cin, cout, k, p, res):
        return eng.conv_desc(N, (1, H, W), cin, cout, (1, k, k), (1, 1, 1), (0, p, p), (1, H, W), (1, H, W), cout, capi.FMT_S32,
                             capi.FMT_S32, relu=True, res_mode=res)
    return [d(4 * planes, planes, 1, 0, capi.RES_NONE), d(planes, planes, 3, 1, capi.RES_NONE),
            d(planes, 4 * planes, 1, 0, capi.RES_BEFORE_RELU)]


def per_layer(x, d, layers, blocks, N, H, W, planes, impl):
    P = N * H * W
    for k in range(blocks):
        y1 = torch.empty(P * 2 * planes, dtype=torch.float16, device=DEV)
        y2 = torch.empty_like(y1)
        out = torch.empty(P * 2 * 4 * planes, dtype=torch.float16, device=DEV)
        (w0, s0, h0), (w1, s1, h1), (w2, s2, h2) = layers[3 * k:3 * k + 3]
        capi.conv_nd(d[0], x, w0, s0, h0, None, y1, impl)
        capi.conv_nd(d[1], y1, w1, s1, h1, None, y2, impl)
        capi.conv_nd(d[2], y2, w2, s2, h2, x, out, impl)
        x = out
    return x


# (blocks, N, H, W, planes)
CASES = {
    "1 block batch 1": (1, 1, 24, 24, 256),
    "2 blocks batch 32": (2, 32, 24, 24, 256),
    "35 blocks batch 32 (config #2 layer 3)": (35, 32, 24, 24, 256),
    "3 blocks 20x12 partial tiles": (3, 1, 12, 20, 256),
    "2 blocks 13x7 batch 3 planes 128": (2, 3, 7, 13, 128),
}


@pytest.mark.parametrize("impl", [capi.CONV_TC, capi.CONV_TC1])
@pytest.mark.parametrize("name", list(CASES))
def test_chain_matches_per_layer_launches(name, impl):
    blocks, N, H, W, planes = CASES[name]
    if impl == capi.CONV_TC1 and blocks > 2:
        pytest.skip("one long chain per product count is enough")
    P, C = N * H * W, 4 * planes
    d = descs(N, H, W, planes)
    layers = make_layers(blocks, planes, seed=blocks * 1000 + N)
    x32 = torch.randn(P, C, generator=torch.Generator().manual_seed(5)).clamp_(min=0).to(DEV)
    x0 = s32(x32, P, C)
    ref = per_layer(x0.clone(), d, layers, blocks, N, H, W, planes, impl)

    xbig, x = guarded(P * 2 * C)
    x.copy_(x0)
    bigs, bufs = zip(*[guarded(P * 2 * planes) for _ in range(4)])
    plan = capi.conv_tc_chain_plan(d, blocks, torch.cuda.get_device_properties(0).multi_processor_count)
    cbig, counters = guarded(2 * plan["counters"])
    counters = counters.view(torch.int32)
    capi.conv_tc_chain(d, blocks, x, list(bufs), [l[0] for l in layers], [l[1] for l in layers], [l[2] for l in layers], counters, impl)
    torch.cuda.synchronize()
    assert torch.isfinite(ref.float()).all()
    assert torch.equal(x.view(torch.int16), ref.view(torch.int16)), name
    for big in (xbig, cbig) + bigs:
        assert torch.isnan(big[:GUARD].float()).all() and torch.isnan(big[-GUARD:].float()).all(), "a guard band was written"
    # every (layer, M tile) counter reached its N tiles; the dispenser handed out every unit once per CTA beyond the last
    cnt = counters.cpu().numpy().astype(np.int64)
    assert cnt[0] == plan["units"] + plan["grid"]
    assert (cnt[1:].reshape(3 * blocks, plan["m_tiles"]) == np.tile(plan["n_tiles"], blocks)[:, None]).all()


def test_chain_repeats_and_graph_replays_bit_identically():
    blocks, N, H, W, planes = 4, 8, 24, 24, 256
    P, C = N * H * W, 4 * planes
    d = descs(N, H, W, planes)
    layers = make_layers(blocks, planes, seed=3)
    x0 = s32(torch.rand(P, C, generator=torch.Generator().manual_seed(1)).to(DEV), P, C)
    bufs = [torch.empty(P * 2 * planes, dtype=torch.float16, device=DEV) for _ in range(4)]
    plan = capi.conv_tc_chain_plan(d, blocks, 132)
    counters = torch.empty(plan["counters"], dtype=torch.int32, device=DEV)
    x = torch.empty_like(x0)

    def run():
        x.copy_(x0)
        capi.conv_tc_chain(d, blocks, x, bufs, [l[0] for l in layers], [l[1] for l in layers], [l[2] for l in layers], counters,
                           capi.CONV_TC)

    run()
    first = x.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            run()
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(3):
        x.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(x.view(torch.int16), first.view(torch.int16))
