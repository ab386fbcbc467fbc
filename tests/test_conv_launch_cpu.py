"""engine.launch_conv without a GPU: the C ABI is stubbed and every lt_conv_nd_fwd call recorded, so each test sees the kernel, filter,
Cout, scale and split-K scratch that one launch of a packed filter would get.  The fold choice is checked against the
conv_fold_supported mirror of test_conv_cpu."""
import pytest
import torch

from lt_b200 import capi, engine as eng_mod
from test_conv_cpu import Launch, fold_supported

S32, F32 = capi.FMT_S32, capi.FMT_F32


@pytest.fixture
def launches(monkeypatch):
    got = []
    monkeypatch.setattr(capi, "lib", lambda: None)
    monkeypatch.setattr(capi, "conv_nd", lambda d, x, w, scale, shift, res, out, impl: got.append((d, w, scale, shift, impl)))
    return got


def pack(k, cout, fold, cin=32, stride=(1, 1, 1), groups=1):
    """A ConvPack as pack_filter lays one out for the tensor-core modes; scale and scale_fold hold different values."""
    pk = eng_mod.ConvPack()
    pk.k, pk.stride, pk.pad = k, stride, tuple(kk // 2 for kk in k)
    pk.taps, pk.cin, pk.cout, pk.groups = k[0] * k[1] * k[2], cin, cout, groups
    pk.cout_p = eng_mod._round_up(cout, 32)
    pk.impl, pk.in_fmt, pk.kmacs = capi.CONV_TC, S32, pk.taps * cin * cout
    pk.w = torch.zeros(pk.taps * cin * pk.cout_p * 2, dtype=torch.float16)
    pk.scale = torch.arange(1, pk.cout_p + 1, dtype=torch.float32)
    pk.shift = torch.zeros(pk.cout_p)
    pk.w_fold = torch.zeros(k[0] ** 3 * 32 * 64, dtype=torch.float16) if fold else None
    pk.scale_fold = pk.scale + 0.5 if fold else pk.scale
    return pk


def x_act(dims, cin=32, N=1):
    return eng_mod.Act(N, *dims, cin, S32, "cpu")


def mirror_fold(d, pk):
    """conv_fold_supported (test_conv_cpu.fold_supported) of the recorded descriptor, for a pack that has a fold filter."""
    L = Launch(d.N, (d.ID, d.IH, d.IW), (d.OD, d.OH, d.OW), (d.KD, d.KH, d.KW), (d.sd, d.sh, d.sw), (d.pd, d.ph, d.pw),
               (d.FD, d.FH, d.FW), (d.osd, d.osh, d.osw), (d.ood, d.ooh, d.oow), (d.ogd, d.ogh, d.ogw), d.Cout, d.FC)
    return pk.w_fold is not None and fold_supported(L, d.Cin, pk.cout, d.in_format)


def check(launch, pk, fold, inv=None):
    d, w, scale, shift, impl = launch
    assert impl == (capi.CONV_TC_FOLD if fold else capi.CONV_TC)
    assert (impl == capi.CONV_TC_FOLD) == mirror_fold(d, pk)
    assert w is (pk.w_fold if fold else pk.w)
    assert d.Cout == (pk.cout if fold else pk.cout_p)
    want = pk.scale_fold if fold else pk.scale
    if inv is None:
        assert scale is want
    else:
        assert torch.equal(scale, want * inv)
    assert shift is pk.shift
    assert d.workspace_bytes == eng_mod.SPLITK_WS_BYTES and d.workspace == eng_mod.splitk_workspace(torch.device("cpu")).data_ptr()


@pytest.mark.parametrize("inv", [None, torch.tensor([0.375])])
@pytest.mark.parametrize("k,W,fold", [(3, 15, False), (3, 16, True), (3, 64, True), (3, 65, False), (7, 16, True), (7, 80, True)])
def test_fold_packed_layer_width(launches, k, W, fold, inv):
    """3^3 layers run on the lines kernel for 16 <= W <= 64, 7^3 layers on conv_fold_kernel from W 16; both on conv_tc_kernel
    otherwise.  With scale_mul (a data gradient's 1 / S) the launch gets the chosen scale times it."""
    pk = pack((k, k, k), 32 if k == 3 else 16, fold=True)
    dims = (4, 5, W)
    out = eng_mod.Act(1, *dims, 32, S32, "cpu")
    impl = eng_mod.launch_conv(x_act(dims), pk, out, scale_mul=inv)
    assert impl == launches[0][4]
    check(launches[0], pk, fold, inv)


@pytest.mark.parametrize("fc,fold", [(32, True), (16, False)])
def test_fold_needs_a_32_channel_output(launches, fc, fold):
    """A 32 -> 16 layer writing a 16-wide float32 map (the training convs' width) stays on conv_tc_kernel."""
    pk = pack((3, 3, 3), 16, fold=True)
    dims = (4, 4, 32)
    eng_mod.launch_conv(x_act(dims), pk, eng_mod.Act(1, *dims, fc, F32, "cpu"))
    check(launches[0], pk, fold)


def test_scaled_output_is_not_folded(launches):
    """An output scale of 2 (a phase of a strided data gradient) takes conv_tc_kernel even for a fold-packed filter."""
    pk = pack((3, 3, 3), 32, fold=True)
    dims = (4, 5, 32)
    out = eng_mod.Act(1, 4, 10, 64, 32, F32, "cpu")
    eng_mod.launch_conv(x_act(dims), pk, out, out_scale=(1, 2, 2), out_off=(0, 1, 0), scale_mul=torch.tensor([2.0]))
    d = launches[0][0]
    assert (d.osd, d.osh, d.osw, d.ood, d.ooh, d.oow) == (1, 2, 2, 0, 1, 0) and (d.FD, d.FH, d.FW, d.FC) == (4, 10, 64, 32)
    check(launches[0], pk, False, torch.tensor([2.0]))


def test_grouped_output(launches):
    """The merged k2 s2 transposed conv: one 1x1x1 launch, N = 8 Cout, each block to its phase of the doubled grid."""
    pk = pack((1, 1, 1), 8 * 32, fold=False, cin=64, groups=8)
    x = x_act((2, 3, 4), cin=64, N=2)
    y = eng_mod.deconv3d_k2s2(x, pk, S32, relu=True)
    assert (y.N, y.D, y.H, y.W, y.C) == (2, 4, 6, 8, 32)
    d = launches[0][0]
    assert (d.OD, d.OH, d.OW, d.ogd, d.ogh, d.ogw, d.osd, d.osh, d.osw) == (2, 3, 4, 2, 2, 2, 2, 2, 2) and d.relu == 1
    assert d.residual == capi.RES_NONE and d.out_format == S32
    check(launches[0], pk, False)


def test_empty_workspace_forces_a_single_pass(launches):
    pk = pack((3, 3, 3), 32, fold=False)
    dims = (2, 2, 2)
    eng_mod.launch_conv(x_act(dims), pk, eng_mod.Act(1, *dims, 32, S32, "cpu"), workspace=torch.empty(0, dtype=torch.uint8))
    assert launches[0][0].workspace_bytes == 0
