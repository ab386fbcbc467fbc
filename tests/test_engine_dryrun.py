"""Host-side planner logic without a GPU: run NativeEngine with the C-ABI launches replaced by a recorder that
re-checks every descriptor the way capi.cu validates it (shapes, output mapping bounds, formats)."""
import numpy as np
import pytest
import torch

import lt_b200
from lt_b200 import capi, engine as eng_mod, testing


class Recorder:
    def __init__(self):
        self.calls = []

    def install(self, monkeypatch):
        def rec(name):
            def f(*a, **k):
                self.calls.append((name, a))
            return f
        monkeypatch.setattr(capi, "conv_fold_weight_bytes", lambda k, co: k * k * k * ((co + 15) // 16 * 16) * 64 * 2)
        monkeypatch.setattr(capi, "conv_pair_weight_bytes", lambda t, ci, co: t * (ci // 32) * ((co + 127) // 128 * 128) * 128)
        # stand-in for lt_conv_pair_eligible (Cout % 128 == 0, output wide enough): the dry run loads no library
        monkeypatch.setattr(capi, "conv_pair_eligible", lambda d: d.Cout % 128 == 0 and d.FC % 32 == 0 and d.Cout <= d.FC and
                            d.N * d.OD * d.OH * d.OW >= 128 * 40)
        for name in ("v2v_tail", "absmax", "conv_gather_weights", "fold_bn", "conv_pair_pack_weights", "conv_fold_pack_weights", "stem_s2d", "coord_volume", "unproject_aggregate", "softargmax3d", "maxpool", "nchw_to_nhwc", "f32_to_s32",
                     "s32_to_f32", "cl_to_cf", "conv_tc_pack_weights"):
            monkeypatch.setattr(capi, name, rec(name))
        def tail_stats(*a, **k):
            self.calls.append(("v2v_tail_stats", a))
            return 444
        monkeypatch.setattr(capi, "v2v_tail_stats", tail_stats)
        monkeypatch.setattr(capi, "softargmax3d_finish", rec("softargmax3d_finish"))
        monkeypatch.setattr(capi, "lib", lambda: None)
        monkeypatch.setattr(capi, "conv_tc_weight_bytes", lambda t, ci, co: t * (ci // 32) * ((co + 15) // 16 * 16) * 64 * 2)
        monkeypatch.setattr(capi, "softargmax3d_workspace_bytes", lambda B, J, n: B * J * ((n + 2047) // 2048 * 5 + 2) * 4)
        monkeypatch.setattr(capi, "conv_nd", self.conv_nd)

    def conv_nd(self, d, x, w, scale, shift, res, out, impl):
        # mirror of the argument checks in csrc/capi.cu + conv_simt.cu + conv_tc.cu
        assert (d.OD - 1) * d.osd + d.ood < d.FD and (d.OH - 1) * d.osh + d.ooh < d.FH and (d.OW - 1) * d.osw + d.oow < d.FW
        assert d.FC % 4 == 0
        elems_in = d.N * d.ID * d.IH * d.IW * d.Cin * (2 if d.in_format == capi.FMT_S32 else 1)
        assert x.numel() == elems_in, (x.shape, elems_in)
        elems_out = d.N * d.FD * d.FH * d.FW * d.FC * (2 if d.out_format == capi.FMT_S32 else 1)
        assert out.numel() == elems_out
        if res is not None:
            assert res.numel() == elems_out and res.dtype == out.dtype
        if impl == capi.CONV_TC_FOLD:
            assert d.Cin == 32 and d.FC == 32 and d.Cout <= 32 and d.IW >= 16 and d.KD == d.KH == d.KW and d.KW in (3, 7)
            assert w.numel() == d.KW ** 3 * ((d.Cout + 15) // 16 * 16) * 64
        elif impl == capi.CONV_TC_PAIR:
            assert d.in_format == capi.FMT_S32 and x.dtype == torch.float16 and d.Cin % 32 == 0 and d.Cout % 128 == 0
            assert w.numel() == d.KD * d.KH * d.KW * (d.Cin // 32) * d.Cout * 64 and scale.numel() >= d.Cout
            assert d.FC % 32 == 0 and d.Cout >= d.FC
        elif impl == capi.CONV_SIMT:
            assert d.in_format == capi.FMT_F32 and x.dtype == torch.float32
            cw = (d.Cout + 3) // 4 * 4
            assert w.numel() == d.KD * d.KH * d.KW * d.Cin * cw and scale.numel() >= cw
        else:
            assert d.in_format == capi.FMT_S32 and x.dtype == torch.float16
            assert d.Cin % 32 == 0
            cp = (d.Cout + 15) // 16 * 16
            assert w.numel() == d.KD * d.KH * d.KW * (d.Cin // 32) * cp * 64 and scale.numel() >= cp
            assert cp <= 128 or cp % 128 == 0
            if d.out_format == capi.FMT_S32:
                assert d.FC % 32 == 0 and cp >= d.FC, "padding channels of a split-fp16 output must be written"
        self.calls.append(("conv_nd", (impl, d.Cin, d.Cout, (d.KD, d.KH, d.KW))))


@pytest.mark.parametrize("mode", ["simt", "tc"])
@pytest.mark.parametrize("layers", [18, 50])
def test_engine_plan_is_consistent(monkeypatch, mode, layers):
    rec = Recorder()
    rec.install(monkeypatch)
    cfg = testing.make_config(num_layers=layers, volume_size=32)
    model = lt_b200.VolumetricTriangulationNet(cfg, device="cpu", backend="native", conv_mode=mode, use_cuda_graph=False).eval()
    e = eng_mod.NativeEngine(model, mode=mode, use_graph=False)
    B, V, S = 2, 2, 64
    images = torch.zeros(B, V, 3, S, S)
    z3 = torch.zeros(B, 3)
    kp, feats, vols, coord = e.forward(images, torch.zeros(B, V, 3, 4), z3, z3, torch.zeros(3), torch.zeros(B, 9))
    assert tuple(kp.shape) == (B, 17, 3) and tuple(vols.shape) == (B, 17, 32, 32, 32)
    assert tuple(feats.shape) == (B, V, 32, S // 4, S // 4) and tuple(coord.shape) == (B, 32, 32, 32, 3)
    convs = [c for c in rec.calls if c[0] == "conv_nd"]
    n_units = {18: 8, 50: 16}[layers]
    per_unit = 2 if layers == 18 else 3
    # stem + trunk convs + 3 (or 4) downsamples + 3 deconvs x 4 phases + process_features
    n_ds = 3 if layers == 18 else 4
    backbone = 1 + n_units * per_unit + n_ds + 12 + 1
    # V2V: front0 + 20 res blocks (2 convs each) + 4 skip convs (16->32, 32->64, 64->128 enc, none else) ...
    v2v = len(convs) - backbone
    tail = sum(1 for c in rec.calls if c[0] in ("v2v_tail", "v2v_tail_stats"))      # tc mode: back1 + back2 + output fused into one launch
    # 32^3 volumes: the fused tail also carries the soft-argmax statistics pass, the soft-argmax itself is merge + normalise (2 launches)
    assert sum(1 for c in rec.calls if c[0] == "softargmax3d_finish") == (1 if mode == "tc" else 0)
    assert tail == (1 if mode == "tc" else 0)
    up = 5 * (1 if mode == "tc" else 8)     # tc: each k2 s2 transposed conv is one grouped-output GEMM; simt: eight phase convs
    assert v2v == 1 + 20 * 2 + 3 + up + (0 if tail else 2 + 1), v2v
    assert e.launches == len(rec.calls) - sum(1 for c in rec.calls if c[0] in ("conv_tc_pack_weights", "conv_fold_pack_weights", "conv_pair_pack_weights", "conv_gather_weights", "fold_bn", "absmax")) + (1 if tail else 2)   # softargmax = 3 launches (2 behind the fused tail)
    if mode == "tc":
        simt = [c for c in convs if c[1][0] == capi.CONV_SIMT]
        assert len(simt) == 0, "every conv runs on the tensor-core kernels"
