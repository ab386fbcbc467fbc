"""Native inference executor for the volumetric path.

Walks the parameter-holding module tree (pose_resnet.PoseResNet, v2v.V2VModel, the 1x1
`process_features` conv) once, folds BatchNorm into per-channel scale/shift, packs the filters
into the layouts the kernels want, and then runs the whole device side of
`VolumetricTriangulationNet.forward` (reference triangulation.py:250-353) as a sequence of
C-ABI launches on the current CUDA stream -- optionally captured into one CUDA graph.

Data layout in HBM: every activation is channels-last ([N][D][H][W][C]); 2-D maps use D = 1.
  mode "simt": float32 activations, exact-fp32 FFMA convs (parity mode / checker)
  mode "tc"  : split-fp16 activations, wgmma convs with 3-term products (fp32-grade)
  mode "tc1" : split-fp16 activations, wgmma convs with high parts only (bf16-grade, fast)
In the tensor-core modes every conv runs on the tensor cores: the 3-channel 7x7 stride-2 stem as a
4x4 stride-1 conv over the 2x2 space-to-depth image, the stride-2 convs through TMA traversal strides.
"""
import math

import torch
from torch import nn

from . import capi
from .capi import FMT_F32, FMT_S32, CONV_SIMT, CONV_TC, CONV_TC1, CONV_TC_FOLD, RES_NONE, RES_BEFORE_RELU, RES_AFTER_RELU


def _round_up(v, m):
    return (v + m - 1) // m * m


def _stream_layout_ok(vs, J, nvox):
    """Logits of voxel stride vs that the streaming soft-argmax kernels read: stream_layout_ok in csrc/softargmax_common.cuh.  The fused
    V2V tail's statistics are merged by those kernels, so the engine fuses only for such a layout."""
    return vs % 4 == 0 and 20 <= vs <= 32 and J <= vs and nvox % 8 == 0 and nvox >= 16384


class Act:
    """Channels-last activation: `data` is float32 [N,D,H,W,C] or bfloat16 [N,D,H,W,2C] (split-fp16)."""
    __slots__ = ("data", "N", "D", "H", "W", "C", "fmt", "stats")

    def __init__(self, N, D, H, W, C, fmt, device, zero=False):
        self.N, self.D, self.H, self.W, self.C, self.fmt = N, D, H, W, C, fmt
        self.stats = None      # (workspace, n_partials): soft-argmax statistics produced together with these logits (fused V2V tail)
        alloc = torch.zeros if zero else torch.empty
        if fmt == FMT_F32:
            self.data = alloc((N, D, H, W, C), dtype=torch.float32, device=device)
        else:
            assert C % 32 == 0
            self.data = alloc((N, D, H, W, 2 * C), dtype=torch.float16, device=device)

    @classmethod
    def view(cls, data):
        """An existing channels-last tensor as an Act, without copying: float32 [N,D,H,W,C] or float16 [N,D,H,W,2C] (split-fp16)."""
        a = cls.__new__(cls)
        a.N, a.D, a.H, a.W, c = data.shape
        a.fmt = FMT_F32 if data.dtype == torch.float32 else FMT_S32
        a.C = c if a.fmt == FMT_F32 else c // 2
        a.data, a.stats = data, None
        return a

    @property
    def pixels(self):
        return self.N * self.D * self.H * self.W


class ConvPack:
    """One (phase of a) convolution, ready to launch: packed filter + folded scale/shift + geometry."""
    __slots__ = ("w", "scale", "shift", "taps", "k", "stride", "pad", "cin", "cout", "cout_p", "impl", "in_fmt", "kmacs", "w_fold", "scale_fold",
                 "groups")


def _f32(t):
    """The module's own tensor as contiguous float32 (no copy for ordinary float32 parameters)."""
    return None if t is None else t.detach().float().contiguous()


class _Timed:
    """CUDA-event bracket around one launch (only when a timeline list is installed; never during graph capture)."""

    def __init__(self, timeline, label, flops, nbytes, desc=""):
        self.tl, self.label, self.flops, self.nbytes, self.desc = timeline, label, flops, nbytes, desc

    def __enter__(self):
        if self.tl is not None:
            self.e0, self.e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *exc):
        if self.tl is not None:
            self.e1.record()
            self.tl.append((self.label, self.flops, self.nbytes, self.e0, self.e1, self.desc))
        return False


_TC_IMPL = {"simt": CONV_SIMT, "tc": CONV_TC, "tc1": CONV_TC1}


def fold_width_ok(k, width):
    """Whether LT_CONV_TC_FOLD takes a layer packed for it at this W: 3^3 (conv_lines_kernel, whole W lines as the m64 rows)
    for 16 <= W <= 64, 7^3 (conv_fold_kernel) for W >= 16.  Wider 3^3 layers run on conv_tc_kernel."""
    return width >= 16 and (k == 7 or width <= 64)


def pack_filter(src, k, stride, pad, cin, cout, bias, bn, mode="tc", cin_pad=None, force_simt=False, out_fmt=None):
    """src = (filter tensor, base, (s_td, s_th, s_tw, s_ci, s_co)): where element (td, th, tw, ci, co) of this (phase of a)
    convolution sits inside the module's own weight tensor.  Everything below is our own kernels: gather to the canonical
    [tap][Cin][Cout] layout (lt_conv_gather_weights_fwd), operand packing, BatchNorm folding (lt_fold_bn_fwd).  mode: the
    engine's conv mode; NativeEngine packs once per parameter version, the training convolutions (autograd_ops) on every call."""
    # a list of sources = column blocks of ONE wider filter (k2 s2 transposed conv: 8 phases side by side along N)
    srcs = src if isinstance(src, list) else [src]
    G = len(srcs)
    w = srcs[0][0]
    dev = w.device
    taps = k[0] * k[1] * k[2]
    act_fmt = FMT_F32 if mode == "simt" else FMT_S32
    out_fmt = act_fmt if out_fmt is None else out_fmt
    pk = ConvPack()
    pk.taps, pk.k, pk.stride, pk.pad, pk.cout, pk.groups = taps, k, stride, pad, G * cout, G
    pk.kmacs = taps * cin * cout * G   # algorithmic MACs per output position
    pk.w_fold = None
    use_tc = (mode != "simt") and not force_simt
    assert G == 1 or (use_tc and cout % 32 == 0), "column blocks need the tensor-core path and 32-channel multiples"
    if use_tc:
        cin_p = _round_up(max(cin, cin_pad or 0), 32)
        cout_p = _round_up(G * cout, 32 if out_fmt == FMT_S32 else 16)
    else:
        cin_p = max(cin, cin_pad or 0)
        cout_p = _round_up(cout, 4)
    blk_p = cout if G > 1 else cout_p
    wp = torch.empty((taps, cin_p, cout_p), dtype=torch.float32, device=dev)
    amax = None
    if use_tc:
        # power-of-two pre-scale of the whole filter tensor (all phases of a transposed conv share it): common.cuh
        amax = torch.empty(1, dtype=torch.int32, device=dev)
        capi.absmax(w, amax)
    for g, (wg, base, strides) in enumerate(srcs):
        capi.conv_gather_weights(wg, base, strides, k, cin, cin_p, cout, blk_p, wp, amax, out_ld=cout_p, out_col0=g * cout)
    if use_tc:
        packed = torch.empty(capi.conv_tc_weight_bytes(taps, cin_p, cout_p) // 2, dtype=torch.float16, device=dev)
        capi.conv_tc_pack_weights(wp, packed, taps, cin_p, cout_p)
        pk.w, pk.cin, pk.cout_p, pk.impl, pk.in_fmt = packed, cin_p, cout_p, _TC_IMPL[mode], FMT_S32
        # narrow cubic stride-1 layers (V2V at full resolution): also pack for the halo-reusing persistent kernel (csrc/conv_fold.cu)
        if (mode == "tc" and cin_p == 32 and cout <= 32 and k[0] == k[1] == k[2] and k[0] in (3, 7)
                and tuple(pad) == (k[0] // 2,) * 3 and max(stride) == 1):
            wf = torch.empty(capi.conv_fold_weight_bytes(k[0], cout) // 2, dtype=torch.float16, device=dev)
            wsrc = wp if cout_p == cout else wp[:, :, :cout].contiguous()
            capi.conv_fold_pack_weights(wsrc, wf, k[0], cout)
            pk.w_fold = wf
    else:
        pk.w, pk.cin, pk.cout_p, pk.impl, pk.in_fmt = wp, cin_p, cout_p, CONV_SIMT, FMT_F32
    # tensor-core accumulation steps on the main fp32 accumulator, which lt_fold_bn_fwd compensates for the expected truncation shrinkage
    # (accum_gain, csrc/common.cuh): one hi*hi MMA per 16 input channels and tap in conv_tc_kernel (its split-K reduce rescales to the
    # steps of one split) and conv_fold_kernel; conv_lines_kernel, the 3^3 layers packed for LT_CONV_TC_FOLD, accumulates each kw column
    # over the 9 (kd, kh) taps and sums the three in fp32.  A fold-packed 3^3 layer keeps both scales: it runs on conv_tc_kernel at
    # widths and output mappings the lines kernel does not take.
    steps = taps * (cin_p // 16) if use_tc else 0
    fold_steps = 9 * (cin_p // 16) if pk.w_fold is not None and k[0] == 3 else steps
    pk.scale, pk.shift = _fold_scale(bn, bias, cout, blk_p, cout_p, G, amax, steps, dev)
    pk.scale_fold = pk.scale if fold_steps == steps else _fold_scale(bn, bias, cout, blk_p, cout_p, G, amax, fold_steps, dev)[0]
    return pk


def _fold_scale(bn, bias, cout, blk_p, cout_p, G, amax, steps, dev):
    """(scale, shift) [cout_p] of lt_fold_bn_fwd for a filter whose kernel accumulates `steps` tensor-core steps per output."""
    scale = torch.empty(cout_p, dtype=torch.float32, device=dev)
    shift = torch.empty(cout_p, dtype=torch.float32, device=dev)
    for g in range(G):     # the per-channel affine repeats for every column block
        sc, sh = scale[g * cout:g * cout + blk_p], shift[g * cout:g * cout + blk_p]
        if bn is not None:
            capi.fold_bn(_f32(bn.weight), _f32(bn.bias), _f32(bn.running_mean), _f32(bn.running_var), _f32(bias), bn.eps, cout, blk_p,
                         sc, sh, amax, accum_steps=steps)
        else:
            capi.fold_bn(None, None, None, None, _f32(bias), 0.0, cout, blk_p, sc, sh, amax, accum_steps=steps)
    return scale, shift


def pack_conv(conv, bn, mode="tc", cin_pad=None, **kw):
    """conv: anything with the nn.Conv2d / nn.Conv3d attributes weight, bias, kernel_size, stride, padding."""
    w = _f32(conv.weight)
    cout, cin = w.shape[:2]
    if w.dim() == 4:   # (Cout, Cin, KH, KW)
        k = (1,) + tuple(conv.kernel_size)
        stride = (1,) + tuple(conv.stride)
        pad = (0,) + tuple(conv.padding)
    else:              # (Cout, Cin, KD, KH, KW)
        k, stride, pad = tuple(conv.kernel_size), tuple(conv.stride), tuple(conv.padding)
    T = k[0] * k[1] * k[2]
    src = (w, 0, (k[1] * k[2], k[2], 1, T, cin * T))
    return pack_filter(src, k, stride, pad, cin, cout, conv.bias, bn, mode=mode, cin_pad=cin_pad, **kw)


def pack_deconv3d_k2s2(deconv, bn, mode="tc"):
    """ConvTranspose3d(k=2, s=2): eight independent 1x1x1 convs scattered to the output parities.

    Tensor-core modes with Cout % 32 == 0: ONE 1x1x1 GEMM with N = 8 x Cout (the phases side by side along N, the epilogue
    writing each 32-channel block to its phase of the output lattice: lt_conv_desc.ogd/ogh/ogw) -- the input is read once
    instead of eight times and a level costs one launch instead of eight."""
    w = _f32(deconv.weight)  # (Cin, Cout, 2, 2, 2)
    cin, cout = w.shape[:2]
    if mode != "simt" and cout % 32 == 0:
        srcs = [(w, a * 4 + b * 2 + c, (0, 0, 0, cout * 8, 8)) for a in (0, 1) for b in (0, 1) for c in (0, 1)]
        return pack_filter(srcs, (1, 1, 1), (1, 1, 1), (0, 0, 0), cin, cout, deconv.bias, bn, mode=mode)
    phases = {}
    for a in (0, 1):
        for b in (0, 1):
            for c in (0, 1):
                src = (w, a * 4 + b * 2 + c, (0, 0, 0, cout * 8, 8))
                phases[(a, b, c)] = pack_filter(src, (1, 1, 1), (1, 1, 1), (0, 0, 0), cin, cout, deconv.bias, bn, mode=mode)
    return phases


def stem_s2d_filter(weight):
    """7x7 stride-2 pad-3 stem filter (Cout, 3, 7, 7) -> canonical [4][4][32][Cout] filter of the equivalent 4x4 stride-1 conv
    (front pad 2) over the 2x2 space-to-depth input (lt_stem_s2d_fwd).

    Input row 2*oy - 3 + ky = 2*(oy + a) + r with a = tap offset in {-2..1}, r = row parity: ky = 2a + r + 3, and likewise kx;
    s2d channel (r*2 + s)*3 + c.  Taps with ky or kx outside [0, 7) and channels 12..31 are zero.  The re-indexing is not affine
    in the s2d channel, so it is a gather on the filter's device (no host round trip)."""
    cout = weight.shape[0]
    dev = weight.device
    a = torch.arange(4, device=dev).view(4, 1, 1)
    b = torch.arange(4, device=dev).view(1, 4, 1)
    ch = torch.arange(32, device=dev).view(1, 1, 32)
    rs, c = ch // 3, ch % 3
    ky, kx = 2 * a + rs // 2 - 1, 2 * b + rs % 2 - 1
    valid = (ch < 12) & (ky >= 0) & (ky < 7) & (kx >= 0) & (kx < 7)
    idx = torch.where(valid, (c * 7 + ky.clamp(0, 6)) * 7 + kx.clamp(0, 6), 0)          # (4, 4, 32) into w[co] flattened
    w = weight.detach().float().reshape(cout, 3 * 49)
    wt = w[:, idx.reshape(-1)].reshape(cout, 4, 4, 32).permute(1, 2, 3, 0)
    return torch.where(valid.unsqueeze(-1), wt, torch.zeros((), dtype=torch.float32, device=dev)).contiguous()


def pack_stem_s2d(conv, bn, mode="tc", **kw):
    """The stem conv as the tensor-core modes run it: stem_s2d_filter packed as a 4x4 stride-1 conv over 32 s2d channels."""
    assert tuple(conv.weight.shape[1:]) == (3, 7, 7) and tuple(conv.stride) == (2, 2) and tuple(conv.padding) == (3, 3)
    cout = conv.weight.shape[0]
    wt = stem_s2d_filter(conv.weight)
    pk = pack_filter((wt, 0, (0, 4 * 32 * cout, 32 * cout, cout, 1)), (1, 4, 4), (1, 1, 1), (0, 2, 2), 32, cout, conv.bias, bn, mode=mode,
                     **kw)
    pk.kmacs = 49 * 3 * cout
    return pk


def deconv2d_k4s2_phase(py, px, cout):
    """Phase (py, px) of ConvTranspose2d(k=4, s=2, p=1) (Cin, Cout, 4, 4) as a 2x2 stride-1 conv: (lt_conv_gather_weights_fwd source
    (base, strides), padding).  out[2m+py] takes ky in {3,1} (input rows m-1, m) for py=0 and {2,0} (rows m, m+1) for py=1: tap i
    reads ky = 3 - py - 2i."""
    return ((3 - py) * 4 + (3 - px), (0, -8, -2, cout * 16, 16)), (0, 1 - py, 1 - px)


def pack_deconv2d_k4s2(deconv, bn, mode="tc", **kw):
    """ConvTranspose2d(k=4, s=2, p=1) as four 2x2 stride-1 convs, one per output parity: {(py, px): ConvPack}."""
    w = _f32(deconv.weight)  # (Cin, Cout, 4, 4)
    assert tuple(deconv.kernel_size) == (4, 4) and tuple(deconv.stride) == (2, 2) and tuple(deconv.padding) == (1, 1)
    cin, cout = w.shape[:2]
    phases = {}
    for py in (0, 1):
        for px in (0, 1):
            (base, strides), pad = deconv2d_k4s2_phase(py, px, cout)
            phases[(py, px)] = pack_filter((w, base, strides), (1, 2, 2), (1, 1, 1), pad, cin, cout, deconv.bias, bn, mode=mode, **kw)
    return phases


def conv_out_dims(dims, k, stride, pad):
    return tuple((n + 2 * p - kk) // s + 1 for n, kk, s, p in zip(dims, k, stride, pad))


def conv_desc(N, in_dims, cin, cout, k, stride, pad, out_dims, out_full, out_c, in_fmt, out_fmt, out_scale=(1, 1, 1), out_off=(0, 0, 0),
              out_groups=(1, 1, 1), relu=False, res_mode=RES_NONE):
    """lt_conv_desc of one launch over an (N, in_dims, cin) input: out_dims is the grid the launch computes, out_full and out_c the
    output tensor's (D, H, W) and channel count.  No workspace: launch_conv attaches the split-K scratch."""
    return capi.ConvDesc(N=N, ID=in_dims[0], IH=in_dims[1], IW=in_dims[2], Cin=cin, OD=out_dims[0], OH=out_dims[1], OW=out_dims[2],
                         Cout=cout, KD=k[0], KH=k[1], KW=k[2], sd=stride[0], sh=stride[1], sw=stride[2], pd=pad[0], ph=pad[1], pw=pad[2],
                         FD=out_full[0], FH=out_full[1], FW=out_full[2], FC=out_c, osd=out_scale[0], osh=out_scale[1], osw=out_scale[2],
                         ood=out_off[0], ooh=out_off[1], oow=out_off[2], relu=int(relu), residual=res_mode, in_format=in_fmt,
                         out_format=out_fmt, ogd=out_groups[0], ogh=out_groups[1], ogw=out_groups[2])


SPLITK_WS_BYTES = 32 << 20
CHAIN_MAX_BLOCKS = 36     # bottleneck blocks per lt_conv_tc_chain_fwd launch (its kernel parameter block holds 3 filter maps per block)
_SPLITK_WS = {}


def splitk_workspace(device):
    """The split-K scratch of every lt_conv_nd_fwd launch on `device` (inference and training): one fixed buffer, so a layer's split
    count, and with it the rounding of its result, depends on its shape only.  Launches on one stream are ordered; the engine's eager
    warm-up forward allocates it before any CUDA-graph capture."""
    ws = _SPLITK_WS.get(device)
    if ws is None:
        ws = _SPLITK_WS[device] = torch.empty(SPLITK_WS_BYTES, dtype=torch.uint8, device=device)
    return ws


def launch_conv(x, pk, out, relu=False, residual=None, res_mode=RES_NONE, out_dims=None, out_scale=(1, 1, 1), out_off=(0, 0, 0),
                out_groups=(1, 1, 1), scale_mul=None, workspace=None):
    """One lt_conv_nd_fwd of packed filter `pk` over Act x into Act out (and residual) -> the impl launched.  out_dims: the grid the
    launch computes (default: the conv's own output), written at out_scale / out_off / out_groups of `out`.  A fold-packed layer runs on
    LT_CONV_TC_FOLD, with the fold filter, its real Cout and scale_fold, when the kernel takes its width and `out` is its own 32-channel
    grid.  scale_mul: device tensor the scale is multiplied by (1 / S of a scaled output gradient).  workspace: split-K scratch
    (default splitk_workspace; an empty tensor forces single-pass launches)."""
    assert x.fmt == pk.in_fmt and x.C == pk.cin, (x.fmt, pk.in_fmt, x.C, pk.cin)
    if residual is not None:
        assert residual.fmt == out.fmt and residual.C == out.C
    in_dims = (x.D, x.H, x.W)
    out_dims = conv_out_dims(in_dims, pk.k, pk.stride, pk.pad) if out_dims is None else tuple(out_dims)
    d = conv_desc(x.N, in_dims, x.C, pk.cout_p, pk.k, pk.stride, pk.pad, out_dims, (out.D, out.H, out.W), out.C, x.fmt, out.fmt,
                  out_scale, out_off, out_groups, relu, res_mode)
    ws = splitk_workspace(x.data.device) if workspace is None else workspace
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    impl, weight, scale = pk.impl, pk.w, pk.scale
    if (pk.w_fold is not None and fold_width_ok(pk.k[2], x.W) and out.C == 32 and tuple(out_scale) == (1, 1, 1)
            and out_dims == in_dims):
        impl, weight, scale = CONV_TC_FOLD, pk.w_fold, pk.scale_fold
        d.Cout = pk.cout
    if scale_mul is not None:
        scale = scale * scale_mul
    capi.conv_nd(d, x.data, weight, scale, pk.shift, None if residual is None else residual.data, out.data, impl)
    return impl


def deconv2d_k4s2(x, phases, out_fmt, relu, conv=launch_conv):
    """ConvTranspose2d(k=4, s=2, p=1) of x from its phase packs (pack_deconv2d_k4s2): each phase a 2x2 stride-1 conv into its (py, px)
    sub-lattice of one (N, 1, 2H, 2W) output.  conv: the launch, with launch_conv's arguments."""
    c = next(iter(phases.values())).cout
    out = Act(x.N, 1, 2 * x.H, 2 * x.W, _round_up(c, 4 if out_fmt == FMT_F32 else 32), out_fmt, x.data.device)
    for (py, px), pk in phases.items():
        conv(x, pk, out=out, relu=relu, out_scale=(1, 2, 2), out_off=(0, py, px), out_dims=(1, x.H, x.W))
    return out


def deconv3d_k2s2(x, pk, out_fmt, relu, residual=None, conv=launch_conv):
    """ConvTranspose3d(k=2, s=2) of x as the one grouped 1x1x1 GEMM of pack_deconv3d_k2s2 (N = 8 Cout, column block g = a 4 + b 2 + c
    written to output phase (a, b, c) of one (N, 2D, 2H, 2W) output); `residual` is added after the ReLU."""
    out = Act(x.N, 2 * x.D, 2 * x.H, 2 * x.W, pk.cout // 8, out_fmt, x.data.device)
    conv(x, pk, out=out, relu=relu, residual=residual, res_mode=RES_NONE if residual is None else RES_AFTER_RELU, out_scale=(2, 2, 2),
         out_dims=(x.D, x.H, x.W), out_groups=(2, 2, 2))
    return out


def pixel_grid(B, h, w, device):
    """(B, h*w, 3) float32 coordinates (x, y, 0) of the pixels of an h x w map: the 2-D soft-argmax runs on the 3-D kernels."""
    ys, xs = torch.meshgrid(torch.arange(h, device=device, dtype=torch.float32), torch.arange(w, device=device, dtype=torch.float32),
                            indexing="ij")
    return torch.stack([xs, ys, torch.zeros_like(xs)], dim=-1).reshape(1, h * w, 3).expand(B, h * w, 3).contiguous()


class NativeEngine:
    _splitk_ws = None              # split-K scratch of the convs: None = splitk_workspace; an empty tensor forces single-pass launches

    def __init__(self, model, mode="tc", use_graph=True):
        assert mode in ("simt", "tc", "tc1")
        self.model = model
        self.mode = mode
        self.use_graph = use_graph
        self.act_fmt = FMT_F32 if mode == "simt" else FMT_S32
        self.tc_impl = _TC_IMPL[mode]
        self._packs = None
        self._packs_version = None
        self._epoch = 0
        self._graphs = {}
        self.captures = 0          # CUDA graphs captured by replay()
        self._grids2d = {}         # (h, w, B*V, device) -> pixel_grid of the algebraic forward's 2-D soft-argmax
        self.launches = 0          # kernels launched by the last eager forward (our own kernels only)
        self.timeline = None       # set to [] to record (label, flops, bytes, start_evt, end_evt) per launch
        self._chain_runs = {}      # (layer, block, input shape) -> _chain_run's answer for the current packs
        capi.lib()                 # fail loudly if the extension is missing

    # ------------------------------------------------------------------ weight packing
    def _param_version(self):
        """Key that changes whenever the packed filters / captured graphs may be stale: in-place updates bump `_version`;
        `p.data = ...`, `.to()/.cuda()/.double()` and `load_state_dict(assign=True)` change storage pointer, device or dtype
        instead.  (`p.data.copy_()` bypasses both: call `invalidate()` after such an update.)"""
        items = list(self.model.parameters()) + list(self.model.buffers())
        return tuple((t._version, t.data_ptr(), t.device, t.dtype) for t in items) + (self._epoch,)

    def invalidate(self):
        """Drop the packed filters and the captured CUDA graphs; the next forward re-packs from the module's tensors."""
        self._epoch += 1
        self._packs = None
        self._graphs = {}

    def _pack(self, *args, **kw):
        return pack_filter(*args, mode=self.mode, **kw)

    def _pack_conv(self, conv, bn, cin_pad=None, **kw):
        return pack_conv(conv, bn, mode=self.mode, cin_pad=cin_pad, **kw)

    def _pack_stem_s2d(self, conv, bn):
        return pack_stem_s2d(conv, bn, mode=self.mode)

    def _pack_deconv2d_k4s2(self, deconv, bn):
        return pack_deconv2d_k4s2(deconv, bn, mode=self.mode)

    def _pack_deconv3d_k2s2(self, deconv, bn):
        return pack_deconv3d_k2s2(deconv, bn, mode=self.mode)

    def prepare(self):
        ver = self._param_version()
        if self._packs is not None and ver == self._packs_version:
            return
        m = self.model
        bb, P = m.backbone, {}
        with torch.no_grad():
            # stem: exact-fp32 mode pads 3 -> 4 channels (float4 per pixel) for the FFMA kernel; the tensor-core modes
            # rewrite the 7x7 stride-2 conv as a 4x4 stride-1 conv over the 2x2 space-to-depth image (12 -> 32 channels)
            if self.mode == "simt":
                P["stem"] = self._pack_conv(bb.conv1, bb.bn1, cin_pad=4, force_simt=True)
            else:
                P["stem_s2d"] = self._pack_stem_s2d(bb.conv1, bb.bn1)
            for li in range(1, 5):
                for ui, unit in enumerate(getattr(bb, "layer%d" % li)):
                    key = "layer%d.%d" % (li, ui)
                    for si, (conv, bn) in enumerate(unit.stages()):
                        P["%s.c%d" % (key, si)] = self._pack_conv(conv, bn)
                    if unit.downsample is not None:
                        P[key + ".ds"] = self._pack_conv(unit.downsample[0], unit.downsample[1])
            for i in (0, 3, 6):
                P["deconv%d" % i] = self._pack_deconv2d_k4s2(bb.deconv_layers[i], bb.deconv_layers[i + 1])
            # 17-channel heatmap head: only the algebraic model evaluates it (the volumetric forward uses its shape only)
            P["final"] = self._pack_conv(bb.final_layer, None, out_fmt=FMT_F32)
            for head_name in ("alg_confidences", "vol_confidences"):
                if hasattr(bb, head_name):
                    head = getattr(bb, head_name)
                    P[head_name + ".c0"] = self._pack_conv(head.features[0], head.features[1])
                    P[head_name + ".c1"] = self._pack_conv(head.features[4], head.features[5])
                    P[head_name + ".mlp"] = [(head.head[i].weight.detach().float().contiguous(), head.head[i].bias.detach().float().contiguous())
                                             for i in (0, 2, 4)]
            if not hasattr(m, "volume_net"):
                self._packs, self._packs_version = P, ver
                self._chain_runs = {}
                self._graphs = {}
                return
            P["process_features"] = self._pack_conv(m.process_features[0], None, out_fmt=FMT_F32)
            v = m.volume_net
            pad16 = 32 if self.mode != "simt" else None   # the 16-channel tensor is stored 32 wide in split-fp16

            def pack_res(name, blk):
                cin_pad = pad16 if blk.res_branch[0].in_channels == 16 else None
                P[name + ".a"] = self._pack_conv(blk.res_branch[0], blk.res_branch[1], cin_pad=cin_pad)
                P[name + ".b"] = self._pack_conv(blk.res_branch[3], blk.res_branch[4])
                if len(blk.skip_con) > 0:
                    P[name + ".s"] = self._pack_conv(blk.skip_con[0], blk.skip_con[1], cin_pad=cin_pad)

            P["front0"] = self._pack_conv(v.front_layers[0].block[0], v.front_layers[0].block[1])
            for i in (1, 2, 3):
                pack_res("front%d" % i, v.front_layers[i])
            ed = v.encoder_decoder
            for lvl in range(1, 6):
                pack_res("skip%d" % lvl, getattr(ed, "skip_res%d" % lvl))
                pack_res("enc%d" % lvl, getattr(ed, "encoder_res%d" % lvl))
                pack_res("dec%d" % lvl, getattr(ed, "decoder_res%d" % lvl))
                up = getattr(ed, "decoder_upsample%d" % lvl)
                P["up%d" % lvl] = self._pack_deconv3d_k2s2(up.block[0], up.block[1])
            pack_res("mid", ed.mid_res)
            pack_res("back0", v.back_layers[0])
            P["back1"] = self._pack_conv(v.back_layers[1].block[0], v.back_layers[1].block[1])
            P["back2"] = self._pack_conv(v.back_layers[2].block[0], v.back_layers[2].block[1])
            P["output"] = self._pack_conv(v.output_layer, None, out_fmt=FMT_F32)
        self._packs, self._packs_version = P, ver
        self._chain_runs = {}
        self._graphs = {}

    # ------------------------------------------------------------------ op helpers
    def _as_f32(self, x):
        if x.fmt == FMT_F32:
            return x
        y = Act(x.N, x.D, x.H, x.W, x.C, FMT_F32, x.data.device)
        capi.s32_to_f32(x.data, y.data, x.pixels, x.C)
        self.launches += 1
        return y

    def _conv(self, x, pk, relu, residual=None, res_mode=RES_NONE, out=None, out_scale=(1, 1, 1), out_off=(0, 0, 0),
              out_dims=None, out_fmt=None, out_c=None, out_groups=(1, 1, 1)):
        """Launch one conv (launch_conv). `out` (with out_scale/out_off) lets transposed-conv phases share an output tensor.

        out_c: channel stride of a float32 output narrower than the padded N tile (the TMA store clips the padding)."""
        if pk.impl == CONV_SIMT:
            x = self._as_f32(x)
        od, oh, ow = conv_out_dims((x.D, x.H, x.W), pk.k, pk.stride, pk.pad) if out_dims is None else out_dims
        if out is None:
            fmt = self.act_fmt if out_fmt is None else out_fmt
            c = _round_up(pk.cout, 32) if fmt == FMT_S32 else pk.cout_p
            if out_c is not None and fmt == FMT_F32 and pk.cout <= out_c <= pk.cout_p:
                c = out_c
            out = Act(x.N, od, oh, ow, c, fmt, x.data.device)
        kd, kh, kw = pk.k
        with self._timed("conv_tc", flops=2.0 * x.N * od * oh * ow * pk.kmacs,
                         desc="N%d %dx%dx%d Cin%d Cout%d k%d%d%d s%d" % (x.N, od, oh, ow, pk.cin, pk.cout, kd, kh, kw, pk.stride[2])) as t:
            impl = launch_conv(x, pk, out, relu, residual, res_mode, (od, oh, ow), out_scale, out_off, out_groups, workspace=self._splitk_ws)
            t.label = {CONV_TC_FOLD: "conv_fold", CONV_SIMT: "conv_ffma"}.get(impl, "conv_tc")
        self.launches += 1
        return out

    def _timed(self, label, flops=0.0, nbytes=0.0, desc=""):
        return _Timed(self.timeline, label, flops, nbytes, desc)

    def _maxpool(self, x, k, s, p):
        od = (x.D + 2 * p[0] - k[0]) // s[0] + 1
        oh = (x.H + 2 * p[1] - k[1]) // s[1] + 1
        ow = (x.W + 2 * p[2] - k[2]) // s[2] + 1
        y = Act(x.N, od, oh, ow, x.C, x.fmt, x.data.device)
        capi.maxpool(x.data, y.data, x.fmt, x.N, x.D, x.H, x.W, x.C, k, s, p, od, oh, ow)
        self.launches += 1
        return y

    def _deconv2d(self, x, phases):
        return deconv2d_k4s2(x, phases, self.act_fmt, relu=True, conv=self._conv)

    def _deconv3d(self, x, phases, skip):
        if isinstance(phases, ConvPack):      # merged: one GEMM, eight output groups
            return deconv3d_k2s2(x, phases, self.act_fmt, relu=True, residual=skip, conv=self._conv)
        c = next(iter(phases.values())).cout
        out = Act(x.N, 2 * x.D, 2 * x.H, 2 * x.W, c, self.act_fmt, x.data.device)
        for (a, b, cc), pk in phases.items():
            self._conv(x, pk, relu=True, residual=skip, res_mode=RES_AFTER_RELU, out=out, out_scale=(2, 2, 2),
                       out_off=(a, b, cc), out_dims=(x.D, x.H, x.W))
        return out

    def _res3d(self, x, name):
        P = self._packs
        skip = self._conv(x, P[name + ".s"], relu=False) if (name + ".s") in P else x
        y = self._conv(x, P[name + ".a"], relu=True)
        return self._conv(y, P[name + ".b"], relu=True, residual=skip, res_mode=RES_BEFORE_RELU)

    # ------------------------------------------------------------------ network stages
    def backbone_features(self, images_nchw, return_trunk=False):
        """(BV, 3, H, W) float32 -> processed features, channels-last float32 Act (BV, 1, h, w, 32).

        = backbone trunk + deconvs (pose_resnet.py:293-313) + process_features (triangulation.py:344-346).
        The 17-channel heatmap head (final_layer) is not evaluated: the volumetric forward uses it
        only for its shape (triangulation.py:257,264-265).
        """
        trunk = self.backbone_trunk(images_nchw)
        feats = self._conv(self.backbone_upsample(trunk), self._packs["process_features"], relu=False, out_fmt=FMT_F32)
        return (feats, trunk) if return_trunk else feats

    def backbone_upsample(self, x):
        """trunk output -> 256-channel features at 1/4 resolution (three k4 s2 transposed convs + BN + ReLU)."""
        for i in (0, 3, 6):
            x = self._deconv2d(x, self._packs["deconv%d" % i])
        return x

    def confidence_head(self, trunk, name):
        """GlobalAveragePoolingHead (pose_resnet.py:140-174) on the trunk output -> float32 (BV, n_classes).

        conv3x3+BN, MaxPool2, ReLU, twice (ReLU and max commute, so ReLU is fused into the conv epilogue), then the
        global-average-pool + 3-layer MLP + sigmoid tail in one small kernel."""
        P = self._packs
        x = self._conv(trunk, P[name + ".c0"], relu=True)
        x = self._maxpool(x, (1, 2, 2), (1, 2, 2), (0, 0, 0))
        x = self._conv(x, P[name + ".c1"], relu=True)
        x = self._maxpool(x, (1, 2, 2), (1, 2, 2), (0, 0, 0))
        lin = P[name + ".mlp"]
        out = torch.empty((x.N, lin[2][0].shape[0]), dtype=torch.float32, device=x.data.device)
        capi.gap_mlp3(x.data, x.fmt, x.N, x.D * x.H * x.W, x.C, lin[0], lin[1], lin[2], out)
        self.launches += 1
        return out

    def backbone_trunk(self, images_nchw):
        """(BV, 3, H, W) float32 -> trunk output Act (BV, 1, H/32, W/32, 512*expansion) (pose_resnet.py:293-302)."""
        P = self._packs
        bv, c, H, W = images_nchw.shape
        dev = images_nchw.device
        if "stem_s2d" in P:
            x = Act(bv, 1, H // 2, W // 2, 32, FMT_S32, dev)
            capi.stem_s2d(images_nchw, x.data, bv, c, H, W)
            self.launches += 1
            x = self._conv(x, P["stem_s2d"], relu=True, out_dims=(1, H // 2, W // 2))
        else:
            x = Act(bv, 1, H, W, 4, FMT_F32, dev)
            capi.nchw_to_nhwc(images_nchw, x.data, bv, c, H, W, 4)
            self.launches += 1
            x = self._conv(x, P["stem"], relu=True)
        x = self._maxpool(x, (1, 3, 3), (1, 2, 2), (0, 1, 1))
        bb = self.model.backbone
        for li in range(1, 5):
            units = getattr(bb, "layer%d" % li)
            ui = 0
            while ui < len(units):
                run = self._chain_run(x, li, ui, units)
                if run:
                    x = self._chain(x, ["layer%d.%d" % (li, ui + i) for i in range(run[0])], run[1])
                    ui += run[0]
                    continue
                unit = units[ui]
                key = "layer%d.%d" % (li, ui)
                n_st = len(unit.stages())
                identity = self._conv(x, P[key + ".ds"], relu=False) if unit.downsample is not None else x
                y = x
                for si in range(n_st - 1):
                    y = self._conv(y, P["%s.c%d" % (key, si)], relu=True)
                x = self._conv(y, P["%s.c%d" % (key, n_st - 1)], relu=True, residual=identity, res_mode=RES_BEFORE_RELU)
                ui += 1
        return x

    def _chain_descs(self, x, pks):
        """The lt_conv_nd_fwd descriptors of one bottleneck block (1x1 reduce, 3x3, 1x1 expansion + residual) over Act x."""
        dims = (x.D, x.H, x.W)
        return [conv_desc(x.N, dims, pk.cin, pk.cout_p, pk.k, pk.stride, pk.pad, dims, dims, pk.cout_p, FMT_S32, FMT_S32, relu=True,
                          res_mode=RES_BEFORE_RELU if i == 2 else RES_NONE) for i, pk in enumerate(pks)]

    def _chain_run(self, x, li, ui, units):
        """(blocks, descs) of the chain launch (lt_conv_tc_chain_fwd) that runs blocks ui.. of backbone layer li, or None: the
        per-layer launches run them.  A run is the longest stretch of bottleneck blocks without downsample whose three layers map the
        grid of x onto itself at N tile 128 (stride 1, Cout a multiple of 128) and whose per-layer launches would not split K: the
        chain runs exactly their products and epilogues, so its outputs are bit-identical to theirs."""
        if not x.data.is_cuda or x.fmt != FMT_S32 or self.tc_impl == CONV_SIMT:
            return None
        P = self._packs
        key = (li, ui, x.N, x.D, x.H, x.W, x.C)
        cache = self._chain_runs
        if key in cache:
            return cache[key]

        def block(i):
            u = units[i]
            if u.downsample is not None or len(u.stages()) != 3:
                return None
            pks = [P["layer%d.%d.c%d" % (li, i, si)] for si in range(3)]
            if any(pk.impl != self.tc_impl or pk.w_fold is not None or pk.cout_p % 128 or tuple(pk.stride) != (1, 1, 1) for pk in pks):
                return None
            return pks

        run, descs = 0, None
        first = block(ui)
        if first is not None and x.C == first[2].cout_p == first[0].cin:
            descs = self._chain_descs(x, first)
            ws = splitk_workspace(x.data.device) if self._splitk_ws is None else self._splitk_ws
            sms = torch.cuda.get_device_properties(x.data.device).multi_processor_count
            plans = []
            for d in descs:
                d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
                plans.append(capi.conv_tc_plan(d, sms, capi.get_options()["tc_splitk"]))
                d.workspace, d.workspace_bytes = None, 0
            if all(p["splits"] == 1 and p["nt"] == 128 for p in plans):
                shape = [(pk.k, pk.pad, pk.cin, pk.cout_p) for pk in first]
                run = 1
                while ui + run < len(units) and run < CHAIN_MAX_BLOCKS:
                    nxt = block(ui + run)
                    if nxt is None or [(pk.k, pk.pad, pk.cin, pk.cout_p) for pk in nxt] != shape:
                        break
                    run += 1
                capi.conv_tc_chain_plan(descs, run, sms)   # the C side's own checks
        cache[key] = (run, descs) if run else None
        return cache[key]

    def _chain(self, x, keys, descs):
        """Blocks `keys` of the backbone as one chain launch, in place on x (lt_conv_tc_chain_fwd)."""
        P = self._packs
        pks = [P["%s.c%d" % (k, si)] for k in keys for si in range(3)]
        dev = x.data.device
        mid = pks[0].cout_p
        bufs = [Act(x.N, x.D, x.H, x.W, mid, FMT_S32, dev).data for _ in range(4)]
        plan = capi.conv_tc_chain_plan(descs, len(keys), 1)
        counters = torch.empty(plan["counters"], dtype=torch.int32, device=dev)
        flops = sum(2.0 * x.N * x.D * x.H * x.W * pk.kmacs for pk in pks)
        with self._timed("conv_tc", flops=flops, desc="chain %s..%s N%d %dx%d Cin%d" % (keys[0], keys[-1], x.N, x.H, x.W, x.C)):
            capi.conv_tc_chain(descs, len(keys), x.data, bufs, [pk.w for pk in pks], [pk.scale for pk in pks], [pk.shift for pk in pks],
                               counters, self.tc_impl)
        self.launches += 1
        return x

    def unproject(self, feats, B, V, proj, coord, agg, conf=None):
        """feats: Act (B*V, 1, h, w, C) float32 -> volume Act (B, n, n, n, C) in the conv operand format."""
        n = coord.shape[1]
        vol = Act(B, n, n, n, feats.C, self.act_fmt, feats.data.device)
        # algorithmic bytes: volume write + compulsory feature read + coordinate read (DESIGN.md)
        nbytes = B * (n ** 3 * feats.C * 4 + V * feats.H * feats.W * feats.C * 4 + n ** 3 * 12)
        with self._timed("unproject", nbytes=nbytes):
            capi.unproject_aggregate(feats.data.view(B, V, feats.H, feats.W, feats.C), proj, coord.view(B, n * n * n, 3), conf,
                                     vol.data, vol.fmt, agg)
        self.launches += 1
        return vol

    def v2v(self, x, softargmax_args=None):
        """volume Act (B, n, n, n, 32) -> logits Act float32 channels-last (v2v.py:164-169).

        softargmax_args = (coord, J, multiplier, softmax): when the fused tail kernel runs, the statistics pass of the volumetric
        soft-argmax is folded into it (logits.stats); `softargmax` then only merges the partials and normalises."""
        P = self._packs
        x = self._conv(x, P["front0"], relu=True)
        for i in (1, 2, 3):
            x = self._res3d(x, "front%d" % i)
        skips = {}
        for lvl in range(1, 6):
            skips[lvl] = self._res3d(x, "skip%d" % lvl)
            x = self._maxpool(x, (2, 2, 2), (2, 2, 2), (0, 0, 0))
            x = self._res3d(x, "enc%d" % lvl)
        x = self._res3d(x, "mid")
        for lvl in range(5, 0, -1):
            x = self._res3d(x, "dec%d" % lvl)
            x = self._deconv3d(x, P["up%d" % lvl], skips.pop(lvl))
        x = self._res3d(x, "back0")
        out_c = _round_up(P["output"].cout, 4)
        b1, b2, b3 = P["back1"], P["back2"], P["output"]
        # the tail kernel reads b1.w / b2.w as 32 rows and b3.w as round_up(out_c, 16) rows of lt_conv_tc_pack_weights
        if (b1.impl == b2.impl == b3.impl == CONV_TC and x.fmt == FMT_S32 and x.C == 32 and b1.cin == b2.cin == b3.cin == 32
                and b1.cout == b2.cout == b1.cout_p == b2.cout_p == 32 and b3.cout <= out_c <= 32 and b3.cout_p == _round_up(out_c, 16)):
            # v2v.py:154-160,168-169 in one kernel: the two hidden activations never leave the SM
            logits = Act(x.N, x.D, x.H, x.W, out_c, FMT_F32, x.data.device)
            rows = x.pixels
            nvox = x.D * x.H * x.W
            # the statistics tile takes at most 20 floats per voxel and the streaming finish no fewer: J 17..20 (out_c 20)
            fuse = (softargmax_args is not None and nvox % 128 == 0 and out_c <= 20 and _stream_layout_ok(out_c, softargmax_args[1], nvox)
                    and softargmax_args[3] in (0, 1, False, True))
            with self._timed("conv_tail", flops=2.0 * rows * (b1.kmacs + b2.kmacs + b3.kmacs), nbytes=rows * (128 + 4 * out_c + (12 if fuse else 0)),
                             desc="N%d %dx%dx%d 32->32->32->%d k111 fused%s" % (x.N, x.D, x.H, x.W, b3.cout, " + soft-argmax statistics" if fuse else "")):
                if fuse:
                    coord, J, mult, softmax = softargmax_args
                    ws = torch.empty(capi.softargmax3d_workspace_bytes(x.N, J, nvox) // 4 + 1, dtype=torch.float32, device=x.data.device)
                    G = capi.v2v_tail_stats(x.data, b1.w, b2.w, b3.w, b1.scale, b1.shift, b2.scale, b2.shift, b3.scale, b3.shift,
                                            logits.data, x.N, nvox, out_c, coord, J, mult, int(softmax), ws)
                    logits.stats = (ws, G)
                else:
                    capi.v2v_tail(x.data, b1.w, b2.w, b3.w, b1.scale, b1.shift, b2.scale, b2.shift, b3.scale, b3.shift, logits.data, rows, out_c)
            self.launches += 1
            return logits
        x = self._conv(x, P["back1"], relu=True)
        x = self._conv(x, P["back2"], relu=True)
        # compact logits: 17 joints stored 20 wide (80-byte voxel rows) instead of the 32-wide N tile -> the soft-argmax
        # streams 37 % fewer bytes; the conv's TMA store clips the 12 padding channels
        return self._conv(x, P["output"], relu=False, out_fmt=FMT_F32, out_c=out_c)

    def softargmax(self, logits, coord, J, multiplier, softmax):
        B, n = logits.N, logits.D
        nvox = n * n * n
        dev = logits.data.device
        volumes = torch.empty((B, J, n, n, n), dtype=torch.float32, device=dev)
        keypoints = torch.empty((B, J, 3), dtype=torch.float32, device=dev)
        if logits.stats is not None:
            # statistics came out of the fused V2V tail: merge + normalise only.  Algorithmic bytes as for the whole op (logits read once,
            # volumes written once, coordinates read once -- by the tail kernel)
            ws, G = logits.stats
            with self._timed("softargmax", nbytes=B * (2 * J * nvox * 4 + nvox * 12)):
                capi.softargmax3d_finish(logits.data, nvox * logits.C, logits.C, coord, volumes, keypoints, ws, B, J, nvox, G, multiplier, int(softmax))
            self.launches += 2
            return keypoints, volumes
        ws = torch.empty(capi.softargmax3d_workspace_bytes(B, J, nvox) // 4 + 1, dtype=torch.float32, device=dev)
        with self._timed("softargmax", nbytes=B * (2 * J * nvox * 4 + nvox * 12)):
            capi.softargmax3d(logits.data, nvox * logits.C, logits.C, 1, coord, volumes, keypoints, ws, B, J, nvox, multiplier, softmax)
        self.launches += 3   # statistics / merge / normalise (streaming or classic kernels, csrc/softargmax.cu)
        return keypoints, volumes

    # ------------------------------------------------------------------ whole device-side forward
    def _device_forward(self, images, proj, position, center, step, rot, conf=None):
        m = self.model
        B, V = images.shape[:2]
        n = m.volume_size
        dev = images.device
        self.launches = 0
        coord = torch.empty((B, n, n, n, 3), dtype=torch.float32, device=dev)
        capi.coord_volume(position, center, step, rot, coord, m.transfer_cmu_to_human36m)
        self.launches += 1
        need_conf = m.volume_aggregation_method.startswith("conf")
        feats, trunk = self.backbone_features(images.reshape(B * V, *images.shape[2:]), return_trunk=True)
        if need_conf:
            conf = self.confidence_head(trunk, "vol_confidences").view(B, V, -1)          # triangulation.py:253-261
            if m.volume_aggregation_method == "conf_norm":
                capi.view_normalize(conf, B, V, conf.shape[2], 0.0)                        # :268-269
                self.launches += 1
        del trunk
        agg = capi.AGG[m.volume_aggregation_method]
        vol = self.unproject(feats, B, V, proj, coord, agg, conf)
        logits = self.v2v(vol, (coord, m.num_joints, m.volume_multiplier, m.volume_softmax))
        keypoints, volumes = self.softargmax(logits, coord, m.num_joints, m.volume_multiplier, m.volume_softmax)
        # (B, V, 32, h, w) view of the channels-last features (values identical, strides permuted)
        features = feats.data.view(B, V, feats.H, feats.W, feats.C).permute(0, 1, 4, 2, 3)
        if need_conf:
            return keypoints, features, volumes, coord, conf
        return keypoints, features, volumes, coord

    # ------------------------------------------------------------------ multi-GPU (view-sharded) step
    def _sh_exchange_state(self, plan, pg, collective, B, feats_shape, planes, nvox, dev):
        """Peer-memory buffers of the `features` / `p2p` exchanges (symmetric memory, allocated once per shape)."""
        from . import dist as lt_dist
        h, w, C = feats_shape
        if collective == "features":
            key = ("feat", B, plan.n_views, h, w, C)
            if getattr(self, "_peer_key", None) != key:
                self._peer = lt_dist.FeatureExchange(plan, pg, B, plan.n_views, h, w, C, dev)
                self._peer_key = key
        elif collective == "p2p":
            key = ("p2p", B, planes, nvox, C)
            if getattr(self, "_peer_key", None) != key:
                self._peer = lt_dist.PeerExchange(plan, pg, B, planes, nvox, C, dev)
                self._peer_key = key
        return getattr(self, "_peer", None)

    def _sh_pre(self, images_local, proj_local, position, center, step, rot, plan, collective):
        """Stage 1 (capturable: our kernels only): coordinate volumes, backbone on this rank's views, and -- for the NCCL
        exchanges -- the packed partial aggregates of those views."""
        m = self.model
        B, Vl = images_local.shape[:2]
        n = m.volume_size
        nvox = n * n * n
        dev = images_local.device
        coord = torch.empty((B, n, n, n, 3), dtype=torch.float32, device=dev)
        capi.coord_volume(position, center, step, rot, coord, m.transfer_cmu_to_human36m)
        self.launches += 1
        feats = self.backbone_features(images_local.reshape(B * Vl, *images_local.shape[2:]))
        partial = None
        if plan.group_size > 1 and collective in ("all_reduce", "reduce_scatter"):
            planes = 2 if m.volume_aggregation_method == "softmax" else 1
            partial = torch.empty((B, planes, nvox, feats.C), dtype=torch.float32, device=dev)
            capi.unproject_partial(feats.data.view(B, Vl, feats.H, feats.W, feats.C), proj_local, coord.view(B, nvox, 3), None, partial,
                                   capi.AGG[m.volume_aggregation_method])
            self.launches += 1
        return coord, feats, partial

    def _sh_exchange(self, coord, feats, partial, proj_local, plan, pg, collective, out=None):
        """Stage 2: the ONE exchange step of the view group (NCCL collective, or peer-memory stores + group barriers)."""
        from . import dist as lt_dist
        m = self.model
        B = coord.shape[0]
        Vl = feats.N // B
        nvox = coord.shape[1] ** 3
        agg = capi.AGG[m.volume_aggregation_method]
        if plan.group_size == 1:
            return None
        if collective == "features":
            fx = self._peer
            fx.barrier()      # every owner has finished reading the previous step's maps
            fx.scatter(feats.data.view(B, Vl, feats.H, feats.W, feats.C))
            self.launches += 1
            fx.barrier()      # all stores of the group have landed
            return None
        if collective == "p2p":
            px = self._peer
            px.barrier()
            capi.unproject_push(feats.data.view(B, Vl, feats.H, feats.W, feats.C), proj_local, coord.view(B, nvox, 3), None,
                                px.peer_ptrs, plan.view_rank, agg)
            self.launches += 1
            px.barrier()
            return None
        return lt_dist.complete_partials(partial, plan, pg, collective, "max" if m.volume_aggregation_method == "max" else "sum", out=out)

    def _sh_post(self, coord, feats, mine, proj_local, proj_all, plan, collective):
        """Stage 3 (capturable): aggregate volume of the samples this rank owns, V2V, soft-argmax."""
        m = self.model
        B = coord.shape[0]
        n = m.volume_size
        nvox = n * n * n
        dev = coord.device
        agg = capi.AGG[m.volume_aggregation_method]
        own = plan.owned_samples(B)
        Bl = len(own)
        coord_own = coord[own[0]:own[-1] + 1]
        vol = Act(Bl, n, n, n, feats.C, self.act_fmt, dev)
        if plan.group_size == 1:
            capi.unproject_aggregate(feats.data.view(B, feats.N // B, feats.H, feats.W, feats.C), proj_local, coord.view(B, nvox, 3), None,
                                     vol.data, vol.fmt, agg)
        elif collective == "features":
            # the owner unprojects all views of its samples with exactly the single-GPU arithmetic
            capi.unproject_aggregate(self._peer.buf, proj_all[own[0]:own[-1] + 1].contiguous(), coord_own.reshape(Bl, nvox, 3), None,
                                     vol.data, vol.fmt, agg)
        elif collective == "p2p":
            capi.unproject_reduce_finalize(self._peer.buf, plan.group_size, vol.data, vol.fmt, Bl, feats.C, nvox, agg)
        else:
            capi.unproject_finalize(mine.contiguous(), vol.data, vol.fmt, Bl, feats.C, nvox, agg)
        self.launches += 1
        coord_own = coord_own.contiguous()
        logits = self.v2v(vol, (coord_own, m.num_joints, m.volume_multiplier, m.volume_softmax))
        kp, volumes = self.softargmax(logits, coord_own, m.num_joints, m.volume_multiplier, m.volume_softmax)
        return kp, volumes

    def forward_view_sharded(self, images_local, proj_local, position, center, step, rot, plan, pg, collective="all_reduce",
                             proj_all=None, use_graph=False):
        """Multi-GPU step of one rank (see dist.py): this rank's views of the group's batch in, all keypoints out.

        images_local (B, V_local, 3, H, W), proj_local (B, V_local, 3, 4); the other inputs cover all B samples.
        backbone (+ unprojection partials) -> ONE exchange over the view group -> V2V + soft-argmax on the
        B / group_size samples this rank owns -> all-gather of the (B, 17, 3) keypoints.

        use_graph: stages 1 and 3 are captured into two CUDA graphs (one pair per input shape and exchange kind); only the
        exchange itself and the key-point all-gather are issued eagerly between / after the replays.
        """
        from . import dist as lt_dist
        self.prepare()
        m = self.model
        B, Vl = images_local.shape[:2]
        n = m.volume_size
        dev = images_local.device
        planes = 2 if m.volume_aggregation_method == "softmax" else 1
        if collective == "features" and plan.group_size > 1:
            assert proj_all is not None, "collective='features' needs the projection matrices of all views"
        if proj_all is None:
            proj_all = proj_local
        ins = (images_local, proj_local, position, center, step, rot, proj_all)
        if not use_graph:
            self.launches = 0
            coord, feats, partial = self._sh_pre(*ins[:6], plan, collective)
            self._sh_exchange_state(plan, pg, collective, B, (feats.H, feats.W, feats.C), planes, n ** 3, dev)
            mine = self._sh_exchange(coord, feats, partial, proj_local, plan, pg, collective)
            kp, volumes = self._sh_post(coord, feats, mine, proj_local, proj_all, plan, collective)
        else:
            key = ("sharded", tuple(images_local.shape), dev.index, collective, plan.group_size, plan.view_rank)
            g = self._graphs.get(key)
            if g is None:
                static_in = [t.clone() for t in ins]
                side = torch.cuda.Stream(device=dev)
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):      # eager warm-up: module load, function attributes, peer buffers, NCCL communicator
                    self.launches = 0
                    c0, f0, p0 = self._sh_pre(*static_in[:6], plan, collective)
                    self._sh_exchange_state(plan, pg, collective, B, (f0.H, f0.W, f0.C), planes, n ** 3, dev)
                    m0 = self._sh_exchange(c0, f0, p0, static_in[1], plan, pg, collective)
                    self._sh_post(c0, f0, m0, static_in[1], static_in[6], plan, collective)
                torch.cuda.current_stream().wait_stream(side)
                torch.cuda.synchronize()
                del c0, f0, p0, m0
                ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                self.launches = 0
                with torch.cuda.graph(ga):
                    coord, feats, partial = self._sh_pre(*static_in[:6], plan, collective)
                la = self.launches
                # stage 3 reads the reduced block from a static address: the in-place all-reduce leaves it in this rank's
                # slice of `partial`; the reduce-scatter writes into a buffer allocated here
                per = B // plan.group_size
                mine_static = None
                if partial is not None:
                    mine_static = (torch.empty((per,) + tuple(partial.shape[1:]), dtype=torch.float32, device=dev)
                                   if collective == "reduce_scatter" else partial[plan.view_rank * per:(plan.view_rank + 1) * per])
                with torch.cuda.graph(gb, pool=ga.pool()):
                    kp, volumes = self._sh_post(coord, feats, mine_static, static_in[1], static_in[6], plan, collective)
                g = (ga, gb, static_in, (coord, feats, partial, mine_static), (kp, volumes), la, self.launches)
                self._graphs[key] = g
            ga, gb, static_in, (coord, feats, partial, mine_static), (kp, volumes), la, lall = g
            for dst, src in zip(static_in, ins):
                if dst.data_ptr() != src.data_ptr():
                    dst.copy_(src, non_blocking=True)
            ga.replay()
            self.launches = lall
            self._sh_exchange(coord, feats, partial, static_in[1], plan, pg, collective,
                              out=mine_static if collective == "reduce_scatter" else None)
            gb.replay()
        kp_all = lt_dist.gather_keypoints(kp, plan, pg)
        features = feats.data.view(B, Vl, feats.H, feats.W, feats.C).permute(0, 1, 4, 2, 3)
        return kp_all, features, volumes, coord

    # ------------------------------------------------------------------ algebraic model (config #5)
    def algebraic_forward(self, images, proj, heatmap_multiplier, use_confidences, heatmap_softmax=True):
        """AlgebraicTriangulationNet.forward (triangulation.py:149-200), device side.

        images (B, V, 3, H, W), proj (B, V, 3, 4) image-space projection matrices.
        -> keypoints_3d (B, J, 3), keypoints_2d (B, V, J, 2) in image pixels, heatmaps (B, V, J, h, w) softmaxed,
           confidences (B, V, J)."""
        self.prepare()
        self.launches = 0
        m = self.model
        B, V = images.shape[:2]
        H, W = images.shape[3:]
        dev = images.device
        J = m.backbone.num_joints
        trunk = self.backbone_trunk(images.reshape(B * V, *images.shape[2:]))
        logits = self._conv(self.backbone_upsample(trunk), self._packs["final"], relu=False, out_fmt=FMT_F32)   # (BV,1,h,w,32)
        h, w = logits.H, logits.W
        # 2-D soft-argmax (op.py:11-47) = the 3-D kernels with pixel-index coordinates (x, y, 0).  One grid per shape, kept: a grid
        # made during a CUDA-graph capture is filled only by a replay, and a captured graph reads its grid at a fixed address
        key = (h, w, B * V, dev)
        grid = self._grids2d.get(key)
        if grid is None:
            grid = self._grids2d[key] = pixel_grid(B * V, h, w, dev)
        heat = torch.empty((B * V, J, h, w), dtype=torch.float32, device=dev)
        kp = torch.empty((B * V, J, 3), dtype=torch.float32, device=dev)
        ws = torch.empty(capi.softargmax3d_workspace_bytes(B * V, J, h * w) // 4 + 1, dtype=torch.float32, device=dev)
        capi.softargmax3d(logits.data, h * w * logits.C, logits.C, 1, grid, heat, kp, ws, B * V, J, h * w, heatmap_multiplier,
                          1 if heatmap_softmax else 2)    # op.py:25-41: ReLU heat-maps, centre of mass / mass
        self.launches += 3
        # the (W / w, H / h) scale (:181-184) is filled on the device: a host-to-device copy cannot be captured
        scale = torch.full((2,), W / w, device=dev, dtype=torch.float32)
        scale[1].fill_(H / h)
        kp2d = (kp[:, :, :2].reshape(B, V, J, 2) * scale).contiguous()
        if use_confidences:
            conf = self.confidence_head(trunk, "alg_confidences").view(B, V, J)
        else:
            conf = torch.ones((B, V, J), dtype=torch.float32, device=dev)
        capi.view_normalize(conf, B, V, J, 1e-5)                                                                 # :173-174
        kp3d = torch.empty((B, J, 3), dtype=torch.float32, device=dev)
        capi.triangulate_dlt(proj.contiguous(), kp2d, conf, kp3d)
        self.launches += 2
        return kp3d, kp2d, heat.view(B, V, J, h, w), conf

    # ------------------------------------------------------------------ RANSAC baseline
    def ransac_forward(self, images, proj, pairs, n_iters, eps, direct):
        """RANSACTriangulationNet.forward (triangulation.py:27-70), device side.

        images (B, V, 3, H, W), proj (B, V, 3, 4) float32 image-space projection matrices, pairs (B, J, n_iters, 2) int32 drawn views.
        -> keypoints_3d (B, J, 3), keypoints_2d (B, V, J, 2) int64 in image pixels, heatmaps (B, V, J, h, w) raw, confidences
           (B, V, J) zeros."""
        self.prepare()
        self.launches = 0
        B, V = images.shape[:2]
        H, W = images.shape[3:]
        dev = images.device
        J = self.model.backbone.num_joints
        trunk = self.backbone_trunk(images.reshape(B * V, *images.shape[2:]))
        logits = self._conv(self.backbone_upsample(trunk), self._packs["final"], relu=False, out_fmt=FMT_F32)   # (BV,1,h,w,C)
        h, w = logits.H, logits.W
        heat = torch.empty((B * V, J, h, w), dtype=torch.float32, device=dev)
        kp2d = torch.empty((B, V, J, 2), dtype=torch.int64, device=dev)
        ws = torch.empty(capi.heatmap_argmax_workspace_bytes(B * V, J, h, w) // 4, dtype=torch.float32, device=dev)
        with self._timed("heatmap_argmax", nbytes=4.0 * B * V * h * w * (logits.C + J)):
            capi.heatmap_argmax(logits.data, logits.C, heat, kp2d, ws, B * V, J, h, w, W / w, H / h)      # :44-52
        kp3d = torch.empty((B, J, 3), dtype=torch.float32, device=dev)
        with self._timed("triangulate_ransac"):
            capi.triangulate_ransac(proj, kp2d, pairs, n_iters, eps, direct, kp3d)                       # :58-65
        self.launches += 3
        conf = torch.zeros((B, V, J), dtype=torch.float32, device=dev)                                     # :59, the "plug"
        return kp3d, kp2d, heat.view(B, V, J, h, w), conf

    def forward(self, images, proj, position, center, step, rot):
        """All inputs are CUDA float32 tensors. Returns (keypoints, features, volumes, coord_volumes)."""
        self.prepare()
        inputs = (images, proj, position, center, step, rot)
        if not self.use_graph:
            return self._device_forward(*inputs)
        return self.replay((tuple(images.shape), images.device.index), self._device_forward, inputs)

    def algebraic_forward_graphed(self, images, proj, heatmap_multiplier, use_confidences, heatmap_softmax=True):
        """algebraic_forward replayed from one CUDA graph per (images shape, device): -> the graph's static outputs."""
        self.prepare()
        fn = lambda im, pr: self.algebraic_forward(im, pr, heatmap_multiplier, use_confidences, heatmap_softmax)
        return self.replay(("algebraic", tuple(images.shape), images.device.index), fn, (images, proj))

    def replay(self, key, fn, inputs):
        """fn(*inputs), a device forward of the prepared packs, replayed from the CUDA graph cached under `key` -> its static
        outputs, overwritten by the next replay.  A miss runs fn eagerly on a side stream first (module loads, function attributes,
        the split-K scratch, the soft-argmax grids), then captures it there, reading static copies of the inputs; `captures` counts
        them.  The capture is thread_local: a DataLoader's pin-memory thread may make CUDA calls meanwhile (a validation pass captures
        at its first batch, when that thread is prefetching).  prepare() and invalidate() drop the graphs with the packs they read."""
        g = self._graphs.get(key)
        if g is None:
            static_in = [t.clone() for t in inputs]
            s = torch.cuda.Stream(device=inputs[0].device)
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                fn(*static_in)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=s, capture_error_mode="thread_local"):
                static_out = fn(*static_in)
            g = self._graphs[key] = (graph, static_in, static_out, self.launches)
            self.captures += 1
        graph, static_in, static_out, launches = g
        for dst, src in zip(static_in, inputs):
            dst.copy_(src, non_blocking=True)
        graph.replay()
        self.launches = launches
        return static_out
