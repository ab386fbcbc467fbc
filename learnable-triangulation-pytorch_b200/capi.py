"""ctypes binding of liblt_b200.so (the C ABI declared in include/lt_b200.h).

This is the stub a maintainer of the (pure-Python) reference would add to call the native
kernels: raw device pointers + sizes in, status code out.  torch tensors are only used as
device-memory owners (`data_ptr()`), never passed through the ABI.
"""
import ctypes
import os

import torch

from . import build as _build

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "liblt_b200.so")

FMT_F32, FMT_S32 = 0, 1
AGG = {"sum": 0, "max": 1, "softmax": 2, "conf": 3, "conf_norm": 3}
CONV_SIMT, CONV_TC, CONV_TC1, CONV_TC_FOLD, CONV_TC_PAIR = 0, 1, 2, 3, 4
RES_NONE, RES_BEFORE_RELU, RES_AFTER_RELU = 0, 1, 2

c_int, c_long, c_float, c_void_p, c_size_t = ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t


class ConvDesc(ctypes.Structure):
    """Mirror of `struct lt_conv_desc` (include/lt_b200.h) -- field order matters."""
    _fields_ = [(n, c_int) for n in (
        "N", "ID", "IH", "IW", "Cin",
        "OD", "OH", "OW", "Cout",
        "KD", "KH", "KW",
        "sd", "sh", "sw",
        "pd", "ph", "pw",
        "FD", "FH", "FW", "FC",
        "osd", "osh", "osw",
        "ood", "ooh", "oow",
        "relu", "residual", "in_format", "out_format", "ogd", "ogh", "ogw", "reserved0")] + [("workspace", c_void_p), ("workspace_bytes", c_size_t)]


class Options(ctypes.Structure):
    """Mirror of `struct lt_options` (include/lt_b200.h): kernel-selection switches, all defaulting to the measured-best path."""
    _fields_ = [(n, c_int) for n in ("tc_persist", "tc_splitk", "tc_bres", "tc_direct_epilogue", "fold_fast_issue", "fold_debug",
                                     "softargmax_stream", "unproject_v2", "unproject_cpl", "unproject_lb", "unproject_brick", "unproject_brick_order", "pair_nt", "pair_stages", "pair_prof", "pair_direct_out", "pair_two_acc", "fold_pair", "fold_direct", "fold_fullw")]


# The ONE place the environment is read (A/B experiments): LT_OPT_<FIELD>=<int>
OPTIONS_ENV_PREFIX = "LT_OPT_"

# every symbol include/lt_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "lt_default_options": (None, [ctypes.POINTER(Options)]),
    "lt_get_options": (c_int, [ctypes.POINTER(Options)]),
    "lt_set_options": (c_int, [ctypes.POINTER(Options)]),
    "lt_version": (c_int, []),
    "lt_last_error_string": (ctypes.c_char_p, []),
    "lt_device_info": (c_int, [ctypes.POINTER(c_int)] * 3),
    "lt_coord_volume_fwd": (c_int, [c_void_p] * 5 + [c_int, c_int, c_int, c_void_p]),
    "lt_unproject_aggregate_fwd": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_long, c_int, c_void_p]),
    "lt_unproject_partial_fwd": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_unproject_finalize_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_int, c_void_p]),
    "lt_unproject_push_fwd": (c_int, [c_void_p] * 4 + [ctypes.POINTER(c_void_p), c_int, c_int] + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_unproject_reduce_finalize_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_long, c_int, c_void_p]),
    "lt_feature_scatter_fwd": (c_int, [c_void_p, ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_long, c_void_p]),
    "lt_unproject_aggregate_bwd": (c_int, [c_void_p] * 7 + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_softargmax3d_bwd": (c_int, [c_void_p] * 6 + [c_int, c_int, c_long, c_float, c_int, c_void_p]),
    "lt_test_unproject_aggregate_bwd_host": (c_int, [c_void_p] * 7 + [c_int] * 5 + [c_long, c_int]),
    "lt_test_softargmax3d_bwd_host": (c_int, [c_void_p] * 5 + [c_int, c_int, c_long, c_float, c_int]),
    "lt_softargmax3d_workspace_bytes": (c_size_t, [c_int, c_int, c_long]),
    "lt_softargmax3d_fwd": (c_int, [c_void_p, c_long, c_long, c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                    c_int, c_int, c_long, c_float, c_int, c_void_p]),
    "lt_conv_nd_fwd": (c_int, [ctypes.POINTER(ConvDesc)] + [c_void_p] * 6 + [c_int, c_void_p]),
    "lt_conv_tc_weight_bytes": (c_size_t, [c_int, c_int, c_int]),
    "lt_conv_tc_pack_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "lt_absmax_fwd": (c_int, [c_void_p, c_long, c_void_p, c_void_p]),
    "lt_conv_gather_weights_fwd": (c_int, [c_void_p] + [c_long] * 6 + [c_int] * 7 + [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "lt_fold_bn_fwd": (c_int, [c_void_p] * 5 + [c_float, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "lt_conv_pair_weight_bytes": (c_size_t, [c_int, c_int, c_int]),
    "lt_conv_pair_pack_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "lt_conv_pair_eligible": (c_int, [ctypes.POINTER(ConvDesc)]),
    "lt_v2v_tail_fwd": (c_int, [c_void_p] * 11 + [c_long, c_int, c_void_p]),
    "lt_v2v_tail_stats_fwd": (c_int, [c_void_p] * 11 + [c_int, c_long, c_int, c_void_p, c_int, c_float, c_int, c_void_p, c_size_t,
                                      ctypes.POINTER(c_int), c_void_p]),
    "lt_softargmax3d_finish_fwd": (c_int, [c_void_p, c_long, c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_long, c_int,
                                           c_float, c_int, c_void_p]),
    "lt_conv_fold_weight_bytes": (c_size_t, [c_int, c_int]),
    "lt_conv_fold_pack_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "lt_maxpool_fwd": (c_int, [c_void_p, c_void_p] + [c_int] * 18 + [c_void_p]),
    "lt_gap_mlp3_fwd": (c_int, [c_void_p] + [c_int] * 7 + [c_void_p] * 7 + [c_void_p]),
    "lt_view_normalize_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p]),
    "lt_triangulate_dlt_fwd": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "lt_nchw_to_nhwc_f32": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "lt_images_hwc_to_nchw_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "lt_stem_s2d_fwd": (c_int, [c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "lt_f32_to_s32": (c_int, [c_void_p, c_void_p, c_long, c_int, c_void_p]),
    "lt_s32_to_f32": (c_int, [c_void_p, c_void_p, c_long, c_int, c_void_p]),
    "lt_cl_to_cf_f32": (c_int, [c_void_p, c_void_p, c_int, c_long, c_int, c_int, c_void_p]),
    "lt_tc_gemm_selftest": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
}

_lib = None


def lib():
    """Load (building first if the .so is missing or stale and nvcc is present) the native library.

    Fails loudly: there is no Python/CPU substitute for these kernels.
    """
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH) or (os.path.exists("/usr/local/cuda/bin/nvcc") and not _build.is_current()):
            _build.build()
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("liblt_b200.so is missing and could not be built -- the native CUDA extension is required")
        handle = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the .so does not export a declared symbol
            fn.restype = res
            fn.argtypes = args
        _lib = handle
        _apply_env_options(handle)
    return _lib


def _apply_env_options(handle):
    """LT_OPT_<FIELD> environment overrides -> lt_set_options, once at load (the C library itself never reads the environment)."""
    o = Options()
    handle.lt_default_options(ctypes.byref(o))
    changed = False
    for name, _ in Options._fields_:
        v = os.environ.get(OPTIONS_ENV_PREFIX + name.upper())
        if v is not None:
            setattr(o, name, int(v))
            changed = True
    if changed and handle.lt_set_options(ctypes.byref(o)) != 0:
        raise RuntimeError("lt_set_options failed: %s" % handle.lt_last_error_string().decode())


def set_options(**kw):
    """Explicit options API: capi.set_options(unproject_cpl=8, ...)."""
    o = Options()
    _check(lib().lt_get_options(ctypes.byref(o)), "lt_get_options")
    for k, v in kw.items():
        if k not in dict(Options._fields_):
            raise KeyError("unknown lt_options field %r" % k)
        setattr(o, k, int(v))
    _check(lib().lt_set_options(ctypes.byref(o)), "lt_set_options")


def get_options():
    o = Options()
    _check(lib().lt_get_options(ctypes.byref(o)), "lt_get_options")
    return {n: getattr(o, n) for n, _ in Options._fields_}


def _check(rc, what):
    if rc != 0:
        raise RuntimeError("%s failed (%d): %s" % (what, rc, lib().lt_last_error_string().decode()))


def _stream():
    """Stream of the CURRENT device: callers that work on another device wrap the call in `torch.cuda.device(...)`
    (VolumetricTriangulationNet.forward does)."""
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    if t is None:
        return None
    assert t.is_cuda and t.is_contiguous(), "native kernels need contiguous CUDA tensors"
    return t.data_ptr()


# ---- thin wrappers -------------------------------------------------------------------------------

def device_info():
    sm, major, minor = c_int(), c_int(), c_int()
    _check(lib().lt_device_info(ctypes.byref(sm), ctypes.byref(major), ctypes.byref(minor)), "lt_device_info")
    return sm.value, major.value, minor.value


def coord_volume(position, center, step, rot, out, transfer_cmu=False):
    B, n = out.shape[0], out.shape[1]
    _check(lib().lt_coord_volume_fwd(_ptr(position), _ptr(center), _ptr(step), _ptr(rot), _ptr(out), B, n,
                                     int(transfer_cmu), _stream()), "lt_coord_volume_fwd")


def unproject_aggregate(features_cl, proj, coord, conf, out, out_format, agg):
    B, V, h, w, C = features_cl.shape
    nvox = coord.shape[1]
    _check(lib().lt_unproject_aggregate_fwd(_ptr(features_cl), _ptr(proj), _ptr(coord), _ptr(conf), _ptr(out), out_format,
                                            B, V, C, h, w, nvox, agg, _stream()), "lt_unproject_aggregate_fwd")


def unproject_partial(features_cl, proj, coord, conf, partial, agg):
    B, V, h, w, C = features_cl.shape
    nvox = coord.shape[1]
    _check(lib().lt_unproject_partial_fwd(_ptr(features_cl), _ptr(proj), _ptr(coord), _ptr(conf), _ptr(partial),
                                          B, V, C, h, w, nvox, agg, _stream()), "lt_unproject_partial_fwd")


def unproject_finalize(partial, out, out_format, B, C, nvox, agg):
    _check(lib().lt_unproject_finalize_fwd(_ptr(partial), _ptr(out), out_format, B, C, nvox, agg, _stream()),
           "lt_unproject_finalize_fwd")


def unproject_push(features_cl, proj, coord, conf, peer_ptrs, src_rank, agg):
    """peer_ptrs: list of int device pointers (one reduction buffer per rank of the view group)."""
    B, V, h, w, C = features_cl.shape
    nvox = coord.shape[1]
    arr = (c_void_p * len(peer_ptrs))(*peer_ptrs)
    _check(lib().lt_unproject_push_fwd(_ptr(features_cl), _ptr(proj), _ptr(coord), _ptr(conf), arr, len(peer_ptrs), src_rank,
                                       B, V, C, h, w, nvox, agg, _stream()), "lt_unproject_push_fwd")


def feature_scatter(feats_local, peer_ptrs, view_rank, n_views):
    """feats_local (B, V_local, h, w, C) float32 -> rows of the owners' peer buffers ([B/G][V][h*w*C] each)."""
    B, Vl = feats_local.shape[:2]
    row = feats_local[0, 0].numel()
    arr = (c_void_p * len(peer_ptrs))(*peer_ptrs)
    _check(lib().lt_feature_scatter_fwd(_ptr(feats_local), arr, len(peer_ptrs), view_rank, B, Vl, n_views, row, _stream()),
           "lt_feature_scatter_fwd")


def unproject_reduce_finalize(slots, nslots, out, out_format, B, C, nvox, agg):
    _check(lib().lt_unproject_reduce_finalize_fwd(_ptr(slots), nslots, _ptr(out), out_format, B, C, nvox, agg, _stream()),
           "lt_unproject_reduce_finalize_fwd")


def softargmax3d(logits, batch_stride, voxel_stride, chan_stride, coord, volumes_out, keypoints_out, workspace,
                 B, J, nvox, multiplier, softmax):
    _check(lib().lt_softargmax3d_fwd(_ptr(logits), batch_stride, voxel_stride, chan_stride, _ptr(coord), _ptr(volumes_out),
                                     _ptr(keypoints_out), _ptr(workspace), workspace.numel() * workspace.element_size(),
                                     B, J, nvox, float(multiplier), int(softmax), _stream()), "lt_softargmax3d_fwd")


def unproject_aggregate_bwd(features_cl, proj, coord, conf, grad_out_cl, grad_features_cl, grad_conf, agg):
    B, V, h, w, C = features_cl.shape
    nvox = coord.shape[1]
    _check(lib().lt_unproject_aggregate_bwd(_ptr(features_cl), _ptr(proj), _ptr(coord), _ptr(conf), _ptr(grad_out_cl), _ptr(grad_features_cl),
                                            _ptr(grad_conf), B, V, C, h, w, nvox, agg, _stream()), "lt_unproject_aggregate_bwd")


def softargmax3d_bwd(probs, coord, grad_keypoints, grad_volumes, grad_logits, scratch, B, J, nvox, multiplier, softmax):
    _check(lib().lt_softargmax3d_bwd(_ptr(probs), _ptr(coord), _ptr(grad_keypoints), _ptr(grad_volumes), _ptr(grad_logits), _ptr(scratch),
                                     B, J, nvox, float(multiplier), int(softmax), _stream()), "lt_softargmax3d_bwd")


def softargmax3d_workspace_bytes(B, J, nvox):
    return lib().lt_softargmax3d_workspace_bytes(B, J, nvox)


def conv_nd(desc, inp, weight, scale, shift, residual, out, impl):
    _check(lib().lt_conv_nd_fwd(ctypes.byref(desc), _ptr(inp), _ptr(weight), _ptr(scale), _ptr(shift), _ptr(residual),
                                _ptr(out), impl, _stream()), "lt_conv_nd_fwd")


def conv_tc_weight_bytes(taps, cin, cout):
    return lib().lt_conv_tc_weight_bytes(taps, cin, cout)


def conv_tc_pack_weights(w_tap_ci_co, packed, taps, cin, cout):
    _check(lib().lt_conv_tc_pack_weights(_ptr(w_tap_ci_co), _ptr(packed), taps, cin, cout, _stream()), "lt_conv_tc_pack_weights")


def absmax(w, out_bits):
    """out_bits: int32[1] device tensor receiving the float bit pattern of max|w|."""
    _check(lib().lt_absmax_fwd(_ptr(w), w.numel(), _ptr(out_bits), _stream()), "lt_absmax_fwd")


def conv_gather_weights(w, base, strides, k, cin, cin_p, cout, cout_p, out, absmax_bits=None, out_ld=0, out_col0=0):
    """w: the module's own filter tensor; strides = element strides of (td, th, tw, ci, co); out float32 [taps][cin_p][out_ld],
    columns [out_col0, out_col0 + cout_p) are written."""
    _check(lib().lt_conv_gather_weights_fwd(_ptr(w), base, *[int(v) for v in strides], k[0], k[1], k[2], cin, cin_p, cout, cout_p,
                                            _ptr(absmax_bits), _ptr(out), out_ld, out_col0, _stream()), "lt_conv_gather_weights_fwd")


def fold_bn(gamma, beta, mean, var, bias, eps, c, cp, scale, shift, absmax_bits=None, accum_steps=0):
    _check(lib().lt_fold_bn_fwd(_ptr(gamma), _ptr(beta), _ptr(mean), _ptr(var), _ptr(bias), float(eps), c, cp, _ptr(absmax_bits),
                                int(accum_steps), _ptr(scale), _ptr(shift), _stream()), "lt_fold_bn_fwd")


def conv_pair_weight_bytes(taps, cin, cout):
    return lib().lt_conv_pair_weight_bytes(taps, cin, cout)


def conv_pair_pack_weights(w_tap_ci_co, packed, taps, cin, cout):
    _check(lib().lt_conv_pair_pack_weights(_ptr(w_tap_ci_co), _ptr(packed), taps, cin, cout, _stream()), "lt_conv_pair_pack_weights")


def conv_pair_eligible(desc):
    return bool(lib().lt_conv_pair_eligible(ctypes.byref(desc)))


def v2v_tail(x, w1, w2, w3, scale1, shift1, scale2, shift2, scale3, bias3, logits, rows, fc):
    _check(lib().lt_v2v_tail_fwd(_ptr(x), _ptr(w1), _ptr(w2), _ptr(w3), _ptr(scale1), _ptr(shift1), _ptr(scale2), _ptr(shift2), _ptr(scale3), _ptr(bias3),
                                 _ptr(logits), rows, fc, _stream()), "lt_v2v_tail_fwd")


def v2v_tail_stats(x, w1, w2, w3, scale1, shift1, scale2, shift2, scale3, bias3, logits, B, nvox, fc, coord, J, multiplier, softmax, workspace):
    """lt_v2v_tail_fwd + the statistics pass of the volumetric soft-argmax; returns the number of partials per sample (for softargmax3d_finish)."""
    n = c_int(0)
    _check(lib().lt_v2v_tail_stats_fwd(_ptr(x), _ptr(w1), _ptr(w2), _ptr(w3), _ptr(scale1), _ptr(shift1), _ptr(scale2), _ptr(shift2), _ptr(scale3),
                                       _ptr(bias3), _ptr(logits), B, nvox, fc, _ptr(coord), J, float(multiplier), int(softmax), _ptr(workspace),
                                       workspace.numel() * workspace.element_size(), ctypes.byref(n), _stream()), "lt_v2v_tail_stats_fwd")
    return n.value


def softargmax3d_finish(logits, batch_stride, voxel_stride, coord, volumes_out, keypoints_out, workspace, B, J, nvox, G, multiplier, softmax):
    _check(lib().lt_softargmax3d_finish_fwd(_ptr(logits), batch_stride, voxel_stride, _ptr(coord), _ptr(volumes_out), _ptr(keypoints_out),
                                            _ptr(workspace), workspace.numel() * workspace.element_size(), B, J, nvox, G, float(multiplier),
                                            int(softmax), _stream()), "lt_softargmax3d_finish_fwd")


def conv_fold_weight_bytes(k, cout):
    return lib().lt_conv_fold_weight_bytes(k, cout)


def conv_fold_pack_weights(w_tap_ci_co, packed, k, cout):
    _check(lib().lt_conv_fold_pack_weights(_ptr(w_tap_ci_co), _ptr(packed), k, cout, _stream()), "lt_conv_fold_pack_weights")


def maxpool(inp, out, fmt, N, ID, IH, IW, C, k, s, p, OD, OH, OW):
    _check(lib().lt_maxpool_fwd(_ptr(inp), _ptr(out), fmt, N, ID, IH, IW, C, k[0], k[1], k[2], s[0], s[1], s[2],
                                p[0], p[1], p[2], OD, OH, OW, _stream()), "lt_maxpool_fwd")


def gap_mlp3(inp, fmt, N, P, C0, lin1, lin2, lin3, out):
    """lin*: (weight [out][in], bias) float32 CUDA tensors."""
    _check(lib().lt_gap_mlp3_fwd(_ptr(inp), fmt, N, P, C0, lin1[0].shape[0], lin2[0].shape[0], lin3[0].shape[0], _ptr(lin1[0]), _ptr(lin1[1]),
                                 _ptr(lin2[0]), _ptr(lin2[1]), _ptr(lin3[0]), _ptr(lin3[1]), _ptr(out), _stream()), "lt_gap_mlp3_fwd")


def view_normalize(conf, B, V, C, eps):
    _check(lib().lt_view_normalize_fwd(_ptr(conf), B, V, C, float(eps), _stream()), "lt_view_normalize_fwd")


def triangulate_dlt(proj, kp2d, conf, out):
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_triangulate_dlt_fwd(_ptr(proj), _ptr(kp2d), _ptr(conf), _ptr(out), B, V, J, _stream()), "lt_triangulate_dlt_fwd")


def nchw_to_nhwc(inp, out, N, C, H, W, Cp):
    _check(lib().lt_nchw_to_nhwc_f32(_ptr(inp), _ptr(out), N, C, H, W, Cp, _stream()), "lt_nchw_to_nhwc_f32")


IMG_DTYPE = {torch.uint8: 0, torch.float32: 1, torch.float64: 2}


def images_hwc_to_nchw(inp, lut, out, N, C, H, W):
    """inp: device tensor [N][H][W][C] uint8/float32/float64; lut: None or float32 [C][256]; out: float32 [N][C][H][W]."""
    _check(lib().lt_images_hwc_to_nchw_fwd(_ptr(inp), IMG_DTYPE[inp.dtype], None if lut is None else _ptr(lut), _ptr(out),
                                           N, C, H, W, _stream()), "lt_images_hwc_to_nchw_fwd")


def stem_s2d(inp, out, N, C, H, W):
    _check(lib().lt_stem_s2d_fwd(_ptr(inp), _ptr(out), N, C, H, W, _stream()), "lt_stem_s2d_fwd")


def f32_to_s32(inp, out, pixels, C):
    _check(lib().lt_f32_to_s32(_ptr(inp), _ptr(out), pixels, C, _stream()), "lt_f32_to_s32")


def s32_to_f32(inp, out, pixels, C):
    _check(lib().lt_s32_to_f32(_ptr(inp), _ptr(out), pixels, C, _stream()), "lt_s32_to_f32")


def cl_to_cf(inp, out, N, P, Cs, C):
    _check(lib().lt_cl_to_cf_f32(_ptr(inp), _ptr(out), N, P, Cs, C, _stream()), "lt_cl_to_cf_f32")


def tc_gemm_selftest(a_fp16, b_fp16, d, M, N, K, variant=0):
    _check(lib().lt_tc_gemm_selftest(_ptr(a_fp16), _ptr(b_fp16), _ptr(d), M, N, K, variant, _stream()), "lt_tc_gemm_selftest")
