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
KIND = {"mpii": 0, "coco": 1}
CONV_SIMT, CONV_TC, CONV_TC1, CONV_TC_FOLD = 0, 1, 2, 3
RES_NONE, RES_BEFORE_RELU, RES_AFTER_RELU = 0, 1, 2

c_int, c_long, c_float, c_double, c_void_p, c_size_t = ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_double, ctypes.c_void_p, ctypes.c_size_t


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


class ConvTcPlan(ctypes.Structure):
    """Mirror of `struct lt_conv_tc_launch_plan` (include/lt_b200.h)."""
    _fields_ = [(n, c_int) for n in ("nt", "m_tiles", "n_tiles", "chunks", "splits", "grid", "stages", "epi_buffers")]


class ConvTcChainPlan(ctypes.Structure):
    """Mirror of `struct lt_conv_tc_chain_launch_plan` (include/lt_b200.h)."""
    _fields_ = [("m_tiles", c_int), ("n_tiles", c_int * 3), ("units", c_int), ("grid", c_int), ("counters", c_int)]


class ConvTcChainUnit(ctypes.Structure):
    """Mirror of `struct lt_conv_tc_chain_unit` (include/lt_b200.h)."""
    _fields_ = [(n, c_int) for n in ("layer", "m_tile", "n_tile", "src_layer", "need", "n_deps")]


class ConvWgradPlan(ctypes.Structure):
    """Mirror of `struct lt_conv_wgrad_launch_plan` (include/lt_b200.h)."""
    _fields_ = [(n, c_int) for n in ("nwg", "ngroups", "m_tiles", "splits", "stages")]


class BatchNormPlan(ctypes.Structure):
    """Mirror of `struct lt_batch_norm_launch_plan` (include/lt_b200.h)."""
    _fields_ = [(n, c_int) for n in ("tc", "ry", "cblocks", "want_splits", "max_splits", "splits")] + [("rows_per_split", c_long),
                                                                                                        ("row_blocks", c_int)]


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
    "lt_cuboid_from_keypoints_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_double, c_void_p, c_void_p, c_void_p]),
    "lt_unproject_aggregate_fwd": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_long, c_int, c_void_p]),
    "lt_unproject_partial_fwd": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_unproject_finalize_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_long, c_int, c_void_p]),
    "lt_unproject_push_fwd": (c_int, [c_void_p] * 4 + [ctypes.POINTER(c_void_p), c_int, c_int] + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_unproject_reduce_finalize_fwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_long, c_int, c_void_p]),
    "lt_feature_scatter_fwd": (c_int, [c_void_p, ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_int, c_int, c_long, c_void_p]),
    "lt_unproject_aggregate_bwd": (c_int, [c_void_p] * 7 + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_softargmax3d_bwd": (c_int, [c_void_p] * 6 + [c_int, c_int, c_long, c_float, c_int, c_void_p]),
    "lt_unproject_aggregate_bwd_geom_workspace_bytes": (c_size_t, [c_int, c_int, c_long]),
    "lt_unproject_aggregate_bwd_geom": (c_int, [c_void_p] * 10 + [c_size_t] + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_softargmax3d_coord_bwd": (c_int, [c_void_p] * 3 + [c_int, c_int, c_long, c_int, c_void_p]),
    "lt_unproject_aggregate_bwd_det_workspace_bytes": (c_size_t, [c_int] * 5 + [c_long, c_int, c_int]),
    "lt_unproject_aggregate_bwd_det": (c_int, [c_void_p] * 10 + [c_size_t] + [c_int] * 5 + [c_long, c_int, c_void_p]),
    "lt_test_unproject_aggregate_bwd_det_host": (c_int, [c_void_p] * 9 + [c_int] * 5 + [c_long, c_int]),
    "lt_maxpool3d_bwd": (c_int, [c_void_p] * 3 + [c_int] * 5 + [c_long] * 10 + [c_int, c_void_p]),
    "lt_test_maxpool3d_bwd_host": (c_int, [c_void_p] * 3 + [c_int] * 5 + [c_long] * 10 + [c_int]),
    "lt_test_unproject_aggregate_bwd_geom_host": (c_int, [c_void_p] * 9 + [c_int] * 5 + [c_long, c_int]),
    "lt_test_softargmax3d_coord_bwd_host": (c_int, [c_void_p] * 3 + [c_int, c_int, c_long]),
    "lt_test_unproject_aggregate_bwd_host": (c_int, [c_void_p] * 7 + [c_int] * 5 + [c_long, c_int]),
    "lt_test_softargmax3d_bwd_host": (c_int, [c_void_p] * 5 + [c_int, c_int, c_long, c_float, c_int]),
    "lt_softargmax3d_workspace_bytes": (c_size_t, [c_int, c_int, c_long]),
    "lt_softargmax3d_fwd": (c_int, [c_void_p, c_long, c_long, c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t,
                                    c_int, c_int, c_long, c_float, c_int, c_void_p]),
    "lt_conv_nd_fwd": (c_int, [ctypes.POINTER(ConvDesc)] + [c_void_p] * 6 + [c_int, c_void_p]),
    "lt_conv_tc_weight_bytes": (c_size_t, [c_int, c_int, c_int]),
    "lt_conv_tc_plan": (c_int, [ctypes.POINTER(ConvDesc), c_int, c_int, ctypes.POINTER(ConvTcPlan)]),
    "lt_conv_tc_pack_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "lt_conv_tc_chain_plan": (c_int, [ctypes.POINTER(ConvDesc), c_int, c_int, ctypes.POINTER(ConvTcChainPlan)]),
    "lt_conv_tc_chain_deps": (c_int, [ctypes.POINTER(ConvDesc), c_int, c_int, ctypes.POINTER(ConvTcChainUnit), ctypes.POINTER(c_int), c_int]),
    "lt_conv_tc_chain_fwd": (c_int, [ctypes.POINTER(ConvDesc), c_int, c_void_p] + [ctypes.POINTER(c_void_p)] * 4 + [c_void_p, c_size_t, c_int,
                                                                                                              c_void_p]),
    "lt_absmax_fwd": (c_int, [c_void_p, c_long, c_void_p, c_void_p]),
    "lt_conv_gather_weights_fwd": (c_int, [c_void_p] + [c_long] * 6 + [c_int] * 7 + [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "lt_fold_bn_fwd": (c_int, [c_void_p] * 5 + [c_float, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "lt_v2v_tail_fwd": (c_int, [c_void_p] * 11 + [c_long, c_int, c_void_p]),
    "lt_v2v_tail_stats_fwd": (c_int, [c_void_p] * 11 + [c_int, c_long, c_int, c_void_p, c_int, c_float, c_int, c_void_p, c_size_t,
                                      ctypes.POINTER(c_int), c_void_p]),
    "lt_softargmax3d_finish_fwd": (c_int, [c_void_p, c_long, c_long, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_int, c_int, c_long, c_int,
                                           c_float, c_int, c_void_p]),
    "lt_conv_wgrad_workspace_bytes": (c_size_t, [ctypes.POINTER(ConvDesc)]),
    "lt_conv_wgrad_plan": (c_int, [ctypes.POINTER(ConvDesc), c_int, ctypes.POINTER(ConvWgradPlan)]),
    "lt_conv_wgrad_fwd": (c_int, [ctypes.POINTER(ConvDesc)] + [c_void_p] * 3 + [c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "lt_test_conv_wgrad_host": (c_int, [ctypes.POINTER(ConvDesc), c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "lt_f32_to_s32_scaled": (c_int, [c_void_p, c_void_p, c_long, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "lt_conv_fold_weight_bytes": (c_size_t, [c_int, c_int]),
    "lt_conv_fold_pack_weights": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "lt_maxpool_fwd": (c_int, [c_void_p, c_void_p] + [c_int] * 18 + [c_void_p]),
    "lt_gap_mlp3_fwd": (c_int, [c_void_p] + [c_int] * 7 + [c_void_p] * 7 + [c_void_p]),
    "lt_view_normalize_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p]),
    "lt_conf_head_tail_fwd": (c_int, [c_void_p] + [c_int] * 4 + [c_long] * 4 + [c_int] * 3 + [c_void_p] * 10 + [c_void_p]),
    "lt_conf_head_tail_bwd_workspace_bytes": (c_size_t, [c_int] * 5),
    "lt_conf_head_tail_bwd": (c_int, [c_void_p] + [c_int] * 4 + [c_long] * 8 + [c_int] * 3 + [c_void_p] * 16 + [c_size_t, c_void_p]),
    "lt_test_conf_head_tail_host": (c_int, [c_void_p] + [c_int] * 4 + [c_long] * 8 + [c_int] * 3 + [c_void_p] * 18),
    "lt_view_normalize_bwd": (c_int, [c_void_p] * 3 + [c_int] * 3 + [c_void_p]),
    "lt_test_view_normalize_bwd_host": (c_int, [c_void_p] * 3 + [c_int] * 3),
    "lt_triangulate_dlt_fwd": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "lt_triangulate_dlt_bwd": (c_int, [c_void_p] * 6 + [c_int] * 3 + [c_void_p]),
    "lt_test_triangulate_dlt_fwd_host": (c_int, [c_void_p] * 4 + [c_int] * 3),
    "lt_test_triangulate_dlt_bwd_host": (c_int, [c_void_p] * 6 + [c_int] * 3),
    "lt_triangulate_dlt_proj_bwd_workspace_bytes": (c_size_t, [c_int] * 3),
    "lt_triangulate_dlt_proj_bwd": (c_int, [c_void_p] * 6 + [c_size_t] + [c_int] * 3 + [c_void_p]),
    "lt_test_triangulate_dlt_proj_bwd_host": (c_int, [c_void_p] * 5 + [c_int] * 3),
    "lt_heatmap_argmax_workspace_bytes": (c_size_t, [c_int] * 4),
    "lt_heatmap_argmax_fwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t] + [c_int] * 4 + [c_float, c_float, c_void_p]),
    "lt_triangulate_ransac_fwd": (c_int, [c_void_p] * 3 + [c_int] * 4 + [c_double, c_int, c_void_p, c_void_p, c_void_p]),
    "lt_test_triangulate_ransac_host": (c_int, [c_void_p] * 3 + [c_int] * 4 + [c_double, c_int, c_void_p, c_void_p]),
    "lt_volumetric_ce_workspace_bytes": (c_size_t, [c_int, c_int, c_long]),
    "lt_volumetric_ce_fwd": (c_int, [c_void_p] * 8 + [c_size_t, c_int, c_int, c_long, c_void_p]),
    "lt_volumetric_ce_bwd": (c_int, [c_void_p] * 5 + [c_int, c_int, c_long, c_void_p]),
    "lt_test_volumetric_ce_host": (c_int, [c_void_p] * 9 + [c_int, c_int, c_long]),
    "lt_keypoints_loss_fwd": (c_int, [c_void_p] * 5 + [c_int, c_double, c_int, c_int, c_void_p]),
    "lt_keypoints_loss_bwd": (c_int, [c_void_p] * 6 + [c_int, c_double, c_int, c_int, c_void_p]),
    "lt_test_keypoints_loss_host": (c_int, [c_void_p] * 7 + [c_int, c_double, c_int, c_int]),
    "lt_batch_norm_workspace_bytes": (c_size_t, [c_long, c_int]),
    "lt_batch_norm_plan": (c_int, [c_long, c_int, c_int, ctypes.POINTER(BatchNormPlan)]),
    "lt_batch_norm_fwd": (c_int, [c_void_p] * 9 + [c_long, c_int, c_float, c_float, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "lt_batch_norm_bwd": (c_int, [c_void_p] * 10 + [c_long, c_int, c_int, c_int, c_void_p, c_size_t, c_void_p]),
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


def cuboid_from_keypoints(keypoints_3d, kind, cuboid_side, center, position):
    """keypoints_3d (B, J, 3) float32 -> center and position (B, 3) float32, written: the base point of skeleton `kind` ("mpii" or
    "coco") and base - cuboid_side / 2 formed in float64, as the host geometry computes them."""
    B, J = keypoints_3d.shape[:2]
    assert keypoints_3d.dtype == center.dtype == position.dtype == torch.float32
    _check(lib().lt_cuboid_from_keypoints_fwd(_ptr(keypoints_3d), B, J, KIND[kind], float(cuboid_side), _ptr(center), _ptr(position),
                                              _stream()), "lt_cuboid_from_keypoints_fwd")


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


def unproject_aggregate_bwd_geom(features_cl, proj, coord, conf, grad_out_cl, grad_features_cl, grad_conf, grad_proj, grad_coord, agg,
                                 workspace):
    """lt_unproject_aggregate_bwd_geom: grad_features_cl / grad_conf accumulated into, grad_proj (B, V, 12) and grad_coord (B, nvox, 3)
    (either None) written; workspace: unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox) bytes."""
    B, V, h, w, C = features_cl.shape
    nvox = coord.shape[1]
    _check(lib().lt_unproject_aggregate_bwd_geom(_ptr(features_cl), _ptr(proj), _ptr(coord), _ptr(conf), _ptr(grad_out_cl),
                                                 _ptr(grad_features_cl), _ptr(grad_conf), _ptr(grad_proj), _ptr(grad_coord), _ptr(workspace),
                                                 workspace.numel() * workspace.element_size(), B, V, C, h, w, nvox, agg, _stream()),
           "lt_unproject_aggregate_bwd_geom")


def unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox):
    return lib().lt_unproject_aggregate_bwd_geom_workspace_bytes(B, V, nvox)


def unproject_aggregate_bwd_det(features_cl, proj, coord, conf, grad_out_cl, grad_features_cl, grad_conf, grad_proj, grad_coord, agg,
                                workspace):
    """lt_unproject_aggregate_bwd_det, the fixed-order backward: arguments as unproject_aggregate_bwd_geom (grad_proj and grad_coord may
    both be None); workspace: unproject_aggregate_bwd_det_workspace_bytes(...) bytes."""
    B, V, h, w, C = features_cl.shape
    nvox = coord.shape[1]
    _check(lib().lt_unproject_aggregate_bwd_det(_ptr(features_cl), _ptr(proj), _ptr(coord), _ptr(conf), _ptr(grad_out_cl),
                                                _ptr(grad_features_cl), _ptr(grad_conf), _ptr(grad_proj), _ptr(grad_coord), _ptr(workspace),
                                                workspace.numel() * workspace.element_size(), B, V, C, h, w, nvox, agg, _stream()),
           "lt_unproject_aggregate_bwd_det")


def unproject_aggregate_bwd_det_workspace_bytes(B, V, C, h, w, nvox, agg, geom):
    n = lib().lt_unproject_aggregate_bwd_det_workspace_bytes(B, V, C, h, w, nvox, agg, int(bool(geom)))
    if n == 0:
        raise RuntimeError("lt_unproject_aggregate_bwd_det_workspace_bytes: sizes out of range or no CUDA device")
    return n


def maxpool3d_bwd(x, grad_y, grad_x, k):
    """lt_maxpool3d_bwd: grad_x (strides of x) written from float32 x and grad_y (N, C, D, H, W) tensors of any strides."""
    N, C, D, H, W = x.shape
    assert x.is_cuda and grad_y.is_cuda and grad_x.is_cuda and x.stride() == grad_x.stride()
    assert x.dtype == grad_y.dtype == grad_x.dtype == torch.float32
    _check(lib().lt_maxpool3d_bwd(x.data_ptr(), grad_y.data_ptr(), grad_x.data_ptr(), N, C, D, H, W, *x.stride(), *grad_y.stride(), int(k),
                                  _stream()), "lt_maxpool3d_bwd")


def softargmax3d_coord_bwd(probs, grad_keypoints, grad_coord, B, J, nvox, softmax):
    """grad_coord (B, nvox, 3) = sum_j probs (B, J, nvox) x grad_keypoints (B, J, 3), written; modes 0 and 1 only."""
    _check(lib().lt_softargmax3d_coord_bwd(_ptr(probs), _ptr(grad_keypoints), _ptr(grad_coord), B, J, nvox, int(softmax), _stream()),
           "lt_softargmax3d_coord_bwd")


def softargmax3d_workspace_bytes(B, J, nvox):
    return lib().lt_softargmax3d_workspace_bytes(B, J, nvox)


def conv_nd(desc, inp, weight, scale, shift, residual, out, impl):
    _check(lib().lt_conv_nd_fwd(ctypes.byref(desc), _ptr(inp), _ptr(weight), _ptr(scale), _ptr(shift), _ptr(residual),
                                _ptr(out), impl, _stream()), "lt_conv_nd_fwd")


def conv_tc_plan(desc, sm_count, splitk=1):
    """Host-only work decomposition of an LT_CONV_TC launch (lt_conv_tc_plan): dict of nt, m_tiles, n_tiles, chunks, splits, grid,
    stages, epi_buffers."""
    plan = ConvTcPlan()
    _check(lib().lt_conv_tc_plan(ctypes.byref(desc), sm_count, splitk, ctypes.byref(plan)), "lt_conv_tc_plan")
    return {name: getattr(plan, name) for name, _ in ConvTcPlan._fields_}


def _chain_descs(descs):
    assert len(descs) == 3
    return (ConvDesc * 3)(*descs)


def conv_tc_chain_plan(descs, blocks, sm_count):
    """Host-only work decomposition of a chain launch (lt_conv_tc_chain_plan) of `blocks` blocks whose three layers the ConvDescs
    `descs` describe: dict of m_tiles, n_tiles (3), units, grid, counters."""
    plan = ConvTcChainPlan()
    _check(lib().lt_conv_tc_chain_plan(_chain_descs(descs), blocks, sm_count, ctypes.byref(plan)), "lt_conv_tc_chain_plan")
    return {"m_tiles": plan.m_tiles, "n_tiles": list(plan.n_tiles), "units": plan.units, "grid": plan.grid, "counters": plan.counters}


def conv_tc_chain_deps(descs, blocks, unit, cap=64):
    """lt_conv_tc_chain_deps: (layer, m_tile, n_tile, src_layer, need, [tiles of src_layer unit `unit` waits for])."""
    info = ConvTcChainUnit()
    tiles = (c_int * cap)()
    _check(lib().lt_conv_tc_chain_deps(_chain_descs(descs), blocks, unit, ctypes.byref(info), tiles, cap), "lt_conv_tc_chain_deps")
    return info.layer, info.m_tile, info.n_tile, info.src_layer, info.need, list(tiles[:info.n_deps])


def conv_tc_chain(descs, blocks, x, bufs, weights, scales, shifts, counters, impl):
    """lt_conv_tc_chain_fwd: `blocks` bottleneck blocks in one launch, in place on tensor x; bufs: the 4 intermediate tensors (Y1 even,
    Y1 odd, Y2 even, Y2 odd); weights / scales / shifts: 3 x blocks tensors; counters: device scratch of plan["counters"] int32."""
    n = 3 * blocks
    assert len(bufs) == 4 and len(weights) == len(scales) == len(shifts) == n
    arr = lambda ts: (c_void_p * len(ts))(*[t.data_ptr() for t in ts])
    _check(lib().lt_conv_tc_chain_fwd(_chain_descs(descs), blocks, _ptr(x), arr(bufs), arr(weights), arr(scales), arr(shifts), _ptr(counters),
                                      counters.numel() * counters.element_size(), impl, _stream()), "lt_conv_tc_chain_fwd")


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


def _map_dims(x):
    """(N, C, H, W) and element strides of a float32 map of any strides (lt_conf_head_tail_*)."""
    assert x.dim() == 4 and x.dtype == torch.float32, "the confidence-head tail takes a float32 (N, C, H, W) map"
    return tuple(x.shape), tuple(x.stride())


def conf_head_tail(x, lin1, lin2, lin3, out, x0, h1, h2):
    """lt_conf_head_tail_fwd: x (N, C0, H, W) float32 CUDA of any element strides, lin* = (weight, bias) of the three nn.Linear layers
    -> out (N, NO), x0 (N, C0), h1 (N, H1), h2 (N, H2) written."""
    (N, C0, H, W), xs = _map_dims(x)
    assert x.is_cuda
    _check(lib().lt_conf_head_tail_fwd(x.data_ptr(), N, C0, H, W, *xs, lin1[0].shape[0], lin2[0].shape[0], lin3[0].shape[0],
                                       _ptr(lin1[0]), _ptr(lin1[1]), _ptr(lin2[0]), _ptr(lin2[1]), _ptr(lin3[0]), _ptr(lin3[1]), _ptr(out),
                                       _ptr(x0), _ptr(h1), _ptr(h2), _stream()), "lt_conf_head_tail_fwd")


def conf_head_tail_bwd_workspace_bytes(N, C0, H1, H2, NO):
    return lib().lt_conf_head_tail_bwd_workspace_bytes(N, C0, H1, H2, NO)


def conf_head_tail_bwd(x, w1, w2, w3, x0, h1, h2, y, grad_y, grad_x, grads, workspace):
    """lt_conf_head_tail_bwd: grad_x (any element strides, the shape of x) and grads = (dW1, db1, dW2, db2, dW3, db3) written."""
    (N, C0, H, W), xs = _map_dims(x)
    assert x.is_cuda and tuple(grad_x.shape) == (N, C0, H, W)
    _check(lib().lt_conf_head_tail_bwd(x.data_ptr(), N, C0, H, W, *xs, *grad_x.stride(), w1.shape[0], w2.shape[0], w3.shape[0], _ptr(w1),
                                       _ptr(w2), _ptr(w3), _ptr(x0), _ptr(h1), _ptr(h2), _ptr(y), _ptr(grad_y), grad_x.data_ptr(),
                                       *[_ptr(t) for t in grads], _ptr(workspace), workspace.numel() * workspace.element_size(), _stream()),
           "lt_conf_head_tail_bwd")


def view_normalize_bwd(conf, grad, grad_conf):
    """lt_view_normalize_bwd: conf, grad, grad_conf (B, V, C) float32 contiguous."""
    B, V, C = conf.shape
    _check(lib().lt_view_normalize_bwd(_ptr(conf), _ptr(grad), _ptr(grad_conf), B, V, C, _stream()), "lt_view_normalize_bwd")


def triangulate_dlt(proj, kp2d, conf, out):
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_triangulate_dlt_fwd(_ptr(proj), _ptr(kp2d), _ptr(conf), _ptr(out), B, V, J, _stream()), "lt_triangulate_dlt_fwd")


def triangulate_dlt_bwd(proj, kp2d, conf, grad_out, grad_kp2d, grad_conf):
    """grad_kp2d (B, V, J, 2) and grad_conf (B, V, J) or None are written, not accumulated into."""
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_triangulate_dlt_bwd(_ptr(proj), _ptr(kp2d), _ptr(conf), _ptr(grad_out), _ptr(grad_kp2d), _ptr(grad_conf), B, V, J,
                                        _stream()), "lt_triangulate_dlt_bwd")


def triangulate_dlt_proj_bwd(proj, kp2d, conf, grad_out, grad_proj, workspace):
    """grad_proj (B, V, 3, 4) is written; workspace: triangulate_dlt_proj_bwd_workspace_bytes(B, V, J) bytes."""
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_triangulate_dlt_proj_bwd(_ptr(proj), _ptr(kp2d), _ptr(conf), _ptr(grad_out), _ptr(grad_proj), _ptr(workspace),
                                             workspace.numel() * workspace.element_size(), B, V, J, _stream()), "lt_triangulate_dlt_proj_bwd")


def triangulate_dlt_proj_bwd_workspace_bytes(B, V, J):
    return lib().lt_triangulate_dlt_proj_bwd_workspace_bytes(B, V, J)


def heatmap_argmax_workspace_bytes(N, J, h, w):
    return lib().lt_heatmap_argmax_workspace_bytes(N, J, h, w)


def heatmap_argmax(logits, C, heatmaps, keypoints_2d, workspace, N, J, h, w, scale_x, scale_y):
    """logits channels-last float32 (N, h, w, C) -> heatmaps (N, J, h, w) float32 and keypoints_2d (N, J, 2) int64, both written;
    scale_x / scale_y: image side over map side (rounded to float32 as the reference's float32 product rounds it)."""
    assert keypoints_2d.dtype == torch.int64
    _check(lib().lt_heatmap_argmax_fwd(_ptr(logits), C, _ptr(heatmaps), _ptr(keypoints_2d), _ptr(workspace),
                                       workspace.numel() * workspace.element_size(), N, J, h, w, float(scale_x), float(scale_y),
                                       _stream()), "lt_heatmap_argmax_fwd")


def triangulate_ransac(proj, kp2d, pairs, n_iters, eps, direct, out, inliers=None):
    """proj (B, V, 3, 4) float32, kp2d (B, V, J, 2) int64, pairs (B, J, n_iters, 2) int32 -> out (B, J, 3) float32 and inliers
    (B, J) int64 bit masks (optional), written."""
    B, V, J = kp2d.shape[:3]
    assert kp2d.dtype == torch.int64 and pairs.dtype == torch.int32 and (inliers is None or inliers.dtype == torch.int64)
    _check(lib().lt_triangulate_ransac_fwd(_ptr(proj), _ptr(kp2d), _ptr(pairs), B, V, J, int(n_iters), float(eps), int(bool(direct)),
                                           _ptr(out), _ptr(inliers), _stream()), "lt_triangulate_ransac_fwd")


def volumetric_ce_workspace_bytes(B, J, nvox):
    return lib().lt_volumetric_ce_workspace_bytes(B, J, nvox)


def volumetric_ce(probs, coord, keypoints_gt, validity, loss, index, picked, workspace):
    """probs (B, J, nvox), coord (B, nvox, 3), keypoints_gt (B, J, 3), validity (B, J) float32 -> loss (1,) float32,
    index (B, J) int32, picked (B, J) float32."""
    B, J, nvox = probs.shape
    _check(lib().lt_volumetric_ce_fwd(_ptr(probs), _ptr(coord), _ptr(keypoints_gt), _ptr(validity), _ptr(loss), _ptr(index), _ptr(picked),
                                      _ptr(workspace), workspace.numel() * workspace.element_size(), B, J, nvox, _stream()),
           "lt_volumetric_ce_fwd")


def volumetric_ce_bwd(grad_loss, index, picked, validity, grad_probs):
    """grad_loss: one float32 on the device; grad_probs (B, J, nvox) is written in full."""
    B, J, nvox = grad_probs.shape
    _check(lib().lt_volumetric_ce_bwd(_ptr(grad_loss), _ptr(index), _ptr(picked), _ptr(validity), _ptr(grad_probs), B, J, nvox, _stream()),
           "lt_volumetric_ce_bwd")


KEYPOINTS_LOSS = {"mse": 0, "mse_smooth": 1, "mae": 2, "l2": 3}


def keypoints_loss(pred, gt, validity, loss, norm, kind, threshold=400.0):
    """pred, gt (n, dim), validity (n,) float32 -> loss (1,) float32 and norm (1,) float64 (the divisor), written."""
    n, dim = pred.shape
    _check(lib().lt_keypoints_loss_fwd(_ptr(pred), _ptr(gt), _ptr(validity), _ptr(loss), _ptr(norm), KEYPOINTS_LOSS[kind],
                                       float(threshold), n, dim, _stream()), "lt_keypoints_loss_fwd")


def keypoints_loss_bwd(grad_loss, pred, gt, validity, norm, grad_pred, kind, threshold=400.0):
    """grad_loss: one float32 on the device; grad_pred (n, dim) is written in full."""
    n, dim = pred.shape
    _check(lib().lt_keypoints_loss_bwd(_ptr(grad_loss), _ptr(pred), _ptr(gt), _ptr(validity), _ptr(norm), _ptr(grad_pred),
                                       KEYPOINTS_LOSS[kind], float(threshold), n, dim, _stream()), "lt_keypoints_loss_bwd")


def batch_norm_workspace_bytes(M, C):
    return lib().lt_batch_norm_workspace_bytes(M, C)


def batch_norm_plan(M, C, sm_count):
    """Host-only launch plan of lt_batch_norm_fwd / _bwd (lt_batch_norm_plan): dict of tc, ry, cblocks, want_splits, max_splits, splits,
    rows_per_split, row_blocks."""
    plan = BatchNormPlan()
    _check(lib().lt_batch_norm_plan(M, C, sm_count, ctypes.byref(plan)), "lt_batch_norm_plan")
    return {name: getattr(plan, name) for name, _ in BatchNormPlan._fields_}


def batch_norm(x, residual, gamma, beta, running_mean, running_var, save_mean, save_invstd, y, M, C, eps, momentum, training, relu,
               workspace):
    """x, residual (or None), y: float32 channels-last [M][C]; per-channel vectors [C]; the running statistics are updated in place
    in training mode."""
    _check(lib().lt_batch_norm_fwd(_ptr(x), _ptr(residual), _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var),
                                   _ptr(save_mean), _ptr(save_invstd), _ptr(y), M, C, float(eps), float(momentum), int(training),
                                   int(relu), _ptr(workspace), workspace.numel() * workspace.element_size(), _stream()),
           "lt_batch_norm_fwd")


def batch_norm_bwd(x, y, grad_y, gamma, save_mean, save_invstd, grad_x, grad_residual, grad_gamma, grad_beta, M, C, training, relu,
                   workspace):
    """grad_x, grad_residual (or None), grad_gamma and grad_beta are written; y (the forward's output) is read with relu only."""
    _check(lib().lt_batch_norm_bwd(_ptr(x), _ptr(y), _ptr(grad_y), _ptr(gamma), _ptr(save_mean), _ptr(save_invstd), _ptr(grad_x),
                                   _ptr(grad_residual), _ptr(grad_gamma), _ptr(grad_beta), M, C, int(training), int(relu),
                                   _ptr(workspace), workspace.numel() * workspace.element_size(), _stream()), "lt_batch_norm_bwd")


def _host_ptr(t):
    if t is None:
        return None
    assert not t.is_cuda and t.is_contiguous() and t.dtype == torch.float32, "test hooks need contiguous float32 CPU tensors"
    return t.data_ptr()


def volumetric_ce_host(probs, coord, keypoints_gt, validity, grad_loss=None, grad_probs=None):
    """lt_test_volumetric_ce_host: the loss kernels' per-voxel, per-term and gradient code run on CPU tensors (test hook, no GPU
    needed).  Returns (loss float, index (B, J) int32, picked (B, J)); grad_probs (B, J, nvox), if given, is written."""
    B, J, nvox = probs.shape
    loss = torch.empty(1, dtype=torch.float32)
    index = torch.empty((B, J), dtype=torch.int32)
    picked = torch.empty((B, J), dtype=torch.float32)
    g = None if grad_loss is None else torch.tensor([float(grad_loss)], dtype=torch.float32)
    _check(lib().lt_test_volumetric_ce_host(_host_ptr(probs), _host_ptr(coord), _host_ptr(keypoints_gt), _host_ptr(validity),
                                            _host_ptr(loss), index.data_ptr(), _host_ptr(picked), _host_ptr(g), _host_ptr(grad_probs),
                                            B, J, nvox), "lt_test_volumetric_ce_host")
    return float(loss[0]), index, picked


def keypoints_loss_host(pred, gt, validity, kind, threshold=400.0, grad_loss=None, grad_pred=None):
    """lt_test_keypoints_loss_host: the criteria kernels' term, derivative and summation order run on CPU tensors (test hook, no GPU
    needed).  Returns (loss float, divisor float); grad_pred (n, dim), if given, is written."""
    n, dim = pred.shape
    loss = torch.empty(1, dtype=torch.float32)
    norm = torch.empty(1, dtype=torch.float64)
    g = None if grad_loss is None else torch.tensor([float(grad_loss)], dtype=torch.float32)
    _check(lib().lt_test_keypoints_loss_host(_host_ptr(pred), _host_ptr(gt), _host_ptr(validity), _host_ptr(loss), norm.data_ptr(),
                                             _host_ptr(g), _host_ptr(grad_pred), KEYPOINTS_LOSS[kind], float(threshold), n, dim),
           "lt_test_keypoints_loss_host")
    return float(loss[0]), float(norm[0])


def triangulate_dlt_host(proj, kp2d, conf, out):
    """lt_test_triangulate_dlt_fwd_host: the forward kernel's per-item code run on CPU tensors (test hook, no GPU needed)."""
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_test_triangulate_dlt_fwd_host(_host_ptr(proj), _host_ptr(kp2d), _host_ptr(conf), _host_ptr(out), B, V, J),
           "lt_test_triangulate_dlt_fwd_host")


def triangulate_dlt_bwd_host(proj, kp2d, conf, grad_out, grad_kp2d, grad_conf):
    """lt_test_triangulate_dlt_bwd_host: the backward kernel's per-item code run on CPU tensors (test hook, no GPU needed)."""
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_test_triangulate_dlt_bwd_host(_host_ptr(proj), _host_ptr(kp2d), _host_ptr(conf), _host_ptr(grad_out),
                                                  _host_ptr(grad_kp2d), _host_ptr(grad_conf), B, V, J), "lt_test_triangulate_dlt_bwd_host")


def triangulate_ransac_host(proj, kp2d, pairs, n_iters, eps, direct, out, inliers=None):
    """lt_test_triangulate_ransac_host: the RANSAC kernel's per-item code on CPU tensors (test hook, no GPU needed).  Dtypes as
    triangulate_ransac."""
    B, V, J = kp2d.shape[:3]
    for t, dt in ((kp2d, torch.int64), (pairs, torch.int32)) + (() if inliers is None else ((inliers, torch.int64),)):
        assert not t.is_cuda and t.is_contiguous() and t.dtype == dt, "test hooks need contiguous CPU tensors of the kernel's dtypes"
    _check(lib().lt_test_triangulate_ransac_host(_host_ptr(proj), kp2d.data_ptr(), pairs.data_ptr(), B, V, J, int(n_iters), float(eps),
                                                 int(bool(direct)), _host_ptr(out), None if inliers is None else inliers.data_ptr()),
           "lt_test_triangulate_ransac_host")


def softargmax3d_bwd_host(probs, coord, grad_keypoints, grad_volumes, grad_logits, B, J, nvox, multiplier, mode):
    """lt_test_softargmax3d_bwd_host: the soft-argmax backward's per-item code run on CPU tensors (test hook, no GPU needed)."""
    _check(lib().lt_test_softargmax3d_bwd_host(_host_ptr(probs), _host_ptr(coord), _host_ptr(grad_keypoints), _host_ptr(grad_volumes),
                                               _host_ptr(grad_logits), B, J, nvox, float(multiplier), int(mode)),
           "lt_test_softargmax3d_bwd_host")


def unproject_aggregate_bwd_det_host(features, proj, coord, conf, grad_out, grad_features, grad_conf, grad_proj, grad_coord, agg):
    """lt_test_unproject_aggregate_bwd_det_host: the fixed-order backward's pass-1, gather and confidence items on CPU tensors (test hook,
    no GPU needed).  Shapes as unproject_aggregate_bwd_det."""
    B, V, h, w, C = features.shape
    nvox = coord.shape[1]
    _check(lib().lt_test_unproject_aggregate_bwd_det_host(_host_ptr(features), _host_ptr(proj), _host_ptr(coord), _host_ptr(conf),
                                                          _host_ptr(grad_out), _host_ptr(grad_features), _host_ptr(grad_conf),
                                                          _host_ptr(grad_proj), _host_ptr(grad_coord), B, V, C, h, w, nvox, agg),
           "lt_test_unproject_aggregate_bwd_det_host")


def maxpool3d_bwd_host(x, grad_y, grad_x, k):
    """lt_test_maxpool3d_bwd_host: the max-pool backward's per-element code on CPU float32 tensors of any strides (grad_x: those of x)."""
    N, C, D, H, W = x.shape
    assert not x.is_cuda and x.stride() == grad_x.stride() and x.dtype == grad_y.dtype == grad_x.dtype == torch.float32
    _check(lib().lt_test_maxpool3d_bwd_host(x.data_ptr(), grad_y.data_ptr(), grad_x.data_ptr(), N, C, D, H, W, *x.stride(), *grad_y.stride(),
                                            int(k)), "lt_test_maxpool3d_bwd_host")


def unproject_aggregate_bwd_geom_host(features, proj, coord, conf, grad_out, grad_features, grad_conf, grad_proj, grad_coord, agg):
    """lt_test_unproject_aggregate_bwd_geom_host: the geometry variant's per-item code and the q / dP / dX arithmetic run on CPU tensors
    (test hook, no GPU needed).  Shapes as unproject_aggregate_bwd_geom."""
    B, V, h, w, C = features.shape
    nvox = coord.shape[1]
    _check(lib().lt_test_unproject_aggregate_bwd_geom_host(_host_ptr(features), _host_ptr(proj), _host_ptr(coord), _host_ptr(conf),
                                                           _host_ptr(grad_out), _host_ptr(grad_features), _host_ptr(grad_conf),
                                                           _host_ptr(grad_proj), _host_ptr(grad_coord), B, V, C, h, w, nvox, agg),
           "lt_test_unproject_aggregate_bwd_geom_host")


def softargmax3d_coord_bwd_host(probs, grad_keypoints, grad_coord):
    """lt_test_softargmax3d_coord_bwd_host: the coordinate gradient's per-item code on CPU tensors (test hook)."""
    B, J, nvox = probs.shape
    _check(lib().lt_test_softargmax3d_coord_bwd_host(_host_ptr(probs), _host_ptr(grad_keypoints), _host_ptr(grad_coord), B, J, nvox),
           "lt_test_softargmax3d_coord_bwd_host")


def triangulate_dlt_proj_bwd_host(proj, kp2d, conf, grad_out, grad_proj):
    """lt_test_triangulate_dlt_proj_bwd_host: the projection gradient's per-item and merge code on CPU tensors (test hook)."""
    B, V, J = kp2d.shape[:3]
    _check(lib().lt_test_triangulate_dlt_proj_bwd_host(_host_ptr(proj), _host_ptr(kp2d), _host_ptr(conf), _host_ptr(grad_out),
                                                       _host_ptr(grad_proj), B, V, J), "lt_test_triangulate_dlt_proj_bwd_host")


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


def f32_to_s32_scaled(inp, out, pixels, C, CP, absmax_bits=None, inv_scale=None):
    """[P][C] float32 -> [P][CP] split-fp16 of S x (S from absmax_bits, 1 without); inv_scale: float32[1] receiving 1 / S, or None."""
    _check(lib().lt_f32_to_s32_scaled(_ptr(inp), _ptr(out), pixels, C, CP, _ptr(absmax_bits), _ptr(inv_scale), _stream()),
           "lt_f32_to_s32_scaled")


def conv_wgrad_workspace_bytes(desc):
    return lib().lt_conv_wgrad_workspace_bytes(ctypes.byref(desc))


def conv_wgrad_plan(desc, sm_count):
    """Host-only work decomposition of an lt_conv_wgrad_fwd launch (lt_conv_wgrad_plan): dict of nwg, ngroups, m_tiles, splits, stages."""
    plan = ConvWgradPlan()
    _check(lib().lt_conv_wgrad_plan(ctypes.byref(desc), sm_count, ctypes.byref(plan)), "lt_conv_wgrad_plan")
    return {name: getattr(plan, name) for name, _ in ConvWgradPlan._fields_}


def conv_wgrad(desc, inp, grad_out, grad_absmax_bits, cin, cout, grad_w, workspace):
    """grad_w float32 [taps][cin][G cout] of the lt_conv_nd_fwd call `desc` describes (both operands split-fp16)."""
    _check(lib().lt_conv_wgrad_fwd(ctypes.byref(desc), _ptr(inp), _ptr(grad_out), _ptr(grad_absmax_bits), cin, cout, _ptr(grad_w),
                                   _ptr(workspace), workspace.numel() * workspace.element_size(), _stream()), "lt_conv_wgrad_fwd")


def conv_wgrad_host(desc, inp, grad_out, cin, cout, grad_w):
    """lt_test_conv_wgrad_host: the weight-gradient kernel's index mapping on CPU float32 channels-last tensors (test hook)."""
    _check(lib().lt_test_conv_wgrad_host(ctypes.byref(desc), _host_ptr(inp), _host_ptr(grad_out), cin, cout, _host_ptr(grad_w)),
           "lt_test_conv_wgrad_host")


def s32_to_f32(inp, out, pixels, C):
    _check(lib().lt_s32_to_f32(_ptr(inp), _ptr(out), pixels, C, _stream()), "lt_s32_to_f32")


def cl_to_cf(inp, out, N, P, Cs, C):
    _check(lib().lt_cl_to_cf_f32(_ptr(inp), _ptr(out), N, P, Cs, C, _stream()), "lt_cl_to_cf_f32")


def tc_gemm_selftest(a_fp16, b_fp16, d, M, N, K, variant=0):
    _check(lib().lt_tc_gemm_selftest(_ptr(a_fp16), _ptr(b_fp16), _ptr(d), M, N, K, variant, _stream()), "lt_tc_gemm_selftest")


def conf_head_tail_host(x, lin1, lin2, lin3, grad_y=None):
    """lt_test_conf_head_tail_host: the confidence-head tail kernels' per-item code on CPU float32 tensors (test hook, no GPU needed).
    x (N, C0, H, W) of any element strides.  -> (out, x0, h1, h2), and with grad_y (N, NO) also (grad_x with the strides of
    torch.empty_like(x), (dW1, db1, dW2, db2, dW3, db3))."""
    (N, C0, H, W), xs = _map_dims(x)
    assert not x.is_cuda
    H1, H2, NO = lin1[0].shape[0], lin2[0].shape[0], lin3[0].shape[0]
    out, x0, h1, h2 = (torch.empty(N, k) for k in (NO, C0, H1, H2))
    gx = torch.empty_like(x) if grad_y is not None else None
    grads = tuple(torch.empty(t.shape) for lin in (lin1, lin2, lin3) for t in lin) if grad_y is not None else (None,) * 6
    _check(lib().lt_test_conf_head_tail_host(x.data_ptr(), N, C0, H, W, *xs, *(gx.stride() if gx is not None else (0,) * 4), H1, H2, NO,
                                             *[_host_ptr(t) for lin in (lin1, lin2, lin3) for t in lin], _host_ptr(out), _host_ptr(x0),
                                             _host_ptr(h1), _host_ptr(h2), _host_ptr(grad_y), None if gx is None else gx.data_ptr(),
                                             *[_host_ptr(t) for t in grads]), "lt_test_conf_head_tail_host")
    return (out, x0, h1, h2) if grad_y is None else (out, x0, h1, h2, gx, grads)


def view_normalize_bwd_host(conf, grad):
    """lt_test_view_normalize_bwd_host: the view-normalisation backward's per-item code on CPU (B, V, C) float32 tensors."""
    B, V, C = conf.shape
    out = torch.empty_like(conf)
    _check(lib().lt_test_view_normalize_bwd_host(_host_ptr(conf), _host_ptr(grad), _host_ptr(out), B, V, C),
           "lt_test_view_normalize_bwd_host")
    return out
