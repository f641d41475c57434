"""ctypes binding of libbevfusion_b200.so (C ABI: include/bevfusion_b200.h).

The library is loaded lazily on first use and the load FAILS LOUDLY: there is no fallback
implementation behind these calls."""
import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libbevfusion_b200.so")
HEADER_PATH = os.path.join(_HERE, "..", "include", "bevfusion_b200.h")

_lib = None

c_void_p, c_int, c_size_t, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t, ctypes.c_float
_P = c_void_p  # every device / host pointer is passed as an address

# symbol -> (restype, argtypes); kept in the same order as the header
_SIGNATURES = {
    "bevb200_version": (c_int, []),
    "bevb200_last_error": (ctypes.c_char_p, []),
    "bevb200_launch_count": (ctypes.c_longlong, []),
    "bevb200_reset_launch_count": (None, []),
    "bevb200_bev_pool_workspace_bytes": (c_size_t, [c_int, c_int]),
    "bevb200_bev_pool": (c_int, [c_int] * 7 + [_P] * 6 + [c_size_t, _P]),
    "bevb200_bev_pool_grad": (c_int, [c_int] * 7 + [_P] * 6),
    "bevb200_bev_pool_perm": (c_int, [c_int] * 7 + [_P] * 7 + [c_size_t, _P]),
    "bevb200_bev_pool_grad_perm": (c_int, [c_int] * 8 + [_P] * 7),
    "bevb200_bev_channels_first": (c_int, [_P, _P, c_int, c_int, c_int, c_int, ctypes.c_longlong, _P]),
    "bevb200_bev_pool_lift": (c_int, [c_int] * 7 + [_P, _P, c_int, c_int] + [_P] * 6 + [c_size_t, _P]),
    "bevb200_bev_pool_lift_prepare_workspace_bytes": (c_size_t, [c_int]),
    "bevb200_bev_pool_lift_prepare": (c_int, [_P, _P] + [c_int] * 6 + [_P] * 7 + [c_size_t, _P]),
    "bevb200_bev_pool_lift_columns_workspace_bytes": (c_size_t, [c_int] * 3),
    "bevb200_bev_pool_lift_columns": (c_int, [c_int] * 7 + [_P, _P] + [c_int] * 4 + [_P] * 7 + [c_int, _P, _P, c_size_t, _P]),
    "bevb200_bev_pool_lift_columns_backward_workspace_bytes": (c_size_t, [c_int] * 3),
    "bevb200_bev_pool_lift_columns_backward": (c_int, [c_int] * 7 + [_P] * 3 + [c_int] * 4 + [_P] * 5
                                               + [c_int, _P, _P, _P, c_size_t, _P]),
    "bevb200_bev_pool_lift_backward_workspace_bytes": (c_size_t, [c_int] * 2),
    "bevb200_bev_pool_lift_backward": (c_int, [c_int] * 8 + [_P] * 3 + [c_int] * 2 + [_P] * 6 + [_P, c_size_t, _P]),
    "bevb200_bev_pool_prepare_workspace_bytes": (c_size_t, [c_int]),
    "bevb200_bev_pool_prepare_geom": (c_int, [_P, c_int, c_int, _P, _P, _P, c_int] + [_P] * 7
                                      + [c_size_t, _P]),
    "bevb200_bev_pool_prepare_cameras": (c_int, [_P, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_int] + [_P] * 8
                                         + [c_size_t, _P]),
    "bevb200_bev_pool_prepare_coords": (c_int, [_P] + [c_int] * 5 + [_P] * 7 + [c_size_t, _P]),
    "bevb200_hard_voxelize_workspace_bytes": (c_size_t, [c_int, c_int]),
    "bevb200_hard_voxelize": (c_int, [_P, c_int, c_int, _P, _P, c_int, c_int] + [_P] * 5
                              + [c_size_t, _P]),
    "bevb200_hard_voxelize_mean": (c_int, [_P, c_int, c_int, _P, _P, c_int, c_int, c_int, _P, _P, _P, _P,
                                           _P, c_size_t, _P]),
    "bevb200_depth_rasterize_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "bevb200_depth_rasterize": (c_int, [_P, c_int, c_int, _P, _P, _P, c_int, c_int, c_int, c_int, c_int,
                                        c_int, _P, _P, c_size_t, _P]),
    "bevb200_dynamic_scatter_workspace_bytes": (c_size_t, [c_int]),
    "bevb200_dynamic_scatter": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P,
                                        c_size_t, _P]),
    "bevb200_dynamic_scatter_backward": (c_int, [_P, _P, _P, _P, _P, _P, c_int, c_int, c_int, c_int,
                                                 c_int, _P, _P]),
    "bevb200_dynamic_voxelize": (c_int, [_P, c_int, c_int, _P, _P, _P, _P]),
    "bevb200_voxel_mean": (c_int, [_P, _P, _P] + [c_int] * 4 + [_P, _P, _P]),
    "bevb200_pillar_packed_bytes": (c_size_t, [c_int] * 3),
    "bevb200_pillar_pack_weights": (c_int, [_P] * 6 + [c_int] * 3 + [_P, _P]),
    "bevb200_pillar_features": (c_int, [_P, _P, _P, c_int, _P, c_int, c_int] + [c_float] * 4 + [_P, _P, _P]),
    "bevb200_hard_voxelize_pillars": (c_int, [_P, c_int, c_int, _P, _P, c_int, c_int] + [c_float] * 4
                                      + [_P, _P, c_int, c_int, _P, _P, c_size_t, _P]),
    "bevb200_radar_packed_bytes": (c_size_t, [c_int, c_int, _P]),
    "bevb200_radar_pack_weights": (c_int, [_P, _P, _P, c_int, c_int, _P, _P, _P]),
    "bevb200_radar_features_workspace_bytes": (c_size_t, [c_int, c_int]),
    "bevb200_radar_features": (c_int, [_P, _P, _P, c_int, _P, c_int, c_int, c_int, _P] + [c_float] * 4
                               + [_P] * 5 + [c_size_t, _P]),
    "bevb200_hard_voxelize_radar_workspace_bytes": (c_size_t, [c_int, c_int]),
    "bevb200_hard_voxelize_radar": (c_int, [_P, c_int, c_int, _P, _P, c_int, c_int, c_int, _P] + [c_float] * 4
                                    + [_P, _P, _P, _P, c_int, c_int, _P, _P, c_size_t, _P]),
    "bevb200_boxes_iou_bev": (c_int, [_P, c_int, _P, c_int, _P, _P]),
    "bevb200_boxes_overlap_bev": (c_int, [_P, c_int, _P, c_int, _P, _P]),
    "bevb200_nms_workspace_bytes": (c_size_t, [c_int, c_int]),
    "bevb200_nms": (c_int, [_P, _P, c_int, c_int, c_int, ctypes.c_double, c_int, _P, _P, _P, _P, c_size_t, _P]),
    "bevb200_head_targets_workspace_bytes": (c_size_t, [c_int, c_int]),
    "bevb200_head_targets": (c_int, [_P, _P, _P, c_int, c_int, c_int, _P, c_int, _P, c_int] + [c_float] * 4
                             + [c_int] * 3 + [ctypes.c_double] + [c_int] * 4 + [_P] * 6 + [c_size_t, _P]),
    "bevb200_draw_heatmap_gaussian": (c_int, [_P] + [c_int] * 5 + [c_float, _P]),
    "bevb200_lsap_workspace_bytes": (c_size_t, [c_int] * 3),
    "bevb200_lsap": (c_int, [_P] * 3 + [c_int] * 3 + [_P] * 5 + [c_size_t, _P]),
    "bevb200_transfusion_assign_workspace_bytes": (c_size_t, [c_int] * 4),
    "bevb200_transfusion_assign": (c_int, [_P] * 6 + [c_int] * 4 + [_P] * 3 + [c_int] * 2 + [ctypes.c_double] * 4
                                   + [c_int] * 2 + [ctypes.c_double] * 10 + [_P] * 13 + [c_size_t, _P]),
    "bevb200_rulebook_workspace_bytes": (c_size_t, [c_int, c_int, _P]),
    "bevb200_rulebook_prepare": (c_int, [_P, c_int, c_int] + [_P] * 6 + [c_int, _P, _P, c_size_t, _P]),
    "bevb200_rulebook_fill": (c_int, [_P, c_int, c_int] + [_P] * 6 + [c_int, c_int, _P, _P, _P,
                                                                       c_size_t, _P]),
    "bevb200_rulebook_fill_subm_sorted": (c_int, [_P, c_int, c_int, _P, _P, _P, _P, _P, c_size_t, _P]),
    "bevb200_rulebook_to_pairs": (c_int, [_P, c_int, c_int, c_int, _P, _P, _P]),
    "bevb200_pairs_to_nbr": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P]),
    "bevb200_spconv_forward": (c_int, [_P, _P, _P] + [c_int] * 5 + [_P, _P, _P, c_int, c_int, _P, _P]),
    "bevb200_spconv_padded_channels": (c_int, [c_int, c_int]),
    "bevb200_spconv_packed_weight_bytes": (c_size_t, [c_int] * 4),
    "bevb200_spconv_pack_weights": (c_int, [_P] + [c_int] * 4 + [_P, _P]),
    "bevb200_spconv_forward_packed": (c_int, [_P, _P, _P] + [c_int] * 5 + [_P, _P, _P, c_int, c_int, _P, _P]),
    "bevb200_spconv_split_channels": (c_int, [c_int]),
    "bevb200_spconv_split_rows": (c_int, [_P, c_int, _P, c_int, _P, _P]),
    "bevb200_spconv_split_weight_bytes": (c_size_t, [c_int] * 3),
    "bevb200_spconv_pack_split_weights": (c_int, [_P] + [c_int] * 3 + [_P, _P]),
    "bevb200_spconv_forward_split": (c_int, [_P, _P, _P, ctypes.c_longlong, c_int, c_int, _P] + [c_int] * 3
                                     + [_P, _P, _P, c_int, _P, _P, _P]),
    "bevb200_rulebook_transpose": (c_int, [_P, c_int, c_int, c_int, _P, _P]),
    "bevb200_spconv_backward_workspace_bytes": (c_size_t, [c_int] * 5),
    "bevb200_spconv_backward": (c_int, [_P] * 5 + [c_int] * 6 + [_P, _P, _P, c_size_t, _P]),
    "bevb200_sparse_to_dense": (c_int, [_P, _P, c_int, c_int, c_int, _P, c_int, ctypes.c_longlong, _P, _P]),
    "bevb200_encoder_create": (c_int, [c_int, _P, _P, c_int, _P]),
    "bevb200_encoder_destroy": (None, [_P]),
    "bevb200_encoder_param_bytes": (c_size_t, [_P]),
    "bevb200_encoder_num_levels": (c_int, [_P]),
    "bevb200_encoder_output_shape": (c_int, [_P, _P, _P]),
    "bevb200_encoder_set_conv": (c_int, [_P, c_int, _P, _P, _P, _P, c_size_t, _P]),
    "bevb200_encoder_level_caps": (c_int, [_P, c_int, c_int, _P, _P]),
    "bevb200_encoder_workspace_bytes": (c_size_t, [_P, c_int, c_int, _P]),
    "bevb200_encoder_forward": (c_int, [_P, _P, _P, _P, c_int, _P, c_int, _P, _P, ctypes.c_longlong, _P, _P,
                                        c_size_t, _P, _P]),
}


def declared_symbols():
    """Names of every function declared in include/bevfusion_b200.h."""
    with open(HEADER_PATH) as f:
        text = f.read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bevb200_[a-z0-9_]+)\s*\(", text)))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libbevfusion_b200.so is missing (%s); build it with `python -m bevfusion_b200.build`"
                " -- there is no fallback implementation" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


class BevB200Error(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        msg = lib().bevb200_last_error()
        raise BevB200Error("%s failed (code %d): %s" % (what, rc, msg.decode() if msg else ""))


def ptr(t):
    """Address of a torch tensor's storage (0 for None)."""
    return 0 if t is None else t.data_ptr()


def current_stream(device=None):
    import torch
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda(t, name, dtype=None, contiguous=True):
    """The library has no CPU path: reject CPU tensors loudly (north star: no CPU fallback)."""
    import torch
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("%s must be a CUDA tensor: bevfusion_b200 has no CPU implementation" % name)
    if dtype is not None and t.dtype != dtype:
        raise TypeError("%s must have dtype %s, got %s" % (name, dtype, t.dtype))
    if contiguous and not t.is_contiguous():
        raise RuntimeError("%s must be contiguous" % name)
    return t


def host_array(ctype, values):
    return (ctype * len(values))(*values)


def launch_count():
    return int(lib().bevb200_launch_count())


def reset_launch_count():
    lib().bevb200_reset_launch_count()
