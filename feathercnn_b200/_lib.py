"""ctypes loader for the in-tree native libraries.

``libfcuda.so`` (CUDA kernels + the C ABI of include/fcuda.h) and ``libfeather_b200.so`` (C++ feather::Net,
C ABI of include/feather_c.h) are built in-tree by ``__graft_entry__.build()`` /
``make -C feathercnn_b200/csrc``.  There is NO fallback: if a library is missing or fails to load this module
raises — the product never routes through PyTorch ops, the oracle or any CPU path.
"""
from __future__ import annotations

import ctypes
from pathlib import Path

_LIBDIR = Path(__file__).resolve().parent / "lib"

c_float_p = ctypes.POINTER(ctypes.c_float)


class NativeLibraryError(RuntimeError):
    pass


def _load(name: str) -> ctypes.CDLL:
    path = _LIBDIR / name
    if not path.exists():
        raise NativeLibraryError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            f"or `make -C feathercnn_b200/csrc` (there is no CPU fallback)")
    try:
        # RTLD_LOCAL: libfeather_b200.so and the oracle's reference build both define feather::Net; keep scopes apart
        return ctypes.CDLL(str(path), mode=ctypes.RTLD_LOCAL)
    except OSError as e:  # pragma: no cover
        raise NativeLibraryError(f"failed to load {path}: {e}") from e


_fcuda = None
_feather = None


class FcudaConvParam(ctypes.Structure):
    """include/fcuda.h FcudaConvParam == booster::ConvParam (booster.h:59-77)."""

    _fields_ = [(n, ctypes.c_int) for n in (
        "output_channels input_channels input_h input_w kernel_h kernel_w output_h output_w stride_h stride_w "
        "pad_left pad_bottom pad_right pad_top group").split()] + [("bias_term", ctypes.c_ubyte),
                                                                   ("activation", ctypes.c_int)]


class FcudaConvOptions(ctypes.Structure):
    """include/fcuda.h FcudaConvOptions: what fcuda_conv_forward_opts fuses beyond fcuda_conv_forward (all zero)."""

    _fields_ = [("residual", ctypes.c_void_p), ("relu_after_add", ctypes.c_int), ("clip_min", ctypes.c_float),
                ("clip_max", ctypes.c_float), ("dilation_h", ctypes.c_int), ("dilation_w", ctypes.c_int),
                ("pool", ctypes.c_int)]


class FcudaDeconvParam(ctypes.Structure):
    """include/fcuda.h FcudaDeconvParam (total channel counts; output_h / output_w filled by fcuda_deconv_output_dim)."""

    _fields_ = [(n, ctypes.c_int) for n in (
        "output_channels input_channels input_h input_w kernel_h kernel_w stride_h stride_w dilation_h dilation_w "
        "pad_left pad_right pad_top pad_bottom output_pad_right output_pad_bottom group bias_term activation "
        "output_h output_w").split()]


class FcudaInterpParam(ctypes.Structure):
    """include/fcuda.h FcudaInterpParam (output_h / output_w filled by fcuda_interp_output_dim)."""

    _fields_ = ([("resize_type", ctypes.c_int), ("align_corner", ctypes.c_int), ("height_scale", ctypes.c_float),
                 ("width_scale", ctypes.c_float)] +
                [(n, ctypes.c_int) for n in "output_height output_width input_h input_w output_h output_w".split()])


class FcudaPad(ctypes.Structure):
    """include/fcuda.h FcudaPad: type 0 constant, 1 replicate, 2 reflect."""

    _fields_ = [(n, ctypes.c_int) for n in "top bottom left right type".split()] + [("value", ctypes.c_float)]


class FcudaPriorBoxParam(ctypes.Structure):
    """include/fcuda.h FcudaPriorBoxParam (fixed arrays of FCUDA_PRIORBOX_MAX = 16)."""

    _fields_ = ([("num_min_sizes", ctypes.c_int), ("num_max_sizes", ctypes.c_int), ("num_aspect_ratios", ctypes.c_int),
                 ("min_sizes", ctypes.c_float * 16), ("max_sizes", ctypes.c_float * 16),
                 ("aspect_ratios", ctypes.c_float * 16), ("variances", ctypes.c_float * 4), ("flip", ctypes.c_int),
                 ("clip", ctypes.c_int), ("step_w", ctypes.c_float), ("step_h", ctypes.c_float),
                 ("offset", ctypes.c_float)])


class FcudaYoloParam(ctypes.Structure):
    """include/fcuda.h FcudaYoloParam (up to 4 scales of 16 boxes, 128 bias floats)."""

    _fields_ = ([(n, ctypes.c_int) for n in "version num_class num_box num_scales".split()] +
                [("confidence_threshold", ctypes.c_float), ("nms_threshold", ctypes.c_float), ("nms_top_k", ctypes.c_int),
                 ("keep_top_k", ctypes.c_int), ("num_biases", ctypes.c_int), ("biases", ctypes.c_float * 128),
                 ("mask", ctypes.c_int * 64), ("anchors_scale", ctypes.c_float * 4), ("grid_h", ctypes.c_int * 4),
                 ("grid_w", ctypes.c_int * 4)])


class FcudaProposalParam(ctypes.Structure):
    """include/fcuda.h FcudaProposalParam."""

    _fields_ = [("feat_stride", ctypes.c_int), ("base_size", ctypes.c_int), ("pre_nms_topN", ctypes.c_int),
                ("after_nms_topN", ctypes.c_int), ("nms_thresh", ctypes.c_float), ("min_size", ctypes.c_int)]


class FcudaRoute(ctypes.Structure):
    """include/fcuda.h FcudaRoute (up to FCUDA_ROUTE_MAX = 8 sources and destinations)."""

    _fields_ = [("outer", ctypes.c_int), ("inner", ctypes.c_int), ("num_src", ctypes.c_int),
                ("src", ctypes.c_void_p * 8), ("src_extent", ctypes.c_int * 8), ("group", ctypes.c_int),
                ("reverse", ctypes.c_int), ("dst_begin", ctypes.c_int), ("num_dst", ctypes.c_int),
                ("dst", ctypes.c_void_p * 8), ("dst_extent", ctypes.c_int * 8)]


def fcuda() -> ctypes.CDLL:
    global _fcuda
    if _fcuda is None:
        lib = _load("libfcuda.so")
        vp, sz, i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        P = ctypes.POINTER(FcudaConvParam)
        szp = ctypes.POINTER(ctypes.c_size_t)
        D = ctypes.POINTER(FcudaDeconvParam)
        R = ctypes.POINTER(FcudaInterpParam)
        PB = ctypes.POINTER(FcudaPriorBoxParam)
        Y = ctypes.POINTER(FcudaYoloParam)
        PP = ctypes.POINTER(FcudaProposalParam)
        f = ctypes.c_float
        sigs = {
            "fcuda_permute_forward": (i, [vp, vp, i, i, i, i, i, vp]),
            "fcuda_softmax_axis_forward": (i, [vp, vp, i, i, i, i, vp]),
            "fcuda_priorbox_per_location": (i, [PB, ctypes.POINTER(i)]),
            "fcuda_priorbox_forward": (i, [vp, PB, i, i, i, i, vp]),
            "fcuda_ssd_decode": (i, [vp, vp, vp, i, i, vp]),
            "fcuda_detection_output_workspace_size": (i, [i, i, i, i, szp]),
            "fcuda_detection_output_forward": (i, [vp, vp, vp, vp, i, i, f, f, i, i, vp, i, vp]),
            "fcuda_yolo_decode": (i, [vp, vp, vp, vp, Y, i, vp]),
            "fcuda_yolo_detection_workspace_size": (i, [Y, i, szp]),
            "fcuda_yolo_detection_forward": (i, [vp, vp, Y, vp, i, vp]),
            "fcuda_proposal_anchors": (i, [PP, vp]),
            "fcuda_proposal_decode": (i, [vp, vp, vp, vp, PP, i, i, i, vp]),
            "fcuda_proposal_workspace_size": (i, [PP, i, i, i, szp]),
            "fcuda_proposal_forward": (i, [vp, vp, vp, vp, vp, PP, i, i, vp, i, vp]),
            "fcuda_roi_pooling_forward": (i, [vp, vp, vp, i, i, i, i, i, i, f, i, vp]),
            "fcuda_psroi_pooling_forward": (i, [vp, vp, vp, i, i, i, i, i, i, i, f, i, vp]),
            "fcuda_route_forward": (i, [ctypes.POINTER(FcudaRoute), i, vp]),
            "fcuda_slice_plan": (i, [i, i, ctypes.POINTER(i), ctypes.POINTER(i), i, ctypes.POINTER(i), ctypes.POINTER(i)]),
            "fcuda_interp_output_dim": (i, [R]),
            "fcuda_interp_forward": (i, [R, vp, vp, i, i, vp]),
            "fcuda_crop_forward": (i, [vp, vp] + [i] * 10 + [vp]),
            "fcuda_pixel_shuffle_forward": (i, [vp, vp, i, i, i, i, i, vp, R, i, vp]),
            "fcuda_binary_op_shape": (i, [i, ctypes.POINTER(i), i] + [ctypes.POINTER(i)] * 5),
            "fcuda_binary_op_forward": (i, [vp, vp, ctypes.POINTER(i), vp, ctypes.POINTER(i), f, i, i, vp]),
            "fcuda_deconv_output_dim": (i, [D]),
            "fcuda_deconv_plan": (i, [D, P, ctypes.POINTER(i)]),
            "fcuda_deconv_get_buffer_size": (i, [D, i, szp, szp]),
            "fcuda_deconv_init": (i, [D, vp, vp, vp]),
            "fcuda_deconv_forward": (i, [D, vp, vp, vp, vp, vp, i, vp]),
            "fcuda_set_precision": (i, [i]),
            "fcuda_get_precision": (i, []),
            "fcuda_set_l2_chunk_bytes": (i, [sz]),
            "fcuda_get_l2_chunk_bytes": (sz, []),
            "fcuda_conv_assign_output_dim": (i, [P]),
            "fcuda_conv_select_algo": (i, [P, ctypes.POINTER(i)]),
            "fcuda_conv_select_algo_tuned": (i, [P, ctypes.POINTER(i)]),
            "fcuda_conv_get_buffer_size": (i, [P, i, i, szp, szp]),
            "fcuda_conv_init": (i, [P, i, vp, vp, vp]),
            "fcuda_conv_forward": (i, [P, i, vp, vp, vp, vp, vp, i, vp]),
            "fcuda_conv_forward_opts": (i, [P, i, vp, vp, vp, vp, vp, ctypes.POINTER(FcudaConvOptions), i, vp]),
            "fcuda_conv_forward_clip": (i, [P, i, vp, vp, vp, vp, vp, ctypes.c_float, ctypes.c_float, i, vp]),
            "fcuda_conv_forward_residual": (i, [P, i, vp, vp, vp, vp, vp, vp, i, i, vp]),
            "fcuda_conv_can_pool": (i, [P, i]),
            "fcuda_igemm_halo_tile": (i, [P, ctypes.POINTER(i)]),
            "fcuda_igemm_presplit_tile": (i, [P, ctypes.POINTER(i)]),
            "fcuda_igemm_wide_tile": (i, [P, ctypes.POINTER(i)]),
            "fcuda_igemm_stem_supported": (i, [P, ctypes.POINTER(FcudaConvOptions)]),
            "fcuda_conv_forward_pool": (i, [P, i, vp, vp, vp, vp, vp, i, vp]),
            "fcuda_conv_forward_ext": (i, [P, i, vp, vp, vp, vp, vp, vp, i, i, i, i, vp]),
            "fcuda_eltwise_forward": (i, [vp, vp, vp, sz, i, ctypes.c_float, ctypes.c_float, i, vp]),
            "fcuda_set_tuning": (i, [ctypes.c_char_p, i]),
            "fcuda_get_tuning": (i, [ctypes.c_char_p]),
            "fcuda_pixel_channels": (i, [i, ctypes.POINTER(i), ctypes.POINTER(i)]),
            "fcuda_from_pixels": (i, [vp, vp, i, i, i, i, i, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float), i, vp]),
            "fcuda_tensor_gemm": (i, [vp, vp, vp, vp, i, i, i, i, vp]),
            "fcuda_split_tf32": (i, [vp, vp, vp, sz, vp]),
            "fcuda_inner_product_get_buffer_size": (i, [i, i, i, szp, szp]),
            "fcuda_inner_product_init": (i, [i, i, vp, vp, vp]),
            "fcuda_inner_product_forward": (i, [i, i, vp, vp, vp, vp, vp, i, i, vp]),
            "fcuda_pooling_out_dim": (i, [i, i, i, i, i]),
            "fcuda_pooling_forward": (i, [vp, vp] + [i] * 14 + [vp]),
            "fcuda_batchnorm_forward": (i, [vp, vp, i, sz, vp, vp, vp, vp, i, i, vp]),
            "fcuda_scale_forward": (i, [vp, vp, i, sz, vp, vp, i, vp]),
            "fcuda_eltwise_add_forward": (i, [vp, vp, vp, sz, i, vp]),
            "fcuda_relu_forward": (i, [vp, vp, sz, vp]),
            "fcuda_clip_forward": (i, [vp, vp, sz, ctypes.c_float, ctypes.c_float, vp]),
            "fcuda_activation_forward": (i, [vp, vp, sz, i, ctypes.c_float, ctypes.c_float, vp]),
            "fcuda_layer_norm_forward": (i, [vp, vp, i, ctypes.c_longlong, vp, vp, f, vp]),
            "fcuda_attention_forward": (i, [vp, vp, i, vp, i, vp, i, i, i, i, i, i, f, vp]),
            "fcuda_prelu_forward": (i, [vp, vp, i, sz, vp, i, i, vp]),
            "fcuda_normalize_workspace_size": (i, [i, i, i, sz, i, szp]),
            "fcuda_normalize_forward": (i, [vp, vp, i, sz, vp, i, i, i, f, i, vp, i, vp]),
            "fcuda_instance_norm_workspace_size": (i, [i, sz, i, szp]),
            "fcuda_instance_norm_forward": (i, [vp, vp, i, i, i, vp, vp, f, i, vp, vp, i, vp]),
            "fcuda_padding_forward": (i, [vp, vp, i, i, i, vp, i, vp]),
            "fcuda_lrn_forward": (i, [vp, vp, i, i, i, i, i, f, f, f, i, vp]),
            "fcuda_softmax_forward": (i, [vp, vp, sz, i, vp]),
            "fcuda_dropout_forward": (i, [vp, vp, sz, ctypes.c_float, vp]),
            "fcuda_copy_channels": (i, [vp, i, i, vp, i, sz, i, vp]),
            "fcuda_profile_tensor_gemm": (None, [i]),
            "fcuda_profile_collect": (i, [ctypes.POINTER(ctypes.c_double)] * 3 + [ctypes.POINTER(ctypes.c_longlong)]),
            "fcuda_profile_collect_kind": (i, [i] + [ctypes.POINTER(ctypes.c_double)] * 4 + [ctypes.POINTER(ctypes.c_longlong)]),
            "fcuda_launch_count": (ctypes.c_ulonglong, []),
            "fcuda_reset_launch_count": (None, []),
        }
        for name, (res, args) in sigs.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _fcuda = lib
    return _fcuda


def feather() -> ctypes.CDLL:
    global _feather
    if _feather is None:
        fcuda()  # dependency, resolved through $ORIGIN rpath as well
        lib = _load("libfeather_b200.so")
        vp, sz, i, cp = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_char_p
        ip = ctypes.POINTER(ctypes.c_int)
        sigs = {
            "fnet_create": (vp, []),
            "fnet_destroy": (None, [vp]),
            "fnet_set_fusion": (None, [vp, i]),
            "fnet_set_cuda_graph": (None, [vp, i]),
            "fnet_set_stream": (None, [vp, vp]),
            "fnet_load_param": (i, [vp, cp]),
            "fnet_load_param_text": (i, [vp, cp]),
            "fnet_load_weights": (i, [vp, cp]),
            "fnet_init_from_path": (i, [vp, cp]),
            "fnet_init_from_buffer": (i, [vp, vp, sz]),
            "fnet_prepare_weight_arena": (i, [vp]),
            "fnet_weight_arena": (i, [vp, ctypes.POINTER(vp), ctypes.POINTER(sz)]),
            "fnet_attach_weights": (i, [vp]),
            "fnet_feed_input_batch": (i, [vp, cp, vp, i, i, i, i]),
            "fnet_feed_input_device": (i, [vp, cp, vp, i, i, i, i]),
            "fnet_feed_input_pixels": (i, [vp, cp, vp, i, i, i, i, i, i, ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_float)]),
            "fnet_forward": (i, [vp]),
            "fnet_forward_batch": (i, [vp, vp, i]),
            "fnet_submit_batch": (i, [vp, vp, i, cp, vp]),
            "fnet_wait_batch": (i, [vp, i]),
            "fnet_synchronize": (i, [vp]),
            "fnet_blob_shape": (i, [vp, cp, ip, ip, ip, ip]),
            "fnet_blob_dims": (i, [vp, cp]),
            "fnet_extract_blob": (i, [vp, cp, vp]),
            "fnet_extract_device": (i, [vp, cp, ctypes.POINTER(vp), ip, ip, ip, ip]),
            "fnet_launches_per_forward": (ctypes.c_ulonglong, [vp]),
            "fnet_input_shape": (i, [vp, ip, ip, ip]),
            "fnet_blob_names": (sz, [vp, cp, sz]),
            "fnet_modelbin_load_mem": (ctypes.c_long, [ctypes.c_char_p, i, i, ctypes.POINTER(ctypes.c_float)]),
            "fnet_fuse_now": (i, [vp]),
            "fnet_layer_fused_away": (i, [vp, cp]),
            "fnet_layer_conv_algo": (i, [vp, cp]),
            "fnet_input_name": (cp, [vp]),
            "fgroup_create": (vp, []),
            "fgroup_destroy": (None, [vp]),
            "fgroup_set_options": (None, [vp, i, i]),
            "fgroup_init_from_path": (i, [vp, cp, ip, i]),
            "fgroup_size": (i, [vp]),
            "fgroup_device": (i, [vp, i]),
            "fgroup_member": (vp, [vp, i]),
            "fgroup_broadcast_transport": (cp, [vp]),
            "fgroup_forward_batch": (i, [vp, vp, i, cp, vp]),
            "fgroup_shard_range": (i, [i, i, i, ip, ip]),
            "fgroup_synchronize": (i, [vp]),
        }
        for name, (res, args) in sigs.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _feather = lib
    return _feather
