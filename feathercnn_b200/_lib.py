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


class FcudaDeconvParam(ctypes.Structure):
    """include/fcuda.h FcudaDeconvParam (total channel counts; output_h / output_w filled by fcuda_deconv_output_dim)."""

    _fields_ = [(n, ctypes.c_int) for n in (
        "output_channels input_channels input_h input_w kernel_h kernel_w stride_h stride_w dilation_h dilation_w "
        "pad_left pad_right pad_top pad_bottom output_pad_right output_pad_bottom group bias_term activation "
        "output_h output_w").split()]


def fcuda() -> ctypes.CDLL:
    global _fcuda
    if _fcuda is None:
        lib = _load("libfcuda.so")
        vp, sz, i = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
        P = ctypes.POINTER(FcudaConvParam)
        szp = ctypes.POINTER(ctypes.c_size_t)
        D = ctypes.POINTER(FcudaDeconvParam)
        sigs = {
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
            "fcuda_conv_forward_residual": (i, [P, i, vp, vp, vp, vp, vp, vp, i, i, vp]),
            "fcuda_conv_can_pool": (i, [P, i]),
            "fcuda_igemm_halo_tile": (i, [P, ctypes.POINTER(i)]),
            "fcuda_igemm_presplit_tile": (i, [P, ctypes.POINTER(i)]),
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
