"""ctypes binding of libgifb200.so (the C ABI declared in include/gifb200.h).

This is the reference-side binding a maintainer would add (INTEGRATION.md): every call passes raw device
pointers (``tensor.data_ptr()``), int shapes and the current CUDA stream; no torch types cross the boundary.
There is NO fallback: if the library is missing it is built with nvcc, and if that is impossible the import
fails; if a kernel returns an error code a ``RuntimeError`` carrying ``gifb200_last_error()`` is raised.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgifb200.so")

_p = ctypes.c_void_p
_i = ctypes.c_int
_f = ctypes.c_float
_d = ctypes.c_double
_ll = ctypes.c_longlong
_sz = ctypes.c_size_t

# name -> (restype, argtypes); mirrors include/gifb200.h one to one (tests/test_abi.py checks the header against it)
SIGNATURES = {
    "gifb200_version": (_i, []),
    "gifb200_last_error": (ctypes.c_char_p, []),
    "gifb200_launch_count": (_ll, []),
    "gifb200_conv2d_workspace_bytes": (_sz, [_i] * 11),
    "gifb200_conv2d": (_i, [_p, _p, _p] + [_i] * 13 + [_p, _f, _f, _i, _p, _sz, _p]),
    "gifb200_conv2d_wgrad_workspace_bytes": (_sz, [_i] * 10),
    "gifb200_conv2d_wgrad_path": (_i, [_i] * 10),
    "gifb200_conv2d_wgrad": (_i, [_p, _p, _p] + [_i] * 12 + [_p, _sz, _p]),
    "gifb200_conv2d_ex_workspace_bytes": (_sz, [_i] * 13),
    "gifb200_conv2d_ex": (_i, [_p, _p, _p] + [_i] * 16 + [_p, _i, _p, _sz, _p]),
    "gifb200_pool2d": (_i, [_p, _p] + [_i] * 12 + [_p]),
    "gifb200_resize_bilinear": (_i, [_p, _p, _i, _i, _i, _ll, _ll, _ll, _ll, _i, _i, _i, _f, _f, _i, _p]),
    "gifb200_resize_bilinear_u8": (_i, [_p, _p, _i, _i, _i, _ll, _i, _i, _i, _f, _f, _i, _p]),
    "gifb200_split_bf16": (_i, [_p, _p, _p, _i, _i, _i, _p]),
    "gifb200_upfirdn2d": (_i, [_p, _p, _p] + [_i] * 14 + [_p]),
    "gifb200_bias_act": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _f, _f, _i, _p]),
    "gifb200_act_bwd": (_i, [_p, _p, _p, _ll, _f, _f, _i, _p]),
    "gifb200_rows_sum": (_i, [_p, _p, _i, _i, _i, _p]),
    "gifb200_chan_scale": (_i, [_p, _p, _p, _i, _i, _i, _i, _p]),
    "gifb200_tail_bwd": (_i, [_p] * 8 + [_i, _i, _i, _f, _f, _i, _p]),
    "gifb200_tail_bwd_planes": (_i, [_p] * 8 + [_i, _i, _i, _f, _f, _p, _p, _p]),
    "gifb200_scale_bwd": (_i, [_p] * 5 + [_i, _i, _i, _i, _p]),
    "gifb200_tail_bwd2": (_i, [_p] * 9 + [_i, _i, _i, _f, _f, _p, _p]),
    "gifb200_adam_step": (_i, [_p, _p, _p, _p, _p, _p, _i, _d, _d, _d, _d, _p]),
    "gifb200_spatial_dot": (_i, [_p, _p, _p, _i, _i, _i, _p]),
    "gifb200_axpby": (_i, [_p, _p, _p, _ll, _f, _f, _i, _p]),
    "gifb200_demod": (_i, [_p, _p, _p, _i, _i, _i, _f, _p]),
    "gifb200_torgb_fwd": (_i, [_p, _p, _p, _i, _i, _i, _p]),
    "gifb200_torgb_bwd_x": (_i, [_p, _p, _p, _i, _i, _i, _p]),
    "gifb200_torgb_bwd_w": (_i, [_p, _p, _p, _i, _i, _i, _p]),
    "gifb200_sgemm": (_i, [_i, _i, _i, _i, _i, _f, _p, _i, _p, _i, _p, _i, _p]),
    "gifb200_cond_down": (_i, [_p, _p, _i, _i, _i, _i, _i, _i, _p]),
    "gifb200_cond_up": (_i, [_p, _p, _i, _i, _i, _i, _i, _i, _p]),
    "gifb200_rasterize_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "gifb200_rasterize_fwd": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p, _sz, _p]),
    "gifb200_rasterize_fwd_ex": (_i, [_p] * 7 + [_i] * 5 + [_p, _sz, _p]),
    "gifb200_rasterize_bwd_ex": (_i, [_p] * 11 + [_i] * 5 + [_p]),
    "gifb200_render_shade": (_i, [_p] * 10 + [_i] * 5 + [_p]),
    "gifb200_vertex_normals": (_i, [_p] * 6 + [_i] * 3 + [_p]),
    "gifb200_rasterize_bwd": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p]),
    "gifb200_flame_lbs_workspace_bytes": (_sz, [_i, _i]),
    "gifb200_flame_lbs": (_i, [_p] * 11 + [_i] * 4 + [_p, _sz, _p]),
    "gifb200_eye_camera": (_i, [_p, _p] + [_i] * 4 + [_f] * 4 + [_p]),
    "gifb200_flametex": (_i, [_p] * 4 + [_i] * 4 + [_p]),
    "gifb200_texture_steal_fwd": (_i, [_p] * 9 + [_i] * 6 + [_p]),
    "gifb200_texture_steal_bwd": (_i, [_p] * 7 + [_i] * 6 + [_p]),
    "gifb200_jpeg_workspace_bytes": (_sz, [_i, _i, _ll]),
    "gifb200_jpeg_decode": (_i, [_p] * 6 + [_i, _i, _i, _ll, _i, _i, _p, _p, _p, _sz, _p]),
    "gifb200_png_unfilter": (_i, [_p, _p, _i, _i, _p, _p, _p]),
    "gifb200_resize_bicubic_u8": (_i, [_p] * 5 + [_i] * 7 + [_p]),
    "gifb200_u8_to_unit": (_i, [_p, _p, _i, _i, _i, _ll, _p]),
    "gifb200_image_to_u8": (_i, [_p, _p, _i, _i, _i, _ll, _ll, _ll, _ll, _p]),
    "gifb200_jpeg_encode_workspace_bytes": (_sz, [_i, _i, _i]),
    "gifb200_jpeg_encode_out_bytes": (_sz, [_i, _i, _i]),
    "gifb200_jpeg_encode": (_i, [_p, _p, _i, _i, _i, _p, _p, _p, _sz, _p]),
}


def _bind(path):
    lib = ctypes.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == the .so does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    return lib


def _load():
    import importlib.util
    spec = importlib.util.spec_from_file_location("_gifb200_build", os.path.join(_HERE, "build.py"))
    _build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(_build)
    # incremental (content-hash stamps): a no-op when the library is current, a rebuild when the sources changed
    # (nvcc cross-compiles without a GPU).  A library that still lacks a declared symbol afterwards fails the import.
    _build.build()
    return _bind(LIB_PATH)


lib = _load()


class GifB200Error(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        msg = lib.gifb200_last_error().decode("utf-8", "replace")
        raise GifB200Error(f"{what} failed with code {rc}: {msg}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise GifB200Error("gif_b200 ops run on CUDA tensors only (there is no CPU fallback); got a "
                               f"{t.device} tensor")
        if t is not None and t.dtype != torch.float32 and t.dtype != torch.int32:
            raise GifB200Error(f"gif_b200 ops take float32 tensors, got {t.dtype}")


def launch_count():
    return int(lib.gifb200_launch_count())
