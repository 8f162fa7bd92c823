"""ctypes binding of ``libdefer_b200.so`` (``include/defer_b200.h``) - thin, no logic.

The library is the product: if it is missing and cannot be built, or no CUDA device is usable,
calls raise ``RuntimeError``; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from pathlib import Path

import numpy as np

ABI_VERSION = 2
LINK_TOKEN_BYTES = 256

# enums (include/defer_b200.h)
FMT_F32, FMT_BF16X2, FMT_BF16 = 0, 1, 2
OP_CONV, OP_MAXPOOL, OP_GAP, OP_DENSE, OP_SOFTMAX, OP_AFFINE, OP_RELU, OP_ADD, OP_PAD, OP_COPY, OP_PREPROCESS, OP_RESIZE = range(1, 13)
FLAG_RELU, FLAG_RESIDUAL = 1, 2
BUF_ACT, BUF_F32, BUF_U8, BUF_JPEG, BUF_PNG, BUF_IMAGE = 0, 1, 2, 3, 4, 5
OP_JPEG_DECODE, OP_PNG_DECODE, OP_IMAGE_DECODE = 13, 14, 15
PRE_CAFFE, PRE_TF = 0, 1
PRE_MODES = {"caffe": PRE_CAFFE, "tf": PRE_TF}
RESIZE_SAMPLE_W, RESIZE_SAMPLE_H = 1, 2
RESIZE_W, RESIZE_H = 4, 5      # fixed tables on the named axis, which may keep its length (a keep_aspect_ratio crop box)
OK, ERR_INVALID, ERR_CUDA, ERR_TIMEOUT, ERR_STATE = 0, -1, -2, -3, -4

FMT_NAMES = {FMT_F32: "f32", FMT_BF16X2: "bf16x2", FMT_BF16: "bf16"}
OP_NAMES = {OP_CONV: "conv", OP_MAXPOOL: "maxpool", OP_GAP: "gap", OP_DENSE: "dense", OP_SOFTMAX: "softmax",
            OP_AFFINE: "affine", OP_RELU: "relu", OP_ADD: "add", OP_PAD: "pad", OP_COPY: "copy",
            OP_PREPROCESS: "preprocess"}
#: OP_NAMES covers the ops of a model and of its preprocess_input; KIND_NAMES adds RESIZE, the load_img resize in front
KIND_NAMES = {**OP_NAMES, OP_RESIZE: "resize", OP_JPEG_DECODE: "jpeg_decode", OP_PNG_DECODE: "png_decode",
              OP_IMAGE_DECODE: "image_decode"}


class BufDesc(C.Structure):
    _fields_ = [("h", C.c_int32), ("w", C.c_int32), ("c", C.c_int32), ("elem", C.c_int32)]


class OpDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("in0", C.c_int32), ("in1", C.c_int32), ("out", C.c_int32),
                ("kh", C.c_int32), ("kw", C.c_int32), ("sh", C.c_int32), ("sw", C.c_int32),
                ("pad_t", C.c_int32), ("pad_l", C.c_int32), ("pad_b", C.c_int32), ("pad_r", C.c_int32),
                ("flags", C.c_uint32), ("w_kernel", C.c_int32), ("w_scale", C.c_int32), ("w_shift", C.c_int32),
                ("mode", C.c_int32)]


class StageConfig(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("device", C.c_int32), ("fmt", C.c_int32), ("batch", C.c_int32),
                ("depth", C.c_int32), ("input_buf", C.c_int32), ("output_buf", C.c_int32),
                ("is_first", C.c_int32), ("is_last", C.c_int32), ("conv_backend", C.c_int32),
                ("use_graph", C.c_int32), ("wait_timeout_ms", C.c_int32)]


_vp, _i, _u64, _f32p = C.c_void_p, C.c_int, C.c_uint64, C.POINTER(C.c_float)

#: every symbol include/defer_b200.h declares: name -> (restype, argtypes)
PROTOTYPES = {
    "defer_last_error": (C.c_char_p, []),
    "defer_abi_version": (_i, []),
    "defer_device_count": (_i, [C.POINTER(_i)]),
    "defer_device_info": (_i, [_i, C.c_char_p, _i, C.POINTER(_i), C.POINTER(_i), C.POINTER(_u64)]),
    "defer_stage_create": (_i, [C.POINTER(StageConfig), C.POINTER(BufDesc), _i, C.POINTER(OpDesc), _i,
                                C.POINTER(_vp), C.POINTER(_u64), _i, C.POINTER(_vp)]),
    "defer_stage_destroy": (_i, [_vp]),
    "defer_stage_describe": (_i, [_vp, C.c_char_p, C.c_size_t]),
    "defer_stage_io_bytes": (_i, [_vp, C.POINTER(_u64), C.POINTER(_u64)]),
    "defer_stage_link": (_i, [_vp, _vp]),
    "defer_stage_export_link": (_i, [_vp, _i, _vp]),
    "defer_stage_import_link": (_i, [_vp, _i, _vp]),
    "defer_stage_unlink": (_i, [_vp]),
    "defer_stage_finalize": (_i, [_vp]),
    "defer_stage_submit": (_i, [_vp, _u64, _vp, _u64]),
    "defer_stage_submit_part": (_i, [_vp, _u64, _i, _i, _vp, _u64]),
    "defer_stage_submit_parts": (_i, [_vp, _u64, _i, _i, _i, C.POINTER(_vp), _u64]),
    "defer_stage_submit_frames": (_i, [_vp, _u64, _i, _i, C.POINTER(_vp), _vp, _vp, _u64]),
    "defer_stage_submit_jpegs": (_i, [_vp, _u64, _i, _i, C.POINTER(_vp), _vp, _vp, _u64]),
    "defer_stage_submit_pngs": (_i, [_vp, _u64, _i, _i, C.POINTER(_vp), _vp, _vp, _u64]),
    "defer_stage_submit_images": (_i, [_vp, _u64, _i, _i, C.POINTER(_vp), _vp, _vp, _u64]),
    "defer_stage_step": (_i, [_vp, _u64]),
    "defer_stage_result": (_i, [_vp, _u64, _vp, _u64]),
    "defer_stage_predict": (_i, [_vp, _vp, _u64, _vp, _u64]),
    "defer_stage_sync": (_i, [_vp]),
    "defer_stage_status": (_i, [_vp]),
    "defer_stage_last_step_us": (_i, [_vp, _i, C.POINTER(C.c_float)]),
    "defer_stage_timer_start": (_i, [_vp]),
    "defer_stage_timer_stop": (_i, [_vp, C.POINTER(C.c_float)]),
    "defer_stage_mark": (_i, [_vp, _u64, _i]),
    "defer_stage_mark_elapsed": (_i, [_vp, C.POINTER(C.c_float)]),
    "defer_stage_num_kernels": (_i, [_vp, C.POINTER(_i)]),
    "defer_stage_read_buffer": (_i, [_vp, _i, _i, _vp, _u64]),
    "defer_stage_stream": (_i, [_vp, _i, C.POINTER(_vp)]),
    "defer_stage_time_op": (_i, [_vp, _i, _i, _i, C.POINTER(C.c_float)]),
    "defer_stage_op_info": (_i, [_vp, _i, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_char_p, _i]),
    "defer_host_alloc": (_i, [C.POINTER(_vp), _u64]),
    "defer_host_free": (_i, [_vp]),
    "defer_host_register": (_i, [_vp, _u64]),
    "defer_host_unregister": (_i, [_vp]),
    "defer_k_conv": (_i, [_i, _i, _vp, _i, _vp, _vp, _vp, _vp, _vp] + [_i] * 13 + [C.c_uint32, _vp]),
    "defer_k_maxpool": (_i, [_i, _vp, _vp] + [_i] * 12 + [_vp]),
    "defer_k_gap": (_i, [_i, _vp, _vp, _i, _i, _i, _i, _vp]),
    "defer_k_dense": (_i, [_i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, C.c_uint32, _vp]),
    "defer_k_softmax": (_i, [_vp, _vp, _i, _i, _vp]),
    "defer_k_eltwise": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, C.c_uint32, _vp]),
    "defer_k_encode": (_i, [_i, _vp, _vp, _u64, _vp]),
    "defer_k_decode": (_i, [_i, _vp, _vp, _u64, _vp]),
    "defer_k_preprocess": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "defer_k_preprocess_tf": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "defer_k_resize": (_i, [_vp, _vp, _vp, _vp] + [_i] * 7 + [_vp]),
    "defer_k_resize_frames": (_i, [_i, _vp, _vp, _vp] + [_i] * 8 + [_vp]),
    "defer_k_jpeg_workspace": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp]),
    "defer_k_jpeg_decode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "defer_k_png_workspace": (_i, [_i, _i, _i, _vp, _vp, _vp]),
    "defer_k_png_decode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "defer_k_image_workspace": (_i, [_i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "defer_k_image_decode": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
}

_LIB = None
_LOCK = threading.Lock()


def lib_path() -> Path:
    return Path(__file__).resolve().parent / "lib" / "libdefer_b200.so"


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load the shared library and bind every prototype.  Raises if it cannot be loaded."""
    global _LIB
    with _LOCK:
        if _LIB is not None:
            return _LIB
        # The hop's device-side flag waits are spin kernels: a waiter must never sit in front of the kernel
        # it waits for in the same hardware work queue.  One stage per GPU uses `depth` streams (<= 8 queues
        # by default); several stages on ONE device (tests, 1-GPU debugging) need more queues.  Only
        # effective if CUDA has not been initialised in this process yet.
        os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
        path = lib_path()
        if not path.exists():
            if not build_if_missing:
                raise RuntimeError(f"{path} is missing; run `python -m defer_b200.build`")
            from . import build as _build
            _build.build()
        lib = C.CDLL(str(path), mode=os.RTLD_LOCAL | os.RTLD_NOW)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(lib, name)  # AttributeError => header / library drift
            fn.restype = res
            fn.argtypes = args
        if lib.defer_abi_version() != ABI_VERSION:
            raise RuntimeError(f"libdefer_b200 ABI {lib.defer_abi_version()} != binding {ABI_VERSION}")
        _LIB = lib
        return lib


class DeferError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libdefer_b200 error {code}: {msg}")
        self.code = code


def check(code: int) -> None:
    if code != OK:
        msg = load().defer_last_error()
        raise DeferError(code, msg.decode(errors="replace") if msg else "?")


def np_ptr(a: np.ndarray) -> C.c_void_p:
    return C.c_void_p(a.ctypes.data)


def device_count() -> int:
    n = C.c_int(0)
    check(load().defer_device_count(C.byref(n)))
    return n.value


def device_info(device: int = 0) -> dict:
    name = C.create_string_buffer(256)
    sm, cc, mem = C.c_int(0), C.c_int(0), C.c_uint64(0)
    check(load().defer_device_info(device, name, 256, C.byref(sm), C.byref(cc), C.byref(mem)))
    return {"name": name.value.decode(), "sm_count": sm.value, "cc": cc.value, "hbm_bytes": mem.value}
