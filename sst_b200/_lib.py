"""ctypes binding of libsstb200.so (the C ABI declared in include/sstb200.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.
torch is used only for device memory / streams (tensor.data_ptr(), torch.cuda.current_stream()).
"""
import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsstb200.so")

_lib = None
_lock = threading.Lock()
_ctx = {}  # (device, stream) -> ctx

vp, i32, i64, f32 = C.c_void_p, C.c_int32, C.c_int64, C.c_float
P_i32, P_i64, P_f32 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_float)

# name -> (restype, argtypes).  Kept in one table so tests can check it against include/sstb200.h.
SIGNATURES = {
    "sstb200_version": (C.c_int, []),
    "sstb200_create": (vp, [C.c_int]),
    "sstb200_destroy": (None, [vp]),
    "sstb200_set_stream": (C.c_int, [vp, vp]),
    "sstb200_last_error": (C.c_char_p, [vp]),
    "sstb200_num_sms": (C.c_int, [vp]),
    "sstb200_dynamic_voxelize": (C.c_int, [vp, vp, C.c_int, C.c_int, P_f32, P_f32, vp]),
    "sstb200_hard_voxelize": (C.c_int, [vp, vp, C.c_int, C.c_int, P_f32, P_f32, C.c_int, C.c_int, vp, vp, vp, vp, P_i32]),
    "sstb200_dynamic_point_to_voxel_forward": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, P_i32, P_i32,
                                                           vp, vp, vp, vp, vp, P_i32]),
    "sstb200_dynamic_point_to_voxel_backward": (C.c_int, [vp, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int,
                                                            C.c_int]),
    "sstb200_unique_rows_i64": (C.c_int, [vp, vp, C.c_int, C.c_int, P_i64, P_i64, vp, vp, vp, vp, P_i32]),
    "sstb200_segment_reduce": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]),
    "sstb200_ingroup_indices": (C.c_int, [vp, vp, C.c_int, C.c_int64, vp]),
}


class SSTB200Error(RuntimeError):
    pass


class _Signatures(dict):
    """name -> (restype, argtypes).  Assigning after the library is loaded binds the prototype immediately, so
    modules imported late (engine, sir, ...) can never call through an un-prototyped (pointer-truncating) symbol."""

    def __setitem__(self, name, sig):
        super().__setitem__(name, sig)
        if _lib is not None:
            _bind(_lib, name, sig)


def _bind(L, name, sig):
    fn = getattr(L, name)  # AttributeError if the symbol is missing -> loud
    fn.restype, fn.argtypes = sig


SIGNATURES = _Signatures(SIGNATURES)


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise SSTB200Error(
                    f"{LIB_PATH} not found - build it with `python -m sst_b200.build` "
                    "(there is no CPU or PyTorch fallback for this path)")
            L = C.CDLL(LIB_PATH)
            for name, sig in SIGNATURES.items():
                _bind(L, name, sig)
            _lib = L
    return _lib


def ctx(device=None):
    """Per-(device, current stream) context."""
    if not torch.cuda.is_available():
        raise SSTB200Error("sst_b200 needs a CUDA device (sm_90a); no CPU fallback exists")
    if device is None:
        device = torch.cuda.current_device()
    elif isinstance(device, torch.device):
        device = device.index if device.index is not None else torch.cuda.current_device()
    stream = torch.cuda.current_stream(device).cuda_stream
    key = (device, stream)
    c = _ctx.get(key)
    if c is None:
        L = lib()
        with torch.cuda.device(device):
            c = L.sstb200_create(device)
        if not c:
            raise SSTB200Error(f"sstb200_create({device}) failed")
        L.sstb200_set_stream(c, stream)
        _ctx[key] = c
    return c


def check(c, rc):
    if rc != 0:
        msg = lib().sstb200_last_error(c)
        raise SSTB200Error(f"libsstb200 error {rc}: {msg.decode() if msg else '?'}")


def ptr(t):
    return 0 if t is None else t.data_ptr()


def arr(ctype, vals):
    return (ctype * len(vals))(*vals)
