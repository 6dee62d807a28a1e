"""ctypes binding of libvil_attn.so (C ABI declared in include/vil_attn.h).

There is deliberately NO fallback: if the library is missing the import-time
loader raises, and every op raises if CUDA is unavailable.  The library is
built in-tree by `__graft_entry__.build()` (nvcc, sm_90a).
"""
from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_NAME = "libvil_attn.so"
LIB_PATH = os.environ.get("VIL_ATTN_LIB") or os.path.join(_HERE, LIB_NAME)   # override: debug builds only

VIL_F32, VIL_BF16, VIL_F16 = 0, 1, 2
VIL_IMPL_AUTO, VIL_IMPL_SIMT, VIL_IMPL_WGMMA = 0, 1, 2
VIL_E_BADARG, VIL_E_UNSUPPORTED, VIL_E_CUDA, VIL_E_WORKSPACE = -1, -2, -3, -4
ABI_VERSION = 3
VIL_FLAG_F32_OUT, VIL_FLAG_UNFUSED, VIL_FLAG_F32_SPLIT, VIL_FLAG_DILATED = 1, 2, 4, 16

# every symbol include/vil_attn.h declares
EXPORTS = (
    "vil_attn_abi_version", "vil_attn_last_error", "vil_attn_launch_count", "vil_attn_last_impl", "vil_attn_last_kernel",
    "vil_attn_workspace_bytes", "vil_attn_wgmma_supported", "vil_attn_fwd_sm100", "vil_attn_bwd_sm100",
    "vil_attn_fwd_sized_sm100", "vil_attn_bwd_sized_sm100",
    "vil_layernorm_workspace_bytes", "vil_layernorm_fwd_sm100", "vil_layernorm_bwd_sm100",
    "vil_addnorm_workspace_bytes", "vil_addnorm_fwd_sm100", "vil_addnorm_bwd_sm100",
    "vil_bias_act_workspace_bytes", "vil_bias_act_fwd_sm100", "vil_bias_act_bwd_sm100",
)
VIL_ACT_NONE, VIL_ACT_GELU = 0, 1


class VilTensor4(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("sb", ctypes.c_int64), ("sh", ctypes.c_int64), ("st", ctypes.c_int64)]


class VilAttnParams(ctypes.Structure):
    _fields_ = [
        ("struct_bytes", ctypes.c_int32), ("dtype", ctypes.c_int32), ("impl", ctypes.c_int32),
        ("B", ctypes.c_int32), ("H", ctypes.c_int32), ("D", ctypes.c_int32),
        ("nx", ctypes.c_int32), ("ny", ctypes.c_int32), ("w", ctypes.c_int32), ("nglo", ctypes.c_int32),
        ("exact", ctypes.c_int32), ("mode", ctypes.c_int32), ("scale", ctypes.c_float), ("skip_mask", ctypes.c_int32),
        ("flags", ctypes.c_int32),
        ("q", VilTensor4), ("k", VilTensor4), ("v", VilTensor4),
        ("qg", VilTensor4), ("kg", VilTensor4), ("vg", VilTensor4),
        ("o", VilTensor4), ("og", VilTensor4),
        ("lse", ctypes.c_void_p), ("lse_g", ctypes.c_void_p),
        ("bias_table", ctypes.c_void_p), ("g2l", ctypes.c_void_p), ("g2g", ctypes.c_void_p),
        ("d_o", VilTensor4), ("d_og", VilTensor4),
        ("dq", VilTensor4), ("dk", VilTensor4), ("dv", VilTensor4),
        ("dqg", VilTensor4), ("dkg", VilTensor4), ("dvg", VilTensor4),
        ("d_bias_table", ctypes.c_void_p), ("d_g2l", ctypes.c_void_p), ("d_g2g", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
        ("dropout_p", ctypes.c_float), ("dilation", ctypes.c_int32),
        ("dropout_seed", ctypes.c_uint64), ("dropout_offset", ctypes.c_uint64),
    ]


class VilLayerNormParams(ctypes.Structure):
    _fields_ = [
        ("struct_bytes", ctypes.c_int32), ("x_dtype", ctypes.c_int32), ("y_dtype", ctypes.c_int32), ("C", ctypes.c_int32),
        ("rows", ctypes.c_int64), ("eps", ctypes.c_float), ("reserved", ctypes.c_int32),
        ("x", ctypes.c_void_p), ("gamma", ctypes.c_void_p), ("beta", ctypes.c_void_p),
        ("y", ctypes.c_void_p), ("mean", ctypes.c_void_p), ("rstd", ctypes.c_void_p),
        ("dy", ctypes.c_void_p), ("dx", ctypes.c_void_p), ("dgamma", ctypes.c_void_p), ("dbeta", ctypes.c_void_p),
        ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
    ]


class VilAddNormParams(ctypes.Structure):
    _fields_ = [
        ("struct_bytes", ctypes.c_int32), ("b_dtype", ctypes.c_int32), ("y_dtype", ctypes.c_int32), ("C", ctypes.c_int32),
        ("rows", ctypes.c_int64), ("rows_per_sample", ctypes.c_int64), ("eps", ctypes.c_float), ("reserved", ctypes.c_int32),
        ("x", ctypes.c_void_p), ("br", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("rowscale", ctypes.c_void_p),
        ("gamma", ctypes.c_void_p), ("beta", ctypes.c_void_p), ("xo", ctypes.c_void_p), ("y", ctypes.c_void_p),
        ("mean", ctypes.c_void_p), ("rstd", ctypes.c_void_p), ("dy", ctypes.c_void_p), ("gres", ctypes.c_void_p),
        ("dx", ctypes.c_void_p), ("dbr", ctypes.c_void_p), ("dgamma", ctypes.c_void_p), ("dbeta", ctypes.c_void_p),
        ("dbias", ctypes.c_void_p), ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
    ]


class VilBiasActParams(ctypes.Structure):
    _fields_ = [
        ("struct_bytes", ctypes.c_int32), ("dtype", ctypes.c_int32), ("C", ctypes.c_int32), ("act", ctypes.c_int32),
        ("rows", ctypes.c_int64),
        ("z", ctypes.c_void_p), ("bias", ctypes.c_void_p), ("a", ctypes.c_void_p), ("da", ctypes.c_void_p),
        ("dz", ctypes.c_void_p), ("dbias", ctypes.c_void_p), ("workspace", ctypes.c_void_p), ("workspace_bytes", ctypes.c_int64),
    ]


_lib = None
_lock = threading.Lock()


def load() -> ctypes.CDLL:
    """Load (once) and type the shared library.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc -gencode arch=compute_90a,code=sm_90a).  There is no CPU / PyTorch fallback.")
        lib = ctypes.CDLL(LIB_PATH)
        lib.vil_attn_abi_version.restype = ctypes.c_int
        lib.vil_attn_last_error.restype = ctypes.c_char_p
        lib.vil_attn_last_impl.restype = ctypes.c_char_p
        lib.vil_attn_last_kernel.restype = ctypes.c_char_p
        lib.vil_attn_launch_count.restype = ctypes.c_int64
        lib.vil_attn_workspace_bytes.restype = ctypes.c_int64
        lib.vil_attn_workspace_bytes.argtypes = [ctypes.POINTER(VilAttnParams), ctypes.c_int]
        lib.vil_attn_wgmma_supported.restype = ctypes.c_int
        lib.vil_attn_wgmma_supported.argtypes = [ctypes.POINTER(VilAttnParams)]
        for fn in (lib.vil_attn_fwd_sm100, lib.vil_attn_bwd_sm100):
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.POINTER(VilAttnParams), ctypes.c_void_p]
        for fn in (lib.vil_attn_fwd_sized_sm100, lib.vil_attn_bwd_sized_sm100):
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.POINTER(VilAttnParams), ctypes.c_void_p, ctypes.c_void_p]
        lib.vil_layernorm_workspace_bytes.restype = ctypes.c_int64
        lib.vil_layernorm_workspace_bytes.argtypes = [ctypes.POINTER(VilLayerNormParams)]
        for fn in (lib.vil_layernorm_fwd_sm100, lib.vil_layernorm_bwd_sm100):
            fn.restype = ctypes.c_int
            fn.argtypes = [ctypes.POINTER(VilLayerNormParams), ctypes.c_void_p]
        for ws, fns, st in ((lib.vil_addnorm_workspace_bytes, (lib.vil_addnorm_fwd_sm100, lib.vil_addnorm_bwd_sm100), VilAddNormParams),
                            (lib.vil_bias_act_workspace_bytes, (lib.vil_bias_act_fwd_sm100, lib.vil_bias_act_bwd_sm100), VilBiasActParams)):
            ws.restype = ctypes.c_int64
            ws.argtypes = [ctypes.POINTER(st)]
            for fn in fns:
                fn.restype = ctypes.c_int
                fn.argtypes = [ctypes.POINTER(st), ctypes.c_void_p]
        if lib.vil_attn_abi_version() != ABI_VERSION:
            raise RuntimeError(f"ABI mismatch: library {lib.vil_attn_abi_version()}, binding {ABI_VERSION}")
        _lib = lib
    return _lib


def last_error() -> str:
    return load().vil_attn_last_error().decode()


def last_impl() -> str:
    return load().vil_attn_last_impl().decode()


def last_kernel() -> str:
    return load().vil_attn_last_kernel().decode()


def launch_count() -> int:
    return int(load().vil_attn_launch_count())


def aligned(t):
    """`t` itself when its data starts on a 16-byte boundary (every caching-allocator tensor does), else an aligned copy.
    The epilogue kernels make 128-bit accesses and the library refuses misaligned pointers; a contiguous view can still
    start at any element (`buf[1:].view(...)`, a parameter that is a view into a flat buffer)."""
    if t is None or t.data_ptr() % 16 == 0:
        return t
    return t.clone()                     # callers pass contiguous tensors: the fresh copy keeps their strides


def raise_for(code: int):
    """Map a C return code to the exception type the reference raises for the same condition
    (asserts / ValueError in longformer2d.py:111, slidingchunk_2d.py:343)."""
    if code == 0:
        return
    msg = last_error()
    if code == VIL_E_BADARG:
        raise ValueError(msg)
    if code == VIL_E_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(f"vil_attn error {code}: {msg}")
