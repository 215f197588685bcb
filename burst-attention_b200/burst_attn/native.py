"""ctypes binding of the C-ABI library ``libburst_attn_b200.so`` (include/burst_attn_b200.h).

There is deliberately NO fallback: if the shared library is missing or the
device is not sm_90 (H100), every entry point raises.  PyTorch is used only for
device memory and streams (``tensor.data_ptr()``, ``torch.cuda.current_stream()``).
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# BA_LIB_PATH: developer hook to A/B a differently built library (tools/); default is the in-tree build
LIB_PATH = os.environ.get("BA_LIB_PATH") or os.path.join(os.path.dirname(_HERE), "lib", "libburst_attn_b200.so")

BA_DTYPE_FP16, BA_DTYPE_BF16 = 0, 1
BA_MASK_NONE, BA_MASK_CAUSAL, BA_MASK_LOWER = 0, 1, 2
BA_FWD_FIRST, BA_FWD_LAST = 1, 2
NCCL_UNIQUE_ID_BYTES = 128
IPC_HANDLE_BYTES = 64


class NativeLibraryError(RuntimeError):
    pass


class ba_tensor4(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("stride_b", ctypes.c_int64),
                ("stride_s", ctypes.c_int64), ("stride_h", ctypes.c_int64)]


class ba_rowstat(ctypes.Structure):
    _fields_ = [("ptr", ctypes.c_void_p), ("stride_b", ctypes.c_int64), ("stride_h", ctypes.c_int64)]


_lib = None

_i, _f, _vp, _i64 = ctypes.c_int, ctypes.c_float, ctypes.c_void_p, ctypes.c_int64
_T4, _RS, _PVP = ba_tensor4, ba_rowstat, ctypes.POINTER(ctypes.c_void_p)
# name -> (restype, argtypes) of every function include/burst_attn_b200.h declares, in its order
# (tests/test_native_abi.py checks each signature against the header)
_EXPORTS = {
    "ba_last_error": (ctypes.c_char_p, []),
    "ba_device_check": (_i, []),
    "ba_version": (_i, []),
    "ba_fwd_chunk": (_i, [_T4, _T4, _T4, _T4, _RS, _T4, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "ba_fwd_chunk_bias": (_i, [_T4, _T4, _T4, _RS, _T4, _RS, _T4, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "ba_fwd_chunk_gqa": (_i, [_T4, _T4, _T4, _RS, _T4, _RS, _T4, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "ba_fwd_chunk_band": (_i, [_T4, _T4, _T4, _RS, _T4, _RS, _T4, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _i, _vp]),
    "ba_fwd_chunk_alibi": (_i, [_T4, _T4, _T4, _T4, _RS, _T4, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i,
                                _vp, _i64, _i64, _i, _i, _i, _vp]),
    "ba_fwd_chunk_doc": (_i, [_T4, _T4, _T4, _T4, _RS, _T4, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i,
                              _vp, _i, _i64, _i64, _i, _i, _i, _vp]),
    "ba_bwd_delta": (_i, [_T4, _T4, _RS, _i, _i, _i, _i, _i, _vp]),
    "ba_bwd_chunk": (_i, [_T4, _T4, _T4, _T4, _RS, _RS, _T4, _T4, _T4, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "ba_bwd_chunk_bias": (_i, [_T4, _T4, _T4, _T4, _RS, _RS, _RS, _T4, _T4, _T4,
                               _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "ba_bwd_chunk_gqa": (_i, [_T4, _T4, _T4, _T4, _RS, _RS, _RS, _T4, _T4, _T4,
                              _i, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _vp]),
    "ba_bwd_chunk_band": (_i, [_T4, _T4, _T4, _T4, _RS, _RS, _RS, _T4, _T4, _T4,
                               _i, _i, _i, _i, _i, _i, _f, _i, _i, _i, _i, _i, _vp]),
    "ba_bwd_chunk_alibi": (_i, [_T4, _T4, _T4, _T4, _RS, _RS, _T4, _T4, _T4, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i,
                                _vp, _i64, _i64, _i, _i, _i, _vp]),
    "ba_bwd_chunk_doc": (_i, [_T4, _T4, _T4, _T4, _RS, _RS, _T4, _T4, _T4, _i, _i, _i, _i, _i, _i, _f, _i, _i, _i,
                              _vp, _i, _i64, _i64, _i, _i, _i, _vp]),
    "ba_cast_from_f32": (_i, [_T4, _T4, _i, _i, _i, _i, _i, _vp]),
    "ba_accumulate_f32": (_i, [_T4, _T4, _i, _i, _i, _i, _vp]),
    "ba_ring_unique_id": (_i, [_vp]),
    "ba_ring_create": (_i, [_vp, _i, _i, _PVP]),
    "ba_ring_post": (_i, [_vp, _PVP, _PVP, ctypes.POINTER(_i64), _i, _vp]),
    "ba_ring_wait": (_i, [_vp, _vp]),
    "ba_ring_rank": (_i, [_vp]),
    "ba_ring_world": (_i, [_vp]),
    "ba_ring_destroy": (_i, [_vp]),
    "ba_ring_arena_create": (_i, [_vp, _i64, _PVP, _vp]),
    "ba_ring_arena_connect": (_i, [_vp, _vp, _vp]),
}
SELFTEST_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libburst_attn_b200_selftest.so")
# the same for include/burst_attn_b200_selftest.h
_SELFTEST_EXPORTS = {
    "ba_selftest_last_error": (ctypes.c_char_p, []),
    "ba_selftest": (_i, [_i, _vp, _vp, _vp, _i, _vp]),
}


def _bind(L: ctypes.CDLL, signatures) -> ctypes.CDLL:
    for name, (restype, argtypes) in signatures.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    return L


def exported_symbols() -> Sequence[str]:
    """Every symbol include/burst_attn_b200.h declares (checked by the CPU tests)."""
    return tuple(_EXPORTS)


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C burst-attention_b200/csrc`).  There is no CPU/PyTorch fallback.")
    _lib = _bind(ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL), _EXPORTS)
    return _lib


_selftest_lib = None


def selftest_lib() -> ctypes.CDLL:
    """The diagnostics library (include/burst_attn_b200_selftest.h); loaded by tests/ and tools/ only."""
    global _selftest_lib
    if _selftest_lib is None:
        if not os.path.exists(SELFTEST_LIB_PATH):
            raise NativeLibraryError(f"{SELFTEST_LIB_PATH} not found: build with __graft_entry__.build()")
        _selftest_lib = _bind(ctypes.CDLL(SELFTEST_LIB_PATH), _SELFTEST_EXPORTS)
    return _selftest_lib


def check_selftest(rc: int, what: str) -> None:
    if rc != 0:
        msg = selftest_lib().ba_selftest_last_error()
        raise NativeLibraryError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = lib().ba_last_error()
        raise NativeLibraryError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")


def dtype_code(dt: torch.dtype) -> int:
    if dt == torch.bfloat16:
        return BA_DTYPE_BF16
    if dt == torch.float16:
        return BA_DTYPE_FP16
    raise TypeError(f"burst_attn_b200 supports float16/bfloat16 inputs, got {dt}")


def t4(t: Optional[torch.Tensor], seq_dim: int) -> ba_tensor4:
    """[b,s,h,d] view descriptor of a 4-D tensor whose sequence axis is ``seq_dim``
    (1 for the flash layout [B,S,H,D], 2 for the normal layout [B,H,S,D])."""
    if t is None:
        return ba_tensor4(None, 0, 0, 0)
    assert t.dim() == 4 and t.stride(3) == 1, "last (head_dim) axis must be contiguous"
    return ba_tensor4(t.data_ptr(), t.stride(0), t.stride(seq_dim), t.stride(3 - seq_dim))


def rs(t: Optional[torch.Tensor]) -> ba_rowstat:
    """[B,H,S] fp32 row statistic (lse / delta / key bias); S contiguous.  None -> null view."""
    if t is None:
        return ba_rowstat(None, 0, 0)
    assert t.dim() == 3 and t.stride(2) == 1 and t.dtype == torch.float32
    return ba_rowstat(t.data_ptr(), t.stride(0), t.stride(1))


def stream_ptr(device=None) -> int:
    return torch.cuda.current_stream(device).cuda_stream
