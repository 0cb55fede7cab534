"""ctypes binding of libcontrollora_b200.so (C ABI: include/controllora_b200.h).

The product path has no CPU or library fallback: if the shared library is missing, or a call fails, this module
raises.  PyTorch is used only as the owner of device memory and streams.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import os

_PKG = Path(__file__).resolve().parent
# CLB_LIB selects another build of the same sources (e.g. one compiled with extra CLB_EXTRA_NVCC flags); never a different
# implementation.
LIB_PATH = Path(os.environ["CLB_LIB"]) if os.environ.get("CLB_LIB") else _PKG / "libcontrollora_b200.so"


class CLError(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Load the shared library (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise CLError(
                f"{LIB_PATH} is missing: run `python -m controllora_b200.build` (or __graft_entry__.build()). "
                "controllora_b200 has no CPU / PyTorch fallback for its CUDA kernels."
            )
        _lib = C.CDLL(str(LIB_PATH))
        _lib.cl_last_error.restype = C.c_char_p
        _lib.cl_launch_count.restype = C.c_int64
        _lib.cl_canny.restype = C.c_int
        _lib.cl_canny.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]
    return _lib


def require_cuda(device, what: str) -> None:
    """Every public entry of the package calls this: the product has no CPU path.  The one exception is the test suite's
    host-logic mode (CLB_DRYRUN=1, set by the checkers under tests/), where the kernel wrappers have been replaced by
    test doubles and only the Python program above the C ABI is being exercised."""
    dev_type = device if isinstance(device, str) else getattr(device, "type", str(device))
    if dev_type != "cuda" and not os.environ.get("CLB_DRYRUN"):
        raise RuntimeError(f"controllora_b200.{what} runs only on CUDA (sm_90a); there is no CPU path")


def check(status: int, what: str = "") -> None:
    if status != 0:
        msg = lib().cl_last_error().decode("utf-8", "replace")
        raise CLError(f"{what} failed with status {status}: {msg}")


def launch_count() -> int:
    return int(lib().cl_launch_count())


class GemmArgs(C.Structure):
    _fields_ = [
        ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("a_mode", C.c_int32),
        ("a", C.c_void_p),
        ("lda", C.c_int64),
        ("n_img", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("C", C.c_int32),
        ("pad_lo", C.c_int32),
        ("b", C.c_void_p),
        ("ldb", C.c_int64),
        ("ext", C.c_void_p),
        ("ldb_ext", C.c_int64),
        ("bias", C.c_void_p),
        ("row_bias", C.c_void_p),
        ("rows_per_group", C.c_int32),
        ("ld_row_bias", C.c_int64),
        ("residual", C.c_void_p),
        ("ldr", C.c_int64),
        ("lora_up", C.c_void_p),
        ("lora_rp", C.c_int32),
        ("lora_scale", C.c_float),
        ("t_add", C.c_void_p),
        ("t_out", C.c_void_p),
        ("out", C.c_void_p),
        ("ldd", C.c_int64),
        ("out_fp32", C.c_int32),
        ("block_n", C.c_int32),
        ("split_k", C.c_int32),
        ("split_ws", C.c_void_p),
    ]


class AttnFwdArgs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("H", C.c_int32), ("Nq", C.c_int32), ("Nk", C.c_int32), ("d", C.c_int32),
        ("q", C.c_void_p), ("ldq", C.c_int64),
        ("k", C.c_void_p), ("ldk", C.c_int64),
        ("v", C.c_void_p), ("ldv", C.c_int64),
        ("o", C.c_void_p), ("ldo", C.c_int64),
        ("lse", C.c_void_p),
        ("scale", C.c_float),
    ]


class AttnBwdArgs(C.Structure):
    _fields_ = [
        ("B", C.c_int32), ("H", C.c_int32), ("Nq", C.c_int32), ("Nk", C.c_int32), ("d", C.c_int32),
        ("q", C.c_void_p), ("ldq", C.c_int64),
        ("k", C.c_void_p), ("ldk", C.c_int64),
        ("v", C.c_void_p), ("ldv", C.c_int64),
        ("o", C.c_void_p), ("ldo", C.c_int64),
        ("d_o", C.c_void_p), ("lddo", C.c_int64),
        ("lse", C.c_void_p),
        ("delta", C.c_void_p),
        ("dq", C.c_void_p), ("lddq", C.c_int64),
        ("dk", C.c_void_p), ("lddk", C.c_int64),
        ("dv", C.c_void_p), ("lddv", C.c_int64),
        ("scale", C.c_float),
    ]


class PackDesc(C.Structure):
    _fields_ = [
        ("src", C.c_void_p),
        ("dst", C.c_void_p),
        ("kind", C.c_int32),
        ("r", C.c_int32), ("K", C.c_int32),
        ("s_j", C.c_int64), ("s_k", C.c_int64),
        ("ld", C.c_int32),
        ("row_off", C.c_int32),
        ("mul", C.c_float),
        ("pad_", C.c_int32),
    ]


class SkinnyDesc(C.Structure):
    _fields_ = [
        ("a", C.c_void_p), ("lda", C.c_int32), ("r", C.c_int32),
        ("b", C.c_void_p), ("ldb", C.c_int64),
        ("out", C.c_void_p), ("so_j", C.c_int64), ("so_c", C.c_int64),
        ("alpha", C.c_float), ("M", C.c_int32), ("C", C.c_int32),
    ]


SKINNY_MAX = 16
