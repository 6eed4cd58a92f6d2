"""ctypes loader of the C-ABI library (include/ct2b200.h).  Fails loudly: there is no CPU fallback."""
from __future__ import annotations

import ctypes
import os
import re

_HERE = os.path.dirname(os.path.abspath(__file__))
# CT2B200_LIB: another build of the same sources (python -m ctranslate2_b200.build --variant NAME), for A/B experiments
LIB_PATH = os.environ.get("CT2B200_LIB") or os.path.join(_HERE, "libct2b200.so")
HEADER_PATH = os.path.join(os.path.dirname(_HERE), "include", "ct2b200.h")
_lib = None


class Ct2B200Error(RuntimeError):
    pass


def declared_symbols():
    """Every function include/ct2b200.h declares."""
    text = open(HEADER_PATH).read()
    return sorted(set(re.findall(r"CT2B200_API[^;(]*?\b(ct2b200_\w+)\s*\(", text)))


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise Ct2B200Error(
                f"{LIB_PATH} is missing: build it with `python -m ctranslate2_b200.build` "
                "(ctranslate2_b200 has no CPU / PyTorch fallback)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.ct2b200_last_error.restype = ctypes.c_char_p
        _lib.ct2b200_version.restype = ctypes.c_char_p
        _lib.ct2b200_kernel_launch_count.restype = ctypes.c_int64
        _lib.ct2b200_generator_open.restype = ctypes.c_void_p
        _lib.ct2b200_translator_open.restype = ctypes.c_void_p
        _lib.ct2b200_attention_decode_workspace.restype = ctypes.c_size_t
    return _lib


def check(rc: int):
    if rc != 0:
        msg = lib().ct2b200_last_error().decode()
        if rc == 2:
            raise ValueError(msg)          # std::invalid_argument on the reference side
        raise Ct2B200Error(msg)            # std::runtime_error


class GeneratorConfig(ctypes.Structure):
    _fields_ = [("device", ctypes.c_int), ("compute_type", ctypes.c_int), ("max_batch", ctypes.c_int64),
                ("max_length", ctypes.c_int64), ("tp_rank", ctypes.c_int), ("tp_size", ctypes.c_int),
                ("use_cuda_graph", ctypes.c_int), ("gemm_impl", ctypes.c_int), ("weight_type", ctypes.c_int)]


def kernel_launch_count() -> int:
    return int(lib().ct2b200_kernel_launch_count())


def set_random_seed(seed: int):
    """ctranslate2.set_random_seed: the process-wide seed of random sampling.  It also restarts the sampling-call counter, so
    the same sequence of sampled calls after the same seed gives the same results."""
    check(lib().ct2b200_set_random_seed(ctypes.c_uint32(int(seed) & 0xFFFFFFFF)))
