"""ctypes binding of libb200sd.so (C ABI declared in include/b200sd.h).

There is NO fallback: if the shared object is missing or a symbol is absent, importing this module raises.
"""
import ctypes
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200sd.so")
HEADER_PATH = os.path.normpath(os.path.join(HERE, "..", "..", "include", "b200sd.h"))


class Epilogue(ctypes.Structure):
    """struct b200sd_epilogue"""
    _fields_ = [
        ("bias", ctypes.c_void_p),
        ("bias_group_rows", ctypes.c_int),
        ("residual", ctypes.c_void_p),
        ("ldr", ctypes.c_longlong),
        ("flags", ctypes.c_int),
    ]


class LoraTarget(ctypes.Structure):
    """struct b200sd_lora_target"""
    _fields_ = [
        ("W", ctypes.c_void_p),
        ("P", ctypes.c_void_p),
        ("U", ctypes.c_void_p),
        ("D", ctypes.c_void_p),
        ("ldw", ctypes.c_longlong),
        ("rows", ctypes.c_int),
        ("cols", ctypes.c_int),
        ("R", ctypes.c_int),
        ("reserved", ctypes.c_int),
    ]


EPI_GEGLU = 1
EPI_SILU = 2
EPI_LRELU = 4
F16 = 0
BF16 = 1

ERRORS = {-1: "invalid argument", -2: "CUDA runtime error", -3: "tensor-map encode failed", -4: "unsupported shape"}


class B200SDError(RuntimeError):
    pass


def declared_symbols(header: str = HEADER_PATH):
    """Every function name declared in include/b200sd.h."""
    text = open(header).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200sd_[a-z0-9_]+)\s*\(", text)))


def load(path: str = LIB_PATH) -> ctypes.CDLL:
    if not os.path.exists(path):
        raise B200SDError(
            f"{path} not found: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "There is no CPU or PyTorch fallback for the hot path.")
    lib = ctypes.CDLL(path)
    for name in declared_symbols():
        if not hasattr(lib, name):
            raise B200SDError(f"{path} does not export {name}")
    lib.b200sd_version.restype = ctypes.c_char_p
    lib.b200sd_groupnorm_stats_floats.restype = ctypes.c_longlong
    lib.b200sd_tome_match_workspace_bytes.restype = ctypes.c_longlong
    return lib


_LIB = None


def lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = load()
    return _LIB


def check(rc: int, what: str):
    if rc != 0:
        raise B200SDError(f"{what} failed: {ERRORS.get(rc, rc)} (rc={rc})")
