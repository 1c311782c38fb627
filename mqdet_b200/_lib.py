"""ctypes binding of libmqdet_b200.so (the C-ABI boundary, see include/mqdet_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` (``make -C mqdet_b200/csrc``).  There is no
CPU or PyTorch fallback: if the shared object is missing, loading raises.
"""
import ctypes
import os
import re
from ctypes import c_char_p, c_float, c_int, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libmqdet_b200.so")

F16, F32 = 0, 1
ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
VEC_NONE, VEC_SCALAR, VEC_PER_COL, VEC_PER_ROW = 0, 1, 2, 3
IMPL_TC, IMPL_SIMT, IMPL_TC_ONESHOT = 0, 1, 2


class GemmArgs(ctypes.Structure):
    """Mirror of ``mqdet_gemm_args`` (include/mqdet_b200.h)."""

    _fields_ = [
        ("A", c_void_p), ("B", c_void_p),
        ("M", c_int64), ("N", c_int64), ("K", c_int64),
        ("lda", c_int64), ("ldb", c_int64),
        ("nb1", c_int64), ("nb2", c_int64),
        ("a_b1", c_int64), ("a_b2", c_int64), ("b_b1", c_int64), ("b_b2", c_int64),
        ("C", c_void_p), ("c_dtype", c_int32),
        ("ldc", c_int64), ("c_b1", c_int64), ("c_b2", c_int64),
        ("alpha", c_float), ("scale_after_bias", c_int32),
        ("bias", c_void_p), ("bias_mode", c_int32), ("bias_b1", c_int64), ("bias_b2", c_int64),
        ("act", c_int32), ("clamp", c_float),
        ("gate", c_void_p), ("gate_mode", c_int32), ("gate_tanh", c_int32),
        ("R", c_void_p), ("r_dtype", c_int32), ("ldr", c_int64), ("r_b1", c_int64), ("r_b2", c_int64),
    ]


_HEADER = os.path.join(_HERE, os.pardir, "include", "mqdet_b200.h")
_SCALAR_TYPES = {"int": c_int, "int32_t": c_int32, "int64_t": c_int64, "float": c_float}


class MqdetError(RuntimeError):
    """Raised when a C-ABI call returns a negative code (mirrors the reference's AT_ERROR -> RuntimeError)."""


def _ctype(symbol, decl, is_return):
    """ctypes type of one header type: the scalar table, ``const char*`` returns as ``c_char_p``, every other pointer as
    ``c_void_p`` (it also takes ``byref(...)`` and ctypes arrays), ``void`` returns as None.  Anything else raises."""
    t = " ".join(decl.replace("*", " * ").split())
    if "*" in t:
        return c_char_p if is_return and t == "const char *" else c_void_p
    if is_return and t == "void":
        return None
    if t in _SCALAR_TYPES:
        return _SCALAR_TYPES[t]
    raise MqdetError(f"{symbol}: header type {decl.strip()!r} has no ctypes binding")


def parse_header(src):
    """The ``mqdet_*`` declarations of a C header -> {name: (restype, argtypes)}."""
    src = re.sub(r"/\*.*?\*/", " ", src, flags=re.S)
    src = re.sub(r"^\s*#.*$", " ", src, flags=re.M)
    src = re.sub(r"typedef\s+struct\s+\w+\s*\{.*?\}\s*\w+\s*;", " ", src, flags=re.S)
    src = re.sub(r'extern\s+"C"\s*\{|^\s*\}\s*$', " ", src, flags=re.M)
    sigs = {}
    for decl in filter(None, (" ".join(d.split()) for d in src.split(";"))):
        m = re.fullmatch(r"(.+?)\b(mqdet_\w+)\s*\((.*)\)", decl)
        if m is None:
            raise MqdetError(f"cannot bind header declaration {decl!r}")
        ret, name, params = m.groups()
        params = [] if params.strip() in ("", "void") else params.split(",")
        sigs[name] = (_ctype(name, ret, True), [_ctype(name, re.sub(r"\w+\s*$", "", p), False) for p in params])
    return sigs


# name -> (restype, argtypes) of every entry point include/mqdet_b200.h declares
with open(_HEADER) as _f:
    SIGNATURES = parse_header(_f.read())

_lib = None

# tools/breakdown.py sets this to a list: every launch through ops is then bracketed by CUDA events -> (symbol, e0, e1)
CALL_PROFILE = None


def load():
    """Load the shared library and bind every declared symbol (raises if the build is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MqdetError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(there is no CPU / PyTorch fallback for the mqdet_b200 hot path)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc, what=""):
    if rc != 0:
        msg = load().mqdet_last_error()
        raise MqdetError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")
