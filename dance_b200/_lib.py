"""ctypes binding of ``libdance_b200.so`` (the C-ABI declared in ``include/dance_b200.h``).

There is no CPU fallback: if the shared library is missing, :func:`lib` raises and tells
the user to run ``python -m dance_b200.build``.  Tensors cross the boundary as raw
device pointers + sizes; the CUDA stream is torch's current stream.

Every function's restype and argtypes are read from the header when the library loads, so
the binding cannot drift from the declarations.
"""
from __future__ import annotations

import ctypes as C
import re
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libdance_b200.so"
_HEADER = Path(__file__).resolve().parent.parent / "include" / "dance_b200.h"
_lib = None

_SCALARS = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint32_t": C.c_uint32, "float": C.c_float,
            "double": C.c_double, "size_t": C.c_size_t}
_DECL = re.compile(r"((?:const\s+)?\w+(?:\s*\*)*)\s*\b(b2_\w+)\s*\(([^()]*)\)")


class B2Error(RuntimeError):
    """A C-ABI call returned a negative status."""


def _ctype(decl: str, where: str, ret: bool = False):
    """ctypes type of a C type: any pointer is c_void_p (a returned ``const char*`` is c_char_p), scalars map by name."""
    if "*" in decl:
        return C.c_char_p if ret and decl.replace(" ", "") == "constchar*" else C.c_void_p
    words = [w for w in decl.split() if w != "const"]
    if ret and words == ["void"]:
        return None
    if len(words) != 1 or words[0] not in _SCALARS:
        raise B2Error(f"{where}: no ctypes mapping for C type {decl!r}")
    return _SCALARS[words[0]]


def parse_header(text: str):
    """{name: (restype, argtypes)} of every function declared in C header text.  Comments and preprocessor lines are
    dropped, the rest is split into declarations at ';'; a declaration that is neither a typedef nor a b2_ function, or
    a type without a ctypes mapping, raises."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    text = re.sub(r"^\s*#.*$", " ", text, flags=re.M)
    text = text.replace('extern "C" {', " ").replace("}", " ")
    sigs = {}
    for decl in (d.strip() for d in text.split(";")):
        if not decl or decl.startswith("typedef "):
            continue
        m = _DECL.fullmatch(decl)
        if m is None:
            raise B2Error(f"cannot bind declaration {' '.join(decl.split())!r}")
        ret, name, params = m.groups()
        args = []
        for p in ([] if params.strip() == "void" else params.split(",")):
            p = p.strip()
            end = p.rfind("*") + 1 or p.rfind(" ")      # the type ends at its last '*', else before the parameter's name
            if end <= 0:
                raise B2Error(f"{name}: parameter {p!r} has no name")
            args.append(_ctype(p[:end], f"{name}: parameter {p!r}"))
        sigs[name] = (_ctype(ret, name, ret=True), args)
    return sigs


def lib_path() -> Path:
    return _LIB_PATH


def declared_symbols():
    return sorted(parse_header(_HEADER.read_text()))


def lib():
    """Return the loaded shared library (loads it on first use; no fallback if absent)."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise B2Error(f"{_LIB_PATH} not found: build the CUDA extension first with "
                          "`python -m dance_b200.build` (there is no CPU fallback).")
        handle = C.CDLL(str(_LIB_PATH))
        for name, (res, args) in parse_header(_HEADER.read_text()).items():
            fn = getattr(handle, name)
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(status: int, what: str = ""):
    if status != 0:
        msg = lib().b2_last_error().decode("utf-8", "replace")
        raise B2Error(f"{what or 'dance_b200'} failed with status {status}: {msg}")
