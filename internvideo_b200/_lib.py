"""ctypes binding of libivb200.so (the C ABI in include/ivb200.h).

The header is the only declaration of the ABI: load() attaches the prototypes parse_prototypes() reads from it.
There is no fallback: if the shared library is missing, or a compute entry point is called without an H100-class
(sm_90) device, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libivb200.so"
HEADER = _PKG.parent / "include" / "ivb200.h"

_SCALARS = {"int": C.c_int, "long": C.c_long, "float": C.c_float, "void": None}


def _ctype(decl: str, ret: bool = False):
    """ctypes type of a C return type, or of a parameter declaration (type and name).  Every pointer is c_void_p, except
    a `const char*` return (c_char_p); a scalar type the binding does not know raises."""
    if "*" in decl:
        return C.c_char_p if ret and "".join(decl.split()) == "constchar*" else C.c_void_p
    words = [w for w in decl.split() if w != "const"]
    base = " ".join(words if ret else words[:-1])
    if base not in _SCALARS:
        raise ValueError(f"unknown C type in {decl!r}")
    return _SCALARS[base]


def parse_prototypes(header: str) -> dict:
    """{name: (restype, argtypes)} for every ivb_* function declared in the C header text."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", "", header, flags=re.S)
    text = re.sub(r"^\s*#[^\n]*", "", text, flags=re.M)
    protos = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\s*\b(ivb_\w+)\s*\(([^()]*)\)\s*;", text):
        params = " ".join(params.split())
        args = [] if params in ("", "void") else [_ctype(p) for p in params.split(",")]
        protos[name] = (_ctype(ret, ret=True), args)
    return protos


PROTOTYPES = parse_prototypes(HEADER.read_text())

_lib = None


class IvbError(RuntimeError):
    pass


def load(build_if_missing: bool = False) -> C.CDLL:
    """Load libivb200.so and attach prototypes. Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        if build_if_missing or os.environ.get("IVB200_AUTOBUILD") == "1":
            from . import build as _b
            _b.build()
        else:
            raise IvbError(
                f"{LIB_PATH} not found: build it with `python -m internvideo_b200.build` "
                "(there is no CPU / PyTorch fallback for the ivb200 compute path)")
    lib = C.CDLL(str(LIB_PATH))
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().ivb_last_error().decode(errors="replace")
        raise IvbError(f"{what} failed (rc={rc}): {msg}")


def header_symbols() -> list[str]:
    """Function names declared in include/ivb200.h (used by the CPU ABI test)."""
    text = re.sub(r"/\*.*?\*/", "", HEADER.read_text(), flags=re.S)
    return sorted(set(re.findall(r"\b(ivb_[a-z0-9_]+)\s*\(", text)))
