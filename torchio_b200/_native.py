"""ctypes binding of the C-ABI library, bound from its header.

The library is built in-tree by ``__graft_entry__.build()`` /
``torchio_b200/csrc/build.py`` (nvcc, sm_90a) and loaded from
``torchio_b200/csrc/libtio_b200.so``.  Every function's argument and return types are read from
``include/tio_b200.h``, which travels with the tree, so the header is the one statement of the ABI.
There is no fallback: if the library is missing or a call fails, a RuntimeError carrying
``tio_last_error()`` is raised.
"""

from __future__ import annotations

import ctypes
import functools
import re
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_uint64, c_void_p
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "csrc" / "libtio_b200.so"
HEADER_PATH = Path(__file__).resolve().parent.parent / "include" / "tio_b200.h"

_SCALARS = {"int": c_int, "int64_t": c_int64, "uint64_t": c_uint64, "size_t": c_size_t, "float": c_float}
_PROTOTYPE = re.compile(r"^[ \t]*([\w ]+?\**)[ \t]*\b(tio_\w+)\s*\(([^)]*)\)\s*;", re.M)


def _ctype(spelling: str, *, result: bool = False):
    """The ctypes type of a C type as the header spells it; raises on one it does not map, so that no
    function is left with ctypes' default int conversions."""
    spelling = re.sub(r"\s*\*", "*", " ".join(spelling.split()))
    if result and spelling == "const char*":
        return c_char_p
    if "*" in spelling and not result:
        return c_void_p
    ctype = _SCALARS.get(spelling.removeprefix("const "))
    if ctype is None:
        raise RuntimeError(f"torchio_b200: {HEADER_PATH.name} uses a C type the binding does not map: {spelling!r}")
    return ctype


@functools.cache
def prototypes() -> dict[str, tuple[type, list[type]]]:
    """name -> (restype, argtypes) of every function declared in include/tio_b200.h."""
    text = re.sub(r"/\*.*?\*/", "", HEADER_PATH.read_text(), flags=re.S)
    out = {}
    for restype, name, params in _PROTOTYPE.findall(text):
        params = " ".join(params.split())
        argtypes = [] if params in ("", "void") else [
            _ctype(re.sub(r"\s*\b\w+$", "", p.strip())) for p in params.split(",")]
        out[name] = (_ctype(restype, result=True), argtypes)
    declared = re.findall(r"\btio_\w+\s*\(", text)
    if len(declared) != len(out):
        raise RuntimeError(f"torchio_b200: {HEADER_PATH.name} declares {len(declared)} functions, but only"
                           f" {len(out)} prototypes could be parsed")
    return out


_lib = None


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(
                f"torchio_b200: CUDA library not built ({LIB_PATH} is missing)."
                " Run `python -c 'import __graft_entry__ as g; g.build()'` at the"
                " repo root (needs nvcc). There is no CPU fallback."
            )
        handle = ctypes.CDLL(str(LIB_PATH))
        for name, (restype, argtypes) in prototypes().items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = restype, argtypes
        _lib = handle
    return _lib


def exported_symbols() -> list[str]:
    return list(prototypes())


def call(name: str, *args) -> None:
    handle = lib()
    rc = getattr(handle, name)(*args)
    if rc != 0:
        msg = handle.tio_last_error().decode(errors="replace")
        raise RuntimeError(f"{name} failed (code {rc}): {msg}")
