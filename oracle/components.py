"""CPU oracle for KeepLargestComponent (Python side): drive ``oracle/c/components.c``.

TEST INFRASTRUCTURE — NOT PRODUCT CODE: used by tests/ and tools/ only; torchio_b200 never imports
it.  The C side is a sequential scan-order union-find written from the definition of connectivity
(equal values, 6 or 26 neighbours, root = the smallest C-order index of a component).
"""

from __future__ import annotations

import ctypes
import subprocess
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
SRC = HERE / "c" / "components.c"
LIB = HERE / "_build" / "libcomponents_oracle.so"

_DTYPES = {
    torch.float32: 0, torch.uint8: 1, torch.int8: 2,
    torch.int16: 3, torch.int32: 4, torch.int64: 5,
}


def build(force: bool = False) -> Path:
    """Compile the C oracle (gcc)."""
    if LIB.exists() and not force and LIB.stat().st_mtime >= SRC.stat().st_mtime:
        return LIB
    LIB.parent.mkdir(exist_ok=True)
    subprocess.run(["gcc", "-O2", "-fPIC", "-shared", "-o", str(LIB), str(SRC)], check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(str(build()))
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _roots(raw: torch.Tensor) -> torch.Tensor:
    """uint32 roots held in int32 -> int64, -1 for a voxel that takes no part."""
    roots = raw.to(torch.int64) & 0xFFFFFFFF
    return torch.where(roots == 0xFFFFFFFF, torch.full_like(roots, -1), roots)


def connected_components(values: torch.Tensor, part: torch.Tensor, fully_connected: bool) -> torch.Tensor:
    """(I, J, K) CPU map and its mask of voxels that take part -> (I, J, K) int64: the smallest C-order
    index of each voxel's component (equal values, 26 or 6 neighbours), -1 outside the mask."""
    values = values.contiguous()
    mask = part.to(torch.uint8).contiguous()
    raw = torch.empty(values.shape, dtype=torch.int32)
    rc = lib().orc_connected_components(_p(values), _DTYPES[values.dtype], *values.shape, _p(mask),
                                        int(bool(fully_connected)), _p(raw))
    assert rc == 0
    return _roots(raw)


def keep_largest(data: torch.Tensor, part: torch.Tensor, fully_connected: bool, fill: torch.Tensor):
    """(B, I, J, K) CPU map -> (map with every component but the largest of each value overwritten by
    the one-element ``fill``, ties to the smallest root; (B, I, J, K) int64 roots as
    `connected_components`)."""
    out = data.clone().contiguous()
    mask = part.to(torch.uint8).contiguous()
    fill = fill.to(data.dtype).reshape(1).contiguous()
    raw = torch.empty(out.shape, dtype=torch.int32)
    rc = lib().orc_keep_largest(_p(out), _DTYPES[out.dtype], *out.shape, _p(mask), int(bool(fully_connected)),
                                _p(fill), _p(raw))
    assert rc == 0
    return out, _roots(raw)
