"""The C-ABI library loads and exports every symbol include/tio_b200.h
declares (no compute calls: runs without a GPU)."""

import ctypes
import re
from pathlib import Path

from torchio_b200 import _native

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    text = (ROOT / "include" / "tio_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(tio_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = _native.lib()
    declared = _declared()
    assert "tio_resample" in declared and len(declared) >= 8
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in tio_b200.h but not exported"
    assert sorted(_native.exported_symbols()) == declared


def test_abi_version_and_error_string():
    lib = _native.lib()
    assert lib.tio_abi_version() == 2
    assert isinstance(lib.tio_last_error(), bytes)


def test_bad_arguments_fail_loudly_without_touching_the_gpu():
    import pytest

    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_intensity_fused", None, None, None, 1, 1, 1, 1, 16, None, 0, 0, 0, None, 0,
                     None, None, 0, 0, None, None, None, None, None, 0, 0, 0, None, None)
    with pytest.raises(RuntimeError, match="alias"):
        buf = ctypes.create_string_buffer(64)
        p = ctypes.addressof(buf)
        sp = (ctypes.c_float * 3)(1, 1, 1)
        _native.call("tio_resample", p, p, 0, 1, 1, 2, 2, 2, 2, 2, 2, p, None, None, 0, 0, 0,
                     ctypes.addressof(sp), ctypes.addressof(sp), 1, 1, None, 0, None, 0, None)


def test_widened_entry_points_validate_before_launching():
    """tio_upload / tio_crop_patches / tio_remap: non-zero return + message, no CUDA call."""
    import pytest

    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_upload", None, None, 16, None)
    with pytest.raises(RuntimeError, match="does not fit"):
        _native.call("tio_crop_patches", p, p + 128, 4, 1, 4, 4, 4, 1, p, 8, 2, 2, None)
    with pytest.raises(RuntimeError, match="element size"):
        _native.call("tio_crop_patches", p, p + 128, 3, 1, 4, 4, 4, 1, p, 2, 2, 2, None)
    with pytest.raises(RuntimeError, match="aliased"):
        _native.call("tio_remap", p, p, 4, 1, 1, 2, 2, 2, 2, 2, 2, 0, 0, 0, 0, None, None, None)
    with pytest.raises(RuntimeError, match="mode"):
        _native.call("tio_remap", p, p + 128, 4, 1, 1, 2, 2, 2, 2, 2, 2, 0, 0, 0, 7, None, None, None)
    with pytest.raises(RuntimeError, match="reflect"):
        _native.call("tio_remap", p, p + 128, 4, 1, 1, 2, 2, 2, 6, 2, 2, 2, 0, 0, 2, None, None, None)
    # an empty upload is a no-op, not an error
    assert _native.lib().tio_upload(p, p + 128, 0, None) == 0


def test_refused_calls_launch_nothing():
    """tio_launch_count counts launches, not calls: entry points that fail their argument checks
    (or have nothing to do) leave it where it was."""
    import pytest

    lib = _native.lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    assert lib.tio_launch_count.restype is ctypes.c_uint64
    before = lib.tio_launch_count()
    assert isinstance(before, int) and before >= 0
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_upload", None, None, 16, None)
    with pytest.raises(RuntimeError, match="does not fit"):
        _native.call("tio_crop_patches", p, p + 128, 4, 1, 4, 4, 4, 1, p, 8, 2, 2, None)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_intensity_fused", None, None, None, 1, 1, 1, 1, 16, None, 0, 0, 0, None, 0,
                     None, None, 0, 0, None, None, None, None, None, 0, 0, 0, None, None)
    assert lib.tio_upload(p, p + 128, 0, None) == 0
    assert lib.tio_launch_count() == before
