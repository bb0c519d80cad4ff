"""ctypes binding of the C-ABI library (include/tio_b200.h).

The library is built in-tree by ``__graft_entry__.build()`` /
``torchio_b200/csrc/build.py`` (nvcc, sm_90a) and loaded from
``torchio_b200/csrc/libtio_b200.so``.  There is no fallback: if the library is
missing or a call fails, a RuntimeError carrying ``tio_last_error()`` is raised.
"""

from __future__ import annotations

import ctypes
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_uint64, c_void_p
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "csrc" / "libtio_b200.so"

# name -> argtypes  (every entry point of include/tio_b200.h that returns int or size_t; lib() binds
# tio_last_error and tio_launch_count itself)
_SIGNATURES = {
    "tio_abi_version": [],
    "tio_resample": [c_void_p, c_void_p, c_int] + [c_int] * 8
    + [c_void_p, c_void_p, c_void_p] + [c_int] * 3
    + [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_size_t, c_void_p],
    "tio_resample_workspace_bytes": [c_int, c_int, c_int, c_int],
    "tio_min_sample0": [c_void_p, c_int, c_int64, c_void_p, c_void_p],
    "tio_upload": [c_void_p, c_void_p, c_size_t, c_void_p],
    "tio_remap": [c_void_p, c_void_p, c_int] + [c_int] * 8 + [c_int] * 3 + [c_int, c_void_p, c_void_p, c_void_p],
    "tio_crop_patches": [c_void_p, c_void_p, c_int] + [c_int] * 5 + [c_void_p, c_int, c_int, c_int, c_void_p],
    "tio_blur": [c_void_p, c_void_p, c_void_p] + [c_int] * 5
    + [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p],
    "tio_moments": [c_void_p, c_void_p, c_int64, c_void_p, c_void_p],
    "tio_quantiles_workspace_bytes": [],
    "tio_quantiles": [c_void_p, c_void_p, c_int64, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                      c_size_t, c_void_p],
    "tio_quantiles_batched_workspace_bytes": [c_int, c_int],
    "tio_quantiles_batched": [c_void_p, c_int, c_void_p, c_int, c_int64, c_void_p, c_int, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    "tio_histogram_tables": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p],
    "tio_histogram_map": [c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p, c_int, c_void_p],
    "tio_rescale": [c_void_p, c_void_p, c_int, c_int64, c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                    c_void_p, c_int, c_void_p],
    "tio_onehot": [c_void_p, c_int, c_int, c_int64, c_void_p, c_int, c_void_p, c_void_p],
    "tio_label_argmax": [c_void_p, c_int, c_int, c_int64, c_void_p, c_float, c_void_p, c_int, c_void_p],
    "tio_mt19937_table_bytes": [],
    "tio_mt19937_build_table": [c_void_p, c_size_t],
    "tio_randn_mt19937_workspace_bytes": [c_uint64, c_uint64],
    "tio_randn_mt19937": [c_uint64, c_uint64, c_uint64, c_void_p, c_void_p, c_void_p, c_size_t,
                          c_void_p],
    "tio_intensity_fused": [c_void_p, c_void_p, c_void_p] + [c_int] * 5
    + [c_void_p, c_int, c_int, c_int, c_void_p, c_int]
    + [c_void_p, c_void_p, c_int, c_int]
    + [c_void_p] * 5 + [c_uint64, c_int, c_int, c_void_p, c_void_p],
    "tio_intensity_pass1_with_normals_workspace_bytes": [c_uint64, c_uint64],
    "tio_intensity_pass1_with_normals": [c_void_p, c_void_p] + [c_int] * 5
    + [c_void_p, c_int, c_int, c_int, c_void_p, c_int]
    + [c_void_p, c_void_p, c_int, c_int]
    + [c_uint64, c_uint64, c_uint64, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p],
    "tio_labels_to_image": [c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                            c_uint64, c_int, c_void_p, c_void_p],
    "tio_label_lut": [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_int, c_int, c_void_p],
    "tio_label_contour": [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "tio_onehot_classes": [c_void_p, c_int, c_int, c_int, c_int64, c_int, c_void_p, c_void_p],
    "tio_label_range": [c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p],
    "tio_channel_argmax": [c_void_p, c_int, c_int, c_int, c_int64, c_void_p, c_void_p],
    "tio_interpolate": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p,
                        c_void_p, c_int, c_void_p],
    "tio_axis_resample": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                          c_void_p, c_void_p, c_int, c_int, c_void_p],
    "tio_clamp": [c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p],
    "tio_mask": [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int64,
                 c_void_p, c_void_p],
    "tio_swap_patches": [c_void_p] + [c_int] * 9 + [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "tio_components": [c_void_p] + [c_int] * 6 + [c_void_p, c_int, c_int64, c_int, c_int] + [c_void_p] * 4,
    "tio_component_roots": [c_void_p, c_int, c_int, c_int64] + [c_void_p] * 4,
    "tio_keep_largest": [c_void_p, c_int, c_int, c_int64, c_int, c_void_p, c_int, c_int64, c_int] + [c_void_p] * 5,
    "tio_permute": [c_void_p, c_void_p] + [c_int] * 10 + [c_void_p],
    "tio_spike_stats_workspace_bytes": [c_int],
    "tio_spike_stats": [c_void_p, c_int, c_int, c_int, c_int64] + [c_void_p] * 4 + [c_size_t, c_void_p],
    "tio_spectrum_peak": [c_void_p] + [c_int] * 6 + [c_void_p] * 4 + [c_size_t, c_void_p],
    "tio_spike": [c_void_p] + [c_int] * 6 + [c_void_p, c_int] + [c_void_p] * 5 + [c_size_t, c_void_p],
    "tio_ghosting": [c_void_p] + [c_int] * 6 + [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p],
    "tio_motion": [c_void_p, c_void_p] + [c_int] * 7 + [c_void_p] * 4,
    "tio_aggregate_patches": [c_void_p] * 3 + [c_int] * 11 + [c_void_p] * 4,
    "tio_aggregate_finish": [c_void_p] * 3 + [c_int, c_int, c_int64, c_void_p],
}

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
        handle.tio_last_error.restype = c_char_p
        handle.tio_last_error.argtypes = []
        handle.tio_launch_count.restype = c_uint64
        handle.tio_launch_count.argtypes = []
        for name, argtypes in _SIGNATURES.items():
            fn = getattr(handle, name)
            fn.argtypes = argtypes
            fn.restype = c_size_t if name.endswith("_bytes") else c_int
        _lib = handle
    return _lib


def exported_symbols() -> list[str]:
    return ["tio_last_error", "tio_launch_count", *_SIGNATURES]


def call(name: str, *args) -> None:
    handle = lib()
    rc = getattr(handle, name)(*args)
    if rc != 0:
        msg = handle.tio_last_error().decode(errors="replace")
        raise RuntimeError(f"{name} failed (code {rc}): {msg}")
