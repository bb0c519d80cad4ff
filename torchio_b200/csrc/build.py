"""Build libtio_b200.so in-tree with nvcc for sm_90a (no JIT cache, no torch headers).

    python torchio_b200/csrc/build.py [--force] [--verbose]

The shared library exports exactly the C-ABI of include/tio_b200.h and is
loaded with ctypes by torchio_b200/_native.py.  nvcc cross-compiles without a
GPU.
"""

from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
SOURCES = ["error.cu", "resample.cu", "resample_tile.cu", "resample_fast.cu", "upload.cu", "fused_intensity.cu",
           "mt19937_jump.cpp", "mt19937.cu", "patches.cu", "stats.cu", "labels.cu", "labels_to_image.cu",
           "label_maps.cu", "interpolate.cu"]
HEADERS = [HERE / "common.cuh", HERE / "resample_common.cuh", HERE / "resample_tile.cuh", HERE / "tma.cuh",
           HERE / "mt19937_layout.h", HERE / "label_lookup.cuh", HERE / "image_dtype.cuh",
           ROOT / "include" / "tio_b200.h",
           Path(__file__).resolve()]  # the flags below: objects built for another architecture are rebuilt
OBJ = HERE / "_obj"
OUT = HERE / "libtio_b200.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *ARCH,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def needs_build() -> bool:
    if not OUT.exists():
        return True
    newest = max(p.stat().st_mtime for p in [*(HERE / s for s in SOURCES), *HEADERS])
    return OUT.stat().st_mtime < newest


def _compile(source: str) -> tuple[str, int, str]:
    """One translation unit -> object file (recompiled only when it or a header changed)."""
    src = HERE / source
    obj = OBJ / (Path(source).stem + ".o")
    newest = max(p.stat().st_mtime for p in [src, *HEADERS])
    if obj.exists() and obj.stat().st_mtime >= newest:
        return source, 0, ""
    proc = subprocess.run(["nvcc", *NVCC_FLAGS, "-c", str(src), "-o", str(obj)],
                          capture_output=True, text=True)
    return source, proc.returncode, proc.stdout + proc.stderr


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return OUT
    OBJ.mkdir(exist_ok=True)
    if force:
        for stale in OBJ.glob("*.o"):
            stale.unlink()
    # the translation units are independent: compile them side by side, then link
    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 1)) as pool:
        results = list(pool.map(_compile, SOURCES))
    log = "".join(f"==== {name}\n{text}" for name, _, text in results)
    failed = [name for name, code, _ in results if code != 0]
    if verbose or failed:
        sys.stderr.write(log)
    if failed:
        raise RuntimeError(f"nvcc failed for {failed}")
    objects = [str(OBJ / (Path(s).stem + ".o")) for s in SOURCES]
    proc = subprocess.run(["nvcc", *ARCH, "-shared", "-o", str(OUT),
                           *objects], capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        raise RuntimeError(f"nvcc link failed with exit code {proc.returncode}")
    previous = (HERE / "ptxas.log").read_text() if (HERE / "ptxas.log").exists() and not force else ""
    (HERE / "ptxas.log").write_text(log if all(t for _, _, t in results) else previous + log)
    return OUT


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
