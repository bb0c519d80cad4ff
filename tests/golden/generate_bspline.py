"""Generate the B-spline (orders 2-7) golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_bspline.py [case name ...]

The reference imports ``interpol`` for orders 2-7.  ``torch-interpol`` is not vendored, so this
generator (and only it) installs the float64 restatement of ``tests/bspline_cases.py`` under that
name; its three assumptions about torch-interpol are listed there.  For every case it records the
JSON history, the output images "t1" (and "seg" when the case has one) with their dtypes, and the
output affines.  The inputs are regenerated from the case seeds; the global torch seed is the case
seed before the call.
"""

from __future__ import annotations

import json
import sys
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "_shim"))
sys.path.insert(1, "/root/reference/src")
sys.path.insert(2, str(HERE.parent))

import bspline_cases as bc  # noqa: E402

sys.modules["interpol"] = types.SimpleNamespace(grid_pull=bc.grid_pull)

import torchio as tio  # noqa: E402  (the reference)


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def run_case(case):
    t1, seg = bc.scalar_image(case), bc.label_map(case)
    subjects = []
    for b in range(bc.BATCH):
        images = {"t1": tio.ScalarImage(t1[b].clone())}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b].clone())
        subjects.append(tio.Subject(**images))
    batch = tio.SubjectsBatch.from_subjects(subjects)
    transform = getattr(tio, case["transform"])(**case["kwargs"])
    torch.manual_seed(bc.seed(case))
    out = transform(batch)
    record = {"history": _json([{"name": t.name, "params": t.params} for t in out.applied_transforms])}
    for key in out.images:
        data = out.images[key].data
        record[f"dtype_{key}"] = _json(str(data.dtype))
        record[f"out_{key}"] = data.numpy()
        record[f"affines_{key}"] = np.stack([np.asarray(a.numpy(), dtype=np.float64)
                                             for a in out.images[key].affines])
    return record


def main():
    torch.set_num_threads(1)
    names = set(sys.argv[1:])
    for name, case in bc.CASES.items():
        if names and name not in names:
            continue
        path = HERE / f"{name}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{name:45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
