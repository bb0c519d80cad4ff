"""Generate the Anisotropy / Resize golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_resolution.py [case name ...]

For every case of ``tests/resolution_cases.py`` it records the JSON history, both images (label map
"seg", scalar image "t1") and their affines after the reference's transform, or the error the
reference raised (at construction or when called).  The inputs are regenerated from the case seeds.
"""

from __future__ import annotations

import json
import sys
import warnings
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "_shim"))
sys.path.insert(1, "/root/reference/src")
sys.path.insert(2, str(HERE.parent))

import torchio as tio  # noqa: E402  (the reference)

from resolution_cases import RESOLUTION_CASES, affines, label_map, scalar_image  # noqa: E402


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def _error(exc) -> dict:
    return {"history": _json([]), "error": _json({"type": type(exc).__name__, "message": str(exc)})}


def run_case(case):
    labels, t1 = label_map(case), scalar_image(case)
    subjects = []
    for b, affine in enumerate(affines(case)):
        subjects.append(tio.Subject(seg=tio.LabelMap(labels[b].clone(), affine=affine.copy()),
                                    t1=tio.ScalarImage(t1[b].clone(), affine=affine.copy())))
    batch = tio.SubjectsBatch.from_subjects(subjects)
    assert batch.images["seg"].data.dtype == case["dtype"]
    name, kwargs = case["transform"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            transform = getattr(tio, name)(**kwargs)
        except Exception as exc:  # noqa: BLE001  (the fixture records what the reference raises)
            return _error(exc)
        torch.manual_seed(case["seed"])
        try:
            out = transform(batch)
        except Exception as exc:  # noqa: BLE001
            return _error(exc)
    history = [{"name": t.name, "params": t.params} for t in out.applied_transforms]
    record = {"history": _json(history)}
    for key in ("seg", "t1"):
        record[f"out_{key}"] = out.images[key].data.contiguous().numpy()
        record[f"aff_{key}"] = np.stack([a.data.numpy() for a in out.images[key].affines])
    return record


def main():
    torch.set_num_threads(1)
    names = set(sys.argv[1:])  # optional: regenerate only these cases
    for case in RESOLUTION_CASES:
        if names and case["name"] not in names:
            continue
        path = HERE / f"{case['name']}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{case['name']:45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
