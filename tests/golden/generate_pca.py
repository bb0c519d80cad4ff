"""Generate the PCA golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_pca.py [case name ...]

For every case of ``tests/pca_cases.py`` it records the JSON history, the images after the
reference's transform (``out_<name>``, bf16 as its int16 bits) with their dtype, its ``repr`` and
``to_hydra``, the error the reference raised, and ``torch.rand(4)`` drawn right after the call (the
state of the generator).  The inputs are regenerated from the case seeds; the global torch seed is
the case seed before the call.  ``pca_compose_normalize`` runs ``Compose([Normalize(), PCA()])``.
"""

from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "_shim"))
sys.path.insert(1, "/root/reference/src")
sys.path.insert(2, str(HERE.parent))

import torchio as tio  # noqa: E402  (the reference)

from pca_cases import CASES, as_stored, images, seed  # noqa: E402


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def _error(exc) -> dict:
    return {"error": _json({"type": type(exc).__name__, "message": str(exc)})}


def run_case(case):
    inputs = images(case)
    subjects = [tio.Subject(**{k: tio.ScalarImage(v[b].clone()) for k, v in inputs.items()})
                for b in range(case["batch"])]
    batch = tio.SubjectsBatch.from_subjects(subjects)
    try:
        transform = tio.PCA(**case["kwargs"])
    except Exception as exc:  # noqa: BLE001  (the fixture records what the reference raises)
        return _error(exc)
    record = {"hydra": _json(transform.to_hydra()), "repr": _json(repr(transform))}
    if case.get("compose"):
        transform = tio.Compose([tio.Normalize(), transform])
    torch.manual_seed(seed(case))
    try:
        out = transform(batch)
    except Exception as exc:  # noqa: BLE001
        return {**record, **_error(exc), "rng_after": _json(torch.rand(4).tolist())}
    record["rng_after"] = _json(torch.rand(4).tolist())
    record["history"] = _json([{"name": t.name, "params": t.params} for t in out.applied_transforms])
    record["dtype"] = _json({k: str(out.images[k].data.dtype) for k in out.images})
    for key in out.images:
        record[f"out_{key}"] = as_stored(out.images[key].data)
    return record


def main():
    torch.set_num_threads(1)
    names = set(sys.argv[1:])  # optional: regenerate only these cases
    for name, case in CASES.items():
        if names and name not in names:
            continue
        path = HERE / f"{name}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{name:45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
