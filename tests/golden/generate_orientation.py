"""Generate the Reorient / Transpose / EnsureShapeMultiple / CopyAffine / ToReferenceSpace golden vectors
by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs), except
that ``nibabel.orientations`` is ``nibabel_orientations.py`` beside this file, a restatement of
nibabel's algorithms, since Reorient reads real orientations:

    python tests/golden/generate_orientation.py [case name ...]

For every case of ``tests/orientation_cases.py`` it records the JSON history (name, params, include,
exclude), every image and its per-element affines after the reference's transform, its ``repr``
and ``to_hydra`` (not for ToReferenceSpace, whose argument is an image), or the error the reference
raised.  The inputs are regenerated from the case seeds; the global torch seed is the case seed
before the call.  One more file holds ``ToReferenceSpace.from_tensor``'s affine.
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

import importlib.util  # noqa: E402

import nibabel  # noqa: E402  (the _shim/ stub)

_spec = importlib.util.spec_from_file_location("nibabel.orientations", HERE / "nibabel_orientations.py")
_orientations = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_orientations)
sys.modules["nibabel.orientations"] = nibabel.orientations = _orientations

import torchio as tio  # noqa: E402  (the reference)

import orientation_cases as oc  # noqa: E402


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def _error(exc) -> dict:
    return {"error": _json({"type": type(exc).__name__, "message": str(exc)})}


def _affine(a) -> np.ndarray:
    m = a.numpy() if hasattr(a, "numpy") else a
    return np.asarray(m._matrix if hasattr(m, "_matrix") else m, dtype=np.float64)


def run_case(case):
    images = oc.inputs(case)
    try:
        transform = oc.transform(case, tio)
    except Exception as exc:  # noqa: BLE001  (the fixture records what the reference raises)
        return _error(exc)
    record = {}
    if case["kind"] != "ToReferenceSpace":
        record = {"hydra": _json(transform.to_hydra()), "repr": _json(repr(transform))}
    batch = oc.batch(case, images, tio)
    torch.manual_seed(oc.seed(case))
    try:
        if case.get("subject"):
            out = transform(batch.unbatch()[0])
            result = {k: (out[k].data[None], [out[k].affine]) for k in images}
            history = out.applied_transforms
        else:
            out = transform(batch)
            result = {k: (ib.data, ib.affines) for k, ib in out.images.items()}
            history = out.applied_transforms
    except Exception as exc:  # noqa: BLE001
        return {**record, **_error(exc)}
    record["history"] = _json([{"name": t.name, "params": t.params, "include": t.include, "exclude": t.exclude}
                               for t in history])
    for key, (data, affines) in result.items():
        record[f"out_{key}"] = oc.as_stored(data)
        record[f"affine_{key}"] = np.stack([_affine(a.data if hasattr(a, "data") else a) for a in affines])
    return record


def main():
    torch.set_num_threads(1)
    names = set(sys.argv[1:])  # optional: regenerate only these cases
    for name, case in oc.CASES.items():
        if names and name not in names:
            continue
        path = HERE / f"orientation_{name}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{name:45s} {path.stat().st_size / 1024:8.1f} KiB")
    if not names or "to_reference_space_from_tensor" in names:
        image = tio.ToReferenceSpace.from_tensor(torch.zeros(8, 5, 6, 7), oc.reference_image(tio))
        path = HERE / "orientation_to_reference_space_from_tensor.npz"
        np.savez_compressed(path, affine=_affine(image.affine.data))
        print(f"{'to_reference_space_from_tensor':45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
