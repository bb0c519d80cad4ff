"""Generate the KeepLargestComponent golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_keep_largest.py

The reference hands connected components to SimpleITK, which the shim only stubs for I/O; before the
reference runs, ``GetImageFromArray``, ``ConnectedComponent``, ``RelabelComponent`` and
``GetArrayFromImage`` of the shim module are set to the scipy restatement of
``tests/keep_largest_cases.py`` (``SitkRestatement``, which states its tie-rule assumption).  For every
case it records the JSON history, the label map and the (untouched) scalar image after the
reference's transforms, or the error the reference raised.  The inputs are regenerated from the case
seeds.
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
sys.path.insert(3, str(HERE.parent.parent))

import SimpleITK  # noqa: E402  (the shim)

from keep_largest_cases import CASES, SitkRestatement, affines, label_map, scalar_image  # noqa: E402

_restated = SitkRestatement()
for _name in ("GetImageFromArray", "ConnectedComponent", "RelabelComponent", "GetArrayFromImage"):
    setattr(SimpleITK, _name, getattr(_restated, _name))

import torchio as tio  # noqa: E402  (the reference)


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def run_case(case):
    labels, t1 = label_map(case), scalar_image(case)
    subjects = []
    for b, affine in enumerate(affines(case)):
        subjects.append(tio.Subject(seg=tio.LabelMap(labels[b].clone(), affine=affine.copy()),
                                    t1=tio.ScalarImage(t1[b].clone(), affine=affine.copy())))
    batch = tio.SubjectsBatch.from_subjects(subjects)
    assert batch.images["seg"].data.dtype == case["dtype"]
    children = [getattr(tio, name)(**kwargs) for name, kwargs in case["transforms"]]
    transform = children[0] if len(children) == 1 else tio.Compose(children)
    torch.manual_seed(case["seed"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        try:
            out = transform(batch)
        except Exception as exc:  # noqa: BLE001  (the fixture records what the reference raises)
            return {"history": _json([]), "error": _json({"type": type(exc).__name__, "message": str(exc)})}
    history = [{"name": t.name, "params": t.params} for t in out.applied_transforms]
    return {
        "out_seg": out.images["seg"].data.contiguous().numpy(),
        "out_t1": out.images["t1"].data.contiguous().numpy(),
        "history": _json(history),
    }


def main():
    torch.set_num_threads(1)
    for case in CASES:
        path = HERE / f"{case['name']}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{case['name']:45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
