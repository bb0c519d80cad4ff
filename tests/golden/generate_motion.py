"""Generate the Motion golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_motion.py [case name ...]

For every case of ``tests/motion_cases.py`` it records the JSON history, the images after the
reference's transform (scalar image "t1" and, when the case has one, label map "seg") with the
output dtype, the reference's ``_affine_matrices`` of every segment of the recorded params
(``theta``, (N, B, 3, 4)), its ``repr`` and ``to_hydra``, the warnings its constructor and its call issued, or
the error the reference raised.  A ``compose`` case runs the reference's
``Compose([Motion, Ghosting, BiasField])``.  The inputs are regenerated from the case seeds; the
global torch seed is the case seed before the call.
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
from torchio.transforms.intensity import motion as reference_motion  # noqa: E402

from motion_cases import CASES, as_stored, label_map, scalar_image, seed  # noqa: E402


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def _error(exc) -> dict:
    return {"error": _json({"type": type(exc).__name__, "message": str(exc)})}


def _transform(case):
    motion = tio.Motion(**case["kwargs"])
    if not case.get("compose"):
        return motion, motion
    return tio.Compose([motion, tio.Ghosting(**case["ghosting"]), tio.BiasField(**case["bias"])]), motion


def _theta(params, batch_size, shape) -> np.ndarray:
    if "_batched_keys" in params:
        n = reference_motion._num_motion_transforms(params["transforms"])
        segments = [reference_motion._per_instance_motion_parameters(params["transforms"], s, "cpu") for s in range(n)]
    else:
        segments = [reference_motion._shared_motion_parameters(t, batch_size, "cpu") for t in params["transforms"]]
    return torch.stack([reference_motion._affine_matrices(d, t, list(shape)) for d, t in segments]).numpy()


def run_case(case):
    t1, seg = scalar_image(case), label_map(case)
    subjects = []
    for b in range(case["batch"]):
        images = {"t1": tio.ScalarImage(t1[b].clone())}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b].clone())
        subjects.append(tio.Subject(**images))
    batch = tio.SubjectsBatch.from_subjects(subjects)
    try:
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            transform, motion = _transform(case)
    except Exception as exc:  # noqa: BLE001  (the fixture records what the reference raises)
        return _error(exc)
    record = {"hydra": _json(motion.to_hydra()), "repr": _json(repr(motion))}
    init_caught = caught
    torch.manual_seed(seed(case))
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        try:
            out = transform(batch)
        except Exception as exc:  # noqa: BLE001
            return {**record, **_error(exc)}
    record["init_warnings"] = _json([str(w.message) for w in init_caught])
    record["warnings"] = _json([str(w.message) for w in caught])
    record["history"] = _json([{"name": t.name, "params": t.params} for t in out.applied_transforms])
    record["dtype"] = _json(str(out.images["t1"].data.dtype))
    for t in out.applied_transforms:
        if t.name == "Motion":
            record["theta"] = _theta(t.params, case["batch"], case["shape"])
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
