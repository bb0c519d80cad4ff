"""Generate the HistogramStandardization golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_histogram.py [case name ...]

For every case of ``tests/histogram_cases.py`` it records the JSON history, both images (scalar
image "t1", label map "seg") after the reference's transform, its ``repr`` and ``to_hydra``, or the
error the reference raised; for every landmark case the result of compute_histogram_landmarks or
its error.  The inputs are regenerated from the case seeds.
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
from torchio.transforms.intensity.histogram_standardization import compute_histogram_landmarks  # noqa: E402

from histogram_cases import (HIST_CASES, LANDMARK_CASES, case_cutoff, label_map, landmarks,  # noqa: E402
                             positive_mask, scalar_image, training_images)


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def _error(exc) -> dict:
    return {"error": _json({"type": type(exc).__name__, "message": str(exc)})}


def run_case(case):
    t1, seg = scalar_image(case), label_map(case)
    subjects = [tio.Subject(t1=tio.ScalarImage(t1[b].clone()), seg=tio.LabelMap(seg[b].clone()))
                for b in range(case["batch"])]
    batch = tio.SubjectsBatch.from_subjects(subjects)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = tio.HistogramStandardization(landmarks(case), cutoff=case_cutoff(case), **case.get("kwargs", {}))
        record = {"hydra": _json(transform.to_hydra()), "repr": _json(repr(transform))}
        torch.manual_seed(case["seed"])
        try:
            out = transform(batch)
        except Exception as exc:  # noqa: BLE001  (the fixture records what the reference raises)
            return {**record, **_error(exc)}
    record["history"] = _json([{"name": t.name, "params": t.params} for t in out.applied_transforms])
    for key in ("t1", "seg"):
        data = out.images[key].data.contiguous()
        record[f"out_{key}"] = (data.view(torch.int16) if data.dtype == torch.bfloat16 else data).numpy()
    return record


def run_landmark_case(case):
    kwargs = {k: case[k] for k in ("quantiles", "cutoff") if k in case}
    if case.get("masked"):
        kwargs["masking_method"] = positive_mask
    images = [tio.ScalarImage(t) for t in training_images(case)]
    try:
        return {"landmarks": compute_histogram_landmarks(images, **kwargs).numpy()}
    except Exception as exc:  # noqa: BLE001
        return _error(exc)


def main():
    torch.set_num_threads(1)
    names = set(sys.argv[1:])  # optional: regenerate only these cases
    for case, run in [*((c, run_case) for c in HIST_CASES), *((c, run_landmark_case) for c in LANDMARK_CASES)]:
        if names and case["name"] not in names:
            continue
        path = HERE / f"{case['name']}.npz"
        np.savez_compressed(path, **run(case))
        print(f"{case['name']:45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
