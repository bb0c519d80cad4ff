"""Generate the LabelsToImage golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_labels_to_image.py

For every case of ``tests/labels_to_image_cases.py`` it records the params the reference sampled
(JSON history) and the image it generated; the label maps are regenerated from the case seeds.
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

from labels_to_image_cases import L2I_CASES, affines, label_map, transform_kwargs  # noqa: E402


def run_case(case):
    labels = label_map(case)
    subjects = []
    for b, affine in enumerate(affines(case)):
        subjects.append(tio.Subject(seg=tio.LabelMap(labels[b].clone(), affine=affine.copy())))
    batch = tio.SubjectsBatch.from_subjects(subjects)
    transform = tio.LabelsToImage(**transform_kwargs(case))
    torch.manual_seed(case["seed"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = transform(batch)
    history = [{"name": t.name, "params": t.params} for t in out.applied_transforms]
    return {
        "out_image": out.images["image_from_labels"].data.contiguous().numpy(),
        "history": np.frombuffer(json.dumps(history).encode(), dtype=np.uint8),
    }


def main():
    torch.set_num_threads(1)
    for case in L2I_CASES:
        path = HERE / f"{case['name']}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{case['name']:40s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
