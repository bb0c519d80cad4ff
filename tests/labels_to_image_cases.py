"""LabelsToImage test infrastructure: the fixture cases, their seeded inputs, and the reference's
op sequence on plain torch ops (labels_to_image.py:182-290 of TorchIO 2.0.0a2), runnable on CPU
and on CUDA tensors.  ``tests/golden/generate_labels_to_image.py`` runs the reference on these
cases; nothing here is imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

# name, batch, channels, spatial shape, label dtype, LabelsToImage kwargs, transform kwargs
L2I_CASES = [
    dict(name="labels_to_image_b1_default", batch=1, channels=1, shape=(24, 20, 16), dtype=torch.int64,
         kwargs={}, seed=101),
    dict(name="labels_to_image_b3_lists", batch=3, channels=1, shape=(16, 18, 20), dtype=torch.int16,
         kwargs={"mean": [(0.0, 0.2), 0.5, (0.6, 0.9), (1.0, 1.5), (2.0, 2.5), 3.0, (4.0, 5.0), 6.0],
                 "std": [(0.01, 0.02), 0.05, (0.1, 0.2)]}, seed=102),
    dict(name="labels_to_image_ignore_background", batch=2, channels=1, shape=(20, 16, 12), dtype=torch.int32,
         kwargs={"ignore_background": True}, seed=103),
    dict(name="labels_to_image_shared", batch=3, channels=1, shape=(16, 16, 16), dtype=torch.int64,
         kwargs={"per_instance": False}, seed=104),
    dict(name="labels_to_image_absent_label", batch=3, channels=1, shape=(12, 14, 16), dtype=torch.int16,
         kwargs={}, seed=105, extra_label=(2, 9)),
    dict(name="labels_to_image_two_channels", batch=2, channels=2, shape=(12, 12, 20), dtype=torch.int64,
         kwargs={"label_key": "seg"}, seed=106),
    dict(name="labels_to_image_u8", batch=2, channels=1, shape=(16, 12, 20), dtype=torch.uint8,
         kwargs={}, seed=107),
    dict(name="labels_to_image_i32", batch=2, channels=1, shape=(20, 12, 16), dtype=torch.int32,
         kwargs={"default_mean": (-1.0, 1.0), "default_std": (-0.2, 0.3)}, seed=108),
    dict(name="labels_to_image_odd_shape", batch=2, channels=1, shape=(37, 29, 23), dtype=torch.int16,
         kwargs={}, seed=109),
    dict(name="labels_to_image_f32_fractional", batch=2, channels=1, shape=(14, 10, 18), dtype=torch.float32,
         kwargs={}, seed=110, fractional=True),
    dict(name="labels_to_image_i8_negative", batch=2, channels=1, shape=(10, 18, 14), dtype=torch.int8,
         kwargs={}, seed=111, offset=-3),
]
L2I_CASES_BY_NAME = {c["name"]: c for c in L2I_CASES}


def label_map(case) -> torch.Tensor:
    """(B, C, I, J, K) labels in 0..5 (shifted by ``offset``) from the case's seed; channel 1 also
    holds label 7, which is drawn but never read; ``extra_label`` = (element, label) puts a label
    absent from element 0 into another element; ``fractional`` adds non-integral values."""
    g = torch.Generator().manual_seed(case["seed"] * 7919)
    b, c = case["batch"], case["channels"]
    data = torch.randint(0, 6, (b, c, *case["shape"]), generator=g) + case.get("offset", 0)
    if c > 1:
        data[:, 1, :2] = 7
    if "extra_label" in case:
        element, label = case["extra_label"]
        data[element, 0, :3, :4] = label
    data = data.to(case["dtype"])
    if case.get("fractional"):
        data[:, :, ::3, 1] += 0.5  # int() of x.5 collides with x: a duplicate in the draw loop
    return data


def affines(case) -> list[np.ndarray]:
    return [np.diag([1.0 + 0.25 * b, 1.0, 1.5, 1.0]) for b in range(case["batch"])]


def transform_kwargs(case) -> dict:
    kwargs = dict(case["kwargs"])
    kwargs.setdefault("label_key", "seg")
    return kwargs


def load_fixture(name):
    """(history, expected image) written by generate_labels_to_image.py."""
    z = np.load(GOLDEN / f"{name}.npz")
    return json.loads(bytes(z["history"]).decode()), torch.from_numpy(z["out_image"])


def reference_image(label_data: torch.Tensor, means, stds) -> torch.Tensor:
    """The reference's synthesis on torch ops, on ``label_data``'s device and generator: per drawn
    label, a full (B, 1, I, J, K) randn_like, ``* std``, ``+ mean``, masked by ``label == l`` and
    summed into a zero image.  Shared params: one value per label, labels in the dict's order,
    skipped when mean and std are both 0.  Per element: (B,) fp32 columns over the sorted union of
    labels, skipped when both columns are all zero."""
    b = label_data.shape[0]
    result = torch.zeros(b, 1, *label_data.shape[2:], device=label_data.device)
    if isinstance(means, list):
        labels = sorted({int(k) for m in means for k in m})
        for label in labels:
            m = torch.tensor([_get(e, label) for e in means], dtype=result.dtype, device=result.device)
            s = torch.tensor([_get(e, label) for e in stds], dtype=result.dtype, device=result.device)
            if int(torch.count_nonzero(m)) == 0 and int(torch.count_nonzero(s)) == 0:
                continue
            mask = (label_data[:, 0:1] == label).to(result.dtype)
            result += (torch.randn_like(result) * s.view(b, 1, 1, 1, 1) + m.view(b, 1, 1, 1, 1)) * mask
        return result
    for key, mean in means.items():
        label = int(key)
        std = _get(stds, label)
        if mean == 0.0 and std == 0.0:
            continue
        mask = (label_data[:, 0:1] == label).float()
        result += (torch.randn_like(result) * std + mean) * mask
    return result


def _get(values: dict, label: int) -> float:
    """values[label] for int keys or their JSON strings, 0.0 when absent."""
    return values.get(label, values.get(str(label), 0.0))
