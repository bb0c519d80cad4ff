"""Label-map utilities test infrastructure: the fixture cases, their seeded inputs, and the
reference's op sequences on plain torch ops (transforms/label/ of TorchIO 2.0.0a2), runnable on CPU
and on CUDA tensors.  ``tests/golden/generate_label_maps.py`` runs the reference's classes on these
cases; nothing here is imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

GOLDEN = Path(__file__).resolve().parent / "golden"

I8, U8, I16, I32, I64, F32 = torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64, torch.float32

# transforms: [(class name, kwargs)], run as one Compose when there are several.
# labels: (low, high) of torch.randint; extra: [(element, value)] written into a corner block of
# that element; fractional: + 0.5 on a lattice; nan: NaN voxels; large: + 2**24 + 1 on a lattice.
LABEL_CASES = [
    dict(name="label_remap_swap_i16", transforms=[("RemapLabels", {"remapping": {1: 2, 2: 1}})],
         batch=3, channels=1, shape=(12, 10, 9), dtype=I16, labels=(0, 5), seed=201),
    dict(name="label_remap_merge_u8",
         transforms=[("RemapLabels", {"remapping": {2: 1, 3: 1, 4: 1, 5: 0, 257: 7, -1: 6, 300.0: 9}})],
         batch=1, channels=1, shape=(11, 9, 8), dtype=U8, labels=(0, 8), extra=[(0, 255)], seed=202),
    dict(name="label_remap_wrapping_i8", transforms=[("RemapLabels", {"remapping": {1: -3, 200: 5, -56.5: 2, 3: 4.7}})],
         batch=3, channels=1, shape=(8, 9, 10), dtype=I8, labels=(-4, 4), extra=[(1, -56)], seed=203),
    dict(name="label_remap_two_channels_i32", transforms=[("RemapLabels", {"remapping": {0: 10, 10: 0, 3: 3, 4: 1}})],
         batch=2, channels=2, shape=(10, 8, 12), dtype=I32, labels=(0, 11), seed=204),
    dict(name="label_remap_odd_shape_i64", transforms=[("RemapLabels", {"remapping": {k: 40 - k for k in range(40)}})],
         batch=1, channels=1, shape=(17, 13, 11), dtype=I64, labels=(0, 45), seed=205),
    dict(name="label_remap_f32", transforms=[("RemapLabels", {"remapping": {16777217: 3, -0.0: 9, 1: 2.5, 2.5: 1}})],
         batch=3, channels=1, shape=(9, 8, 7), dtype=F32, labels=(-1, 4), fractional=True,
         extra=[(1, 16777216.0), (2, -0.0)], seed=206),
    dict(name="label_remap_overflow_i16", transforms=[("RemapLabels", {"remapping": {1: 70000}})],
         batch=1, channels=1, shape=(6, 5, 4), dtype=I16, labels=(0, 3), seed=207),
    dict(name="label_remap_key_overflow_i16", transforms=[("RemapLabels", {"remapping": {70000: 2, 2: 7}})],
         batch=2, channels=1, shape=(6, 7, 8), dtype=I16, labels=(0, 5), extra=[(0, 4464)], seed=208),
    dict(name="label_remove_i32", transforms=[("RemoveLabels", {"labels": [1, 3], "background_label": 9})],
         batch=3, channels=1, shape=(10, 9, 8), dtype=I32, labels=(0, 5), seed=209),
    dict(name="label_remove_u8", transforms=[("RemoveLabels", {"labels": [2, 258]})],
         batch=1, channels=2, shape=(7, 8, 9), dtype=U8, labels=(0, 5), seed=210),
    dict(name="label_sequential_i16_missing", transforms=[("SequentialLabels", {})],
         batch=3, channels=1, shape=(10, 9, 11), dtype=I16, labels=(3, 9), extra=[(1, 20), (2, 1)], seed=211),
    dict(name="label_sequential_f32_fractional", transforms=[("SequentialLabels", {})],
         batch=2, channels=1, shape=(9, 10, 8), dtype=F32, labels=(0, 6), fractional=True, seed=212),
    dict(name="label_sequential_i8_negative", transforms=[("SequentialLabels", {})],
         batch=1, channels=2, shape=(8, 8, 8), dtype=I8, labels=(-5, 3), seed=213),
    dict(name="label_sequential_u8", transforms=[("SequentialLabels", {})],
         batch=3, channels=1, shape=(9, 7, 8), dtype=U8, labels=(10, 14), extra=[(0, 250)], seed=214),
    dict(name="label_sequential_i64", transforms=[("SequentialLabels", {})],
         batch=2, channels=1, shape=(7, 6, 9), dtype=I64, labels=(-2, 4), extra=[(0, 2**40)], seed=215),
    dict(name="label_onehot_auto_i64", transforms=[("OneHot", {})],
         batch=3, channels=1, shape=(10, 9, 8), dtype=I64, labels=(0, 5), extra=[(2, 6)], seed=216),
    dict(name="label_onehot_explicit_u8", transforms=[("OneHot", {"num_classes": 7})],
         batch=1, channels=1, shape=(11, 7, 9), dtype=U8, labels=(0, 5), seed=217),
    dict(name="label_onehot_u8_300_classes", transforms=[("OneHot", {"num_classes": 300})],
         batch=2, channels=1, shape=(5, 4, 6), dtype=U8, labels=(0, 4), extra=[(1, 255)], seed=218),
    dict(name="label_onehot_f32_truncated", transforms=[("OneHot", {})],
         batch=2, channels=1, shape=(8, 9, 7), dtype=F32, labels=(0, 4), fractional=True, seed=219),
    dict(name="label_onehot_two_channels_i16", transforms=[("OneHot", {"num_classes": 5})],
         batch=2, channels=2, shape=(6, 8, 7), dtype=I16, labels=(0, 5), seed=220),
    dict(name="label_onehot_i8_negative", transforms=[("OneHot", {})],
         batch=2, channels=1, shape=(5, 6, 7), dtype=I8, labels=(-2, 3), seed=221),
    dict(name="label_onehot_too_large_i32", transforms=[("OneHot", {"num_classes": 3})],
         batch=2, channels=1, shape=(5, 6, 7), dtype=I32, labels=(0, 4), seed=222),
    dict(name="label_contour_touching_i16", transforms=[("Contour", {})],
         batch=3, channels=1, shape=(12, 11, 10), dtype=I16, labels=(0, 3), blocks=True, seed=223),
    dict(name="label_contour_negative_i8", transforms=[("Contour", {})],
         batch=2, channels=1, shape=(9, 10, 11), dtype=I8, labels=(-3, 2), blocks=True, seed=224),
    dict(name="label_contour_nan_f32", transforms=[("Contour", {})],
         batch=2, channels=1, shape=(10, 9, 12), dtype=F32, labels=(-2, 3), blocks=True, nan=True, seed=225),
    dict(name="label_contour_large_i32", transforms=[("Contour", {})],
         batch=1, channels=1, shape=(9, 9, 9), dtype=I32, labels=(0, 3), blocks=True, large=True, seed=226),
    dict(name="label_contour_two_channels_u8", transforms=[("Contour", {})],
         batch=2, channels=2, shape=(7, 37, 41), dtype=U8, labels=(0, 4), blocks=True, seed=227),
    dict(name="label_contour_odd_shape_i64", transforms=[("Contour", {})],
         batch=1, channels=1, shape=(70, 19, 35), dtype=I64, labels=(0, 4), blocks=True, seed=228),
    dict(name="label_compose_remap_sequential_onehot_i16",
         transforms=[("RemapLabels", {"remapping": {7: 1, 8: 1, 9: 2}}), ("SequentialLabels", {}), ("OneHot", {})],
         batch=3, channels=1, shape=(10, 8, 9), dtype=I16, labels=(0, 10), seed=229),
]
LABEL_CASES_BY_NAME = {c["name"]: c for c in LABEL_CASES}


def label_map(case) -> torch.Tensor:
    """(B, C, I, J, K) labels of the case's dtype from its seed."""
    g = torch.Generator().manual_seed(case["seed"] * 7919)
    b, c = case["batch"], case["channels"]
    lo, hi = case["labels"]
    shape = case["shape"]
    if case.get("blocks"):  # piecewise-constant blocks, so labels touch along planes
        coarse = torch.randint(lo, hi, (b, c, *(s // 3 + 1 for s in shape)), generator=g)
        data = coarse.repeat_interleave(3, 2).repeat_interleave(3, 3).repeat_interleave(3, 4)
        data = data[:, :, :shape[0], :shape[1], :shape[2]].clone()
    else:
        data = torch.randint(lo, hi, (b, c, *shape), generator=g)
    data = data.to(torch.float64 if case["dtype"] == F32 else torch.int64)
    for element, value in case.get("extra", []):
        data[element, 0, :2, :3] = value
    if case.get("large"):
        data[:, :, ::2, 1::3] += 2**24 + 1  # rounds to 2**24 in fp32: merges with + 2**24 + 0
        data[:, :, 1::2, 1::3] += 2**24
    data = data.to(case["dtype"])
    if case.get("fractional"):
        data[:, :, ::3, 1] += 0.5
        data[:, :, 1::4, 2] -= 0.25
    if case.get("nan"):
        data[0, 0, 4, 4, 4] = float("nan")
        data[-1, 0, 0, 0, 0] = float("nan")
    return data


def scalar_image(case) -> torch.Tensor:
    g = torch.Generator().manual_seed(case["seed"] * 31)
    return torch.rand((case["batch"], 1, *case["shape"]), generator=g)


def affines(case) -> list[np.ndarray]:
    return [np.diag([1.0 + 0.25 * b, 1.0, 1.5, 1.0]) for b in range(case["batch"])]


def load_fixture(name) -> dict:
    """{"history", "out_seg", "out_t1", "inv_seg" (invertible cases), "error" / "inv_error" (what the
    reference raised, forward or inverse: {"type", "message"})}."""
    z = np.load(GOLDEN / f"{name}.npz")
    out = {"history": json.loads(bytes(z["history"]).decode())}
    for key in ("error", "inv_error"):
        if key in z:
            out[key] = json.loads(bytes(z[key]).decode())
    for key in ("out_seg", "out_t1", "inv_seg"):
        if key in z:
            out[key] = torch.from_numpy(z[key])
    return out


# ---- the reference's op sequences ---------------------------------------------------------------


def remap(data, remapping):
    """remap_labels.py:50-58"""
    out = data.clone()
    for old, new in remapping.items():
        out[data == old] = new
    return out


def remove(data, labels, background_label=0):
    """remove_labels.py:54-61"""
    out = data.clone()
    for label in labels:
        out[data == label] = background_label
    return out


def renumber(data, remapping):
    """sequential_labels.py:53-61 and the inverse :97-105"""
    out = torch.zeros_like(data)
    for old, new in remapping.items():
        out[data == old] = new
    return out


def sequential_params(data):
    """sequential_labels.py:38-45 for one map"""
    unique = sorted(int(v) for v in data[0].unique().tolist())
    return {old: new for new, old in enumerate(unique)}


def one_hot(data, num_classes):
    """one_hot.py:58-69"""
    encoded = F.one_hot(data.long()[:, 0], num_classes=num_classes)
    return encoded.permute(0, 4, 1, 2, 3).float()


def one_hot_inverse(data):
    """one_hot.py:92-97"""
    return data.argmax(dim=1, keepdim=True).float() if data.shape[1] > 1 else data


def contour(data):
    """contour.py:52-71"""
    padded = F.pad(data.float(), [1] * 6, mode="constant", value=-1)
    eroded = -F.max_pool3d(-padded, kernel_size=3, stride=1, padding=0)
    return (eroded != data.float()).float()


def apply(name, kwargs, params, data, image_name="seg"):
    """One transform of the case on a label map, from its recorded params."""
    if name == "RemapLabels":
        return remap(data, params["remapping"])
    if name == "RemoveLabels":
        return remove(data, kwargs["labels"], kwargs.get("background_label", 0))
    if name == "SequentialLabels":
        return renumber(data, params["remappings"][image_name])
    if name == "OneHot":
        return one_hot(data, params["num_classes"])
    if name == "Contour":
        return contour(data)
    raise KeyError(name)


def inverse(name, params, data, image_name="seg"):
    if name == "RemapLabels":
        return remap(data, {v: k for k, v in params["remapping"].items()})
    if name == "SequentialLabels":
        return renumber(data, {v: k for k, v in params["remappings"][image_name].items()})
    if name == "OneHot":
        return one_hot_inverse(data)
    return data


def reference_output(case, data):
    """(output, inverse of the output, params per transform) of the case's transforms on ``data``,
    with params made as the reference makes them (none of them draws random numbers)."""
    history = []
    for name, kwargs in case["transforms"]:
        if name == "RemapLabels":
            params = {"remapping": kwargs["remapping"]}
        elif name == "SequentialLabels":
            params = {"remappings": {"seg": sequential_params(data)}}
        elif name == "OneHot":
            params = {"num_classes": kwargs.get("num_classes", -1)}
        else:
            params = {}
        data = apply(name, kwargs, params, data)
        history.append((name, params))
    undone = data
    for name, params in reversed(history):
        undone = inverse(name, params, undone)
    return data, undone, history


def json_keys(obj):
    """Params as the JSON history stores them (int dict keys become strings)."""
    return json.loads(json.dumps(obj))
