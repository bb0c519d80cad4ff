"""Clamp / Mask / Swap test infrastructure: the fixture cases, their seeded inputs, and the reference's
op sequences (transforms/intensity/clamp.py:47-57, mask.py:61-102 and swap.py:195-364 of TorchIO
2.0.0a2) restated on plain torch ops, runnable on CPU and on CUDA tensors.
``tests/golden/generate_intensity_utilities.py`` runs the reference's classes on these cases;
nothing here is imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

F32, F16, BF16, F64 = torch.float32, torch.float16, torch.bfloat16, torch.float64
U8, I8, I16, I32, I64 = torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64
DTYPES = [F32, F16, BF16, F64, U8, I8, I16, I32, I64]
SHORT = {F32: "f32", F16: "f16", BF16: "bf16", F64: "f64", U8: "u8", I8: "i8", I16: "i16", I32: "i32", I64: "i64"}


def positive(x: torch.Tensor) -> torch.Tensor:
    """The callable masking method of the cases."""
    return x > 0


# Inputs: "t1" (ScalarImage, (B, C, *shape) of `dtype`: 40 % zeros, the rest over about [-100, 400],
# integers for integer dtypes, clipped to the dtype; kind "nonfinite" adds NaN, +-Inf and -0 voxels)
# and, with `seg`, a LabelMap "seg" (B, seg_channels, *shape): "int16" labels 0..3 that differ per
# element, "float32" values {0, 0.5, 1, 2.25, NaN}.
SWAP_CASES = [
    dict(name="swap_b1_f32", batch=1, shape=(10, 9, 8), dtype=F32, kwargs=dict(patch_size=3, num_iterations=6)),
    dict(name="swap_b3_p05_f32", batch=3, shape=(10, 9, 8), dtype=F32,
         kwargs=dict(patch_size=3, num_iterations=6, p=0.5)),
    dict(name="swap_b3_shared_f32", batch=3, shape=(10, 9, 8), dtype=F32,
         kwargs=dict(patch_size=3, num_iterations=6, per_instance=False)),
    dict(name="swap_b3_range_f32", batch=3, shape=(10, 9, 8), dtype=F32,
         kwargs=dict(patch_size=(2, 3, 4), num_iterations=(2, 7))),
    dict(name="swap_b3_overlap_f32", batch=3, shape=(10, 10, 10), dtype=F32, kwargs=dict(patch_size=8, num_iterations=5)),
    dict(name="swap_b1_full_f32", batch=1, shape=(6, 5, 4), dtype=F32, kwargs=dict(patch_size=(6, 5, 4), num_iterations=2)),
    dict(name="swap_b1_2d_f32", batch=1, shape=(12, 10, 1), dtype=F32, kwargs=dict(patch_size=(3, 3, 1), num_iterations=8)),
    dict(name="swap_b3_c2_seg_f32", batch=3, channels=2, shape=(10, 9, 8), dtype=F32, seg="int16",
         kwargs=dict(patch_size=3, num_iterations=4)),
    dict(name="swap_error_too_large", batch=1, shape=(10, 9, 8), dtype=F32, kwargs=dict(patch_size=(20, 3, 3))),
    *[dict(name=f"swap_b3_{SHORT[d]}", batch=3, shape=(9, 8, 7), dtype=d, kwargs=dict(patch_size=3, num_iterations=5))
      for d in DTYPES if d != F32],
]

CLAMP_CASES = [
    dict(name="clamp_min_f32", batch=3, shape=(9, 8, 7), dtype=F32, kwargs=dict(out_min=0.0)),
    dict(name="clamp_max_f32", batch=3, shape=(9, 8, 7), dtype=F32, kwargs=dict(out_max=100.5)),
    dict(name="clamp_both_f32", batch=3, shape=(9, 8, 7), dtype=F32, kwargs=dict(out_min=-20, out_max=150)),
    dict(name="clamp_error_none_f32", batch=3, shape=(9, 8, 7), dtype=F32, kwargs=dict()),
    dict(name="clamp_error_init", batch=1, shape=(9, 8, 7), dtype=F32, kwargs=dict(out_min=5.0, out_max=1.0)),
    dict(name="clamp_i16_float_bounds", batch=3, shape=(9, 8, 7), dtype=I16, kwargs=dict(out_min=-20.5, out_max=150.25)),
    dict(name="clamp_u8_min_wraps", batch=3, shape=(9, 8, 7), dtype=U8, kwargs=dict(out_min=-1)),
    dict(name="clamp_error_u8_max_300", batch=3, shape=(9, 8, 7), dtype=U8, kwargs=dict(out_max=300)),
    dict(name="clamp_nonfinite_f32", batch=3, shape=(9, 8, 7), dtype=F32, kind="nonfinite",
         kwargs=dict(out_min=0.0, out_max=50.0)),
    dict(name="clamp_nonfinite_min_f32", batch=3, shape=(9, 8, 7), dtype=F32, kind="nonfinite",
         kwargs=dict(out_min=-0.0)),
    dict(name="clamp_f16_unrepresentable", batch=3, shape=(9, 8, 7), dtype=F16, kwargs=dict(out_min=0.1, out_max=100.3)),
    dict(name="clamp_bf16_unrepresentable", batch=3, shape=(9, 8, 7), dtype=BF16, kwargs=dict(out_min=0.1, out_max=100.3)),
    *[dict(name=f"clamp_b3_{SHORT[d]}", batch=3, shape=(9, 8, 7), dtype=d, kwargs=dict(out_min=10, out_max=100))
      for d in DTYPES if d != F32],
    dict(name="clamp_b1_f32", batch=1, shape=(9, 8, 7), dtype=F32, kwargs=dict(out_min=10, out_max=100)),
]

MASK_CASES = [
    dict(name="mask_key_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16", kwargs=dict(masking_method="seg")),
    dict(name="mask_labels_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16",
         kwargs=dict(masking_method="seg", labels=[1, 3])),
    dict(name="mask_absent_label_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16",
         kwargs=dict(masking_method="seg", labels=[7])),
    dict(name="mask_empty_labels_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16",
         kwargs=dict(masking_method="seg", labels=[])),
    dict(name="mask_fp32_map_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="float32", kwargs=dict(masking_method="seg")),
    dict(name="mask_fp32_map_labels_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="float32",
         kwargs=dict(masking_method="seg", labels=[0.5, 2])),
    dict(name="mask_callable_f32", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16", kwargs=dict(masking_method=positive)),
    dict(name="mask_c2_one_channel_f32", batch=3, channels=2, shape=(9, 8, 7), dtype=F32, seg="int16",
         kwargs=dict(masking_method="seg", outside_value=-3.5)),
    dict(name="mask_c2_two_channel_f32", batch=3, channels=2, seg_channels=2, shape=(9, 8, 7), dtype=F32, seg="int16",
         kwargs=dict(masking_method="seg")),
    dict(name="mask_i16_default_outside", batch=3, shape=(9, 8, 7), dtype=I16, seg="int16",
         kwargs=dict(masking_method="seg")),
    dict(name="mask_i16_int_outside", batch=3, shape=(9, 8, 7), dtype=I16, seg="int16",
         kwargs=dict(masking_method="seg", outside_value=-5)),
    dict(name="mask_error_u8_300", batch=3, shape=(9, 8, 7), dtype=U8, seg="int16",
         kwargs=dict(masking_method="seg", outside_value=300)),
    dict(name="mask_error_missing_key", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16", kwargs=dict()),
    dict(name="mask_error_not_label_map", batch=3, shape=(9, 8, 7), dtype=F32, seg="int16",
         kwargs=dict(masking_method="t1")),
    dict(name="mask_b1_f32", batch=1, shape=(9, 8, 7), dtype=F32, seg="int16", kwargs=dict(masking_method="seg")),
    *[dict(name=f"mask_b3_{SHORT[d]}", batch=3, shape=(9, 8, 7), dtype=d, seg="int16", kwargs=dict(masking_method="seg"))
      for d in DTYPES if d != F32],
]

CASES = {c["name"]: c for c in [*SWAP_CASES, *CLAMP_CASES, *MASK_CASES]}


def transform_name(case) -> str:
    return {"swap": "Swap", "clamp": "Clamp", "mask": "Mask"}[case["name"].split("_")[0]]


def seed(case) -> int:
    return 500 + sorted(CASES).index(case["name"])


def random_values(rng: np.random.Generator, shape, dtype: torch.dtype, kind: str = "background") -> torch.Tensor:
    n = int(np.prod(shape))
    x = rng.uniform(-100.0, 400.0, n)
    x[rng.random(n) < 0.4] = 0.0
    if not dtype.is_floating_point:
        x = np.round(x)
        info = torch.iinfo(dtype)
        x = np.clip(x, info.min, info.max)
    t = torch.as_tensor(x, dtype=torch.float64)
    if kind == "nonfinite":
        t[rng.random(n) < 0.05] = float("nan")
        t[rng.random(n) < 0.03] = float("inf")
        t[rng.random(n) < 0.03] = float("-inf")
        t[rng.random(n) < 0.05] = -0.0
    return t.to(dtype).reshape(shape)


def scalar_image(case) -> torch.Tensor:
    rng = np.random.default_rng(seed(case))
    return random_values(rng, (case["batch"], case.get("channels", 1), *case["shape"]), case["dtype"],
                         case.get("kind", "background"))


def label_map(case) -> torch.Tensor | None:
    kind = case.get("seg")
    if kind is None:
        return None
    rng = np.random.default_rng(seed(case) + 1000)
    shape = (case["batch"], case.get("seg_channels", 1), *case["shape"])
    if kind == "int16":
        return torch.as_tensor(rng.integers(0, 4, shape), dtype=torch.int16)
    values = np.asarray([0.0, 0.5, 1.0, 2.25, np.nan])
    return torch.as_tensor(values[rng.integers(0, 5, shape)], dtype=torch.float32)


# ---- the reference's op sequences ---------------------------------------------------------------

def clamp_reference(data: torch.Tensor, out_min, out_max) -> torch.Tensor:
    return data.clamp(min=out_min, max=out_max)


def mask_reference(data: torch.Tensor, seg: torch.Tensor | None, masking_method, labels, outside_value) -> torch.Tensor:
    if callable(masking_method):
        mask = masking_method(data[0]).bool()
    else:
        mask_data = seg[0]
        if labels is not None:
            mask = torch.zeros_like(mask_data, dtype=torch.bool)
            for label in labels:
                mask = mask | (mask_data == label)
        else:
            mask = mask_data.bool()
    return torch.where(mask.expand_as(data), data, outside_value)


def swap_reference(data: torch.Tensor, locations, patch_size, per_instance: bool) -> torch.Tensor:
    """_apply_swaps (one list for the batch) or, per element, that element's list: the result of
    _apply_swaps_per_instance, whose padded (0, 0, 0) self-swaps change nothing."""
    if isinstance(patch_size, int):
        patch_size = (patch_size,) * 3
    pi, pj, pk = patch_size
    result = data.clone()
    rows = [(slice(e, e + 1), locs) for e, locs in enumerate(locations)] if per_instance else [(slice(None), locations)]
    for rows_slice, locs in rows:
        view = result[rows_slice]
        for (ai, aj, ak), (bi, bj, bk) in locs:
            patch_a = view[:, :, ai:ai + pi, aj:aj + pj, ak:ak + pk].clone()
            patch_b = view[:, :, bi:bi + pi, bj:bj + pj, bk:bk + pk].clone()
            view[:, :, ai:ai + pi, aj:aj + pj, ak:ak + pk] = patch_b
            view[:, :, bi:bi + pi, bj:bj + pj, bk:bk + pk] = patch_a
    return result


def reference_output(case, data: torch.Tensor, seg: torch.Tensor | None, params: dict) -> torch.Tensor:
    """The case's op sequence on ``data`` (any device) with the recorded ``params``."""
    kwargs = case["kwargs"]
    kind = transform_name(case)
    if kind == "Clamp":
        return clamp_reference(data, params["out_min"], params["out_max"])
    if kind == "Mask":
        return mask_reference(data, seg, kwargs.get("masking_method", "brain"), kwargs.get("labels"),
                              kwargs.get("outside_value", 0.0))
    return swap_reference(data, params["locations"], kwargs.get("patch_size", 15), "_batched_keys" in params)


def as_stored(t: torch.Tensor) -> np.ndarray:
    """A tensor as the fixtures store it (bf16 as its int16 bits)."""
    t = t.detach().cpu().contiguous()
    return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).numpy()


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"{name}.npz") as z:
        out = {k: z[k] for k in z.files}
    for key in ("history", "error", "hydra", "repr", "warnings", "dtype"):
        if key in out:
            out[key] = json.loads(out[key].tobytes().decode())
    return out
