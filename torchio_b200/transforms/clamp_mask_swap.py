"""Clamp, Mask and Swap (transforms/intensity/clamp.py, mask.py and swap.py of TorchIO 2.0.0a2).

Constructors, errors, warnings, ``make_params`` (Swap's RNG calls included), gating, history,
``repr`` and ``to_hydra`` are the reference's.  Each ``apply_transform`` is one kernel launch per
image batch:
- `Clamp`: `ops.clamp`, with the bounds converted to the result dtype by torch itself (its
  promotion of an integer image to fp32, its overflow errors, its wrap of ``uint8`` bounds);
- `Mask`: `ops.mask`, the mask of batch element 0 read once per voxel for every element; in place
  when the dtype is kept, so only the outside voxels are written;
- `Swap`: `ops.swap_patches`, every element's swap list in one launch, in place instead of the
  reference's clone + two gathers and two ``index_put_`` per step.

Mask and Swap overwrite the batch's own tensors: a transform called with ``copy=True`` (the
default) or inside a `Compose` has already copied them.
"""

from __future__ import annotations

import warnings
from collections.abc import Callable
from typing import Any

import numpy as np
import torch
from torch import Tensor

from .. import ops, tables
from ..data import LabelMap, SubjectsBatch
from ..params import to_nonneg_range
from .base import IntensityTransform
from .intensity import label_map_element0


# ---- Clamp --------------------------------------------------------------------------------------

def clamp_bounds(dtype: torch.dtype, out_min, out_max) -> tuple[Tensor | None, Tensor | None]:
    """The bounds of ``x.clamp(min=out_min, max=out_max)`` for an image of ``dtype`` as one-element
    CPU tensors of the result dtype, converted as ATen converts the scalars (``Scalar::to``); torch
    raises its own errors here (no bound, a bound the dtype cannot hold)."""
    result = torch.zeros(1, dtype=dtype).clamp(min=out_min, max=out_max).dtype
    lo = None if out_min is None else torch.full((1,), out_min, dtype=result)
    hi = None if out_max is None else torch.full((1,), out_max, dtype=result)
    return lo, hi


class Clamp(IntensityTransform):
    """Clamp intensities into ``[out_min, out_max]``; ``None`` leaves that side open
    (intensity/clamp.py:11-57)."""

    def __init__(self, *, out_min: float | None = None, out_max: float | None = None, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        if out_min is not None and out_max is not None and out_min > out_max:
            raise ValueError(f"out_min ({out_min}) must be <= out_max ({out_max})")
        self.out_min = out_min
        self.out_max = out_max

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {"out_min": self.out_min, "out_max": self.out_max}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for _, img_batch in self._get_images(batch).items():
            lo, hi = clamp_bounds(img_batch.data.dtype, params["out_min"], params["out_max"])
            img_batch.data = ops.clamp(img_batch.data, lo, hi)
        return batch


# ---- Mask ---------------------------------------------------------------------------------------

def where_outside(dtype: torch.dtype, outside_value) -> Tensor:
    """``outside_value`` as ``torch.where(mask, x, outside_value)`` stores it for an image of
    ``dtype``: a one-element CPU tensor of the result dtype (fp32 for an integer image and a float
    value); torch raises its own error for a value the dtype cannot hold."""
    return torch.where(torch.zeros(1, dtype=torch.bool), torch.zeros(1, dtype=dtype), outside_value)


class Mask(IntensityTransform):
    """Set the voxels outside a mask to ``outside_value`` (intensity/mask.py:16-102).  The mask is
    batch element 0 of the `LabelMap` named by ``masking_method`` (nonzero voxels, or those equal to
    one of ``labels``), or ``masking_method(data[0])`` of the first selected image; it applies to
    every element.

    Never streamed in slices: element 0 of a slice is not element 0 of the batch."""

    def __init__(self, *, masking_method: str | Callable = "brain", outside_value: float = 0.0,
                 labels: list[int] | None = None, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.masking_method = masking_method
        self.outside_value = outside_value
        self.labels = labels

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        mask, keys = self._resolve_mask(batch)
        for _, img_batch in self._get_images(batch).items():
            data = img_batch.data
            element = mask.to(data.device).expand_as(data)[0]  # torch's error for shapes it rejects
            if element.shape[0] == 1 or element.stride(0) == 0:
                element = element[:1]
            outside = where_outside(data.dtype, self.outside_value)
            work = data if data.is_contiguous() else data.contiguous()
            img_batch.data = ops.mask(work, element, keys, outside)
        return batch

    def _resolve_mask(self, batch: SubjectsBatch) -> tuple[Tensor, np.ndarray | None]:
        """(mask of one element, label keys or None for "nonzero"), mask.py:73-102."""
        if callable(self.masking_method) and not isinstance(self.masking_method, str):
            first_img = next(iter(self._get_images(batch).values()))
            return self.masking_method(first_img.data[0]).bool(), None
        if isinstance(self.masking_method, str):
            mask_data = label_map_element0(self.masking_method, batch)
            if self.labels is None:
                return mask_data, None
            if mask_data.dtype not in ops.DTYPE_CODES:
                raise TypeError(f"Mask: labels on a {mask_data.dtype} label map are not supported")
            keys, _ = tables.label_lut([(label, 1) for label in self.labels], mask_data.dtype, mask_data.device)
            return mask_data, keys
        raise TypeError(f"masking_method must be a str or callable, got {type(self.masking_method)}")


# ---- Swap ---------------------------------------------------------------------------------------

def _random_origin(max_ini: list[int]) -> tuple[int, int, int]:
    coords = [0 if m == 0 else int(torch.randint(m + 1, (1,)).item()) for m in max_ini]
    return coords[0], coords[1], coords[2]


def _patches_overlap(a, b, patch_size) -> bool:
    return all(not (ai + p <= bi or bi + p <= ai) for ai, bi, p in zip(a, b, patch_size))


def sample_swap_locations(spatial_shape, patch_size, num_iterations: int) -> list:
    """Pairs of patch origins, the second redrawn up to 100 times until it does not overlap the
    first (swap.py:134-192, the same torch.randint calls)."""
    max_ini = [s - p for s, p in zip(spatial_shape, patch_size, strict=True)]
    if any(m < 0 for m in max_ini):
        raise ValueError(f"Patch size {patch_size} cannot be larger than spatial shape {tuple(spatial_shape)}")
    locations = []
    for _ in range(num_iterations):
        first = _random_origin(max_ini)
        for _ in range(100):
            second = _random_origin(max_ini)
            if not _patches_overlap(first, second, patch_size):
                break
        locations.append((first, second))
    return locations


def swap_table(rows, patch_size) -> np.ndarray:
    """(len(rows), steps, 8) int32 lists of `ops.swap_patches` from one location list per row; a
    shorter row is padded with no-op steps (the reference's (0, 0, 0) self-swaps)."""
    steps = max((len(row) for row in rows), default=0)
    table = np.zeros((len(rows), steps, 8), dtype=np.int32)
    table[..., 6] = ops.SWAP_NOOP
    patch = np.asarray(patch_size, dtype=np.int64)
    for e, row in enumerate(rows):
        if not row:
            continue
        pairs = np.asarray(row, dtype=np.int64).reshape(len(row), 2, 3)
        a, b = pairs[:, 0], pairs[:, 1]
        overlap = np.all((a + patch > b) & (b + patch > a), axis=1)
        table[e, : len(row), :6] = pairs.reshape(len(row), 6)
        table[e, : len(row), 6] = np.where(overlap, ops.SWAP_STAGED, ops.SWAP_EXCHANGE)
    return table


class Swap(IntensityTransform):
    """Swap ``num_iterations`` random pairs of ``patch_size`` patches, in order, in each scalar
    image (intensity/swap.py:22-131), for context-restoration pretraining."""

    def __init__(self, *, patch_size: int | tuple[int, int, int] = 15, num_iterations: int | tuple[int, int] = 100,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        if isinstance(patch_size, int):
            patch_size = (patch_size, patch_size, patch_size)
        self.patch_size = patch_size
        self.num_iterations = to_nonneg_range(num_iterations)

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return True

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        for _, img_batch in batch.images.items():
            if issubclass(img_batch._image_class, LabelMap):
                warnings.warn(
                    "Swap is applied to a subject containing LabelMap images. The spatial rearrangement"
                    " will make labels inconsistent with the swapped image. This transform is intended"
                    " for self-supervised learning.", stacklevel=2)
                break
        spatial_shape = next(iter(batch.images.values())).data.shape[2:]
        n = self._resolve_n(batch)
        if n is None:
            iterations = max(1, round(self.num_iterations.sample_1d()))
            return {"locations": sample_swap_locations(spatial_shape, self.patch_size, iterations)}
        keep = self._keep_mask(batch, n)
        locations: list[Any] = []
        for index in range(n):
            if keep is not None and not keep[index]:
                locations.append([])
                continue
            iterations = max(1, round(self.num_iterations.sample_1d()))
            locations.append(sample_swap_locations(spatial_shape, self.patch_size, iterations))
        params = {"locations": locations}
        self._tag_batched(params, batch, n, keep, ["locations"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        rows = params["locations"] if self._is_per_instance_params(params) else [params["locations"]]
        table = swap_table(rows, self.patch_size)
        for _, img_batch in self._get_images(batch).items():
            data = img_batch.data
            work = data if data.is_contiguous() else data.contiguous()
            ops.swap_patches(work, table, self.patch_size)
            img_batch.data = work
        return batch
