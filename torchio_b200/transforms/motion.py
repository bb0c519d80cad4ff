"""Motion (transforms/intensity/motion.py of TorchIO 2.0.0a2): MRI motion artefacts as k-space
segments along the first spatial axis, each taken from a rigidly moved copy of the image.

Constructor, ``make_params`` (its RNG calls and quirks), gating, history, ``repr`` and ``to_hydra``
are the reference's.  The reference resamples the whole batch once per segment with
``affine_grid`` + ``grid_sample``, takes a 3-D FFT of each copy and splices one band of first-axis
k-space rows from each; the segments vary along the first axis only, so the FFTs over the other
two axes cancel and `ops.motion` computes each line along it in one pass, gathering the moved
copies tile by tile.  The affine matrices are built on the host by `motion_theta`, with the
reference's fp32 operations.

A new tensor is written: the caller's tensor is never updated.
"""

from __future__ import annotations

import warnings
from typing import Any

import numpy as np
import torch
from torch import Tensor

from .. import ops
from ..data import SubjectsBatch
from ..params import to_range
from .base import IntensityTransform

_IDENTITY = {"degrees": (0.0, 0.0, 0.0), "translation": (0.0, 0.0, 0.0)}
_UNIT_GRID_WARNING = ("Since version 1.3.0, affine_grid behavior has changed for unit-size grids when"
                      " align_corners=True. This is not an intended use case of affine_grid. See the documentation"
                      " of affine_grid for details.")


def _axis_rotations(angles: Tensor, axis: int) -> Tensor:
    cos, sin = torch.cos(angles), torch.sin(angles)
    m = torch.zeros(angles.shape[0], 3, 3, dtype=angles.dtype)
    a, b = [(1, 2), (0, 2), (0, 1)][axis]
    m[:, axis, axis] = 1
    m[:, a, a] = cos
    m[:, b, b] = cos
    # x and z: [[c, -s], [s, c]] on (a, b); y: [[c, s], [-s, c]] (motion.py:539-558)
    m[:, a, b] = sin if axis == 1 else -sin
    m[:, b, a] = -sin if axis == 1 else sin
    return m


def affine_matrices(degrees: Tensor, translation: Tensor, spatial_shape) -> Tensor:
    """fp32 (B, 3, 4) ``_affine_matrices`` (motion.py:452-514) on CPU: ``r_z @ r_y @ r_x`` of the
    fp32 ``deg2rad`` angles, and ``translation / (shape / 2)`` with ``shape = (I, J, K)``."""
    rx, ry, rz = torch.deg2rad(degrees).unbind(dim=-1)
    theta = torch.zeros(degrees.shape[0], 3, 4, dtype=degrees.dtype)
    theta[:, :3, :3] = _axis_rotations(rz, 2) @ _axis_rotations(ry, 1) @ _axis_rotations(rx, 0)
    theta[:, :3, 3] = translation / (torch.as_tensor(list(spatial_shape), dtype=translation.dtype) / 2)
    return theta


def motion_theta(transforms: list[list[dict]], spatial_shape) -> np.ndarray:
    """fp32 (B, N, 12) tables of `ops.motion` from one list of N rigid transforms per element; an
    empty list (a gated-out element) gets the identity, as in the reference."""
    n = max(len(t) for t in transforms)
    segments = []
    for s in range(n):
        chosen = [t[s] if t else _IDENTITY for t in transforms]
        degrees = torch.as_tensor(tuple(t["degrees"] for t in chosen), dtype=torch.float32)
        translation = torch.as_tensor(tuple(t["translation"] for t in chosen), dtype=torch.float32)
        segments.append(affine_matrices(degrees, translation, spatial_shape).reshape(-1, 12))
    return torch.stack(segments, dim=1).numpy()


def _num_transforms(transforms: list[list[dict]]) -> int:
    lengths = {len(t) for t in transforms} - {0}
    if len(lengths) > 1:
        raise ValueError(f"Expected uniform motion transform counts, got {sorted(lengths)}")
    return max(lengths, default=0)


class Motion(IntensityTransform):
    """Simulate MRI motion artefacts (intensity/motion.py:30-137): ``num_transforms`` rigid motions
    each fill one band of first-axis k-space rows.  A scalar ``degrees`` / ``translation`` is a
    fixed value on every axis, not a range, as in the reference; translations are in voxels and
    move along (K, J, I) while scaled by (I, J, K), as in the reference."""

    def __init__(self, *, degrees: float | tuple[float, float] = 10.0,
                 translation: float | tuple[float, float] = 10.0, num_transforms: int = 2, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.degrees = to_range(degrees)
        self.translation = to_range(translation)
        if not isinstance(num_transforms, int) or num_transforms < 1:
            raise ValueError(f"num_transforms must be a positive int, got {num_transforms}")
        self.num_transforms = num_transforms

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return True

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def _sample_transforms(self) -> list[dict]:
        return [{"degrees": self.degrees.sample(), "translation": self.translation.sample()}
                for _ in range(self.num_transforms)]

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        n = self._resolve_n(batch)
        if n is None:
            return {"transforms": self._sample_transforms()}
        keep = self._keep_mask(batch, n)
        transforms = [[] if keep is not None and not keep[e] else self._sample_transforms() for e in range(n)]
        params = {"transforms": transforms}
        self._tag_batched(params, batch, n, keep, ["transforms"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        per_instance = self._is_per_instance_params(params)
        for _, img_batch in self._get_images(batch).items():
            data = img_batch.data
            b = data.shape[0]
            if per_instance:
                transforms = params["transforms"]
                if len(transforms) != b:
                    raise ValueError(f"Expected {b} motion parameter lists, got {len(transforms)}")
                active = np.array([bool(t) for t in transforms])
                if not active.any():
                    continue  # the reference returns the data itself
                n = _num_transforms(transforms)
            else:
                if not params["transforms"]:
                    continue
                transforms = [params["transforms"]] * b
                active = np.ones(b, dtype=bool)
                n = len(params["transforms"])
            first = int(data.shape[2])
            if first // (n + 1) == 0:
                raise ValueError(
                    f"Cannot split {first} k-space slices into {n + 1} motion segments; reduce num_transforms or"
                    " use a larger image along the first spatial axis.")
            if min(data.shape[2:]) == 1:  # what the reference's affine_grid call issues, once per segment
                for _ in range(n):
                    warnings.warn(_UNIT_GRID_WARNING, stacklevel=2)
            work = data if data.is_contiguous() else data.contiguous()
            img_batch.data = ops.motion(work, motion_theta(transforms, data.shape[2:]), active)
        return batch
