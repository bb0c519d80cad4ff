"""Reorient, Transpose, EnsureShapeMultiple, CopyAffine, ToReferenceSpace (host-side mirror of
transforms/spatial/reorient.py, transpose.py, ensure_shape_multiple.py, copy_affine.py and
to_reference_space.py, TorchIO 2.0.0a2).

Same constructors, validation messages, ``params``, gating draws, history and inverses as the
reference.  The voxel moves of `Reorient` and `Transpose` (the reference's ``torch.flip`` per axis
then ``permute(...).contiguous()``) are one `ops.permute` launch per image; affines are computed
in float64 with the reference's op order.  `EnsureShapeMultiple` is `CropOrPad` with a computed
target; `CopyAffine` and `ToReferenceSpace` only change affines.  None of them streams a host batch
in slices: each changes a shape or an affine that later transforms read when they sample."""

from __future__ import annotations

import math
from typing import Any

import numpy as np
import torch
from torch import Tensor

from .. import ops
from ..data import (AffineMatrix, Image, Subject, SubjectsBatch, _axcodes2ornt, _inv_ornt_aff, _io_orientation,
                    _ornt_transform)
from .base import SpatialTransform
from .neighbours import _PADDING_MODES, CropOrPad


def _validate_orientation(orientation: str) -> str:
    """Three letters, case-insensitive, one of each of R/L, A/P, S/I (reorient.py:17-45)."""
    if not isinstance(orientation, str) or len(orientation) != 3:
        raise ValueError(f'Orientation must be a 3-letter string, got "{orientation}"')
    orientation = orientation.upper()
    valid_codes = set("RLAPIS")
    if not all(c in valid_codes for c in orientation):
        raise ValueError(
            "Orientation code must be composed of three distinct characters"
            f' in {valid_codes} but got "{orientation}"'
        )
    pairs = [{"R", "L"}, {"A", "P"}, {"S", "I"}]
    if not all(set(orientation) & pair for pair in pairs):
        raise ValueError(
            "Orientation code must include one character for each axis"
            f' direction: R or L, A or P, and S or I, but got "{orientation}"'
        )
    return orientation


def ornt_permutation(ornt: np.ndarray) -> tuple[tuple[int, int, int], int]:
    """(output axis -> input axis, flip bits by input axis) of an ornt: nibabel's
    ``apply_orientation``, flips on the input axes then ``transpose(argsort(ornt[:, 0]))``."""
    perm = np.argsort(ornt[:, 0]).astype(int)
    bits = sum(1 << ax for ax in range(3) if ornt[ax, 1] == -1)
    return (int(perm[0]), int(perm[1]), int(perm[2])), bits


class Reorient(SpatialTransform):
    """Reorder voxel axes to a target orientation such as "RAS" or "LPS" (reorient.py:94-179)."""

    def __init__(self, orientation: str = "RAS", **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.orientation = _validate_orientation(orientation)

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        # element 0 of the first image of the batch, whatever include / exclude select
        affine = next(iter(batch.images.values())).affines[0].numpy()
        current = _io_orientation(affine)
        codes = "".join(AffineMatrix(affine).orientation)
        ornt = _ornt_transform(current, _axcodes2ornt(tuple(self.orientation)))
        return {"ornt": ornt.tolist(), "original_orientation": codes}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        ornt = np.asarray(params["ornt"])
        if np.array_equal(ornt[:, 0], [0, 1, 2]) and np.all(ornt[:, 1] == 1):
            return batch
        perm, bits = ornt_permutation(ornt)
        for ib in self._get_images(batch).values():
            original_shape = ib.data.shape[-3:]
            ib.data = ops.permute(ib.data, perm, bits)
            inv_aff = _inv_ornt_aff(ornt, original_shape)
            for index, affine in enumerate(ib.affines):
                ib.affines[index] = type(affine)(affine.numpy() @ inv_aff)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> Reorient:
        return Reorient(orientation=params["original_orientation"], copy=False)


class Transpose(SpatialTransform):
    """Swap the first and last spatial axes of every image, include / exclude notwithstanding
    (transpose.py:11-59)."""

    def __init__(self, **kwargs: Any) -> None:
        super().__init__(**kwargs)

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for ib in batch.images.values():
            ib.data = ops.permute(ib.data, (2, 1, 0))
            for index, affine in enumerate(ib.affines):
                matrix = affine.numpy().copy()
                matrix[:, [0, 2]] = matrix[:, [2, 0]]
                ib.affines[index] = type(affine)(matrix)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> Transpose:
        return Transpose(copy=False)


def _parse_target_multiple(value) -> tuple[int, int, int]:
    """int or 3 values, each >= 1 (ensure_shape_multiple.py:23-38)."""
    if isinstance(value, int):
        if value < 1:
            raise ValueError(f"target_multiple must be >= 1, got {value}")
        return (value, value, value)
    values = tuple(value)
    if len(values) != 3:
        raise ValueError(f"target_multiple must have 1 or 3 values, got {len(values)}")
    for v in values:
        if v < 1:
            raise ValueError(f"All target_multiple values must be >= 1, got {v}")
    return (values[0], values[1], values[2])


def _compute_target_shape(current_shape, target_multiple, method: str) -> tuple[int, int, int]:
    """Next (pad) or previous (crop) multiple per axis, at least 1 (ensure_shape_multiple.py:41-55)."""
    result = []
    for size, multiple in zip(current_shape, target_multiple, strict=True):
        rounding = math.ceil if method == "pad" else math.floor
        result.append(max(rounding(size / multiple) * multiple, 1))
    return (result[0], result[1], result[2])


class EnsureShapeMultiple(SpatialTransform):
    """Pad or crop so that every spatial size is a multiple of ``target_multiple``
    (ensure_shape_multiple.py:58-178).  A `Subject` or `Image` is handed to a `CropOrPad`, whose
    records the history then holds; a batch records ``{"target_shape": ...}``."""

    def __init__(self, target_multiple, *, method: str = "pad", padding_mode: str = "constant", fill: float = 0,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.target_multiple = _parse_target_multiple(target_multiple)
        if method not in ("crop", "pad"):
            raise ValueError(f"method must be 'crop' or 'pad', got {method!r}")
        self.method = method
        if padding_mode not in _PADDING_MODES:
            raise ValueError(f"padding_mode must be one of {_PADDING_MODES}, got {padding_mode!r}")
        self.padding_mode = padding_mode
        self.fill = fill

    def _crop_or_pad(self, target_shape, **kwargs: Any) -> CropOrPad:
        return CropOrPad(target_shape=target_shape, padding_mode=self.padding_mode, fill=self.fill,
                         only_crop=self.method == "crop", only_pad=self.method == "pad",
                         include=self.include, exclude=self.exclude, **kwargs)

    def forward(self, data: Any) -> Any:
        if isinstance(data, (Subject, Image)):
            target = _compute_target_shape(data.spatial_shape, self.target_multiple, self.method)
            return self._crop_or_pad(target, p=self.p, copy=self.copy).forward(data)
        return super().forward(data)

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        current = tuple(int(v) for v in next(iter(batch.images.values())).data.shape[-3:])
        return {"target_shape": _compute_target_shape(current, self.target_multiple, self.method)}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        crop_or_pad = self._crop_or_pad(params["target_shape"], copy=False)
        inner = crop_or_pad.make_params(batch)
        # the reference runs Compose([Pad, Crop]) here: one gate draw for each (p = 1)
        for _ in range((inner["padding"] is not None) + (inner["cropping"] is not None)):
            torch.rand(1)
        return crop_or_pad.apply_transform(batch, inner)


class CopyAffine(SpatialTransform):
    """Copy each element's affine of image ``target`` to every other image, include / exclude
    notwithstanding (copy_affine.py:12-57)."""

    def __init__(self, target: str, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.target = target

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        if self.target not in batch.images:
            raise KeyError(f"Reference image '{self.target}' not found. Available: {list(batch.images.keys())}")
        reference = batch.images[self.target].affines
        for name, ib in batch.images.items():
            if name == self.target:
                continue
            for index in range(len(ib.affines)):
                ib.affines[index] = reference[index].clone()
        return batch


class ToReferenceSpace(SpatialTransform):
    """Give each selected image the affine that spreads its grid over the field of view of
    ``reference`` with the same centre and orientation (to_reference_space.py:17-132)."""

    def __init__(self, reference: Image, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        if not isinstance(reference, Image):
            raise TypeError(f"reference must be a TorchIO Image, got {type(reference).__name__}")
        self.reference = reference

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for ib in self._get_images(batch).values():
            shape = (int(ib.data.shape[2]), int(ib.data.shape[3]), int(ib.data.shape[4]))
            new_affine = reference_space_affine(self.reference, shape)
            ib.affines[:] = [new_affine.clone() for _ in ib.affines]
        return batch

    @staticmethod
    def from_tensor(tensor: Tensor, reference: Image) -> Image:
        """An image of ``reference``'s class holding ``tensor`` (C, I, J, K) in the reference space."""
        shape = (int(tensor.shape[-3]), int(tensor.shape[-2]), int(tensor.shape[-1]))
        return type(reference)(tensor, affine=reference_space_affine(reference, shape))


def reference_space_affine(reference: Image, output_shape) -> AffineMatrix:
    """Same centre and direction as ``reference``, spacing scaled by the size ratio
    (to_reference_space.py:98-132, float64)."""
    ref_affine = reference.affine
    rotation = np.asarray(ref_affine.direction, dtype=np.float64)
    ref_spacing = np.asarray(ref_affine.spacing, dtype=np.float64)
    ref_origin = np.asarray(ref_affine.origin, dtype=np.float64)
    ref_shape = np.asarray(reference.spatial_shape, dtype=np.float64)
    new_shape = np.asarray(output_shape, dtype=np.float64)
    new_spacing = ref_spacing * (ref_shape / new_shape)
    center = ref_origin + rotation @ (((ref_shape - 1) / 2) * ref_spacing)
    new_origin = center - rotation @ (((new_shape - 1) / 2) * new_spacing)
    matrix = np.eye(4, dtype=np.float64)
    matrix[:3, :3] = rotation * new_spacing
    matrix[:3, 3] = new_origin
    return AffineMatrix(matrix)
