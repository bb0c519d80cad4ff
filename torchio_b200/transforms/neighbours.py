"""Flip, Crop, Pad — the index-remap neighbours of the augmentation chain
(host-side mirror of transforms/spatial/flip.py, crop.py, pad.py, _padding.py,
TorchIO 2.0.0a2; SURVEY §8 f-3).

Same constructor arguments, ``params`` and RNG draws as the reference (Flip draws
``torch.rand(3)`` per element, spatial/flip.py:133,173); the data movement is one
`ops.remap` launch per image (flip + crop + pad are the same kernel with different
offsets), and affines are updated exactly as the reference does (crop/pad shift the
origin, flip leaves the affine untouched).
"""

from __future__ import annotations

import math
import warnings
from collections.abc import Sequence
from typing import Any

import numpy as np
import torch

from .. import ops
from ..data import SubjectsBatch
from .base import SpatialTransform

_LABEL_TO_AXIS = {"L": ("L", "R"), "R": ("L", "R"), "A": ("A", "P"), "P": ("A", "P"),
                  "I": ("I", "S"), "S": ("I", "S")}


def _resolve_axes(axes, orientation=None) -> tuple[int, ...]:
    """ints / anatomical strings -> sorted unique ints in {0,1,2} (flip.py:25-66)."""
    if isinstance(axes, (int, str)):
        axes = (axes,)
    result: list[int] = []
    for axis in axes:
        if isinstance(axis, int):
            if axis not in (0, 1, 2):
                raise ValueError(f"Axis must be 0, 1, or 2; got {axis}")
            result.append(axis)
        elif isinstance(axis, str):
            letter = axis[0].upper()
            if letter not in _LABEL_TO_AXIS:
                raise ValueError(
                    f"Unknown anatomical label {axis!r}."
                    " Use L, R, A, P, I, S or full names"
                    " like 'Left', 'Right', etc."
                )
            if orientation is None:
                raise ValueError(
                    "Cannot resolve anatomical axis label"
                    f" {axis!r} without image orientation"
                )
            pair = _LABEL_TO_AXIS[letter]
            for dim, code in enumerate(orientation):
                if code in pair:
                    result.append(dim)
                    break
        else:
            raise TypeError(f"Axis must be int or str, got {type(axis).__name__}")
    return tuple(sorted(set(result)))


def _flip_images(transform, batch, axes_per_element) -> None:
    """axes_per_element: one iterable of spatial axes per batch element."""
    bits = np.asarray([sum(1 << int(a) for a in set(axes)) for axes in axes_per_element], dtype=np.uint8)
    if not bits.any():
        return
    for ib in transform._get_images(batch).values():
        (flags,) = ops.upload(ib.data.device, bits)
        ib.data = ops.remap(ib.data, ib.data.shape[2:], (0, 0, 0), flip=flags)


class Flip(SpatialTransform):
    """Reverse voxel order along spatial axes (flip.py:69-214)."""

    def __init__(self, *, axes: int | str | Sequence[int | str] = 0, flip_probability: float = 1.0,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.axes = axes
        if not 0 <= flip_probability <= 1:
            raise ValueError(f"flip_probability must be in [0, 1], got {flip_probability}")
        self.flip_probability = flip_probability

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        images = self._get_images(batch)
        if not images:
            return {"axes": ()}
        first = next(iter(images.values()))
        n = self._resolve_n(batch)
        if n is None:
            orientation = first.affines[0].orientation if first.batch_size > 0 else None
            resolved = _resolve_axes(self.axes, orientation)
            mask = torch.rand(3) < self.flip_probability
            return {"axes": tuple(a for a in resolved if mask[a].item())}
        keep = self._keep_mask(batch, n)
        axes_list: list[list[int]] = []
        for index in range(n):
            if keep is not None and not keep[index]:
                axes_list.append([])
                continue
            resolved = _resolve_axes(self.axes, first.affines[index].orientation)
            mask = torch.rand(3) < self.flip_probability
            axes_list.append([a for a in resolved if mask[a].item()])
        params = {"axes": axes_list}
        self._tag_batched(params, batch, n, keep, ["axes"])
        return params

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return True

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        axes = params["axes"]
        if self._is_per_instance_params(params):
            _flip_images(self, batch, axes)
        elif axes:
            _flip_images(self, batch, [axes] * batch.batch_size)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]):
        """Flip is its own inverse (flip.py:206-214)."""
        if self._is_per_instance_params(params):
            return _FlipInverse(axes_per_element=params["axes"], copy=False)
        return Flip(axes=params["axes"], copy=False)


class _FlipInverse(SpatialTransform):
    def __init__(self, *, axes_per_element, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self._axes_per_element = axes_per_element

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        _flip_images(self, batch, self._axes_per_element)
        return batch


def _parse_six(value, what: str) -> tuple[int, int, int, int, int, int]:
    """int / 3-tuple / 6-tuple -> (i_ini, i_fin, j_ini, j_fin, k_ini, k_fin) (crop.py:20-33)."""
    if isinstance(value, int):
        return (value,) * 6
    values = list(value)
    if len(values) == 3:
        i, j, k = values
        return (i, i, j, j, k, k)
    if len(values) == 6:
        return tuple(values)
    raise ValueError(f"{what} must have 1, 3, or 6 values, got {len(values)}")


def _shift_origins(ib, voxels) -> None:
    """origin += direction·spacing @ voxels for every affine of the batch (crop.py:96-101)."""
    shift = np.asarray(voxels, dtype=np.float64)
    for index, affine in enumerate(ib.affines):
        matrix = affine.numpy().copy()
        matrix[:3, 3] = matrix[:3, 3] + matrix[:3, :3] @ shift
        ib.affines[index] = type(affine)(matrix)


class Crop(SpatialTransform):
    """Remove a border of voxels from each side of the volume (crop.py:36-112)."""

    def __init__(self, *, cropping, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.cropping = _parse_six(cropping, "Cropping")

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {"cropping": self.cropping}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        i0, i1, j0, j1, k0, k1 = params["cropping"]
        for ib in self._get_images(batch).values():
            si, sj, sk = ib.data.shape[-3:]
            out = (si - i0 - i1, sj - j0 - j1, sk - k0 - k1)
            if min(out) <= 0:
                raise ValueError(f"cropping {tuple(params['cropping'])} leaves no voxels of {(si, sj, sk)}")
            ib.data = ops.remap(ib.data, out, (-i0, -j0, -k0))
            _shift_origins(ib, (i0, j0, k0))
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]):
        return Pad(padding=params["cropping"], copy=False)


_PADDING_MODES = ("constant", "reflect", "replicate", "circular", "mean", "median", "minimum")


def _padding_statistics(data, mode: str) -> list:
    """One whole-volume statistic per batch element (`_compute_padding_statistic`,
    _padding.py:41-68), computed where the batch lives: minimum = `tio_min_sample0` over the
    element, mean = `tio_moments` (fp64 sums; the reference's fp32 `mean()` agrees to rounding),
    median = the exact radix select behind `compute_quantile(values, 0.5)`.  fp64 data keeps its
    mean and median in fp64 as the reference does, through torch's own ops (kthvalue + lerp)."""
    from .intensity import _lerp_f32

    b = data.shape[0]
    if mode == "minimum":
        if data.dtype == torch.float32:
            mins = [ops.min_sample0(data[i:i + 1].reshape(1, 1, -1, 1, 1)) for i in range(b)]
            return torch.cat(mins).tolist()
        return data.flatten(start_dim=1).amin(dim=1).tolist()
    if data.dtype == torch.float64:
        flat = data.flatten(start_dim=1)
        if mode == "mean":
            return flat.mean(dim=1).tolist()
        index = 0.5 * (flat.shape[1] - 1)
        lower = math.floor(index)
        values = []
        for row in flat:
            median = row.kthvalue(lower + 1).values
            if index != lower:
                median = median.lerp(row.kthvalue(lower + 2).values, index - lower)
            values.append(float(median))
        return values
    if not torch.is_floating_point(data):
        warnings.warn(
            f'The constant value computed for padding mode "{mode}"'
            " might be truncated in the output, as the data type of the input"
            " image is not float. Consider converting the image to a floating"
            " point type before applying this transform.",
            RuntimeWarning, stacklevel=4)
    flat = data if data.dtype == torch.float32 else data.float()
    values = []
    for i in range(b):
        element = flat[i].reshape(-1)
        if mode == "mean":
            total, _, count = ops.moments(element)
            values.append(float(np.float32(total / count)))
        else:
            neighbours, weights, _ = ops.quantile_neighbours(element, [0.5])
            values.append(neighbours[0] if weights[0] == 0
                          else _lerp_f32(neighbours[0], neighbours[1], weights[0]))
    return values


def _remap_padded(data, out_shape, offsets, mode: str, fill):
    """`ops.remap` with F.pad's modes, or a constant pad per element with its own whole-volume
    statistic (`pad_tensor`, _padding.py:71-110)."""
    if mode in ops.PAD_MODES:
        return ops.remap(data, out_shape, offsets, mode=mode, fill=fill)
    statistics = _padding_statistics(data, mode)
    out = torch.empty((*data.shape[:2], *out_shape), dtype=data.dtype, device=data.device)
    for i, value in enumerate(statistics):
        ops.remap(data[i:i + 1], out_shape, offsets, mode="constant", fill=value, out=out[i:i + 1])
    return out


class Pad(SpatialTransform):
    """Add a border of voxels to each side of the volume (pad.py:37-122)."""

    def __init__(self, *, padding, padding_mode: str = "constant", fill: float = 0, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.padding = _parse_six(padding, "Padding")
        if padding_mode not in _PADDING_MODES:
            raise ValueError(f"padding_mode must be one of {_PADDING_MODES}, got {padding_mode!r}")
        self.padding_mode = padding_mode
        self.fill = fill

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {"padding": self.padding, "padding_mode": self.padding_mode, "fill": self.fill}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        i0, i1, j0, j1, k0, k1 = params["padding"]
        mode = params["padding_mode"]
        for ib in self._get_images(batch).values():
            si, sj, sk = ib.data.shape[-3:]
            ib.data = _remap_padded(ib.data, (si + i0 + i1, sj + j0 + j1, sk + k0 + k1), (i0, j0, k0),
                                    mode, params["fill"])
            _shift_origins(ib, (-i0, -j0, -k0))
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]):
        return Crop(cropping=params["padding"], copy=False)


# ---- CropOrPad (spatial/crop_or_pad.py, batched path) --------------------------------


def _parse_target_shape(target_shape):
    """int/float or 3-tuple (None = keep that axis) -> 3-tuple of float|None (crop_or_pad.py:50-66)."""
    if isinstance(target_shape, (int, float)):
        return (float(target_shape),) * 3
    values = list(target_shape)
    if len(values) == 3:
        return tuple(None if v is None else float(v) for v in values)
    raise ValueError(f"target_shape must have 1 or 3 values, got {len(values)}")


def _to_voxels(target, units, spacing, current_shape):
    """Target in voxels / mm / cm -> integer voxels per axis (crop_or_pad.py:69-88)."""
    result = []
    for t, sp, cur in zip(target, spacing, current_shape, strict=True):
        if t is None:
            result.append(cur)
        elif units == "voxels":
            result.append(round(t))
        else:
            result.append(round(t * (10.0 if units == "cm" else 1.0) / sp))
    return tuple(result)


def _split_per_axis(diff: int, location: str):
    """((pad_ini, pad_fin), (crop_ini, crop_fin)) for one axis (crop_or_pad.py:91-107);
    a random crop position draws one ``torch.randint`` per cropped axis."""
    import math

    if diff > 0:
        return (math.ceil(diff / 2), math.floor(diff / 2)), (0, 0)
    if diff < 0:
        amount = -diff
        ini = int(torch.randint(0, amount + 1, (1,)).item()) if location == "random" else math.ceil(amount / 2)
        return (0, 0), (ini, amount - ini)
    return (0, 0), (0, 0)


class CropOrPad(SpatialTransform):
    """Crop and/or pad to a target spatial shape (crop_or_pad.py:381-635, tensor-backed
    batched path).  The reference applies ``Compose([Pad, Crop])`` — two copies and two
    history records; here both index moves are one `ops.remap` launch per image, and the
    same ``Pad`` and ``Crop`` records are appended to the history so that replay and
    inversion behave identically."""

    def __init__(self, target_shape, *, units: str = "voxels", padding_mode: str = "constant",
                 fill: float = 0, only_crop: bool = False, only_pad: bool = False,
                 location: str = "center", **kwargs: Any) -> None:
        super().__init__(**kwargs)
        if only_crop and only_pad:
            raise ValueError("only_crop and only_pad cannot both be True")
        if units not in ("voxels", "mm", "cm"):
            raise ValueError(f"units must be 'voxels', 'mm', or 'cm', got {units!r}")
        if location not in ("center", "random"):
            raise ValueError(f"location must be 'center' or 'random', got {location!r}")
        if padding_mode not in _PADDING_MODES:
            raise ValueError(f"padding_mode must be one of {_PADDING_MODES}, got {padding_mode!r}")
        self.target_shape = _parse_target_shape(target_shape)
        self.units = units
        self.padding_mode = padding_mode
        self.fill = fill
        self.only_crop = only_crop
        self.only_pad = only_pad
        self.location = location

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        first = next(iter(batch.images.values()))
        current = tuple(int(v) for v in first.data.shape[-3:])
        target = _to_voxels(self.target_shape, self.units, first.affines[0].spacing, current)
        pad_values: list[int] = []
        crop_values: list[int] = []
        for cur, tgt in zip(current, target, strict=True):
            pad, crop = _split_per_axis(tgt - cur, self.location)
            pad_values.extend(pad)
            crop_values.extend(crop)
        padding = tuple(pad_values) if any(v > 0 for v in pad_values) and not self.only_crop else None
        cropping = tuple(crop_values) if any(v > 0 for v in crop_values) and not self.only_pad else None
        return {"padding": padding, "cropping": cropping}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        padding, cropping = params["padding"], params["cropping"]
        if padding is None and cropping is None:
            return batch
        p = padding or (0,) * 6
        c = cropping or (0,) * 6
        for ib in self._get_images(batch).values():
            si, sj, sk = ib.data.shape[-3:]
            out = (si + p[0] + p[1] - c[0] - c[1], sj + p[2] + p[3] - c[2] - c[3], sk + p[4] + p[5] - c[4] - c[5])
            ib.data = _remap_padded(ib.data, out, (p[0] - c[0], p[2] - c[2], p[4] - c[4]),
                                    self.padding_mode if padding is not None else "constant", self.fill)
            _shift_origins(ib, (c[0] - p[0], c[2] - p[2], c[4] - p[4]))
        # the records Compose([Pad, Crop]) leaves behind (crop_or_pad.py:609-633)
        from .base import AppliedTransform

        include = None if self.include is None else list(self.include)
        exclude = None if self.exclude is None else list(self.exclude)
        if padding is not None:
            batch.applied_transforms.append(AppliedTransform(
                name="Pad", params={"padding": tuple(padding), "padding_mode": self.padding_mode, "fill": self.fill},
                include=include, exclude=exclude))
        if cropping is not None:
            batch.applied_transforms.append(AppliedTransform(
                name="Crop", params={"cropping": tuple(cropping)}, include=include, exclude=exclude))
        return batch
