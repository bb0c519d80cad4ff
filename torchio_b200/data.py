"""Tensor-backed data model the hot path reads and writes.

Host-side mirror of the reference containers (TorchIO 2.0.0a2, paths relative
to src/torchio/):
  AffineMatrix   data/affine.py:20      Image/ScalarImage/LabelMap  data/image.py:104,1238,1251
  Subject        data/subject.py:25     ImagesBatch/SubjectsBatch   data/batch.py:21,124
  Invertible     data/invertible.py:10
Only what the augmentation path touches is provided: tensor-backed images,
metadata, history and batching.  File-backed lazy loading, points and bounding
boxes are out of scope (SURVEY.md §2 rows 10, 18, 19).

Design difference: affines always live on the host as float64 numpy arrays
(the reference keeps them as torch tensors that follow the image to the GPU,
which costs a device sync per ``.spacing`` read).
"""

from __future__ import annotations

import copy
import dataclasses
from typing import Any

import numpy as np
import torch
from torch import Tensor

_BATCH_META_KEYS = ("_batch_size", "_batched_keys", "_keep")

# ---- nibabel.orientations, restated (the reference's Reorient and AffineMatrix.orientation) ----
# An "ornt" is a (3, 2) float64 array: row = input axis, [output axis, +1 / -1 direction].
_AXIS_LABELS = (("L", "R"), ("P", "A"), ("I", "S"))


def _io_orientation(affine: np.ndarray) -> np.ndarray:
    """Axis permutation and flips closest to the direction part of ``affine``: polar decomposition
    by SVD, then per input axis the output axis of largest magnitude, taken greedily."""
    rzs = np.asarray(affine, dtype=np.float64)[:3, :3]
    zooms = np.sqrt(np.sum(rzs * rzs, axis=0))
    zooms[zooms == 0] = 1
    rs = rzs / zooms
    p, s, qs = np.linalg.svd(rs, full_matrices=False)
    keep = s > s.max() * 3 * np.finfo(s.dtype).eps
    r = np.dot(p[:, keep], qs[keep])
    ornt = np.ones((3, 2), dtype=np.int8) * np.nan
    for in_ax in range(3):
        col = r[:, in_ax]
        if not np.allclose(col, 0):
            out_ax = np.argmax(np.abs(col))
            ornt[in_ax, 0] = out_ax
            ornt[in_ax, 1] = -1 if col[out_ax] < 0 else 1
            r[out_ax, :] = 0
    return ornt


def _axcodes2ornt(axcodes) -> np.ndarray:
    """Orientation of axis codes such as "RAS" (L/P/I = −1, R/A/S = +1)."""
    ornt = np.ones((len(axcodes), 2), dtype=np.int8) * np.nan
    for code_idx, code in enumerate(axcodes):
        for label_idx, codes in enumerate(_AXIS_LABELS):
            if code in codes:
                ornt[code_idx, :] = [label_idx, -1 if code == codes[0] else 1]
                break
    return ornt


def _ornt_transform(start_ornt: np.ndarray, end_ornt: np.ndarray) -> np.ndarray:
    """The orientation that takes data in ``start_ornt`` to ``end_ornt``."""
    result = np.empty_like(start_ornt)
    for end_in_idx, (end_out_idx, end_flip) in enumerate(end_ornt):
        for start_in_idx, (start_out_idx, start_flip) in enumerate(start_ornt):
            if end_out_idx == start_out_idx:
                result[start_in_idx, :] = [end_in_idx, 1 if start_flip == end_flip else -1]
                break
        else:
            raise ValueError("Unable to find out axis %d in start_ornt" % end_out_idx)
    return result


def _inv_ornt_aff(ornt: np.ndarray, shape) -> np.ndarray:
    """Affine from the voxel grid after applying ``ornt`` to an array of ``shape`` back to the
    original grid: undo the transpose, then the flips about the array's centre."""
    shape = np.array(shape)[:3]
    axis_transpose = [int(v) for v in ornt[:, 0]]
    undo_reorder = np.eye(4)[axis_transpose + [3], :]
    undo_flip = np.diag(list(ornt[:, 1]) + [1.0])
    center_trans = -(shape - 1) / 2.0
    undo_flip[:3, 3] = (ornt[:, 1] * center_trans) - center_trans
    return np.dot(undo_flip, undo_reorder)


class AffineMatrix:
    """4x4 voxel->world matrix (float64, host)."""

    __slots__ = ("_m", "_spacing")

    def __init__(self, matrix: Any = None) -> None:
        if matrix is None:
            m = np.eye(4, dtype=np.float64)
        elif isinstance(matrix, AffineMatrix):
            m = matrix._m.copy()
        elif isinstance(matrix, Tensor):
            m = matrix.detach().to("cpu", torch.float64).numpy().copy()
        else:
            m = np.array(matrix, dtype=np.float64)
        if m.shape != (4, 4):
            raise ValueError(f"AffineMatrix must be 4x4, got {tuple(m.shape)}")
        self._m = m
        self._spacing = None  # cached; treat the matrix as immutable after construction

    @classmethod
    def from_spacing(cls, spacing, *, origin=(0.0, 0.0, 0.0), direction=None):
        m = np.eye(4, dtype=np.float64)
        if direction is not None:
            m[:3, :3] = np.asarray(direction, dtype=np.float64)
        m[:3, :3] *= np.asarray(spacing, dtype=np.float64)
        m[:3, 3] = origin
        return cls(m)

    @property
    def data(self) -> Tensor:
        return torch.from_numpy(self._m)

    def numpy(self) -> np.ndarray:
        return self._m

    @property
    def spacing(self) -> tuple[float, float, float]:
        if self._spacing is None:
            sp = np.sqrt(np.sum(self._m[:3, :3] ** 2, axis=0))
            self._spacing = (float(sp[0]), float(sp[1]), float(sp[2]))
        return self._spacing

    @property
    def origin(self) -> tuple[float, float, float]:
        o = self._m[:3, 3]
        return (float(o[0]), float(o[1]), float(o[2]))

    @property
    def direction(self) -> np.ndarray:
        rz = self._m[:3, :3]
        return rz / np.sqrt(np.sum(rz**2, axis=0))

    @property
    def orientation(self) -> tuple[str, str, str]:
        """Anatomical axis codes, e.g. ('R','A','S') (data/affine.py:124-128 = nibabel's
        aff2axcodes: closest axis permutation/flips of the direction part, via its SVD)."""
        codes: list[str | None] = [None, None, None]
        for in_ax, (out_ax, direction) in enumerate(_io_orientation(self._m)):
            if not np.isnan(out_ax):
                codes[in_ax] = _AXIS_LABELS[int(out_ax)][0 if direction < 0 else 1]
        return (codes[0], codes[1], codes[2])

    def to(self, *args: Any, **kwargs: Any) -> AffineMatrix:
        return self  # host-resident by design

    def clone(self) -> AffineMatrix:
        return AffineMatrix(self._m)

    def inverse(self) -> AffineMatrix:
        return AffineMatrix(np.linalg.inv(self._m))

    def __matmul__(self, other: object) -> AffineMatrix:
        if not isinstance(other, AffineMatrix):
            return NotImplemented
        return AffineMatrix(self._m @ other._m)

    def __array__(self, dtype=None, copy=None):
        return self._m.astype(dtype) if dtype is not None else self._m

    def __eq__(self, other: object) -> bool:
        if not isinstance(other, AffineMatrix):
            return NotImplemented
        return bool(np.array_equal(self._m, other._m))

    def __repr__(self) -> str:
        sp = ", ".join(f"{s:.2f}" for s in self.spacing)
        o = ", ".join(f"{v:.2f}" for v in self.origin)
        return f"AffineMatrix(spacing=({sp}), origin=({o}))"

    def __deepcopy__(self, memo: dict) -> AffineMatrix:
        return self.clone()

    __copy__ = clone


def _clone_keeping_pin(t: torch.Tensor) -> torch.Tensor:
    """``t.clone()``, but a page-locked host tensor stays page-locked: a deep copy of a pinned
    batch (Transform(copy=True)) must still stream to the device with asynchronous copies."""
    if t.device.type == "cpu" and t.is_pinned():
        return torch.empty_like(t, pin_memory=True).copy_(t)
    return t.clone()


class Invertible:
    """History carrier (data/invertible.py:10-75)."""

    applied_transforms: list[Any]

    def get_inverse_transform(self, *, warn: bool = True, ignore_intensity: bool = False):
        from .transforms.inverse import get_inverse_transform

        return get_inverse_transform(
            self.applied_transforms, warn=warn, ignore_intensity=ignore_intensity
        )

    def apply_inverse_transform(self, **kwargs: Any):
        result = self.get_inverse_transform(**kwargs)(self)
        if hasattr(result, "applied_transforms"):
            result.applied_transforms = []
        return result

    def clear_history(self) -> None:
        self.applied_transforms = []


class Image(Invertible):
    """A (C, I, J, K) tensor plus its affine and free-form metadata."""

    def __init__(self, source: Any = None, *, affine: Any = None, **metadata: Any):
        if source is None:
            raise ValueError("torchio_b200 images are tensor-backed: pass a 4D tensor")
        if isinstance(source, np.ndarray):
            source = torch.as_tensor(source.copy())
        if not isinstance(source, Tensor):
            raise TypeError(
                "torchio_b200 images are tensor-backed (file I/O is out of scope);"
                f" got {type(source).__name__}"
            )
        if source.ndim != 4:
            raise ValueError(f"Tensor must be 4D (C, I, J, K), got {source.ndim}D")
        self._data = source
        self._affine = affine if isinstance(affine, AffineMatrix) else AffineMatrix(affine)
        self._metadata = dict(metadata)
        self.applied_transforms: list[Any] = []

    @property
    def data(self) -> Tensor:
        return self._data

    def set_data(self, tensor: Tensor) -> None:
        if tensor.ndim != 4:
            raise ValueError(f"Tensor must be 4D (C, I, J, K), got {tensor.ndim}D")
        self._data = tensor

    @property
    def affine(self) -> AffineMatrix:
        return self._affine

    @property
    def metadata(self) -> dict[str, Any]:
        return self._metadata

    @property
    def shape(self) -> tuple[int, int, int, int]:
        return tuple(self._data.shape)  # type: ignore[return-value]

    @property
    def spatial_shape(self) -> tuple[int, int, int]:
        return tuple(self._data.shape[1:])  # type: ignore[return-value]

    @property
    def num_channels(self) -> int:
        return int(self._data.shape[0])

    @property
    def spacing(self) -> tuple[float, float, float]:
        return self._affine.spacing

    @property
    def origin(self) -> tuple[float, float, float]:
        return self._affine.origin

    @property
    def dtype(self) -> torch.dtype:
        return self._data.dtype

    @property
    def device(self) -> torch.device:
        return self._data.device

    @property
    def is_loaded(self) -> bool:
        return True

    def load(self) -> None:
        return None

    def to(self, *args: Any, **kwargs: Any):
        self._data = self._data.to(*args, **kwargs)
        return self

    def numpy(self) -> np.ndarray:
        return self._data.detach().cpu().numpy()

    def new_like(self, *, data: Tensor, affine: Any = None):
        return type(self)(
            data, affine=self._affine.clone() if affine is None else affine, **self._metadata
        )

    def __getitem__(self, index):
        """Spatial slicing image[:, i, j, k] -> view + origin-shifted affine
        (data/image.py:832-899); the channel axis must be a full slice."""
        if not isinstance(index, tuple):
            index = (index,)
        index = index + (slice(None),) * (4 - len(index))
        starts = []
        for ax in range(1, 4):
            s = index[ax]
            if not isinstance(s, slice) or s.step not in (None, 1):
                raise IndexError("only contiguous spatial slices are supported")
            starts.append(s.indices(self._data.shape[ax])[0])
        m = self._affine.numpy().copy()
        m[:3, 3] = m[:3, 3] + m[:3, :3] @ np.asarray(starts, dtype=np.float64)
        return type(self)(self._data[index], affine=m, **self._metadata)

    def __getattr__(self, name: str) -> Any:
        if name.startswith("_"):
            raise AttributeError(name)
        meta = self.__dict__.get("_metadata", {})
        if name in meta:
            return meta[name]
        raise AttributeError(f"{type(self).__name__} has no attribute {name!r}")

    def __deepcopy__(self, memo: dict):
        new = type(self)(_clone_keeping_pin(self._data), affine=self._affine.clone(), **self._metadata)
        new.applied_transforms = list(self.applied_transforms)
        memo[id(self)] = new
        return new

    def __copy__(self):
        return self.new_like(data=self._data.clone())

    def __repr__(self) -> str:
        return (
            f"{type(self).__name__}(shape={tuple(self._data.shape)},"
            f" dtype={self._data.dtype}, device={self._data.device})"
        )


class ScalarImage(Image):
    """Intensity image (trilinear resampling, intensity transforms apply)."""


class LabelMap(Image):
    """Segmentation (nearest-neighbour resampling, intensity transforms skip)."""


class Subject(Invertible):
    """Named images + metadata (data/subject.py:25-100)."""

    def __init__(self, **kwargs: Any) -> None:
        if not kwargs:
            raise ValueError("A Subject must contain at least one entry")
        self._images: dict[str, Image] = {}
        self._metadata: dict[str, Any] = {}
        for key, value in kwargs.items():
            (self._images if isinstance(value, Image) else self._metadata)[key] = value
        self.applied_transforms: list[Any] = []

    @property
    def images(self) -> dict[str, Image]:
        return self._images

    @property
    def metadata(self) -> dict[str, Any]:
        return self._metadata

    def __getattr__(self, name: str) -> Any:
        if name.startswith("_"):
            raise AttributeError(name)
        for store in ("_images", "_metadata"):
            d = self.__dict__.get(store, {})
            if name in d:
                return d[name]
        raise AttributeError(f"{type(self).__name__} has no attribute {name!r}")

    def __getitem__(self, item: str) -> Any:
        if item in self._images:
            return self._images[item]
        return self._metadata[item]

    def __contains__(self, name: object) -> bool:
        return name in self._images or name in self._metadata

    def __iter__(self):
        return iter([*self._images, *self._metadata])

    def __len__(self) -> int:
        return len(self._images) + len(self._metadata)

    def _first(self) -> Image:
        return next(iter(self._images.values()))

    @property
    def spatial_shape(self):
        return self._first().spatial_shape

    @property
    def shape(self):
        return self._first().shape

    @property
    def spacing(self):
        return self._first().spacing

    @property
    def device(self) -> torch.device:
        return self._first().device

    def load(self) -> None:
        return None

    def to(self, *args: Any, **kwargs: Any):
        for img in self._images.values():
            img.to(*args, **kwargs)
        return self

    def __deepcopy__(self, memo: dict):
        kwargs = {k: copy.deepcopy(v, memo) for k, v in self._images.items()}
        kwargs.update({k: copy.deepcopy(v, memo) for k, v in self._metadata.items()})
        new = type(self)(**kwargs)
        new.applied_transforms = list(self.applied_transforms)
        return new

    def __repr__(self) -> str:
        return f"Subject(images=[{', '.join(self._images)}])"


class ImagesBatch(Invertible):
    """(B, C, I, J, K) tensor + one affine per sample (data/batch.py:21-121)."""

    def __init__(self, data: Tensor, affines: list[AffineMatrix], *, image_class=ScalarImage):
        if data.ndim != 5:
            raise ValueError(f"Expected 5D tensor (B, C, I, J, K), got {data.ndim}D")
        if len(affines) != data.shape[0]:
            raise ValueError(f"Expected {data.shape[0]} affines, got {len(affines)}")
        self._data = data
        self._affines = affines
        self._image_class = image_class
        self.applied_transforms: list[Any] = []

    @classmethod
    def from_images(cls, images: list[Image]):
        if not images:
            raise ValueError("Cannot create batch from empty list")
        data = torch.stack([img.data for img in images])
        return cls(data, [img.affine.clone() for img in images], image_class=type(images[0]))

    @property
    def data(self) -> Tensor:
        return self._data

    @data.setter
    def data(self, value: Tensor) -> None:
        if value.ndim != 5:
            raise ValueError(f"Expected 5D tensor, got {value.ndim}D")
        self._data = value

    @property
    def affines(self) -> list[AffineMatrix]:
        return self._affines

    @property
    def batch_size(self) -> int:
        return int(self._data.shape[0])

    @property
    def device(self) -> torch.device:
        return self._data.device

    def to(self, *args: Any, **kwargs: Any):
        self._data = self._data.to(*args, **kwargs)
        return self

    def __getitem__(self, index: int) -> Image:
        return self._image_class(self._data[index], affine=self._affines[index].clone())

    def __len__(self) -> int:
        return self.batch_size

    def unbatch(self) -> list[Image]:
        return [self[i] for i in range(self.batch_size)]

    def __deepcopy__(self, memo: dict):
        new = type(self)(
            _clone_keeping_pin(self._data), [a.clone() for a in self._affines], image_class=self._image_class
        )
        new.applied_transforms = list(self.applied_transforms)
        return new

    def __repr__(self) -> str:
        b, c, i, j, k = self._data.shape
        return (
            f"ImagesBatch({self._image_class.__name__}, batch_size={b},"
            f" shape=({c}, {i}, {j}, {k}))"
        )


class SubjectsBatch(Invertible):
    """Dict of ImagesBatch + per-sample metadata lists (data/batch.py:124-330)."""

    def __init__(self, images: dict[str, ImagesBatch], *, metadata=None) -> None:
        self._images = images
        self._metadata: dict[str, list[Any]] = metadata or {}
        self.applied_transforms: list[Any] = []
        self._per_element_history: list[list[Any]] | None = None

    @classmethod
    def from_subjects(cls, subjects: list[Subject]):
        if not subjects:
            raise ValueError("Cannot create batch from empty list")
        first = subjects[0]
        images = {
            name: ImagesBatch.from_images([s.images[name] for s in subjects])
            for name in first.images
        }
        metadata = {k: [s.metadata[k] for s in subjects] for k in first.metadata}
        return cls(images, metadata=metadata)

    @property
    def batch_size(self) -> int:
        return next(iter(self._images.values())).batch_size

    @property
    def images(self) -> dict[str, ImagesBatch]:
        return self._images

    @property
    def metadata(self) -> dict[str, list[Any]]:
        return self._metadata

    @property
    def device(self) -> torch.device:
        return next(iter(self._images.values())).device

    def to(self, *args: Any, **kwargs: Any):
        for b in self._images.values():
            b.to(*args, **kwargs)
        return self

    def __getitem__(self, key: str) -> ImagesBatch:
        return self._images[key]

    def __getattr__(self, name: str) -> ImagesBatch:
        if name.startswith("_"):
            raise AttributeError(name)
        images = self.__dict__.get("_images", {})
        if name in images:
            return images[name]
        raise AttributeError(f"SubjectsBatch has no attribute {name!r}")

    def __len__(self) -> int:
        return self.batch_size

    def set_per_element_history(self, histories: list[list[Any]]) -> None:
        if len(histories) != self.batch_size:
            raise ValueError(
                f"Expected {self.batch_size} per-element histories, got {len(histories)}"
            )
        self._per_element_history = [list(h) for h in histories]
        self.applied_transforms = []

    def clear_history(self) -> None:
        self.applied_transforms = []
        self._per_element_history = None

    def unbatch(self) -> list[Subject]:
        """Split into Subjects; per-instance history is sliced per element and
        gated-out transforms are dropped (data/batch.py:239-264,365-399)."""
        subjects = []
        for i in range(self.batch_size):
            kwargs: dict[str, Any] = {n: ib[i] for n, ib in self._images.items()}
            kwargs.update({k: v[i] for k, v in self._metadata.items()})
            sub = Subject(**kwargs)
            suffix = slice_history(self.applied_transforms, i)
            if self._per_element_history is not None:
                suffix = list(self._per_element_history[i]) + suffix
            sub.applied_transforms = suffix
            subjects.append(sub)
        return subjects

    def __deepcopy__(self, memo: dict):
        new = type(self)(
            {k: copy.deepcopy(v, memo) for k, v in self._images.items()},
            metadata={k: list(v) for k, v in self._metadata.items()},
        )
        new.applied_transforms = list(self.applied_transforms)
        if self._per_element_history is not None:
            new._per_element_history = [list(h) for h in self._per_element_history]
        return new

    def __repr__(self) -> str:
        return f"SubjectsBatch(batch_size={self.batch_size}, images=[{', '.join(self._images)}])"


StudiesBatch = SubjectsBatch


def slice_history(history: list[Any], index: int) -> list[Any]:
    """Per-subject view of a batch history (data/batch.py:337-399)."""
    out: list[Any] = []
    for trace in history:
        params = getattr(trace, "params", None)
        if not isinstance(params, dict) or "_batched_keys" not in params:
            out.append(trace)
            continue
        size = params.get("_batch_size")
        if size is not None and not 0 <= index < size:
            raise IndexError(
                f"Cannot extract per-instance history for element {index}: the transform"
                f" was recorded for a batch of size {size}"
            )
        keep = params.get("_keep")
        if keep is not None and not keep[index]:
            continue
        batched = params["_batched_keys"]
        sliced = {
            k: (v[index] if k in batched and isinstance(v, list) else v)
            for k, v in params.items()
            if k not in _BATCH_META_KEYS
        }
        out.append(dataclasses.replace(trace, params=sliced))
    return out
