"""Patch path: samplers, Queue and loaders (host-side mirror of
data/patch.py, data/sampler.py, data/queue.py and loader.py, TorchIO 2.0.0a2).

Same classes, constructor arguments, iteration order and RNG draws as the
reference (patch corners come from the global torch CPU generator, three
``torch.randint`` calls per patch in i, j, k order — data/sampler.py:218-223;
subject and buffer shuffles use Python's ``random`` — data/queue.py:167,177).

Difference by design: when a subject's tensors live on the GPU, a `Queue` holds
its patches in a pre-allocated device ring (`PatchRing`): one `ops.crop_patches`
launch per image writes the ``patches_per_volume`` patches of a subject straight into
consecutive slots, the buffer shuffle permutes slot indices, and `collate_subjects`
builds a batch with one ``index_select`` per image — no per-patch `Subject`, no
``torch.stack``.  Host-resident subjects keep the reference's zero-copy views.
``Queue(device=...)`` (extension) moves each loaded subject to that device before
the transform, so augmentation and patch extraction run resident.
"""

from __future__ import annotations

import random as _random
import weakref
from collections import deque
from collections.abc import Iterator, Sequence, Sized
from concurrent.futures import Future, ThreadPoolExecutor
from dataclasses import dataclass
from itertools import islice
from typing import Any

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset, IterableDataset, Sampler

from . import ops
from .data import AffineMatrix, ImagesBatch, Subject, SubjectsBatch


@dataclass(frozen=True)
class PatchLocation:
    """Corner index and size of a patch inside its volume (data/patch.py:11-63)."""

    index: tuple[int, int, int]
    size: tuple[int, int, int]
    subject_index: int | None = None

    @property
    def index_ini(self) -> tuple[int, int, int]:
        return self.index

    @property
    def index_fin(self) -> tuple[int, int, int]:
        return (self.index[0] + self.size[0], self.index[1] + self.size[1],
                self.index[2] + self.size[2])

    def to_slices(self) -> tuple[slice, slice, slice]:
        ini, fin = self.index_ini, self.index_fin
        return (slice(ini[0], fin[0]), slice(ini[1], fin[1]), slice(ini[2], fin[2]))

    def scaled(self, factor: tuple[float, float, float]) -> PatchLocation:
        return PatchLocation(
            index=tuple(round(self.index[a] * factor[a]) for a in range(3)),
            size=tuple(round(self.size[a] * factor[a]) for a in range(3)),
            subject_index=self.subject_index,
        )


class PatchSampler:
    """Base class of patch samplers (data/sampler.py:25-67)."""

    def __init__(self, patch_size) -> None:
        if isinstance(patch_size, int):
            patch_size = (patch_size, patch_size, patch_size)
        self.patch_size = tuple(int(v) for v in patch_size)

    def __call__(self, subject: Subject, num_patches: int | None = None) -> Iterator[Subject]:
        raise NotImplementedError(f"{type(self).__name__} must implement __call__")

    def _extract_patch(self, subject: Subject, location: PatchLocation) -> Subject:
        si, sj, sk = location.to_slices()
        kwargs: dict[str, Any] = {name: image[:, si, sj, sk] for name, image in subject.images.items()}
        kwargs.update(subject.metadata)
        kwargs["patch_location"] = location
        return Subject(**kwargs)

    def _extract_patches(self, subject: Subject, locations: list[PatchLocation]) -> list[Subject]:
        """All ``locations`` of one subject.  Device-resident images: one gather launch
        per image; host-resident: the reference's views."""
        if not locations:
            return []
        images = subject.images
        on_device = all(img.data.is_cuda for img in images.values())
        same_size = all(loc.size == locations[0].size for loc in locations)
        fits = all(p <= s for p, s in zip(locations[0].size, subject.spatial_shape))
        if not (on_device and same_size and fits):  # (an oversized patch is a clamped view, as upstream)
            return [self._extract_patch(subject, loc) for loc in locations]
        corners = np.asarray([loc.index for loc in locations], dtype=np.int32)
        blocks = {name: ops.crop_patches(img.data, corners, locations[0].size) for name, img in images.items()}
        patches = []
        for row, loc in enumerate(locations):
            kwargs: dict[str, Any] = {}
            for name, img in images.items():
                matrix = img.affine.numpy().copy()
                matrix[:3, 3] = matrix[:3, 3] + matrix[:3, :3] @ np.asarray(loc.index, dtype=np.float64)
                kwargs[name] = type(img)(blocks[name][row], affine=matrix, **img.metadata)
            kwargs.update(subject.metadata)
            kwargs["patch_location"] = loc
            patches.append(Subject(**kwargs))
        return patches


class UniformSampler(PatchSampler, IterableDataset):
    """Uniformly random patches (data/sampler.py:165-223)."""

    def __init__(self, subject: Subject, patch_size, num_patches: int | None = None) -> None:
        super().__init__(patch_size)
        self.subject = subject
        self.num_patches = num_patches

    def __call__(self, subject: Subject, num_patches: int | None = None) -> Iterator[Subject]:
        limit = num_patches or self.num_patches
        count = 0
        while limit is None or count < limit:
            loc = PatchLocation(index=self._random_index(subject.spatial_shape), size=self.patch_size)
            yield self._extract_patch(subject, loc)
            count += 1

    def __iter__(self) -> Iterator[Subject]:
        return self(self.subject, self.num_patches)

    def draw_locations(self, subject: Subject, count: int) -> list[PatchLocation]:
        """The locations of the first ``count`` patches ``self(subject)`` would yield (same draws)."""
        shape = subject.spatial_shape
        return [PatchLocation(index=self._random_index(shape), size=self.patch_size) for _ in range(count)]

    def sample(self, subject: Subject, num_patches: int) -> list[Subject]:
        """``list(islice(self(subject), num_patches))`` with the same RNG draws, the
        patches of a device-resident subject gathered in one launch per image."""
        count = num_patches if not self.num_patches else min(num_patches, self.num_patches)
        return self._extract_patches(subject, self.draw_locations(subject, count))

    def _random_index(self, spatial_shape) -> tuple[int, int, int]:
        def _rand(d: int) -> int:
            hi = max(spatial_shape[d] - self.patch_size[d], 0) + 1
            return int(torch.randint(0, hi, (1,)).item())

        return (_rand(0), _rand(1), _rand(2))


class GridSampler(PatchSampler, Dataset):
    """Patches on a regular grid for dense inference (data/sampler.py:70-162)."""

    def __init__(self, subject: Subject, patch_size, patch_overlap=0, padding_mode: str | None = None,
                 fill: float = 0) -> None:
        super().__init__(patch_size)
        if isinstance(patch_overlap, int):
            patch_overlap = (patch_overlap, patch_overlap, patch_overlap)
        self.patch_overlap = tuple(int(v) for v in patch_overlap)
        self.padding_mode = padding_mode
        self.fill = fill
        self.subject = self._maybe_pad(subject)
        self.locations = self._compute_locations(self.subject.spatial_shape)

    def __len__(self) -> int:
        return len(self.locations)

    def __getitem__(self, index: int) -> Subject:
        return self._extract_patch(self.subject, self.locations[index])

    def _maybe_pad(self, subject: Subject) -> Subject:
        if self.padding_mode is None:
            return subject
        from .transforms.neighbours import Pad

        border = tuple(v // 2 for v in self.patch_overlap)
        padding = (border[0], border[0], border[1], border[1], border[2], border[2])
        return Pad(padding=padding, padding_mode=self.padding_mode, fill=self.fill, copy=False)(subject)

    def _compute_locations(self, spatial_shape) -> list[PatchLocation]:
        per_axis: list[list[int]] = []
        for dim in range(3):
            size, patch, overlap = spatial_shape[dim], self.patch_size[dim], self.patch_overlap[dim]
            step = max(patch - overlap, 1)
            indices = list(range(0, size - patch + 1, step))
            if not indices or indices[-1] != size - patch:
                indices.append(max(size - patch, 0))
            per_axis.append(indices)
        return [PatchLocation(index=(i, j, k), size=self.patch_size)
                for i in per_axis[0] for j in per_axis[1] for k in per_axis[2]]


# ---------------------------------------------------------------------------------------
# PatchAggregator: stitch inference patches back into a volume (data/aggregator.py:12-245)
#
# The reference moves every batch to the host and adds its patches one at a time.  Here the
# buffers stay on the device and each `add_batch` is one `tio_aggregate_patches` launch per key:
# the boxes are resolved on the host from the locations alone (Python slice rules, as the
# reference's slicing), checked against the patch shape for the whole batch, and uploaded as one
# table.  Counts are kept as one channel: their update does not depend on the channel.
# ---------------------------------------------------------------------------------------

_AGGREGATOR_MODES = ("crop", "average", "hann")
_ATEN_NAMES = {torch.uint8: "Byte", torch.int8: "Char", torch.int16: "Short", torch.int32: "Int",
               torch.int64: "Long", torch.bool: "Bool"}


def _resolved(start: int, stop: int, n: int) -> tuple[int, int]:
    """``t[start:stop]`` of an axis of ``n`` points as (first index, length)."""
    first, last, _ = slice(start, stop).indices(n)
    return first, max(0, last - first)


class PatchAggregator:
    """Reassemble patches into a full volume (data/aggregator.py:12-245).

    Same constructor, attributes, modes ("crop", "average", "hann") and results as the reference,
    which it reproduces bit for bit.  The buffers live on the device of the first batch added (on
    `execution_device()` when that batch is on the host); `get_output` returns a tensor on the device
    of that first batch.  Differences: a batch is checked as a whole before anything is added, a
    box that only broadcasting would fit and a batch whose dtype differs from the buffer's raise
    `NotImplementedError`, and the counts are one channel instead of C equal ones."""

    def __init__(self, spatial_shape, overlap_mode: str = "crop", patch_overlap=0, output_shape=None) -> None:
        if overlap_mode not in _AGGREGATOR_MODES:
            raise ValueError(f"overlap_mode must be one of {_AGGREGATOR_MODES}, got {overlap_mode!r}")
        self.input_spatial_shape = spatial_shape
        self.overlap_mode = overlap_mode
        if isinstance(patch_overlap, int):
            patch_overlap = (patch_overlap, patch_overlap, patch_overlap)
        self.patch_overlap = patch_overlap
        if output_shape is not None:
            self.spatial_shape = output_shape
            self._scale = tuple(output_shape[a] / spatial_shape[a] for a in range(3))
        else:
            self.spatial_shape = spatial_shape
            self._scale = (1.0, 1.0, 1.0)
        self._outputs: dict[str, torch.Tensor] = {}
        self._counts: dict[str, torch.Tensor] = {}
        self._device: torch.device | None = None
        self._host_caller = False

    def _box(self, location: PatchLocation, patch_shape) -> tuple[tuple[int, int, int], tuple[int, int, int],
                                                                  tuple[int, int, int], tuple[int, int, int]]:
        """Where the reference writes a patch of spatial shape ``patch_shape`` added at ``location``:
        (first destination voxel, destination extent, first source voxel, source extent) per axis,
        the location scaled first when there is an ``output_shape`` (aggregator.py:93-96, 153-237)."""
        if self._scale != (1.0, 1.0, 1.0):
            location = location.scaled(self._scale)
        ini, fin = list(location.index_ini), list(location.index_fin)
        crop_ini, crop_fin = [0, 0, 0], list(patch_shape)
        if self.overlap_mode == "crop":
            crop_fin = list(location.size)
            for a in range(3):
                half = round(self.patch_overlap[a] * self._scale[a]) // 2
                if ini[a] > 0:
                    ini[a] += half
                    crop_ini[a] += half
                if fin[a] < self.spatial_shape[a]:
                    fin[a] -= half
                    crop_fin[a] -= half
        dst = [_resolved(ini[a], fin[a], self.spatial_shape[a]) for a in range(3)]
        src = [_resolved(crop_ini[a], crop_fin[a], patch_shape[a]) for a in range(3)]
        return (tuple(d[0] for d in dst), tuple(d[1] for d in dst), tuple(s[0] for s in src),
                tuple(s[1] for s in src))

    def _device_for(self, tensor: torch.Tensor) -> torch.device:
        if self._device is None:
            self._host_caller = not tensor.is_cuda
            if tensor.is_cuda:
                self._device = tensor.device
            else:
                from .transforms.base import execution_device

                self._device = execution_device()
        return self._device

    def _check_dtype(self, key: str, tensor: torch.Tensor) -> None:
        dtype, mode = tensor.dtype, self.overlap_mode
        if mode == "hann" and not dtype.is_floating_point:
            raise RuntimeError(f"result type Float can't be cast to the desired output type {_ATEN_NAMES[dtype]}")
        if mode == "average" and dtype == torch.bool:
            raise RuntimeError("result type Long can't be cast to the desired output type Bool")
        if key in self._outputs and self._outputs[key].dtype != dtype:
            raise NotImplementedError(
                f"PatchAggregator: a batch of {dtype} for key {key!r}, whose buffer is {self._outputs[key].dtype};"
                f" the reference casts it by type promotion, cast it before add_batch")

    def _table(self, key: str, tensor: torch.Tensor, locations) -> np.ndarray:
        """The batch's box table (n, 10), every box checked against its patch first."""
        if tensor.ndim != 5:
            raise ValueError(f"PatchAggregator.add_batch expects (B, C, I, J, K) tensors, got {tuple(tensor.shape)}"
                             f" for key {key!r}")
        if len(locations) > tensor.shape[0]:
            raise IndexError(f"index {tensor.shape[0]} is out of bounds for dimension 0 with size {tensor.shape[0]}")
        self._check_dtype(key, tensor)
        channels = self._outputs[key].shape[0] if key in self._outputs else tensor.shape[1]
        patch_shape = tuple(tensor.shape[2:])
        rows = []
        for row, location in enumerate(locations):
            dst_lo, dst_len, src_lo, src_len = self._box(location, patch_shape)
            target, value = (channels, *dst_len), (tensor.shape[1], *src_len)
            if target != value:
                bad = [d for d in range(4) if value[d] not in (target[d], 1)]
                if bad:
                    raise RuntimeError(
                        f"The size of tensor a ({target[bad[0]]}) must match the size of tensor b ({value[bad[0]]})"
                        f" at non-singleton dimension {bad[0]}: patch {row} of key {key!r} has shape {list(value)},"
                        f" its box {list(target)}")
                raise NotImplementedError(
                    f"PatchAggregator: patch {row} of key {key!r} has shape {list(value)} and fits its box"
                    f" {list(target)} only by broadcasting, which the aggregator does not do")
            if min(dst_len) > 0 and channels > 0:
                rows.append([*dst_lo, *(dst_lo[a] + dst_len[a] for a in range(3)), *src_lo, row])
        return np.asarray(rows, dtype=np.int32).reshape(-1, 10)

    def add_batch(self, batch, locations) -> None:
        """Add a batch of model outputs, a (B, C, I, J, K) tensor or a dict of them keyed by name, whose
        first ``len(locations)`` patches lie at ``locations`` (aggregator.py:75-100).  The whole batch
        is checked before any of it is added; device batches take one launch per key, no host sync."""
        tensors = {"__default__": batch} if isinstance(batch, torch.Tensor) else dict(batch)
        if not tensors or not len(locations):
            return
        tables = {key: self._table(key, tensor, locations) for key, tensor in tensors.items()}
        device = self._device_for(next(iter(tensors.values())))
        staged = []
        for key, tensor in tensors.items():
            tensor = tensor if tensor.device == device else tensor.to(device)
            ops._check(tensor, "aggregate_patches")
            staged.append((key, tensor, tables[key]))
        for key, tensor, table in staged:
            if key not in self._outputs:
                self._outputs[key] = torch.zeros((tensor.shape[1], *self.spatial_shape), dtype=tensor.dtype,
                                                 device=device)
                if self.overlap_mode != "crop":
                    self._counts[key] = torch.zeros((1, *self.spatial_shape), dtype=tensor.dtype, device=device)
            window = None
            if self.overlap_mode == "hann":
                window = torch.cat([torch.hann_window(n + 2, periodic=False)[1:-1] for n in tensor.shape[2:]])
            ops.aggregate_patches(tensor, self._outputs[key], self._counts.get(key), table, self.overlap_mode,
                                  window)

    def get_output(self, key: str | None = None) -> torch.Tensor:
        """The aggregated (C, I, J, K) volume (aggregator.py:102-123): "crop" returns the buffer itself
        (a host copy for a caller whose first batch was on the host), "average" and "hann" a new
        tensor ``out / counts.clamp(min=1)``, fp32 for integer buffers."""
        resolve_key = key if key is not None else "__default__"
        if resolve_key not in self._outputs:
            available = [k for k in self._outputs if k != "__default__"]
            raise KeyError(f"No output for key {key!r}. Available: {available}")
        output = self._outputs[resolve_key]
        if self.overlap_mode != "crop":
            output = ops.aggregate_finish(output, self._counts[resolve_key])
        return output.cpu() if self._host_caller else output


def _mask_borders(prob: torch.Tensor, spatial_shape, patch_size) -> torch.Tensor:
    """Zero probability where a patch centre cannot be placed (data/sampler.py:340-360)."""
    prob = prob.clone()
    for d in range(3):
        half = patch_size[d] // 2
        if half > 0:
            lo: list[slice] = [slice(None)] * 3
            lo[d] = slice(0, half)
            prob[tuple(lo)] = 0
        tail = spatial_shape[d] - half
        if tail < spatial_shape[d]:
            hi: list[slice] = [slice(None)] * 3
            hi[d] = slice(tail, None)
            prob[tuple(hi)] = 0
    return prob


def _center_to_corner(center, spatial_shape, patch_size) -> tuple[int, int, int]:
    """Centre voxel -> patch corner, clamped into the volume (data/sampler.py:363-375)."""
    result = []
    for d in range(3):
        corner = max(0, center[d] - patch_size[d] // 2)
        result.append(min(corner, spatial_shape[d] - patch_size[d]))
    return (result[0], result[1], result[2])


class WeightedSampler(PatchSampler, IterableDataset):
    """Random patches weighted by a probability map (data/sampler.py:226-283).

    The centre voxels are drawn with ``torch.multinomial`` on the flattened map.  For a
    device-resident subject the map is brought to the host once per subject and drawn there,
    so the draws are those of the reference (global CPU generator), whatever the device."""

    def __init__(self, subject: Subject, patch_size, probability_map: str, num_patches: int | None = None) -> None:
        super().__init__(patch_size)
        self.subject = subject
        self.probability_map = probability_map
        self.num_patches = num_patches

    def _flat_map(self, subject: Subject):
        prob = self._build_probability_map_for(subject)
        flat = prob.flatten()
        if flat.sum() == 0:
            raise RuntimeError(f"Probability map '{self.probability_map}' is all zeros")
        return flat.cpu(), tuple(prob.shape)

    def _draw(self, flat, shape, subject: Subject) -> PatchLocation:
        idx_flat = torch.multinomial(flat, 1).item()
        center = tuple(int(x) for x in np.unravel_index(int(idx_flat), shape))
        return PatchLocation(index=_center_to_corner(center, subject.spatial_shape, self.patch_size),
                             size=self.patch_size)

    def __call__(self, subject: Subject, num_patches: int | None = None) -> Iterator[Subject]:
        flat, shape = self._flat_map(subject)
        limit = num_patches or self.num_patches
        count = 0
        while limit is None or count < limit:
            yield self._extract_patch(subject, self._draw(flat, shape, subject))
            count += 1

    def __iter__(self) -> Iterator[Subject]:
        return self(self.subject, self.num_patches)

    def draw_locations(self, subject: Subject, count: int) -> list[PatchLocation]:
        """The locations of the first ``count`` patches ``self(subject)`` would yield (same draws)."""
        flat, shape = self._flat_map(subject)
        return [self._draw(flat, shape, subject) for _ in range(count)]

    def sample(self, subject: Subject, num_patches: int) -> list[Subject]:
        """``list(islice(self(subject), num_patches))``, same draws, one gather launch per
        image for a device-resident subject."""
        count = num_patches if not self.num_patches else min(num_patches, self.num_patches)
        return self._extract_patches(subject, self.draw_locations(subject, count))

    def _build_probability_map_for(self, subject: Subject) -> torch.Tensor:
        prob_data = subject.images[self.probability_map].data[0].float()
        return _mask_borders(prob_data, subject.spatial_shape, self.patch_size)

    def _build_probability_map(self) -> torch.Tensor:
        return self._build_probability_map_for(self.subject)


class LabelSampler(WeightedSampler):
    """Random patches centred on labelled voxels (data/sampler.py:286-333)."""

    def __init__(self, subject: Subject, patch_size, label_name: str,
                 label_probabilities: dict[int, float] | None = None, num_patches: int | None = None) -> None:
        super().__init__(subject, patch_size, probability_map=label_name, num_patches=num_patches)
        self.label_name = label_name
        self.label_probabilities = label_probabilities

    def _build_probability_map_for(self, subject: Subject) -> torch.Tensor:
        label_data = subject.images[self.label_name].data[0]
        if self.label_probabilities is not None:
            prob = torch.zeros_like(label_data, dtype=torch.float32)
            for label, weight in self.label_probabilities.items():
                prob[label_data == label] = weight
        else:
            prob = (label_data > 0).float()
        return _mask_borders(prob, subject.spatial_shape, self.patch_size)


# samplers whose ``__call__`` the ring path may bypass (a subclass that overrides it is iterated)
_STOCK_CALLS = {"UniformSampler": UniformSampler.__call__, "WeightedSampler": WeightedSampler.__call__,
                "LabelSampler": WeightedSampler.__call__}


# ---------------------------------------------------------------------------------------
# Queue: patch buffer for stochastic patch-based training (data/queue.py:21-208)
#
# What the reference does per epoch: subjects (optionally shuffled with `random.shuffle`, or in
# the order of `subject_sampler`) are loaded and transformed one by one, `patches_per_volume`
# patches of each are appended to a buffer, and whenever the buffer holds `max_length` patches
# or more it is shuffled (`random.shuffle`) and handed out from the back until it is empty.
# That order is the contract (tests/golden/patches_*.npz).  How the patches are held is not:
#
#   * host-resident subjects: the buffer holds the sampler's zero-copy views, as upstream;
#   * device-resident subjects (or `device=`): the buffer is a pre-allocated RING of patch
#     slots per image, `(max_length + patches_per_volume - 1, C, *patch_size)` on the device.
#     One `tio_crop_patches` launch per image writes a subject's patches straight into
#     consecutive slots; the shuffle permutes slot indices (same `random.shuffle` call on a
#     list of the same length, hence the same order); the queue hands out `PatchHandle`s
#     (slot + location + a reference to the per-subject record) and `collate_subjects` turns a
#     list of handles into a `SubjectsBatch` with ONE `index_select` per image.  No per-patch
#     `Subject`, no per-patch tensor, no `torch.stack`.
# ---------------------------------------------------------------------------------------


class _SubjectRecord:
    """What the patches of one subject share: image classes / affines / metadata / history."""

    __slots__ = ("kinds", "affines", "image_metadata", "metadata", "history")

    def __init__(self, subject: Subject) -> None:
        self.kinds = {name: type(img) for name, img in subject.images.items()}
        self.affines = {name: img.affine.numpy() for name, img in subject.images.items()}
        self.image_metadata = {name: dict(img.metadata) for name, img in subject.images.items()}
        self.metadata = dict(subject.metadata)
        self.history = list(subject.applied_transforms)

    def patch_affine(self, name: str, index) -> np.ndarray:
        matrix = self.affines[name].copy()
        matrix[:3, 3] = matrix[:3, 3] + matrix[:3, :3] @ np.asarray(index, dtype=np.float64)
        return matrix


class PatchRing:
    """Device-side patch slots of one Queue: ``data[name]`` is ``(capacity, C, *patch_size)``."""

    def __init__(self, capacity: int, patch_size, subject: Subject) -> None:
        self.capacity = int(capacity)
        self.patch_size = tuple(patch_size)
        self.data = {
            name: torch.empty((self.capacity, img.data.shape[0], *self.patch_size), dtype=img.data.dtype,
                              device=img.data.device)
            for name, img in subject.images.items()
        }
        self.filled = 0
        self._handed_out: weakref.WeakSet = weakref.WeakSet()  # handles whose slot is still theirs

    def recycle(self) -> None:
        """Start refilling from slot 0.  Handles of the previous fill that the caller still holds
        (e.g. ``list(queue)``) take a private copy of their slot first, so they stay valid."""
        for handle in list(self._handed_out):
            handle.detach()
        self._handed_out = weakref.WeakSet()
        self.filled = 0

    def matches(self, subject: Subject) -> bool:
        return (set(subject.images) == set(self.data) and all(
            self.data[n].dtype == img.data.dtype and self.data[n].device == img.data.device
            and self.data[n].shape[1] == img.data.shape[0] for n, img in subject.images.items()))

    def write(self, subject: Subject, locations: list[PatchLocation]) -> range:
        """One gather launch per image into the next ``len(locations)`` slots."""
        n = len(locations)
        if self.filled + n > self.capacity:
            raise RuntimeError("PatchRing overflow (queue invariant broken)")
        corners = np.asarray([loc.index for loc in locations], dtype=np.int32)
        slots = range(self.filled, self.filled + n)
        for name, img in subject.images.items():
            ops.crop_patches(img.data, corners, self.patch_size, out=self.data[name][slots.start:slots.stop])
        self.filled += n
        return slots


class PatchHandle:
    """A patch that lives in a `PatchRing` slot.  `collate_subjects` batches handles without
    materialising them; any `Subject` attribute (``handle.t1``, ``handle.patch_location``,
    ``handle.sid`` ...) materialises a `Subject` of VIEWS of the slot on first use.  When the
    queue refills the ring, handles that are still referenced copy their slot out first
    (`detach`), so a patch stays valid for as long as it is held, like the reference's views."""

    __slots__ = ("ring", "slot", "location", "record", "_subject", "__weakref__")

    def __init__(self, ring: PatchRing, slot: int, location: PatchLocation, record: _SubjectRecord) -> None:
        self.ring, self.slot, self.location, self.record = ring, slot, location, record
        self._subject = None
        ring._handed_out.add(self)

    def detach(self) -> None:
        """Own the data: a private copy of the slot replaces the views."""
        if self.ring is not None:
            self._subject = self.subject(copy=True)
            self.ring = None

    def subject(self, copy: bool = False) -> Subject:
        if self.ring is None:
            return self._subject
        if self._subject is None or copy:
            rec = self.record
            kwargs: dict[str, Any] = {}
            for name, block in self.ring.data.items():
                data = block[self.slot].clone() if copy else block[self.slot]
                kwargs[name] = rec.kinds[name](data, affine=rec.patch_affine(name, self.location.index),
                                               **rec.image_metadata[name])
            kwargs.update(rec.metadata)
            kwargs["patch_location"] = self.location
            built = Subject(**kwargs)
            built.applied_transforms = list(rec.history)
            if copy:
                return built
            self._subject = built
        return self._subject

    def __getattr__(self, name: str):
        if name.startswith("_"):
            raise AttributeError(name)
        return getattr(self.subject(), name)


class _ViewBuffer:
    """Reference behaviour: the buffer is a list of patch Subjects (views of their volume)."""

    def __init__(self) -> None:
        self.items: list[Any] = []

    def __len__(self) -> int:
        return len(self.items)

    def add(self, patches: list[Any]) -> None:
        self.items.extend(patches)

    def drain(self, shuffle: bool) -> Iterator[Any]:
        if shuffle:
            _random.shuffle(self.items)
        while self.items:
            yield self.items.pop()


class _RingBuffer(_ViewBuffer):
    """Same order of hand-out, patches held as ring slots."""

    def __init__(self, ring: PatchRing) -> None:
        super().__init__()
        self.ring = ring

    def add_subject(self, subject: Subject, locations: list[PatchLocation]) -> None:
        self.add_subject_check()
        record = _SubjectRecord(subject)
        slots = self.ring.write(subject, locations)
        self.items.extend(PatchHandle(self.ring, slot, loc, record) for slot, loc in zip(slots, locations))

    def add_subject_check(self) -> None:
        if not self.items and self.ring.filled:  # everything was handed out: refill from the start
            self.ring.recycle()


class Queue(IterableDataset):
    """Same constructor, same order of patches as the reference's Queue; ``device=`` (extension)
    moves a copy of each loaded subject to that device before the transform, so augmentation and
    patch extraction run resident and the buffer is a device patch ring (see above)."""

    def __init__(self, subjects: Sequence[Subject], patch_sampler: PatchSampler, max_length: int = 300,
                 patches_per_volume: int = 10, num_workers: int = 0, shuffle_subjects: bool = True,
                 shuffle_patches: bool = True, transform: Any | None = None,
                 subject_sampler: Sampler | None = None, device: str | torch.device | None = None) -> None:
        if subject_sampler is not None and shuffle_subjects:
            raise ValueError(
                "shuffle_subjects must be False when subject_sampler"
                " is provided (the sampler controls the order)"
            )
        self.subjects = subjects
        self.patch_sampler = patch_sampler
        self.max_length = max_length
        self.patches_per_volume = patches_per_volume
        self.num_workers = num_workers
        self.shuffle_subjects = shuffle_subjects
        self.shuffle_patches = shuffle_patches
        self.transform = transform
        self.subject_sampler = subject_sampler
        self.device = None if device is None else torch.device(device)
        self._ring: PatchRing | None = None

    # ---- iteration -------------------------------------------------------------------

    def __iter__(self) -> Iterator[Any]:
        buffer: _ViewBuffer | None = None
        for subject in self._prepared():
            locations = self._ring_locations(subject)
            if locations is not None:
                if not isinstance(buffer, _RingBuffer):
                    if buffer:  # a host-resident stretch came first: hand it out before switching
                        yield from buffer.drain(self.shuffle_patches)
                    buffer = _RingBuffer(self._ring_for(subject))
                buffer.add_subject(subject, locations)
            else:
                if isinstance(buffer, _RingBuffer) or buffer is None:
                    if buffer:
                        yield from buffer.drain(self.shuffle_patches)
                    buffer = _ViewBuffer()
                buffer.add(self._view_patches(subject))
            if len(buffer) >= self.max_length:
                yield from buffer.drain(self.shuffle_patches)
        if buffer:
            yield from buffer.drain(self.shuffle_patches)

    def _prepared(self) -> Iterator[Subject]:
        """Loaded (+ moved, + transformed) subjects in epoch order.  ``num_workers`` threads
        prepare ahead; results are consumed strictly in order, so the patch order does not depend
        on thread timing (the reference's threaded mode flushes at timing-dependent points)."""
        order = self._epoch_order()
        if self.num_workers <= 0:
            for subject in order:
                yield self._prepare(subject)
            return
        window = 2 * self.num_workers
        with ThreadPoolExecutor(max_workers=self.num_workers) as pool:
            pending: deque[Future[Subject]] = deque()
            for subject in order:
                pending.append(pool.submit(self._prepare, subject))
                if len(pending) >= window:
                    yield pending.popleft().result()
            while pending:
                yield pending.popleft().result()

    def _epoch_order(self) -> Iterator[Subject]:
        if self.subject_sampler is not None:
            return (self.subjects[i] for i in list(self.subject_sampler))
        subjects = list(self.subjects)
        if self.shuffle_subjects:
            _random.shuffle(subjects)
        return iter(subjects)

    def _prepare(self, subject: Subject) -> Subject:
        subject.load()
        if self.device is not None:  # a moved copy: the dataset's own subject stays where it is
            kwargs: dict[str, Any] = {
                name: img.new_like(data=img.data.to(self.device, non_blocking=True))
                for name, img in subject.images.items()}
            kwargs.update(subject.metadata)
            moved = Subject(**kwargs)
            moved.applied_transforms = list(subject.applied_transforms)
            subject = moved
        if self.transform is not None:
            subject = self.transform(subject)
        return subject

    # ---- patches of one subject ------------------------------------------------------

    def _count(self) -> int:
        """``islice(sampler(subject), patches_per_volume)`` stops at the sampler's own
        ``num_patches`` when that is smaller."""
        own = getattr(self.patch_sampler, "num_patches", None)
        return self.patches_per_volume if not own else min(self.patches_per_volume, int(own))

    def _ring_locations(self, subject: Subject) -> list[PatchLocation] | None:
        """Patch locations drawn exactly as iterating the sampler would, when the ring applies:
        device-resident subject, a stock sampler (its ``__call__`` not overridden), patches that
        fit the volume.  None = take the sampler's own patches (views)."""
        sampler = self.patch_sampler
        draw = getattr(sampler, "draw_locations", None)
        stock = _STOCK_CALLS.get(type(sampler).__mro__[0].__name__)
        if draw is None or stock is None or type(sampler).__call__ is not stock:
            return None
        if not all(img.data.is_cuda for img in subject.images.values()):
            return None
        if any(p > s for p, s in zip(sampler.patch_size, subject.spatial_shape)):
            return None
        return draw(subject, self._count())

    def _view_patches(self, subject: Subject) -> list[Subject]:
        return list(islice(iter(self.patch_sampler(subject)), self.patches_per_volume))

    def _ring_for(self, subject: Subject) -> PatchRing:
        ring = self._ring
        if ring is None or not ring.matches(subject) or ring.patch_size != tuple(self.patch_sampler.patch_size):
            capacity = self.max_length + self.patches_per_volume - 1
            ring = self._ring = PatchRing(capacity, self.patch_sampler.patch_size, subject)
        ring.recycle()
        return ring

    # ---- bookkeeping the reference exposes -------------------------------------------

    @property
    def num_subjects(self) -> int:
        sampler = self.subject_sampler
        if sampler is not None:
            if not isinstance(sampler, Sized):
                raise TypeError("subject_sampler must have a __len__ method")
            return len(sampler)
        return len(self.subjects)

    @property
    def patches_per_epoch(self) -> int:
        return self.num_subjects * self.patches_per_volume

    @property
    def max_memory(self) -> int:
        """Bytes of ``max_length`` fp32 patches of the first subject's channels (queue.py:195-203)."""
        channels = sum(img.num_channels for img in self.subjects[0].images.values())
        return 4 * channels * int(np.prod(self.patch_sampler.patch_size)) * self.max_length

    @property
    def max_memory_pretty(self) -> str:
        value, units = float(self.max_memory), ("Bytes", "KiB", "MiB", "GiB", "TiB")
        step = 0
        while value >= 1024 and step < len(units) - 1:
            value, step = value / 1024, step + 1
        return f"{value:.0f} Bytes" if step == 0 else f"{value:.1f} {units[step]}"


def collate_subjects(batch: Sequence[Any]) -> SubjectsBatch:
    """List of patches/subjects -> SubjectsBatch (loader.py:15-24).  Handles of one patch ring are
    batched with one ``index_select`` per image; anything else goes through ``from_subjects``."""
    items = list(batch)
    if items and all(isinstance(item, PatchHandle) for item in items) and items[0].ring is not None and all(
            item.ring is items[0].ring for item in items):
        ring = items[0].ring
        slots = torch.tensor([item.slot for item in items], dtype=torch.int64)
        images = {}
        for name, block in ring.data.items():
            data = block.index_select(0, slots.to(block.device, non_blocking=True))
            affines = [AffineMatrix(item.record.patch_affine(name, item.location.index)) for item in items]
            images[name] = ImagesBatch(data, affines, image_class=items[0].record.kinds[name])
        keys = list(items[0].record.metadata)
        metadata = {k: [item.record.metadata[k] for item in items] for k in keys}
        metadata["patch_location"] = [item.location for item in items]
        return SubjectsBatch(images, metadata=metadata)
    return SubjectsBatch.from_subjects([item.subject() if isinstance(item, PatchHandle) else item for item in items])


def collate_images(batch: Sequence[Any]) -> ImagesBatch:
    return ImagesBatch.from_images(list(batch))


class SubjectsLoader(DataLoader):
    """DataLoader that returns `SubjectsBatch` instances (loader.py:38-65)."""

    def __init__(self, dataset: Dataset, **kwargs: Any) -> None:
        if "collate_fn" in kwargs:
            raise ValueError(
                "SubjectsLoader sets collate_fn automatically; "
                "pass a plain DataLoader if you need a custom collate_fn"
            )
        super().__init__(dataset, collate_fn=collate_subjects, **kwargs)


class ImagesLoader(DataLoader):
    """DataLoader that returns `ImagesBatch` instances (loader.py:68-90)."""

    def __init__(self, dataset: Dataset, **kwargs: Any) -> None:
        if "collate_fn" in kwargs:
            raise ValueError(
                "ImagesLoader sets collate_fn automatically; "
                "pass a plain DataLoader if you need a custom collate_fn"
            )
        super().__init__(dataset, collate_fn=collate_images, **kwargs)


StudiesLoader = SubjectsLoader
collate_studies = collate_subjects
