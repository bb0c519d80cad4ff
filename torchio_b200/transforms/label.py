"""Label-map utilities (transforms/label/ of TorchIO 2.0.0a2): RemapLabels, RemoveLabels,
SequentialLabels, OneHot, Contour, KeepLargestComponent and the private inverses.

Constructors, ``make_params``, params schema, gating (one batch-wide coin) and history are the
reference's; only `LabelMap` batches are touched, and, as in the reference, ``include`` /
``exclude`` are recorded but not applied.  Each ``apply_transform`` is one pass of a CUDA kernel:
a table lookup (`ops.label_lut`, tables built by `tables.label_lut` with torch's own scalar
rules), the 27-point contour stencil, the one-hot expansion, the channel argmax, or (KeepLargestComponent)
a batched connected-component union-find.
"""

from __future__ import annotations

from collections.abc import Sequence
from typing import Any

from .. import ops, tables
from ..data import LabelMap, SubjectsBatch
from .base import Transform


def _label_batches(batch: SubjectsBatch):
    return [(name, ib) for name, ib in batch.images.items() if issubclass(ib._image_class, LabelMap)]


def _lookup(data, pairs, *, identity: bool):
    keys, values = tables.label_lut(pairs, data.dtype, data.device)
    return ops.label_lut(data, keys, values, identity=identity)


class RemapLabels(Transform):
    """Replace each key of ``remapping`` by its value in label maps; other labels are unchanged,
    and every match is taken on the original map, so ``{1: 2, 2: 1}`` swaps
    (label/remap_labels.py:12-69)."""

    def __init__(self, remapping: dict[int, int], **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.remapping = remapping

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {"remapping": self.remapping}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        pairs = list(params["remapping"].items())
        for _, ib in _label_batches(batch):
            ib.data = _lookup(ib.data, pairs, identity=True)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> RemapLabels:
        remapping = params["remapping"]
        return RemapLabels(remapping={v: k for k, v in remapping.items()}, copy=False)


class RemoveLabels(Transform):
    """Set ``labels`` to ``background_label`` in label maps (label/remove_labels.py:13-61)."""

    def __init__(self, labels: Sequence[int], *, background_label: int = 0, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.labels = list(labels)
        self.background_label = background_label

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        pairs = [(label, self.background_label) for label in self.labels]
        for _, ib in _label_batches(batch):
            ib.data = _lookup(ib.data, pairs, identity=True)
        return batch


class SequentialLabels(Transform):
    """Renumber the labels of each label map to 0, 1, 2, ... in ascending order of the values of
    batch element 0; values absent from element 0 become 0 (label/sequential_labels.py:14-74).

    Never streamed in slices: ``make_params`` reads the labels as the transforms before it in a
    `Compose` left them, and a streamed `Compose` samples every child's params up front."""

    def __init__(self, **kwargs: Any) -> None:
        super().__init__(**kwargs)

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        remappings: dict[str, dict[int, int]] = {}
        for name, ib in _label_batches(batch):
            unique = sorted(int(v) for v in ib.data[0].unique().tolist())
            remappings[name] = {old: new for new, old in enumerate(unique)}
        return {"remappings": remappings}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        return _renumber(batch, params["remappings"], invert=False)

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _SequentialLabelsInverse:
        return _SequentialLabelsInverse(remappings=params["remappings"], copy=False)


class _SequentialLabelsInverse(Transform):
    """Inverse of SequentialLabels: the inverted tables, unlisted values -> 0
    (label/sequential_labels.py:77-105)."""

    def __init__(self, *, remappings: dict[str, dict[int, int]], **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self._remappings = remappings

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        return _renumber(batch, self._remappings, invert=True)


def _renumber(batch: SubjectsBatch, remappings: dict, *, invert: bool) -> SubjectsBatch:
    for name, ib in batch.images.items():
        if name not in remappings:
            continue
        table = remappings[name]
        if invert:
            table = {v: k for k, v in table.items()}
        ib.data = _lookup(ib.data, list(table.items()), identity=False)
    return batch


class OneHot(Transform):
    """(B, 1, I, J, K) label maps -> (B, num_classes, I, J, K) fp32 one-hot channels of
    ``long(label)`` on channel 0; ``num_classes=-1`` takes the batch's maximum + 1
    (label/one_hot.py:14-78).  Classes out of range raise the CPU reference's errors before any
    launch (the reference on a CUDA batch hits a device-side assert instead)."""

    def __init__(self, *, num_classes: int = -1, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.num_classes = num_classes

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return self.num_classes != -1  # -1: the class count depends on every element

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {"num_classes": self.num_classes}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        num_classes = params["num_classes"]
        for _, ib in _label_batches(batch):
            lo, hi = ops.label_range(ib.data)
            if lo < 0:
                raise RuntimeError("Class values must be non-negative.")
            count = hi + 1 if num_classes == -1 else num_classes
            if hi >= count:
                raise RuntimeError("Class values must be smaller than num_classes.")
            ib.data = ops.onehot_classes(ib.data, count)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _OneHotInverse:
        return _OneHotInverse(copy=False)


class _OneHotInverse(Transform):
    """Inverse of OneHot: ``argmax(dim=1, keepdim=True).float()`` of label maps with more than one
    channel (label/one_hot.py:81-97)."""

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for _, ib in _label_batches(batch):
            if ib.data.shape[1] > 1:
                ib.data = ops.channel_argmax(ib.data)
        return batch


class Contour(Transform):
    """Label maps -> fp32 boundary masks: 1 where some voxel of the 3x3x3 neighbourhood (-1 outside
    the volume) is smaller, or NaN (label/contour.py:15-71)."""

    def __init__(self, **kwargs: Any) -> None:
        super().__init__(**kwargs)

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for _, ib in _label_batches(batch):
            ib.data = ops.label_contour(ib.data)
        return batch


class KeepLargestComponent(Transform):
    """Within each label of each single-channel label map, set every connected component but the
    largest to ``background_label`` (label/keep_largest.py:17-125).  ``labels=None`` takes every
    value with ``int(v) != background_label``; ``fully_connected`` selects 26 neighbours, else 6.
    Among components of equal size the one whose first voxel in C order comes first is kept.

    Every label of every element is labelled in one union-find on the device (`ops.keep_largest`),
    in place: a transform called with ``copy=True`` (the default) or inside a `Compose` has already
    copied the batch."""

    def __init__(self, labels: Sequence[int] | None = None, *, background_label: int = 0,
                 fully_connected: bool = True, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.labels = list(labels) if labels is not None else None
        self.background_label = background_label
        self.fully_connected = fully_connected

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True  # elements are independent

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for _, ib in _label_batches(batch):
            channels = ib.data.shape[1]
            if channels != 1:
                raise RuntimeError(f"KeepLargestComponent requires single-channel label maps, got {channels} channels")
            ib.data, _ = ops.keep_largest(ib.data, self.labels, self.background_label, self.fully_connected)
        return batch
