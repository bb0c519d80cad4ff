"""Resolution changes (transforms/spatial/{anisotropy,resize}.py of TorchIO 2.0.0a2): Anisotropy and
Resize.

Constructors, ``make_params`` RNG order, params schema, gating and history are the reference's.
Both walk every image of the batch (``include`` / ``exclude`` are recorded, not applied, as in the
reference).  Each ``apply_transform`` is one CUDA pass per image on the data's fp32 image, cast back
to its dtype as the reference's ``data.float()`` ... ``.to(dtype)`` do:
- Resize and Anisotropy's shared path (B = 1 or ``per_instance=False``): `ops.interpolate`, ATen's
  CUDA trilinear / nearest resize from `tables.resize_tables` / `tables.anisotropy_shared_tables`
  (Anisotropy's nearest-down map composed into the up table, so the downsampled tensor never exists);
- Anisotropy's per-instance path: `ops.axis_resample` from `tables.anisotropy_instance_tables`, which
  restate that path's own int64 / fp32 index arithmetic (it picks different planes than ATen's).

With `set_differentiable(True)`, a scalar image that requires grad goes through the same calls as
graph nodes (`autograd.interpolate`, `autograd.axis_resample`), whose backwards are the transposes of
these tables (`tables.*_adjoint_tables`), gathered in a fixed order; a label map that requires grad
is refused.
"""

from __future__ import annotations

import functools
from typing import Any

import torch

from .. import autograd, ops, tables
from ..data import LabelMap, SubjectsBatch
from ..params import to_nonneg_range
from .base import SpatialTransform, Transform


class Anisotropy(Transform):
    """Downsample along a randomly chosen axis and upsample back to the original shape
    (spatial/anisotropy.py:17-129): label maps nearest, scalar images ``image_interpolation``
    (``"nearest"``, anything else linear)."""

    def __init__(self, *, axes: tuple[int, ...] = (0, 1, 2), downsampling: float | tuple[float, float] = 1.0,
                 image_interpolation: str = "linear", **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.axes = axes
        self.downsampling = to_nonneg_range(downsampling)
        self.image_interpolation = image_interpolation
        _lo, hi = self.downsampling._ranges[0]
        if hi < 1.0:
            raise ValueError(f"downsampling range upper bound must be >= 1, got {hi}")
        self._warn_if_noop(is_noop=self.downsampling.is_constant(1.0), hint="downsampling=(1.5, 5)")

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return True

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        n = self._resolve_n(batch)
        if n is None:
            axis = self.axes[int(torch.randint(len(self.axes), (1,)).item())]
            factor = max(1.0, self.downsampling.sample_1d())
            return {"axis": axis, "factor": factor}
        keep = self._keep_mask(batch, n)
        axis_list: list[int] = []
        factor_list: list[float] = []
        for index in range(n):
            if keep is not None and not keep[index]:
                axis_list.append(self.axes[0])
                factor_list.append(1.0)
                continue
            axis_list.append(self.axes[int(torch.randint(len(self.axes), (1,)).item())])
            factor_list.append(max(1.0, self.downsampling.sample_1d()))
        params = {"axis": axis_list, "factor": factor_list}
        self._tag_batched(params, batch, n, keep, ["axis", "factor"])
        return params

    differentiable = True  # scalar images: autograd.interpolate / autograd.axis_resample

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        per_instance = self._is_per_instance_params(params)
        for name, ib in batch.images.items():
            is_label = issubclass(ib._image_class, LabelMap)
            linear = not is_label and self.image_interpolation != "nearest"
            graph, data = _graph_input("Anisotropy", name, ib.data, is_label)
            if per_instance:
                ib.data = _degrade_per_instance(data, params["axis"], params["factor"], linear, graph)
            elif params["factor"] > 1.0:
                args = (data.shape[2:], params["axis"], params["factor"], linear)
                idx, lam = tables.anisotropy_shared_tables(*args)
                if graph:
                    ib.data = autograd.interpolate(data, data.shape[2:], idx, lam,
                                                   functools.partial(tables.anisotropy_shared_adjoint_tables, *args))
                else:
                    ib.data = ops.interpolate(data, data.shape[2:], idx, lam)
        return batch


def _graph_input(transform: str, name: str, data, is_label: bool):
    """(records a graph node, the tensor to pass on) for image ``name``: a label map that requires
    grad is refused, and with grad mode off an image that requires grad runs the usual kernels."""
    graph = autograd.records_graph(data)
    if graph and is_label:
        autograd.refuse(transform, f'label map "{name}"')
    if not graph and data.requires_grad and ops.differentiable_default():
        data = data.detach()
    return graph, data


def _degrade_per_instance(data, axes: list[int], factors: list[float], linear: bool, graph: bool = False):
    """_simulate_anisotropy_per_instance (anisotropy.py:132-177): untouched when no element has a
    factor > 1, an error for an active axis outside {0, 1, 2}."""
    active = [f > 1.0 for f in factors]
    if not any(active):
        return data
    if any(a < 0 or a > 2 for a, on in zip(axes, active) if on):
        raise ValueError(f"Anisotropy axis must be in {{0, 1, 2}}, got {sorted(set(axes))}")
    axis, lo, hi, w = tables.anisotropy_instance_tables(data.shape[2:], axes, factors, linear)
    if graph:
        adjoint = functools.partial(tables.anisotropy_instance_adjoint_tables, data.shape[2:], axes, factors, linear)
        return autograd.axis_resample(data, axis, lo, hi, w, adjoint, linear=linear)
    return ops.axis_resample(data, axis, lo, hi, w, linear=linear)


class Resize(SpatialTransform):
    """Resize every image to ``target_shape`` (an int N means (N, N, N)) keeping the field of view:
    trilinear (align_corners=True) unless the interpolation is ``"nearest"``, and each affine's
    column ``axis`` scaled by old / target (spatial/resize.py:13-80).  Not invertible.

    Never streamed in slices: it changes the shape the ``make_params`` of later transforms in a
    `Compose` read, and a streamed `Compose` samples every child's params up front."""

    def __init__(self, target_shape: int | tuple[int, int, int], *, image_interpolation: str = "linear",
                 label_interpolation: str = "nearest", **kwargs: Any) -> None:
        super().__init__(**kwargs)
        if isinstance(target_shape, int):
            target_shape = (target_shape, target_shape, target_shape)
        self.target_shape = target_shape
        self.image_interpolation = image_interpolation
        self.label_interpolation = label_interpolation

    differentiable = True  # scalar images: autograd.interpolate

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {"target_shape": self.target_shape}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        target = [int(s) for s in params["target_shape"]]
        for name, ib in batch.images.items():
            is_label = issubclass(ib._image_class, LabelMap)
            mode = self.label_interpolation if is_label else self.image_interpolation
            graph, data = _graph_input("Resize", name, ib.data, is_label)
            old_shape = tuple(data.shape[2:])
            idx, lam = tables.resize_tables(old_shape, target, mode != "nearest")
            if graph:
                adjoint = functools.partial(tables.resize_adjoint_tables, old_shape, target, mode != "nearest")
                ib.data = autograd.interpolate(data, target, idx, lam, adjoint)
            else:
                ib.data = ops.interpolate(data, target, idx, lam)
            for index, affine in enumerate(ib.affines):
                matrix = affine.numpy().copy()
                for axis in range(3):
                    matrix[:3, axis] *= old_shape[axis] / target[axis]
                ib.affines[index] = type(affine)(matrix)
        return batch
