"""Ghosting (transforms/intensity/ghosting.py of TorchIO 2.0.0a2): MRI ghosting artefacts along the
phase-encode axis.

Constructor, warnings, ``make_params`` (its RNG calls and quirks), gating, history, ``repr`` and
``to_hydra`` are the reference's.  The reference multiplies ``fftshift(fftn(x))`` by a mask that
varies along one axis and inverts the FFT; the FFTs over the other two axes cancel, so here each
line along the chosen axis is filtered by a line FFT, a multiply and an inverse line FFT in one
pass of `ops.ghosting`, with the mask built on the host by `ghosting_filter`.

The batch's own tensors are written in place: a transform called with ``copy=True`` (the default)
or inside a `Compose` has already copied them; with ``copy=False`` on a CUDA batch the caller's
tensor is updated.
"""

from __future__ import annotations

from typing import Any

import numpy as np
import torch

from .. import ops
from ..data import SubjectsBatch
from ..params import to_nonneg_range
from .base import IntensityTransform


def ghosting_filter(n: int, num_ghosts: int, intensity: float, restore: float) -> np.ndarray:
    """fp32 (n,) ``ifftshift(line_mask)``: the reference's mask (ghosting.py:190-197, 250-271) in
    unshifted frequency order.  Ones, ``1 - intensity`` at every ``max(n // num_ghosts, 1)``-th
    point from 0, then, when ``restore > 0``, ones over the Python slice ``[n // 2 - h : n // 2 + h]``
    with ``h = max(int(n * restore / 2), 1)`` (a negative start wraps, as in the reference)."""
    mask = np.ones(n, dtype=np.float32)
    mask[:: max(n // num_ghosts, 1)] = 1 - intensity
    if restore > 0:
        mid, half = n // 2, max(int(n * restore / 2), 1)
        mask[mid - half: mid + half] = 1
    return np.fft.ifftshift(mask)


def ghosting_table(num_ghosts, axes, intensities, restore: float, spatial_shape) -> tuple[np.ndarray, ...]:
    """(fp32 (B, n_max) filters, int32 (B,) axes, bool (B,) active) of `ops.ghosting`; an element with
    no ghosts or intensity 0 is not active (``torch.where`` keeps its data in the reference)."""
    b = len(num_ghosts)
    active = np.array([bool(g) and v != 0 for g, v in zip(num_ghosts, intensities, strict=True)], dtype=bool)
    axis = np.array(axes, dtype=np.int32).reshape(b)
    for a in axis[active]:
        if a not in (0, 1, 2):
            raise ValueError(f"Ghosting: axis {a} is not a spatial axis (0, 1 or 2)")
    n_max = max((int(spatial_shape[a]) for a in axis[active]), default=0)
    table = np.zeros((b, n_max), dtype=np.float32)
    for e in np.flatnonzero(active):
        n = int(spatial_shape[axis[e]])
        table[e, :n] = ghosting_filter(n, int(num_ghosts[e]), float(intensities[e]), restore)
    return table, axis, active


class Ghosting(IntensityTransform):
    """Add random MRI ghosting artefacts (intensity/ghosting.py:16-146): ``num_ghosts`` replicas along
    one of ``axes``, by scaling every ``n // num_ghosts``-th k-space plane by ``1 - intensity`` and
    restoring the central ``restore`` fraction (``None``: nothing is restored, as in the reference)."""

    def __init__(self, *, num_ghosts: int | tuple[int, int] = 4, axes: tuple[int, ...] = (0, 1, 2),
                 intensity: float | tuple[float, float] = 0.0, restore: float | None = None,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.num_ghosts = to_nonneg_range(num_ghosts)
        self.axes = axes
        self.intensity = to_nonneg_range(intensity)
        self.restore = restore
        self._warn_if_noop(
            is_noop=self.intensity.is_constant(0.0) or self.num_ghosts.is_constant(0.0),
            hint="intensity=(0.5, 1)",
        )

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return True

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        restore = self.restore if self.restore is not None else 0.0
        n = self._resolve_n(batch)
        if n is None:
            num_ghosts = max(1, round(self.num_ghosts.sample_1d()))
            axis = self.axes[int(torch.randint(len(self.axes), (1,)).item())]
            return {"num_ghosts": num_ghosts, "axis": axis, "intensity": self.intensity.sample_1d(),
                    "restore": restore}
        keep = self._keep_mask(batch, n)
        num_ghosts_list: list[int] = []
        axis_list: list[int] = []
        intensity_list: list[float] = []
        for index in range(n):
            if keep is not None and not keep[index]:
                num_ghosts_list.append(0)
                axis_list.append(self.axes[0])
                intensity_list.append(0.0)
                continue
            num_ghosts_list.append(max(1, round(self.num_ghosts.sample_1d())))
            axis_list.append(self.axes[int(torch.randint(len(self.axes), (1,)).item())])
            intensity_list.append(self.intensity.sample_1d())
        params = {"num_ghosts": num_ghosts_list, "axis": axis_list, "intensity": intensity_list, "restore": restore}
        self._tag_batched(params, batch, n, keep, ["num_ghosts", "axis", "intensity"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        per_instance = self._is_per_instance_params(params)
        for _, img_batch in self._get_images(batch).items():
            data = img_batch.data
            b = data.shape[0]
            if per_instance:
                ghosts, axes, strengths = params["num_ghosts"], params["axis"], params["intensity"]
            else:
                ghosts, axes, strengths = [params["num_ghosts"]] * b, [params["axis"]] * b, [params["intensity"]] * b
            table, axis, active = ghosting_table(ghosts, axes, strengths, params["restore"], data.shape[2:])
            if not active.any():
                continue  # the reference returns the data itself
            work = data if data.is_contiguous() else data.contiguous()
            img_batch.data = ops.ghosting(work, table, axis, active)
        return batch
