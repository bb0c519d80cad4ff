"""Spike (transforms/intensity/spike.py of TorchIO 2.0.0a2): MRI k-space spike (herringbone) artefacts.

Constructor, warnings, ``make_params`` (its RNG calls and quirks), gating, history, ``repr`` and
``to_hydra`` are the reference's.  The reference adds ``peak * intensity`` at each spike of
``fftshift(fftn(x))`` and inverts the FFT; here each spike is the plane wave that point impulse
becomes, added in one pass by `ops.spike`, and the peak comes from a sum (no negative voxel) or a
forward half-spectrum FFT, decided on the device.

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
from ..params import to_nonneg_range, to_range
from .base import IntensityTransform


def spike_frequencies(positions, spatial_shape) -> list[tuple[int, int, int]]:
    """The frequency of each spike: the reference's fftshift index ``int(p * n) % n`` per axis
    (spike.py:155), shifted back by ``n // 2`` as ifftshift does."""
    return [tuple((int(p * n) % n - n // 2) % n for p, n in zip(pos, spatial_shape, strict=True))
            for pos in positions]


def spike_table(rows, intensities, spatial_shape) -> tuple[np.ndarray, np.ndarray]:
    """(int32 (len(rows), S, 4) ``u, v, w, 1`` rows padded with zeros, fp32 intensities) of
    `ops.spike`; an element without spikes or with intensity 0 gets intensity 0 (left untouched)."""
    steps = max((len(row) for row in rows), default=0)
    table = np.zeros((len(rows), steps, 4), dtype=np.int32)
    ratio = np.zeros(len(rows), dtype=np.float32)
    for e, (row, value) in enumerate(zip(rows, intensities, strict=True)):
        if not row or value == 0:
            continue
        table[e, : len(row), :3] = spike_frequencies(row, spatial_shape)
        table[e, : len(row), 3] = 1
        ratio[e] = value
    return table, ratio


class Spike(IntensityTransform):
    """Add random MRI spike artefacts (intensity/spike.py:17-121): ``num_spikes`` point impulses of
    ``intensity`` times the spectrum's peak, at random k-space positions."""

    def __init__(self, *, num_spikes: int | tuple[int, int] = 1, intensity: float | tuple[float, float] = 0.0,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.num_spikes = to_nonneg_range(num_spikes)
        self.intensity = to_range(intensity)
        self._warn_if_noop(
            is_noop=self.intensity.is_constant(0.0) or self.num_spikes.is_constant(0.0),
            hint="intensity=(1, 3)",
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
        n = self._resolve_n(batch)
        if n is None:
            num_spikes = max(1, round(self.num_spikes.sample_1d()))
            positions = torch.rand(num_spikes, 3).tolist()
            return {"positions": positions, "intensity": self.intensity.sample_1d()}
        keep = self._keep_mask(batch, n)
        positions_list: list[list[list[float]]] = []
        intensity_list: list[float] = []
        for should_keep in [True] * n if keep is None else keep.tolist():
            if not should_keep:
                positions_list.append([])
                intensity_list.append(0.0)
                continue
            num_spikes = max(1, round(self.num_spikes.sample_1d()))
            positions_list.append(torch.rand(num_spikes, 3).tolist())
            intensity_list.append(self.intensity.sample_1d())
        params = {"positions": positions_list, "intensity": intensity_list}
        self._tag_batched(params, batch, n, keep, ["positions", "intensity"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        per_instance = self._is_per_instance_params(params)
        for _, img_batch in self._get_images(batch).items():
            data = img_batch.data
            b = data.shape[0]
            if per_instance:
                rows, intensities = params["positions"], params["intensity"]
            else:
                rows, intensities = [params["positions"]] * b, [params["intensity"]] * b
            table, ratio = spike_table(rows, intensities, data.shape[2:])
            if not ratio.any():
                continue  # the reference returns the data itself
            work = data if data.is_contiguous() else data.contiguous()
            img_batch.data = ops.spike(work, table, ratio)
        return batch
