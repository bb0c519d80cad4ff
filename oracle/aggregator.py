"""PatchAggregator's op sequence (data/aggregator.py of TorchIO 2.0.0a2) on torch tensors.

TEST INFRASTRUCTURE.  The reference stitches patches back into a volume one patch at a time with
plain tensor ops: a slice assignment of the patch's centre (crop), or ``out[box] += patch`` and
``counts[box] += 1`` (average), or ``out[box] += patch * window`` and ``counts[box] += window``
(hann), with C-channel buffers in the patch's dtype, and divides by ``counts.clamp(min=1)`` at the
end.  `OpSequence` issues the same ops in the same order, on whatever device the patches are on (the
reference always moves them to the host), so the GPU tests can compare the CUDA kernels with it on
the same CUDA tensors.  The product never imports this module.
"""

from __future__ import annotations

import torch


def hann_window_3d(patch_shape) -> torch.Tensor:
    """The fp32 weight of each voxel of a patch: the three 1-D windows
    ``hann_window(n + 2, periodic=False)[1:-1]`` multiplied in i, j, k order onto ``ones(1)``."""
    weight = torch.ones(1)
    for axis, n in enumerate(patch_shape):
        view = [1, 1, 1]
        view[axis] = n
        weight = weight * torch.hann_window(n + 2, periodic=False)[1:-1].reshape(view)
    return weight


class OpSequence:
    """Same constructor and methods as the reference's PatchAggregator; locations are anything with
    ``index`` and ``size`` triples."""

    def __init__(self, spatial_shape, overlap_mode: str = "crop", patch_overlap=0, output_shape=None) -> None:
        if overlap_mode not in ("crop", "average", "hann"):
            raise ValueError(f"overlap_mode must be one of ('crop', 'average', 'hann'), got {overlap_mode!r}")
        self.mode = overlap_mode
        self.overlap = (patch_overlap,) * 3 if isinstance(patch_overlap, int) else tuple(patch_overlap)
        self.shape = tuple(spatial_shape if output_shape is None else output_shape)
        self.factor = (1.0, 1.0, 1.0) if output_shape is None else tuple(
            output_shape[a] / spatial_shape[a] for a in range(3))
        self.buffers: dict[str, torch.Tensor] = {}
        self.weights: dict[str, torch.Tensor] = {}

    def add_batch(self, batch, locations) -> None:
        named = {"__default__": batch} if isinstance(batch, torch.Tensor) else batch
        for key, tensor in named.items():
            for row, location in enumerate(locations):
                self._add(key, tensor[row], location)

    def get_output(self, key: str | None = None) -> torch.Tensor:
        name = "__default__" if key is None else key
        if name not in self.buffers:
            raise KeyError(f"No output for key {key!r}. Available: {[k for k in self.buffers if k != '__default__']}")
        if self.mode == "crop":
            return self.buffers[name]
        return self.buffers[name] / self.weights[name].clamp(min=1)

    def _add(self, key: str, patch: torch.Tensor, location) -> None:
        index, size = tuple(location.index), tuple(location.size)
        if self.factor != (1.0, 1.0, 1.0):
            index = tuple(round(index[a] * self.factor[a]) for a in range(3))
            size = tuple(round(size[a] * self.factor[a]) for a in range(3))
        if key not in self.buffers:
            self.buffers[key] = torch.zeros((patch.shape[0], *self.shape), dtype=patch.dtype, device=patch.device)
            if self.mode != "crop":
                self.weights[key] = torch.zeros((patch.shape[0], *self.shape), dtype=patch.dtype,
                                                device=patch.device)
        start = list(index)
        stop = [index[a] + size[a] for a in range(3)]
        if self.mode == "crop":
            first, last = [0, 0, 0], list(size)
            for a in range(3):
                trim = round(self.overlap[a] * self.factor[a]) // 2
                if start[a] > 0:
                    start[a] += trim
                    first[a] += trim
                if stop[a] < self.shape[a]:
                    stop[a] -= trim
                    last[a] -= trim
            box = (slice(None), *(slice(start[a], stop[a]) for a in range(3)))
            self.buffers[key][box] = patch[(slice(None), *(slice(first[a], last[a]) for a in range(3)))]
            return
        box = (slice(None), *(slice(start[a], stop[a]) for a in range(3)))
        if self.mode == "average":
            self.buffers[key][box] += patch
            self.weights[key][box] += 1
        else:
            window = hann_window_3d(tuple(patch.shape[-3:])).to(patch.device)
            self.buffers[key][box] += patch * window
            self.weights[key][box] += window
