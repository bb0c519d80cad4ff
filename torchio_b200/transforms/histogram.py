"""Histogram standardization (transforms/intensity/histogram_standardization.py of TorchIO 2.0.0a2):
`HistogramStandardization` and `compute_histogram_landmarks` (Nyúl and Udupa, 1999).

Constructor, errors, ``make_params`` (``{}``), gating, history, ``repr`` and ``to_hydra`` are the
reference's.  Where the reference copies every element to the host for ``np.percentile`` and maps
it with about twelve torch ops, each image batch here is three device steps with no host sync:
- `ops.quantiles_batched`: the two order statistics around every percentile of every element
  (all channels together), one exact radix select for the whole batch;
- `ops.histogram_tables`: numpy's "linear" interpolation and the reference's fp32 map tables,
  built on the device;
- `ops.histogram_map`: ``slopes[bin] * x + intercepts[bin]`` in place in the batch's own tensor and
  dtype, as the reference's ``img_batch.data[i] = result`` writes it.
"""

from __future__ import annotations

from collections.abc import Callable, Sequence
from pathlib import Path
from typing import Any

import numpy as np
import torch
from torch import Tensor

from .. import ops
from ..data import ScalarImage, SubjectsBatch
from .base import IntensityTransform, execution_device

DEFAULT_CUTOFF: tuple[float, float] = (0.01, 0.99)
STANDARD_RANGE: tuple[float, float] = (0.0, 100.0)
# cutoff endpoints, deciles and quartiles: 13 positions with the default cutoff
_DEFAULT_QUANTILES: tuple[float, ...] = (0.01, 0.10, 0.20, 0.25, 0.30, 0.40, 0.50, 0.60, 0.70, 0.75, 0.80, 0.90,
                                         0.99)

# training-image dtypes whose values fp32 holds exactly, with the numpy dtype np.percentile
# subtracts the two neighbours in (bf16 has no numpy dtype: its difference is taken in fp32)
_PERCENTILE_DTYPES = {torch.float32: np.float32, torch.float16: np.float16, torch.bfloat16: np.float32,
                      torch.uint8: np.uint8, torch.int8: np.int8, torch.int16: np.int16}


def _build_quantiles(cutoff: tuple[float, float]) -> tuple[float, ...]:
    return tuple(sorted({*_DEFAULT_QUANTILES, cutoff[0], cutoff[1]}))


def _validate_quantiles(quantiles: tuple[float, ...], cutoff: tuple[float, float]) -> None:
    if len(quantiles) < 2:
        raise ValueError(f"Need at least 2 quantiles, got {len(quantiles)}")
    if any(q < 0 or q > 1 for q in quantiles):
        raise ValueError("All quantiles must be in [0, 1]")
    if cutoff[0] not in quantiles or cutoff[1] not in quantiles:
        raise ValueError(f"Cutoff values {cutoff} must be included in quantiles. Got quantiles: {quantiles}")


def _fractions(quantiles: Sequence[float]) -> np.ndarray:
    """The q that np.percentile uses for the reference's ``100.0 * q`` percentiles: ``p / 100`` in
    float64."""
    return np.asarray([100.0 * q for q in quantiles], dtype=np.float64) / 100.0


def percentiles_from_neighbours(values: np.ndarray, weights: np.ndarray, has_nan: bool,
                                dtype: torch.dtype) -> np.ndarray:
    """np.percentile's "linear" result from the order statistics a, b around each position and
    g = index - floor(index): ``a + d*g`` (``b - d*(1 - g)`` when g >= 0.5) in float64, with
    ``d = b - a`` taken in the array's own dtype (fp16 rounding, integer wrap-around); NaN
    everywhere when a selected value is NaN."""
    npdt = _PERCENTILE_DTYPES[dtype]
    values = np.asarray(values, dtype=np.float32).reshape(-1, 2)
    a, b = values[:, 0].astype(npdt), values[:, 1].astype(npdt)
    with np.errstate(over="ignore", invalid="ignore"):
        d = np.subtract(b, a).astype(np.float64)
        g = np.asarray(weights, dtype=np.float64).reshape(-1)
        out = np.where(g >= 0.5, b.astype(np.float64) - d * (1 - g), a.astype(np.float64) + d * g)
    if has_nan:
        out[:] = np.nan
    return out


def _average_mapping(database: np.ndarray) -> np.ndarray:
    """Each image's percentiles mapped linearly so that its cutoff percentiles land on
    STANDARD_RANGE, averaged over the images (float64, as the reference's
    _compute_average_mapping)."""
    low, high = STANDARD_RANGE
    scale = np.nan_to_num((high - low) / (database[:, -1] - database[:, 0]))
    offset = float(np.mean(low - scale * database[:, 0]))
    return scale @ database / len(database) + offset


def _load_tensor(source: ScalarImage | Path | str) -> Tensor:
    if isinstance(source, ScalarImage):
        return source.data
    return ScalarImage(source).data  # tensor-backed images: a path raises the package's TypeError


def compute_histogram_landmarks(images: Sequence[ScalarImage | Path | str], *,
                                quantiles: Sequence[float] | None = None,
                                cutoff: tuple[float, float] = DEFAULT_CUTOFF,
                                masking_method: Callable[[Tensor], Tensor] | None = None) -> Tensor:
    """Average standard-space landmarks of training images (histogram_standardization.py:48-113):
    each image's percentiles (all channels together, ``masking_method(tensor)`` voxels only when
    given) come from the exact select on the execution device; the float64 averaging runs on the
    host.  Returns an fp32 CPU tensor for `HistogramStandardization`."""
    quantiles = _build_quantiles(cutoff) if quantiles is None else tuple(sorted(set(quantiles)))
    _validate_quantiles(quantiles, cutoff)
    qs = _fractions(quantiles)
    rows = []
    for source in images:
        tensor = _load_tensor(source)
        if tensor.dtype not in _PERCENTILE_DTYPES:
            raise NotImplementedError(
                f"compute_histogram_landmarks: {tensor.dtype} training images are not supported (their"
                " percentiles need the neighbours in their own dtype, which fp32 does not hold exactly)")
        mask = None if masking_method is None else masking_method(tensor).bool()
        device = execution_device()
        data = tensor.to(device)[None]
        if mask is not None:
            mask = mask.to(device).expand_as(tensor)[None]
            if not bool(mask.any()):
                raise IndexError("index -1 is out of bounds for axis 0 with size 0")
        values, weights, _, has_nan = ops.quantiles_batched(data, qs, mask)
        rows.append(percentiles_from_neighbours(values[0].cpu().numpy(), weights[0].cpu().numpy(),
                                                bool(has_nan[0]), tensor.dtype))
    return torch.as_tensor(_average_mapping(np.vstack(rows)), dtype=torch.float32)


def _load_landmarks(source: Tensor | Path | str) -> Tensor:
    if isinstance(source, Tensor):
        return source.float()
    path = Path(source)
    if path.suffix == ".npy":
        return torch.as_tensor(np.load(path), dtype=torch.float32)
    if path.suffix in (".pt", ".pth"):
        data = torch.load(path, weights_only=True)
        if isinstance(data, Tensor):
            return data.float()
        raise TypeError(f"Expected a Tensor in {path}, got {type(data).__name__}")
    raise ValueError(f"Unsupported landmarks file extension: {path.suffix}")


class HistogramStandardization(IntensityTransform):
    """Piecewise-linear map of every scalar image element's percentiles onto ``landmarks``
    (histogram_standardization.py:164-303).  ``landmarks``: a tensor, or a ``.npy`` / ``.pt`` /
    ``.pth`` file, as `compute_histogram_landmarks` returns them."""

    def __init__(self, landmarks: Tensor | Path | str, *, cutoff: tuple[float, float] = DEFAULT_CUTOFF,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.landmarks = _load_landmarks(landmarks)
        self.cutoff = cutoff

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        quantiles = _build_quantiles(self.cutoff)
        for _, img_batch in self._get_images(batch).items():
            data = img_batch.data
            if data.shape[0] == 0:
                continue
            if len(self.landmarks) != len(quantiles):
                raise ValueError(
                    f"Number of landmarks ({len(self.landmarks)}) does not match the number of quantile"
                    f" positions ({len(quantiles)}). Ensure the same quantile scheme was used for training.")
            work = data if data.is_contiguous() else data.contiguous()
            values, weights, _, has_nan = ops.quantiles_batched(work, _fractions(quantiles))
            (landmarks,) = ops.upload(work.device, np.ascontiguousarray(self.landmarks.numpy()))
            tables = ops.histogram_tables(values, weights, has_nan, landmarks)
            ops.histogram_map(work, tables, len(quantiles))
            if work is not data:
                data.copy_(work)
        return batch
