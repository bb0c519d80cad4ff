"""BiasField / Blur / Noise / Gamma / LabelsToImage behind the reference API.

Host-side mirror of transforms/intensity/{bias_field,blur,noise,gamma}.py
(TorchIO 2.0.0a2): constructor signatures, ``make_params`` RNG order and the
``params`` schema are the reference's; ``apply_transform`` runs the CUDA
kernels K2-K5 (`torchio_b200.ops`).
"""

from __future__ import annotations

import os
import warnings
from typing import Any

import numpy as np
import torch
from torch import Tensor

from .. import ops, tables
from ..data import ImagesBatch, LabelMap, ScalarImage, SubjectsBatch
from ..params import to_nonneg_range, to_range
from .base import IntensityTransform, Transform, chunk_info, staged_derived


def _as_f32(data: Tensor) -> Tensor:
    return data if data.dtype == torch.float32 else data.float()


# ---- BiasField (intensity/bias_field.py:22-197) ------------------------------


class BiasField(IntensityTransform):
    def __init__(self, *, std=0.5, scale: float = 0.025, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.std = to_nonneg_range(std)
        if scale <= 0 or scale > 1:
            raise ValueError(f"scale must be in (0, 1], got {scale}")
        self.scale = scale

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
            std = self.std.sample_1d()
            seed = int(torch.randint(0, 2**31, (1,)).item())
            return {"std": std, "seed": seed, "scale": self.scale}
        keep = self._keep_mask(batch, n)
        std = self._mask_identity(self.std.sample_1d(n), keep, identity=0.0)
        seeds = [int(torch.randint(0, 2**31, (1,)).item()) for _ in range(n)]
        params = {"std": self._serialize_param(std), "seed": seeds, "scale": self.scale}
        self._tag_batched(params, batch, n, keep, ["std", "seed"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        _apply_bias(self, batch, params["std"], params["seed"], params["scale"], divide=False)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _BiasFieldInverse:
        return _BiasFieldInverse(std=params["std"], seed=params["seed"], scale=params["scale"],
                                 copy=False)


def _bias_stage(data_shape, affines, std, seed, scale, *, divide: bool):
    """Host tables of the bias stage, or None when the transform is a no-op
    (bias_field.py:105-107,223-225)."""
    per_element = isinstance(std, list)
    if (not per_element and std == 0) or (per_element and all(s == 0 for s in std)):
        return None
    b = data_shape[0]
    if per_element and len(std) != b:
        raise RuntimeError(
            f"Per-instance parameters were recorded for {len(std)} elements"
            f" but the batch has {b}"
        )
    info = chunk_info()
    if info is not None and not per_element:
        # one generator draws the coarse fields of the whole batch: keep this slice's rows
        full = tables.coarse_bias_fields((info.total, *data_shape[1:]), std, seed, scale)
        coarse = full[info.b0:info.b1].contiguous()
    else:
        coarse = tables.coarse_bias_fields(data_shape, std, seed, scale)
    return {
        "coarse": coarse,
        "bias_identity": np.asarray([s == 0 for s in std], dtype=np.uint8) if per_element else None,
        "bias_divide": divide,
    }


def _apply_bias(transform, batch, std, seed, scale, *, divide: bool) -> None:
    run_stages(transform._get_images(batch),
               [lambda ib, index: _bias_stage(ib.data.shape, ib.affines, std, seed, scale,
                                              divide=divide)])


class _BiasFieldInverse(IntensityTransform):
    def __init__(self, *, std, seed, scale: float, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self._std, self._seed, self._scale = std, seed, scale

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        _apply_bias(self, batch, self._std, self._seed, self._scale, divide=True)
        return batch


# ---- Blur (intensity/blur.py:19-126) ------------------------------------------


class Blur(IntensityTransform):
    def __init__(self, *, std=0.0, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.std = to_nonneg_range(std)
        self._warn_if_noop(is_noop=self.std.is_constant(0.0), hint="std=(0, 2)")

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
            return {"std": self.std.sample()}
        keep = self._keep_mask(batch, n)
        std = self.std.sample(n)
        if keep is not None:
            std[~keep] = 0.0
        params = {"std": self._serialize_param(std)}
        self._tag_batched(params, batch, n, keep, ["std"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        run_stages(self._get_images(batch), [lambda ib, index: _blur_stage(ib, params, index)])
        return batch

    def prepare_stream(self, batch: SubjectsBatch, params: dict[str, Any], cache: dict, step: int) -> None:
        # taps of the whole batch: the mm -> voxel conversion of shared sigmas reads batch element
        # 0's spacing (blur.py:87), and shared-vs-stacked taps are chosen over ALL rows
        for index, ib in enumerate(self._get_images(batch).values()):
            cache[("blur", step, index)] = {"tables": _blur_stage(ib, params, index, whole=True)}


def _blur_stage(ib, params, index: int = 0, whole: bool = False):
    """Host tables of the blur stage, or None when every sigma <= 0 (the
    reference then returns the input tensor itself, blur.py:143-144).  While a batch is streamed
    in slices the rows come from the whole-batch tables `prepare_stream` cached."""
    info = None if whole else chunk_info()
    if info is not None:
        cached = info.cache.get(("blur", info.step, index))
        if cached is not None:
            full = cached["tables"]
            if full is None:
                return None
            return {"taps": full["taps"][:, info.b0:info.b1].contiguous(),
                    "radius": full["radius"][:, info.b0:info.b1].contiguous(),
                    "big_r": full["big_r"], "axes_mask": full["axes_mask"]}
    if "_batched_keys" in params:
        mm = np.asarray(params["std"], dtype=np.float64)
        sp = np.asarray([a.spacing for a in ib.affines], dtype=np.float64)
        vox = np.divide(mm, sp, out=np.zeros_like(mm), where=sp > 0)
    else:
        sp = np.asarray(ib.affines[0].spacing, dtype=np.float64)
        vox = [s / q if q > 0 else 0.0 for s, q in zip(params["std"], sp, strict=True)]
    t = tables.blur_tables(vox, ib.data.shape[0])
    if t is None:
        return None
    return {"taps": t.taps, "radius": t.radius, "big_r": t.big_r, "axes_mask": t.axes_mask}


# ---- Noise (intensity/noise.py:18-178) -----------------------------------------


def _noise_mode() -> str:
    """"exact" (default): the normals are the torch.randn draws of the recorded
    CPU-generator seed — the reference's stream (noise.py:166-178) — replayed on
    the device by `ops.randn_mt19937`, or under the first pass of the fused chain
    (host torch.randn only for draws below 16 values or beyond the jump table's reach).
    "philox": in-kernel counter-based normals — same distribution, other stream."""
    mode = os.environ.get("TIO_B200_NOISE", "exact").lower()
    if mode not in ("exact", "philox"):
        raise ValueError(f"TIO_B200_NOISE must be 'exact' or 'philox', got {mode!r}")
    return mode


class Noise(IntensityTransform):
    def __init__(self, *, mean=0.0, std=0.25, rician: bool = False, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.mean = to_range(mean)
        self.std = to_nonneg_range(std)
        self.rician = rician

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return True

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        # a slice's normals are a window of the draw over the whole batch, which the device
        # replay makes for draws of 16 or more values; the counter-based stream indexes voxels of
        # the tensor it is given
        if _noise_mode() != "exact":
            return False
        sizes = [int(np.prod(ib.data.shape)) for ib in self._get_images(batch).values()]
        if any(n < 16 for n in sizes):
            return False
        # one stream per application, continued across images and the second Rician draw: all of
        # it must lie inside the jump table's reach, or the one-shot path (host draws) takes over
        return sum(ops.mt_draw_words(n) for n in sizes) * (2 if self.rician else 1) <= ops.MT_MAX_WORDS

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        seed = int(torch.randint(0, 2**31, (1,)).item())  # drawn first (noise.py:75)
        n = self._resolve_n(batch)
        keep = self._keep_mask(batch, n)
        mean = self._mask_identity(self.mean.sample_1d(n), keep, identity=0.0)
        std = self._mask_identity(self.std.sample_1d(n), keep, identity=0.0)
        params = {
            "mean": self._serialize_param(mean), "std": self._serialize_param(std),
            "seed": seed, "rician": self.rician,
        }
        self._tag_batched(params, batch, n, keep, ["mean", "std"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        run_stages(self._get_images(batch), [_noise_stage_factory(params)])
        return batch


def _noise_stage_factory(params):
    """One CPU generator per transform application, consumed in flat
    (B,C,I,J,K) order and continuing across images and across the second
    Rician draw (noise.py:109-118,166-178)."""
    mode = _noise_mode()
    generator = torch.Generator(device="cpu")
    generator.manual_seed(params["seed"])
    rician = bool(params.get("rician", False))
    keep = params.get("_keep")

    consumed = [0]  # words of the seed's stream used so far (across images and draws)

    def draw(shape, device, defer=False):
        """Normals of the next draw of the stream for a tensor of ``shape``: the draw of
        ``prod(shape)`` values, or, while `Compose` streams slices, rows [b0, b1) of the draw over
        the whole batch (its outputs [per * b0, per * b1)).  On the device for draws of 16 or more
        values within the jump table's reach, else with torch.randn on the host, which the
        generator object keeps at ``consumed``.  ``defer``: a device draw is returned as
        (seed, start, n, lo) for `ops.intensity_fused` to make (``z_replay``)."""
        n = int(np.prod(shape))
        info = chunk_info()
        lo, n_full = (0, n) if info is None else (n // shape[0] * info.b0, n // shape[0] * info.total)
        start = consumed[0]
        on_device = (not on_host[0] and n_full >= 16 and start + ops.mt_draw_words(n_full) <= ops.MT_MAX_WORDS
                     and device.type == "cuda")
        if info is not None and not on_device:
            raise RuntimeError("Noise: this batch cannot be streamed in slices (host normal stream)")
        if n_full < 16:
            on_host[0] = True  # torch's scalar path: its word count is not followed, stay on the host
        consumed[0] += ops.mt_draw_words(n_full) if n_full >= 16 else n_full
        if on_device:
            if defer:
                return (params["seed"], start, n_full, lo), None
            return ops.randn_mt19937(params["seed"], start, n_full, device, lo=lo, hi=lo + n).view(shape), None
        # host path: fast-forward the CPU generator to `start` past the device draws, each of which
        # took 16k words or m + 16 >= 33 (a draw of m % 16 != 0): skip is 16k or >= 33
        if host_state[0] != start:
            skip = start - host_state[0]
            if skip % 16 == 0:
                torch.randn(skip, generator=generator)
            elif skip >= 33:
                torch.randn(skip - 16, generator=generator)  # ragged: skip - 16 values, 16 more words
            else:
                raise RuntimeError("Noise: cannot realign the host generator")
        pin = torch.cuda.is_available()
        z = torch.empty(shape, dtype=torch.float32, pin_memory=pin)
        torch.randn(shape, generator=generator, out=z)
        host_state[0] = consumed[0]
        return None, z

    host_state = [0]
    on_host = [False]

    def stage(ib, index):
        shape = ib.data.shape
        b = shape[0]
        out = {
            "mean": tables.per_element_vector(params["mean"], b),
            "std": tables.per_element_vector(params["std"], b),
            "keep": None if keep is None else np.asarray(keep, dtype=np.uint8),
            "rician": rician,
        }
        if mode == "philox":
            out["noise_mode"] = 2
            out["philox_seed"] = (int(params["seed"]) << 8) | (index & 0xFF)
            return out
        out["noise_mode"] = 1
        # a single device draw is left to the fused call, which can make it under its first
        # pass; the two draws of Rician noise are made here, one after the other
        z_dev, z_host = draw(shape, ib.data.device, defer=not rician)
        if z_host is not None:
            out["z_host"] = z_host
        else:
            out["z" if rician else "z_replay"] = z_dev
        if rician:
            z_dev, z_host = draw(shape, ib.data.device)
            out["z2" if z_dev is not None else "z2_host"] = z_dev if z_dev is not None else z_host
        return out

    return stage


# ---- Gamma (intensity/gamma.py:17-149) ------------------------------------------


class Gamma(IntensityTransform):
    def __init__(self, *, log_gamma=0.0, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.log_gamma = to_range(log_gamma)
        self._warn_if_noop(is_noop=self.log_gamma.is_constant(0.0), hint="log_gamma=(-0.3, 0.3)")

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
        keep = self._keep_mask(batch, n)
        log_gamma = self._mask_identity(self.log_gamma.sample_1d(n), keep, identity=0.0)
        params = {"log_gamma": self._serialize_param(log_gamma)}
        self._tag_batched(params, batch, n, keep, ["log_gamma"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        _apply_gamma(self, batch, params["log_gamma"])
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _GammaInverse:
        return _GammaInverse(log_gamma=params["log_gamma"], copy=False)


def _apply_gamma(transform, batch, log_gamma) -> None:
    run_stages(transform._get_images(batch),
               [lambda ib, index: {"gamma": tables.gamma_values(log_gamma, ib.data.shape[0])}])


class _GammaInverse(IntensityTransform):
    def __init__(self, *, log_gamma, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self._log_gamma = log_gamma

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        lg = self._log_gamma
        _apply_gamma(self, batch, [-v for v in lg] if isinstance(lg, list) else -lg)
        return batch


# ---- LabelsToImage (intensity/labels_to_image.py:19-290) ---------------------------------------


class LabelsToImage(Transform):
    """Synthetic image from a label map: per label, Gaussian tissue with a sampled mean and std,
    added to the batch as a new `ScalarImage` under ``image_key`` (existing images are untouched).

    ``make_params`` is the reference's (labels of batch element 0, RNG order, params schema).  The
    image is one `ops.labels_to_image` pass that recomputes, per voxel, the element of the
    reference's ``torch.randn_like`` draw on the label map's CUDA device that the voxel keeps: a
    device-resident batch gives the reference's image bit for bit and advances the CUDA generator
    as it does.  A host-resident batch is synthesised on the execution device from that device's
    CUDA generator (the reference would draw from the CPU generator) and the image is returned on
    the host, pinned when the label map is."""

    def __init__(self, label_key: str | None = None, *, image_key: str = "image_from_labels", mean=None,
                 std=None, default_mean=(0.1, 0.9), default_std=(0.01, 0.1), ignore_background: bool = False,
                 **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.label_key = label_key
        self.image_key = image_key
        self.mean_ranges = [to_range(m) for m in mean] if mean is not None else None
        self.std_ranges = [to_range(s) for s in std] if std is not None else None
        self.default_mean = to_range(default_mean)
        self.default_std = to_range(default_std)
        self.ignore_background = ignore_background

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        _, label_batch = self._find_label_batch(batch)
        unique = sorted(int(v) for v in label_batch.data[0].unique().tolist())
        n = self._resolve_n(batch)
        if n is None:
            means, stds = self._sample_label_values(unique)
            return {"means": means, "stds": stds}
        means_list, stds_list = [], []
        for _ in range(n):
            means, stds = self._sample_label_values(unique)
            means_list.append(means)
            stds_list.append(stds)
        params = {"means": means_list, "stds": stds_list}
        self._tag_batched(params, batch, n, None, ["means", "stds"])
        return params

    def _sample_label_values(self, unique: list[int]) -> tuple[dict[int, float], dict[int, float]]:
        """mean then std per label, in ascending order (labels_to_image.py:105-132)."""
        means: dict[int, float] = {}
        stds: dict[int, float] = {}
        for idx, label in enumerate(unique):
            if self.ignore_background and label == 0:
                means[label] = 0.0
                stds[label] = 0.0
                continue
            if self.mean_ranges is not None and idx < len(self.mean_ranges):
                means[label] = self.mean_ranges[idx].sample_1d()
            else:
                means[label] = self.default_mean.sample_1d()
            if self.std_ranges is not None and idx < len(self.std_ranges):
                stds[label] = self.std_ranges[idx].sample_1d()
            else:
                stds[label] = abs(self.default_std.sample_1d())
        return means, stds

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        name, label_batch = self._find_label_batch(batch)
        data = label_batch.data
        if not data.is_cuda:
            from .base import execution_device

            data = data.to(execution_device())
        values, draw, mean, std = tables.label_synthesis_tables(params["means"], params["stds"], data.shape[0])
        generated = ops.labels_to_image(data, values, mean, std, draw)
        batch.images[self.image_key] = ImagesBatch(generated, label_batch.affines, image_class=ScalarImage)
        staged_derived(self.image_key, name)
        return batch

    def _find_label_batch(self, batch: SubjectsBatch):
        """(name, label map batch): ``label_key``, or the first `LabelMap` (labels_to_image.py:164-179)."""
        if self.label_key is not None:
            if self.label_key not in batch.images:
                raise KeyError(f"Label key '{self.label_key}' not found. Available: {list(batch.images.keys())}")
            return self.label_key, batch.images[self.label_key]
        for name, img_batch in batch.images.items():
            if issubclass(img_batch._image_class, LabelMap):
                return name, img_batch
        raise KeyError("No LabelMap found in the subject")


# ---- Standardize / Normalize (intensity/standardize.py:17-170, normalize.py:35-369) -----------
#
# Both read their parameters off batch element 0 (optionally masked) and then apply one affine map
# to every element.  The statistics run where the data lives (`ops.moments`: fp64 sums in one
# pass; `ops.quantile_neighbours`: exact radix select instead of torch.kthvalue's sort) and the
# map is `ops.rescale`, which rounds step by step like the reference's elementwise ops.


def _resolve_mask(masking_method, img_batch, batch) -> Tensor | None:
    """None | LabelMap key | callable -> boolean mask of sample 0 (standardize.py:144-170)."""
    if masking_method is None:
        return None
    if callable(masking_method) and not isinstance(masking_method, str):
        return masking_method(img_batch.data[0]).bool()
    if isinstance(masking_method, str):
        return label_map_element0(masking_method, batch).bool()
    raise TypeError(f"masking_method must be None, str, or callable, got {type(masking_method)}")


def label_map_element0(key: str, batch) -> Tensor:
    """Batch element 0 of the `LabelMap` named ``key``, with the reference's errors for a missing key
    or an image of another class (standardize.py:144-170, mask.py:79-91)."""
    if key not in batch.images:
        raise KeyError(f'Masking method "{key}" not found in batch images.'
                       f" Available: {list(batch.images.keys())}")
    mask_batch = batch.images[key]
    from ..data import LabelMap

    if not issubclass(mask_batch._image_class, LabelMap):
        raise TypeError(f'Masking method "{key}" must refer to a LabelMap.')
    return mask_batch.data[0]


def _sample0(img_batch, mask, warn_empty: str) -> tuple[Tensor, Tensor | None]:
    """Sample 0 as a contiguous fp32 tensor plus its mask; an empty mask falls back to all voxels
    with the reference's warning."""
    tensor = _as_f32(img_batch.data[0]).contiguous()
    if mask is not None:
        mask = mask.to(tensor.device).expand_as(tensor)
        if not bool(mask.any()):
            warnings.warn(warn_empty, RuntimeWarning, stacklevel=4)
            mask = None
    return tensor, mask


class Standardize(IntensityTransform):
    """(v - mean) / std with the statistics of the (masked) first sample (standardize.py:17-107)."""

    def __init__(self, *, masking_method=None, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.masking_method = masking_method

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        stats: dict[str, tuple[float, float]] = {}
        for name, img_batch in self._get_images(batch).items():
            mask = _resolve_mask(self.masking_method, img_batch, batch)
            with _Staged(img_batch) as staged:
                tensor, mask = _sample0(staged, mask, f'Mask is empty for "{name}". Using all voxels.')
                s, dev, n = ops.moments(tensor, mask)
            mean = s / n
            var = dev / (n - 1) if n > 1 else float("nan")  # torch.std: Bessel's correction
            stats[name] = (float(np.float32(mean)), float(np.float32(np.sqrt(var))))
        return {"stats": stats}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        stats = params["stats"]
        for name, img_batch in self._get_images(batch).items():
            if name not in stats:
                continue
            mean, std = stats[name]
            if std == 0:
                raise RuntimeError(f'Standard deviation is zero for masked values in "{name}".'
                                   " Cannot standardize.")
            img_batch.data = ops.rescale(_as_f32(img_batch.data), sub=mean, div=std)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _StandardizeInverse:
        return _StandardizeInverse(stats=params["stats"], copy=False)


class _StandardizeInverse(IntensityTransform):
    def __init__(self, *, stats, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self._stats = stats

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for name, img_batch in self._get_images(batch).items():
            if name not in self._stats:
                continue
            mean, std = self._stats[name]
            if std == 0:
                continue
            img_batch.data = ops.rescale(_as_f32(img_batch.data), mul=std, add=mean)
        return batch


def _lerp_f32(a: float, b: float, weight: float) -> float:
    """Tensor.lerp(end, weight) on fp32 scalars (ATen: a + w (b - a) below 0.5, b - (b - a)(1 - w) above)."""
    a32, b32, w32 = np.float32(a), np.float32(b), np.float32(weight)
    diff = np.float32(b32 - a32)
    if w32 < np.float32(0.5):
        return float(np.float32(a32 + np.float32(w32 * diff)))
    return float(np.float32(b32 - np.float32(diff * np.float32(np.float32(1.0) - w32))))


class Normalize(IntensityTransform):
    """Clip to an input range, then map it linearly onto [out_min, out_max] (normalize.py:35-232)."""

    def __init__(self, *, out_min=-1.0, out_max=1.0, in_min=None, in_max=None, percentile_low=0.0,
                 percentile_high=100.0, masking_method=None, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.out_min = _value_range(out_min)
        self.out_max = _value_range(out_max)
        self.in_min = _value_range(in_min) if in_min is not None else None
        self.in_max = _value_range(in_max) if in_max is not None else None
        self.percentile_low = _value_range(percentile_low)
        self.percentile_high = _value_range(percentile_high)
        self.masking_method = masking_method

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        n = self._resolve_n(batch)
        out_min = self.out_min.sample_1d(n)
        out_max = self.out_max.sample_1d(n)
        pct_low = self.percentile_low.sample_1d()
        pct_high = self.percentile_high.sample_1d()
        params: dict[str, Any] = {"out_min": self._serialize_param(out_min),
                                  "out_max": self._serialize_param(out_max)}
        if self.in_min is not None and self.in_max is not None:
            params["in_min"] = self.in_min.sample_1d()
            params["in_max"] = self.in_max.sample_1d()
        else:
            in_ranges: dict[str, tuple[float, float]] = {}
            for name, img_batch in self._get_images(batch).items():
                mask = _resolve_mask(self.masking_method, img_batch, batch)
                with _Staged(img_batch) as staged:
                    tensor, mask = _sample0(staged, mask, f'Cannot compute percentiles for "{name}": mask is'
                                                          " empty. Using full range.")
                    values, weights, _ = ops.quantile_neighbours(tensor, [pct_low / 100.0, pct_high / 100.0], mask)
                low = values[0] if weights[0] == 0 else _lerp_f32(values[0], values[1], weights[0])
                high = values[2] if weights[1] == 0 else _lerp_f32(values[2], values[3], weights[1])
                in_ranges[name] = (low, high)
            params["in_ranges"] = in_ranges
        if n is not None:
            self._tag_batched(params, batch, n, None, ["out_min", "out_max"])
        return params

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for name, img_batch in self._get_images(batch).items():
            if "in_min" in params:
                in_min, in_max = params["in_min"], params["in_max"]
            else:
                in_ranges = params.get("in_ranges", {})
                if name not in in_ranges:
                    continue
                in_min, in_max = in_ranges[name]
            in_range = in_max - in_min
            if in_range == 0:
                warnings.warn(f'Cannot rescale "{name}": input range is zero.', RuntimeWarning, stacklevel=2)
                continue
            out_min, out_range = _out_min_and_range(params["out_min"], params["out_max"])
            img_batch.data = ops.rescale(_as_f32(img_batch.data), lo=in_min, hi=in_max, sub=in_min, div=in_range,
                                         mul=out_range, add=out_min)
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _RescaleInverse:
        return _RescaleInverse(out_min=params["out_min"], out_max=params["out_max"], in_min=params.get("in_min"),
                               in_max=params.get("in_max"), in_ranges=params.get("in_ranges"), copy=False)


RescaleIntensity = Normalize  # the reference's backwards-compatible alias (normalize.py:369)
ZNormalization = Standardize  # the reference's backwards-compatible alias (standardize.py:178)


def _value_range(value):
    if isinstance(value, (int, float)):
        return to_range(float(value))
    if isinstance(value, (tuple, list)):
        return to_range(tuple(float(v) for v in value))
    return to_range(value)


def _out_min_and_range(out_min, out_max):
    """Scalar pair, or per-element fp32 arrays whose difference is taken in fp32 like the
    reference's tensors (normalize.py:300-329)."""
    if isinstance(out_min, list):
        lo = np.asarray(out_min, dtype=np.float32)
        return lo, (np.asarray(out_max, dtype=np.float32) - lo).astype(np.float32)
    return out_min, out_max - out_min


class _RescaleInverse(IntensityTransform):
    def __init__(self, *, out_min, out_max, in_min, in_max, in_ranges, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self._out_min, self._out_max = out_min, out_max
        self._in_min, self._in_max, self._in_ranges = in_min, in_max, in_ranges

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for name, img_batch in self._get_images(batch).items():
            if self._in_min is not None and self._in_max is not None:
                in_min, in_max = self._in_min, self._in_max
            elif self._in_ranges is not None and name in self._in_ranges:
                in_min, in_max = self._in_ranges[name]
            else:
                continue
            in_range = in_max - in_min
            if in_range == 0:
                continue
            out_min, out_range = _out_min_and_range(self._out_min, self._out_max)
            keep = None
            if isinstance(out_range, float):
                if out_range == 0:
                    continue
            else:  # per element: rows whose output range was zero stay as they are
                keep = (out_range != 0).astype(np.uint8)
                out_range = np.where(out_range == 0, np.float32(1.0), out_range)
            data = _as_f32(img_batch.data)
            # (data - out_min) / out_range * in_range + in_min
            img_batch.data = ops.rescale(data, sub=out_min, div=out_range, mul=in_range, add=in_min, keep=keep)
        return batch


class _Staged:
    """Sample 0 of an image batch on the execution device for the statistics kernels (make_params
    runs before `Transform` stages a host batch)."""

    def __init__(self, img_batch) -> None:
        self.img_batch = img_batch

    def __enter__(self):
        data = self.img_batch.data
        if data.is_cuda:
            return self.img_batch
        from .base import execution_device

        class _View:
            pass

        view = _View()
        view.data = data[:1].to(execution_device(), non_blocking=True)
        return view

    def __exit__(self, *exc) -> None:
        return None


# ---- shared runner: 1..4 stages -> one fused launch pair per image ---------------

_TABLE_KEYS = ("coarse", "bias_identity", "taps", "radius", "mean", "std", "keep", "gamma")


def run_stages(images, stage_builders) -> None:
    """Build the host tables of every stage for every selected image, upload
    them with one staging copy per image and run `ops.intensity_fused`.

    ``stage_builders``: callables ``(images_batch, image_index) -> dict | None``
    in pipeline order bias < blur < noise < gamma (None = that stage is a no-op
    for this image).  Used by the individual transforms (one stage) and by
    `Compose` when it fuses consecutive intensity transforms."""
    for index, ib in enumerate(images.values()):
        kwargs: dict[str, Any] = {}
        for build in stage_builders:
            stage = build(ib, index)
            if stage:
                kwargs.update(stage)
        if not kwargs:
            continue
        data = ib.data
        device = data.device
        uploaded = ops.upload(device, *[kwargs.get(k) for k in _TABLE_KEYS])
        for key, value in zip(_TABLE_KEYS, uploaded, strict=True):
            if key in kwargs:
                kwargs[key] = value
        z_host, z2_host = kwargs.pop("z_host", None), kwargs.pop("z2_host", None)
        if z_host is not None:
            kwargs["z"] = z_host.to(device, non_blocking=True)
        if z2_host is not None:
            kwargs["z2"] = z2_host.to(device, non_blocking=True)
        out = ops.intensity_fused(_as_f32(data), **kwargs)
        # bias/blur return the input dtype (bias_field.py:245, blur.py:204,248);
        # noise/gamma follow torch type promotion against their fp32 operands
        promotes = ("gamma" in kwargs or "mean" in kwargs) and data.dtype != torch.float64
        ib.data = out if promotes or out.dtype == data.dtype else out.to(data.dtype)
