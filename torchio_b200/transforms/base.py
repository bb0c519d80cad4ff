"""Transform base classes (host-side mirror of transforms/transform.py,
TorchIO 2.0.0a2).

Same contract as the reference: ``forward`` = copy -> wrap to a
``SubjectsBatch`` -> probability gate -> ``make_params`` -> ``apply_transform``
-> history -> unwrap to the caller's type (transform.py:212-254).  The RNG call
order on torch's global CPU generator is reproduced call for call
(SURVEY.md Appendix B) so a shared ``torch.manual_seed`` yields the same
``params`` as the reference.

Difference by design: ``apply_transform`` runs hand-written CUDA kernels.  A
batch that lives on the CPU is staged to the execution device for the call and
copied back, so the output device always matches the input device (what the
reference guarantees, docs/concepts/transforms.md:289-306).  Without a CUDA
device the call raises; there is no CPU fallback.
"""

from __future__ import annotations

import contextlib
import copy as _copy
import inspect
import threading
import warnings
from dataclasses import dataclass, field
from typing import Any

import numpy as np
import torch
from torch import Tensor, nn

from .. import autograd, ops
from ..data import Image, ImagesBatch, ScalarImage, Subject, SubjectsBatch
from ..params import _ParameterRange


@dataclass
class AppliedTransform:
    """History record (transform.py:29-43)."""

    name: str
    params: dict[str, Any] = field(default_factory=dict)
    include: list[str] | None = None
    exclude: list[str] | None = None


_TRANSFORM_REGISTRY: dict[str, type[Transform]] = {}
_EXEC_DEVICE: list[torch.device | None] = [None]


def set_execution_device(device: str | torch.device | None) -> None:
    """Device on which CPU-resident batches are augmented (default: current CUDA)."""
    _EXEC_DEVICE[0] = None if device is None else torch.device(device)


def execution_device() -> torch.device:
    if _EXEC_DEVICE[0] is not None:
        return _EXEC_DEVICE[0]
    if not torch.cuda.is_available():
        raise RuntimeError(
            "torchio_b200 needs a CUDA device: its transforms are CUDA kernels and"
            " there is no CPU fallback (torch.cuda.is_available() is False)"
        )
    return torch.device("cuda", torch.cuda.current_device())


@dataclass
class ChunkInfo:
    """Set while `Compose` streams a host batch through the device in slices of
    the batch axis: the transform is being applied to elements ``[b0, b1)`` of a
    batch of ``total``.  ``cache`` is shared by all slices of one call (values
    the reference derives from batch element 0, warnings already issued);
    ``step`` is the position of the transform in the pipeline."""

    b0: int
    b1: int
    total: int
    cache: dict
    step: int = 0


_chunk_local = threading.local()


def chunk_info() -> ChunkInfo | None:
    return getattr(_chunk_local, "info", None)


@contextlib.contextmanager
def chunk_scope(info: ChunkInfo | None):
    previous = getattr(_chunk_local, "info", None)
    _chunk_local.info = info
    try:
        yield info
    finally:
        _chunk_local.info = previous


_staging_local = threading.local()


def staged_derived(name: str, source: str) -> None:
    """Register an image a transform adds to a staged batch (see `_Staging.derive`); a no-op when
    the batch was not staged."""
    staging = getattr(_staging_local, "active", None)
    if staging is not None:
        staging.derive(name, source)


def staged_source_device(name: str, data: Tensor) -> torch.device:
    """The device image ``name`` had before the call staged it on the execution device (a host
    batch's CPU), or ``data``'s device when it was not staged: random draws the reference makes on
    the data's device come from that device's generator."""
    staging = getattr(_staging_local, "active", None)
    if staging is not None and name in staging.origin:
        return staging.origin[name][0]
    return data.device


def refuse_host_grad(batch: SubjectsBatch) -> None:
    """With `set_differentiable(True)`, refuse a host-resident image that requires grad: a graph
    is recorded for CUDA tensors only, never across the staging copies."""
    if not ops.differentiable_default():
        return
    for name, ib in batch.images.items():
        t = ib.data
        if t.requires_grad and not t.is_cuda:
            raise NotImplementedError(
                f'image "{name}" requires grad and lives on {t.device}: gradients are computed for'
                " CUDA tensors only; move the batch to the GPU first")


class _Staging:
    """Move a CPU batch to the execution device and back, preserving pinning.  Images a transform
    adds during the call are brought back like the image they were derived from."""

    def __init__(self, batch: SubjectsBatch) -> None:
        self.batch = batch
        self.origin: dict[str, tuple[torch.device, bool]] = {}

    def __enter__(self):
        refuse_host_grad(self.batch)
        dev = None
        for name, ib in self.batch.images.items():
            t = ib.data
            if t.is_cuda:
                continue
            dev = dev or execution_device()
            self.origin[name] = (t.device, t.is_pinned())
            ib.data = t.to(dev, non_blocking=True)
        self.previous = getattr(_staging_local, "active", None)
        _staging_local.active = self
        return self.batch

    def derive(self, name: str, source: str) -> None:
        """Image ``name``, created on the device from image ``source``, goes back to where
        ``source`` came from (device and pinning) when the call ends."""
        if source in self.origin:
            self.origin[name] = self.origin[source]

    def __exit__(self, exc_type, exc, tb):
        _staging_local.active = self.previous
        if exc_type is not None or not self.origin:
            return False
        for name, (device, pinned) in self.origin.items():
            ib = self.batch.images[name]
            t = ib.data
            if not t.is_cuda:
                continue
            t = t.contiguous()
            host = torch.empty(t.shape, dtype=t.dtype, device=device, pin_memory=pinned)
            host.copy_(t, non_blocking=pinned)
            ib.data = host
        torch.cuda.current_stream().synchronize()
        return False


def _all_gated_out(params: dict[str, Any]) -> bool:
    keep = params.get("_keep")
    return keep is not None and not any(keep)


class Transform(nn.Module):
    """Abstract base of every transform (transform.py:69-130)."""

    def __init__(self, *, p: float = 1.0, copy: bool = True, per_instance: bool = True,
                 include: list[str] | None = None, exclude: list[str] | None = None) -> None:
        super().__init__()
        if not 0 <= p <= 1:
            raise ValueError(f"Probability must be in [0, 1], got {p}")
        self.p = p
        self.copy = copy
        self.per_instance = per_instance
        self.include = include
        self.exclude = exclude

    def __init_subclass__(cls, **kwargs: Any) -> None:
        super().__init_subclass__(**kwargs)
        _TRANSFORM_REGISTRY[cls.__name__] = cls

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        """True when ``apply_transform`` on a slice of the batch axis (with
        `params.slice_params` and an active `ChunkInfo`) equals the same rows
        of the whole-batch result."""
        return False

    def prepare_stream(self, batch: SubjectsBatch, params: dict[str, Any], cache: dict, step: int) -> None:
        """Called once on the WHOLE host batch before `Compose` streams it in slices: host tables
        that depend on more than the slice's own rows (values the reference takes from batch
        element 0, dispatch decisions over all rows) go into ``cache`` here."""

    def _warn_if_noop(self, *, is_noop: bool, hint: str) -> None:
        if is_noop:
            warnings.warn(
                f"{type(self).__name__} is a no-op with the given parameters and will not"
                f" change the data. Pass arguments to apply an effect (e.g. {hint}), or a"
                " range like (a, b) for random augmentation.",
                stacklevel=3,
            )

    def __repr__(self) -> str:
        parts = []
        for name, default in _init_defaults(type(self)).items():
            value = getattr(self, name, default)
            if isinstance(value, _ParameterRange):
                if value._original == default:
                    continue
            elif value == default:
                continue
            parts.append(f"{name}={value!r}")
        return f"{type(self).__name__}({', '.join(parts)})"

    def __add__(self, other: object):
        if not isinstance(other, Transform):
            return NotImplemented
        from .compose import Compose

        left = self.transforms if isinstance(self, Compose) else [self]
        right = other.transforms if isinstance(other, Compose) else [other]
        return Compose([*left, *right])

    # -- the call path ----------------------------------------------------

    def forward(self, data: Any) -> Any:
        if self.copy:
            data = _copy.deepcopy(data)
        batch, unwrap = wrap_input(data)
        with _Staging(batch):
            batch = self._forward_batch(batch)
        return _finish(batch, unwrap)

    def _forward_batch(self, batch: SubjectsBatch) -> SubjectsBatch:
        """Gate, sample, apply, record — on an already wrapped/staged batch."""
        # torch.rand(1) is drawn even when p == 1 (transform.py:227)
        if not self._per_instance_p_active(batch) and torch.rand(1).item() >= self.p:
            return batch
        self._check_differentiable(batch)
        params = self.make_params(batch)
        batch = self.apply_transform(batch, params)
        self._record(batch, params)
        return batch

    #: The transform has a differentiable path (`torchio_b200.autograd`).
    differentiable = False

    def _check_differentiable(self, batch: SubjectsBatch) -> None:
        """With `set_differentiable(True)` and grad mode on, refuse to modify an image that
        requires grad unless the transform has a differentiable path: never detach silently."""
        if self.differentiable or not ops.differentiable_default() or not torch.is_grad_enabled():
            return
        if any(ib.data.requires_grad for ib in self._get_images(batch).values()):
            autograd.refuse(type(self).__name__)

    def _record(self, batch: SubjectsBatch, params: dict[str, Any]) -> None:
        if _all_gated_out(params):
            return
        batch.applied_transforms.append(
            AppliedTransform(
                name=type(self).__name__,
                params=params,
                include=None if self.include is None else list(self.include),
                exclude=None if self.exclude is None else list(self.exclude),
            )
        )

    # -- per-instance plumbing (transform.py:256-393) ------------------------

    @property
    def supports_per_instance_params(self) -> bool:
        return False

    @property
    def supports_per_instance_p(self) -> bool:
        return False

    def _per_instance_active(self, batch: SubjectsBatch) -> bool:
        return self.per_instance and self.supports_per_instance_params and batch.batch_size > 1

    def _per_instance_p_active(self, batch: SubjectsBatch) -> bool:
        return (
            self.per_instance
            and self.supports_per_instance_p
            and batch.batch_size > 1
            and 0.0 < self.p < 1.0
        )

    def _resolve_n(self, batch: SubjectsBatch) -> int | None:
        return batch.batch_size if self._per_instance_active(batch) else None

    def _keep_mask(self, batch: SubjectsBatch, n: int | None) -> Tensor | None:
        if n is None or not self._per_instance_p_active(batch):
            return None
        return torch.rand(n) < self.p

    @staticmethod
    def _mask_identity(value, keep: Tensor | None, *, identity: float):
        if keep is None or not isinstance(value, Tensor):
            return value
        return torch.where(keep, value, torch.full_like(value, identity))

    @staticmethod
    def _serialize_param(value):
        return value.tolist() if isinstance(value, Tensor) else value

    @staticmethod
    def _is_per_instance_params(params: dict[str, Any]) -> bool:
        return "_batched_keys" in params

    def _tag_batched(self, params, batch, n, keep, batched_keys) -> None:
        if n is None:
            return
        params["_batch_size"] = batch.batch_size
        params["_batched_keys"] = list(batched_keys)
        if keep is not None:
            params["_keep"] = keep.tolist()

    # -- to override -------------------------------------------------------------

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        raise NotImplementedError

    @property
    def invertible(self) -> bool:
        return False

    def inverse(self, params: dict[str, Any]) -> Transform:
        raise NotImplementedError(f"{type(self).__name__} is not invertible")

    def _get_images(self, batch: SubjectsBatch) -> dict[str, ImagesBatch]:
        images = batch.images
        if self.include is not None:
            images = {k: v for k, v in images.items() if k in self.include}
        if self.exclude is not None:
            images = {k: v for k, v in images.items() if k not in self.exclude}
        return images

    def to_hydra(self) -> dict[str, Any]:
        cfg: dict[str, Any] = {"_target_": f"torchio.{type(self).__qualname__}"}
        for name, default in _init_defaults(type(self)).items():
            value = getattr(self, name, default)
            if isinstance(value, _ParameterRange):
                if value._original == default:
                    continue
                value = value._original
            elif value == default:
                continue
            if isinstance(value, tuple):
                value = list(value)
            elif isinstance(value, (Tensor, np.ndarray)):
                value = value.tolist()
            cfg[name] = value
        return cfg


class SpatialTransform(Transform):
    """Transforms that change geometry: apply to images and label maps."""


class IntensityTransform(Transform):
    """Transforms that change intensities: ScalarImage batches only
    (transform.py:677-693)."""

    def _get_images(self, batch: SubjectsBatch) -> dict[str, ImagesBatch]:
        images = {k: v for k, v in batch.images.items() if v._image_class is ScalarImage}
        if self.include is not None:
            images = {k: v for k, v in images.items() if k in self.include}
        if self.exclude is not None:
            images = {k: v for k, v in images.items() if k not in self.exclude}
        return images


def _init_defaults(cls: type) -> dict[str, Any]:
    """{name: default} over the MRO's __init__ signatures (transform.py:566-591)."""
    out: dict[str, Any] = {}
    for klass in cls.__mro__:
        if klass is object or klass is nn.Module:
            break
        init = klass.__dict__.get("__init__")
        if init is None:
            continue
        for name, prm in inspect.signature(init).parameters.items():
            if name == "self" or prm.kind in (prm.VAR_POSITIONAL, prm.VAR_KEYWORD):
                continue
            out.setdefault(name, prm.default)
    return out


# -- input type round-tripping (transform.py:487-665) ---------------------------

_DEFAULT = "tio_default_image"


def wrap_input(data: Any):
    """Any supported input -> (SubjectsBatch, unwrap)."""
    if isinstance(data, SubjectsBatch):
        return data, lambda b: b
    if isinstance(data, ImagesBatch):
        return SubjectsBatch({_DEFAULT: data}), lambda b: b.images[_DEFAULT]
    if isinstance(data, Subject):
        return SubjectsBatch.from_subjects([data]), lambda b: b.unbatch()[0]
    if isinstance(data, dict):
        keys = [str(k) for k in data]
        kwargs = {k: (ScalarImage(v) if isinstance(v, Tensor) else v) for k, v in data.items()}
        sb = SubjectsBatch.from_subjects([Subject(**kwargs)])

        def unwrap_dict(b):
            sub = b.unbatch()[0]
            out = {}
            for k in keys:
                entry = sub[k] if k in sub else None
                out[k] = entry.data if isinstance(entry, Image) else entry
            return out

        return sb, unwrap_dict
    if isinstance(data, Image):
        sb = SubjectsBatch.from_subjects([Subject(**{_DEFAULT: data})])
        return sb, lambda b: b.unbatch()[0][_DEFAULT]
    if isinstance(data, Tensor):
        sb = SubjectsBatch.from_subjects([Subject(**{_DEFAULT: ScalarImage(data)})])
        return sb, lambda b: b.unbatch()[0][_DEFAULT].data
    if isinstance(data, np.ndarray):
        t = torch.as_tensor(data.copy(), dtype=torch.float32)
        if t.ndim == 3:
            t = t[None]
        sb = SubjectsBatch.from_subjects([Subject(**{_DEFAULT: ScalarImage(t)})])
        return sb, lambda b: b.unbatch()[0][_DEFAULT].data.cpu().numpy()
    raise TypeError(
        "Expected Subject, Image, Tensor, ndarray, dict, ImagesBatch, or SubjectsBatch,"
        f" got {type(data).__name__}"
    )


def _finish(batch: SubjectsBatch, unwrap) -> Any:
    result = unwrap(batch)
    if not isinstance(result, (SubjectsBatch, Tensor, np.ndarray, dict)):
        with contextlib.suppress(AttributeError):
            if isinstance(result, (Image, ImagesBatch)):
                result.applied_transforms = list(batch.applied_transforms)
    return result
