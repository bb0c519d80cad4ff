"""Differentiable path of the transforms: `torch.autograd.Function`s around the `ops` kernels.

Enabled by `torchio_b200.set_differentiable(True)`.  A transform records a graph node only when
``torch.is_grad_enabled()`` and an image it modifies requires grad; otherwise it runs its usual
kernels and saves nothing.  Gradients flow to image data only, as in the reference: matrices,
control points and fill values are constants.

Differentiable set: `Spatial` and its wrappers (`Affine`, `ElasticDeformation`, `Resample`) and
their inverses, with interpolation orders 0-1 and no anti-aliasing, on scalar images.  Every other
transform that would modify an image requiring grad raises NotImplementedError naming itself.

The `ops` calls below receive detached tensors: `ops` stays forward-only.  Casts of fp16 / bf16 /
fp64 images to fp32 and back happen outside these Functions with the differentiable ``.float()`` /
``.to(dtype)`` the reference uses.
"""

from __future__ import annotations

import warnings

import torch
from torch import Tensor
from torch.autograd.function import once_differentiable

from . import ops


def records_graph(data: Tensor) -> bool:
    """True when a transform modifying ``data`` must take the differentiable path."""
    return ops.differentiable_default() and torch.is_grad_enabled() and data.requires_grad


def refuse(transform: str, why: str = "") -> None:
    """Raise for a transform (or a configuration of one) outside the differentiable set."""
    detail = f" ({why})" if why else ""
    raise NotImplementedError(
        f"{transform}{detail} has no GPU gradient: it cannot modify an image that requires grad."
        " Transforms with gradients: Spatial, Affine, ElasticDeformation, Resample (orders 0-1,"
        " no antialias) and their inverses"
    )


def _alert_not_deterministic(op: str) -> None:
    """What ATen does for its own non-deterministic CUDA backwards (grid_sampler_3d_backward_cuda):
    raise under ``torch.use_deterministic_algorithms(True)``, warn with ``warn_only=True``."""
    if not torch.are_deterministic_algorithms_enabled():
        return
    message = (f"{op} does not have a deterministic implementation: it adds the gradient with atomics."
               " Turn off torch.use_deterministic_algorithms, or call it with warn_only=True")
    if torch.is_deterministic_algorithms_warn_only_enabled():
        warnings.warn(message, UserWarning, stacklevel=3)
    else:
        raise RuntimeError(message)


class _Resample(torch.autograd.Function):
    """K1 forward (`ops.resample`), K1ᵀ backward (`ops.resample_backward`).  ``geometry`` holds the
    device tables and keyword arguments of the forward call; the backward needs no saved tensor."""

    @staticmethod
    def forward(ctx, src: Tensor, geometry: dict) -> Tensor:
        ctx.geometry = geometry
        ctx.in_shape = tuple(src.shape[2:])
        g = geometry
        return ops.resample(src.detach(), g["mat"], g["cp"], g["flags"], g["spacing_in"], g["spacing_out"],
                            affine_first=g["affine_first"], mode=g["mode"], fill=g["fill"],
                            out_shape=g["out_shape"], box_hint=g["box_hint"], tiers=g["tiers"])

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out: Tensor):
        _alert_not_deterministic("tio_resample_backward")
        g = ctx.geometry
        grad_in = ops.resample_backward(
            grad_out.float(), ctx.in_shape, g["mat"], g["cp"], g["flags"], g["spacing_in"], g["spacing_out"],
            affine_first=g["affine_first"], mode=g["mode"], fill=g["fill"], box_hint=g["box_hint"])
        return grad_in, None


def resample(src: Tensor, **geometry) -> Tensor:
    """`ops.resample` of fp32 ``src`` as a graph node; keyword arguments as `ops.resample`."""
    if src.dtype != torch.float32:
        raise TypeError(f"autograd.resample: expected a float32 image, got {src.dtype}")
    if geometry["mode"] not in (ops.NEAREST, ops.LINEAR):
        raise ValueError(f"autograd.resample: mode {geometry['mode']} has no adjoint")
    return _Resample.apply(src, geometry)
