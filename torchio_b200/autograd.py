"""Differentiable path of the transforms: `torch.autograd.Function`s around the `ops` kernels.

Enabled by `torchio_b200.set_differentiable(True)`.  A transform records a graph node only when
``torch.is_grad_enabled()`` and an image it modifies requires grad; otherwise it runs its usual
kernels and saves nothing.  Gradients flow to image data only, as in the reference: matrices,
control points and fill values are constants.

Differentiable set: `Spatial` and its wrappers (`Affine`, `ElasticDeformation`, `Resample`) and
their inverses, with interpolation orders 0-1 and no anti-aliasing, on scalar images; `Resize` and
`Anisotropy`, linear and nearest, on scalar images.  Every other transform that would modify an
image requiring grad raises NotImplementedError naming itself.

The `ops` calls below receive detached tensors: `ops` stays forward-only.  For the spatial path,
casts of fp16 / bf16 / fp64 images to fp32 and back happen outside these Functions with the
differentiable ``.float()`` / ``.to(dtype)`` the reference uses.  The resolution Functions take the
image in its own dtype and run the very forward call made without grad (which converts inside the
kernel, and copies an Anisotropy element that is not degraded bit for bit, fp64 included); their
backward makes the same two casts, ``grad.float()`` before the fp32 adjoint kernel and ``.to(dtype)``
after it.  Their backwards are gathers in a fixed order, deterministic, so they run under
``torch.use_deterministic_algorithms(True)``.
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
        " no antialias) and their inverses, Resize and Anisotropy (scalar images)"
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


class _Interpolate(torch.autograd.Function):
    """`ops.interpolate` forward, `ops.interpolate_backward` backward.  The map is linear: only the
    tables, the input shape and dtype are kept; ``adjoint`` builds the CSR tables on first use."""

    @staticmethod
    def forward(ctx, src: Tensor, out_shape, idx, lam, adjoint) -> Tensor:
        ctx.in_shape, ctx.dtype, ctx.adjoint = tuple(src.shape[2:]), src.dtype, adjoint
        return ops.interpolate(src.detach(), out_shape, idx, lam)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out: Tensor):
        grad_in = ops.interpolate_backward(grad_out.float(), ctx.in_shape, *ctx.adjoint())
        return grad_in.to(ctx.dtype), None, None, None, None


class _AxisResample(torch.autograd.Function):
    """`ops.axis_resample` forward, `ops.axis_resample_backward` backward; keeps the forward's
    axis and weight rows and ``adjoint``, which builds the per-element CSR rows on first use."""

    @staticmethod
    def forward(ctx, src: Tensor, axis, lo, hi, w, linear: bool, adjoint) -> Tensor:
        ctx.dtype, ctx.axis, ctx.w, ctx.linear, ctx.adjoint = src.dtype, axis, w, linear, adjoint
        return ops.axis_resample(src.detach(), axis, lo, hi, w, linear=linear)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out: Tensor):
        grad_in = ops.axis_resample_backward(grad_out.float(), ctx.axis, ctx.w, *ctx.adjoint(), linear=ctx.linear)
        return grad_in.to(ctx.dtype), None, None, None, None, None, None


def interpolate(src: Tensor, out_shape, idx, lam, adjoint) -> Tensor:
    """`ops.interpolate` of a floating ``src`` as a graph node; ``adjoint()`` returns the
    (ptr, ent, wt) tables of the same pass (`tables.resize_adjoint_tables`,
    `tables.anisotropy_shared_adjoint_tables`)."""
    if not src.dtype.is_floating_point:
        raise TypeError(f"autograd.interpolate: expected a floating-point image, got {src.dtype}")
    return _Interpolate.apply(src, out_shape, idx, lam, adjoint)


def axis_resample(src: Tensor, axis, lo, hi, w, adjoint, *, linear: bool) -> Tensor:
    """`ops.axis_resample` of a floating ``src`` as a graph node; ``adjoint()`` returns the
    (ptr, ent) rows of `tables.anisotropy_instance_adjoint_tables` for the same arguments."""
    if not src.dtype.is_floating_point:
        raise TypeError(f"autograd.axis_resample: expected a floating-point image, got {src.dtype}")
    return _AxisResample.apply(src, axis, lo, hi, w, linear, adjoint)
