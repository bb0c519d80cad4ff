"""Spatial / Affine / ElasticDeformation behind the reference API.

Host-side mirror of transforms/spatial/spatial.py (TorchIO 2.0.0a2):
constructor signatures, validation messages, ``make_params`` RNG order and the
``params`` schema are the reference's (spatial.py:307-369, 436-558,
2219-2375, 2427-2484); ``apply_transform`` packs the sampled geometry into
three small tables and runs ONE fused CUDA pass per image
(`ops.resample`, K1) instead of materialising a sampling grid and calling
``grid_sample`` twice (spatial.py:1110-1272, 1504-1857).

Supported natively: interpolation orders 0-1 (``"nearest"``/``"linear"``) through K1, B-spline
orders 2-7 (``"quadratic"`` ... ``"seventh"``) through a separable prefilter and an (n+1)^3-tap pull
at K1's sampling coordinates (the reference's ``interpol.grid_pull(bound="dct2",
extrapolate=False, prefilter=True)``, spatial.py:1734-1761, 1860-1878), and the partial-volume
``label_interpolation="label"`` with any one-hot order; ``target=None``, a concrete
``(shape, affine)`` space, an image, an image name or (random) spacings; ``antialias``; fills
``"minimum"``, ``"mean"``, ``"otsu"`` or numeric (orders 2-7 ignore them, as the reference does:
their out-of-bounds voxels are 0; their prefilter refuses an axis longer than 51199 voxels).
Raise NotImplementedError: file-path targets.
"""

from __future__ import annotations

import warnings
from numbers import Number
from pathlib import Path
from typing import Any

import numpy as np
import torch
from torch import Tensor
from torch.distributions import Distribution

from .. import autograd, ops, tables
from ..data import AffineMatrix, Image, ImagesBatch, LabelMap, SubjectsBatch
from ..params import Choice, LazyParams, _ParameterRange, to_range, uniform_from_unit
from .base import SpatialTransform, chunk_info

_ORDERS = {
    "nearest": 0, "linear": 1, "quadratic": 2, "cubic": 3,
    "fourth": 4, "fifth": 5, "sixth": 6, "seventh": 7,
}
_NAMES = {v: k for k, v in _ORDERS.items()}
LABEL_INTERPOLATION = "label"
_PAD_MODES = ("minimum", "mean", "otsu")
_SPLINE_ORDER = 3



# ---- argument parsing (messages follow spatial.py:2592-2762) -----------------


def _range(value) -> _ParameterRange:
    if isinstance(value, (Distribution, Choice)):
        return _ParameterRange(value)
    if isinstance(value, (int, float)):
        return _ParameterRange(float(value))
    if isinstance(value, tuple) and all(isinstance(v, (int, float)) for v in value):
        return _ParameterRange(tuple(float(v) for v in value))
    return _ParameterRange(value)


def _positive_range(value) -> _ParameterRange:
    r = _range(value)
    if r._distribution is None and any(lo <= 0 or hi <= 0 for lo, hi in r._ranges):
        raise ValueError(f"Scale factors must be strictly positive, got {value}")
    return r


def _nonnegative_range(value) -> _ParameterRange:
    r = _range(value)
    if r._distribution is None and any(lo < 0 or hi < 0 for lo, hi in r._ranges):
        raise ValueError(f"Value must be non-negative, got {value}")
    return r


def _interpolation(value) -> str:
    if isinstance(value, int) and not isinstance(value, bool):
        if value not in _NAMES:
            raise ValueError(f"Interpolation order {value} is not supported. Must be 0-7.")
        return _NAMES[value]
    if not isinstance(value, str):
        raise TypeError(f"Interpolation must be a string or int, got {type(value)}")
    lowered = value.lower()
    supported = (*_ORDERS, LABEL_INTERPOLATION)
    if lowered not in supported:
        raise ValueError(
            f'Interpolation "{lowered}" is not supported. Supported values are {supported}'
        )
    return lowered


def _control_points(value) -> Tensor:
    t = (
        value.clone().detach().to(torch.float32)
        if isinstance(value, Tensor)
        else torch.as_tensor(np.asarray(value), dtype=torch.float32)
    )
    if t.ndim != 4 or t.shape[-1] != 3:
        raise ValueError(
            f"control_points must have shape (n_i, n_j, n_k, 3), got {tuple(t.shape)}"
        )
    for axis, size in enumerate(t.shape[:-1]):
        if size < 4:
            raise ValueError(
                "Each control-point axis must have at least 4 elements;"
                f" axis {axis} got {size}"
            )
    return t.contiguous()


def _max_abs(cp: Tensor) -> tuple[float, float, float]:
    a = cp.abs()
    return (float(a[..., 0].max()), float(a[..., 1].max()), float(a[..., 2].max()))


# ---- geometry (float64 host math, spatial.py:2269-2375) ------------------------


def _close3(values, target: float) -> bool:
    """np.allclose(values, target) for three finite scalars (rtol 1e-5, atol 1e-8)."""
    tol = 1e-8 + 1e-5 * abs(target)
    return all(abs(v - target) <= tol for v in values)


def _rotation(degrees: np.ndarray) -> np.ndarray:
    rx, ry, rz = np.radians(degrees)
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    mx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]], dtype=np.float64)
    my = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]], dtype=np.float64)
    mz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]], dtype=np.float64)
    return mz @ my @ mx


def build_forward_affine(scales, degrees, translation, center: str, shape, affine) -> np.ndarray:
    """World-space T = [R S | c - R S c + t], pivot at the image centre."""
    scaling = np.array(scales, dtype=np.float64)
    rotation = np.array(degrees, dtype=np.float64)
    shift = np.array(translation, dtype=np.float64)
    if shape[-1] == 1:  # 2-D input: suppress out-of-plane terms
        scaling[2] = 1.0
        rotation[0] = rotation[1] = 0.0
        shift[2] = 0.0
    rs = _rotation(rotation) @ np.diag(scaling)
    t = np.eye(4, dtype=np.float64)
    t[:3, :3] = rs
    if center == "image":
        m = affine.numpy()
        c = m[:3, 3] + m[:3, :3] @ ((np.asarray(shape, dtype=np.float64) - 1) / 2)
        t[:3, 3] = c - rs @ c
    t[:3, 3] += shift
    return t


def build_forward_affines(scales, degrees, translation, center: str, shape, affine) -> np.ndarray:
    """`build_forward_affine` for (n, 3) parameter arrays -> (n, 4, 4).  Stacked
    `np.matmul` runs the same inner kernel per matrix, so the result is
    bit-identical to the per-element version (tests/test_host_params.py)."""
    scaling = np.array(scales, dtype=np.float64)
    rotation = np.array(degrees, dtype=np.float64)
    shift = np.array(translation, dtype=np.float64)
    if shape[-1] == 1:
        scaling[:, 2] = 1.0
        rotation[:, :2] = 0.0
        shift[:, 2] = 0.0
    n = len(scaling)
    r = np.radians(rotation)
    cx, sx, cy, sy, cz, sz = (np.cos(r[:, 0]), np.sin(r[:, 0]), np.cos(r[:, 1]), np.sin(r[:, 1]),
                              np.cos(r[:, 2]), np.sin(r[:, 2]))
    z, o = np.zeros(n), np.ones(n)
    row = lambda a, b, c: np.stack([a, b, c], axis=-1)  # noqa: E731
    mx = np.stack([row(o, z, z), row(z, cx, -sx), row(z, sx, cx)], axis=-2)
    my = np.stack([row(cy, z, sy), row(z, o, z), row(-sy, z, cy)], axis=-2)
    mz = np.stack([row(cz, -sz, z), row(sz, cz, z), row(z, z, o)], axis=-2)
    diag = np.zeros((n, 3, 3))
    diag[:, 0, 0], diag[:, 1, 1], diag[:, 2, 2] = scaling[:, 0], scaling[:, 1], scaling[:, 2]
    rs = (mz @ my @ mx) @ diag
    t = np.zeros((n, 4, 4))
    t[:, 3, 3] = 1.0
    t[:, :3, :3] = rs
    if center == "image":
        m = affine.numpy()
        c = m[:3, 3] + m[:3, :3] @ ((np.asarray(shape, dtype=np.float64) - 1) / 2)
        t[:, :3, 3] = c - rs @ c
    t[:, :3, 3] += shift
    return t


def _sample_control_points(grid_shape, max_displacement, locked_borders: int) -> Tensor:
    """U(-max, +max) per axis, outer shells zeroed (spatial.py:2241-2266)."""
    field = torch.rand(*grid_shape, 3, dtype=torch.float32)
    field -= 0.5
    field *= 2
    for axis in range(3):
        field[..., axis] *= max_displacement[axis]
    for border in range(locked_borders):
        field[border, :] = 0
        field[-1 - border, :] = 0
        field[:, border] = 0
        field[:, -1 - border] = 0
        field[:, :, border] = 0
        field[:, :, -1 - border] = 0
    return field


def _check_folding(cp_shape, max_displacement, shape, spacing) -> None:
    """RuntimeWarning heuristic of spatial.py:2192-2216."""
    mesh = np.asarray(cp_shape, dtype=np.float64) - _SPLINE_ORDER
    grid_spacing = np.asarray(shape, dtype=np.float64) * spacing / mesh
    conflicts = np.asarray(max_displacement, dtype=np.float64) > grid_spacing / 2
    if np.any(conflicts):
        (where,) = np.where(conflicts)
        warnings.warn(
            "The maximum displacement is larger than half the coarse-grid spacing for"
            f" dimensions {where.tolist()}, so folding may occur",
            RuntimeWarning,
            stacklevel=4,
        )


def _folding_warning(cps, max_displacements, out_shape, a_out) -> None:
    """One warning for the batch: test the largest displacement of any element."""
    sp_out = np.asarray(a_out.spacing, dtype=np.float64)
    worst, grid_shape = None, None
    for index, cp in enumerate(cps):
        if cp is None:
            continue
        disp = max_displacements[index] if max_displacements else None
        if disp is None:
            disp = np.abs(cp).reshape(-1, 3).max(axis=0)
        disp = np.asarray(disp, dtype=np.float64)
        worst = disp if worst is None else np.maximum(worst, disp)
        grid_shape = cp.shape[:3]
    if worst is not None:
        _check_folding(grid_shape, worst, out_shape, sp_out)


def _shape_of(ib: ImagesBatch) -> tuple[int, int, int]:
    s = ib.data.shape
    return (int(s[-3]), int(s[-2]), int(s[-1]))


def _check_shared_space(images, shape, affine: AffineMatrix) -> None:
    ref = affine.numpy()
    for name, ib in images.items():
        if _shape_of(ib) != shape:
            raise RuntimeError(f'Image "{name}" has shape {_shape_of(ib)}, expected {shape}')
        stacked = np.stack([a.numpy() for a in ib.affines])
        if np.allclose(stacked, ref, rtol=1e-6, atol=1e-6):
            continue
        for a in ib.affines:
            if not np.allclose(a.numpy(), ref, rtol=1e-6, atol=1e-6):
                raise RuntimeError(
                    "Spatial transforms with affine or elastic components require"
                    " selected images to share the same affine"
                )


def _space_to_json(space):
    if space is None:
        return None
    shape, affine = space
    return {"shape": list(shape), "affine": affine.numpy().tolist()}


def _space_from_json(d):
    if d is None:
        return None
    s = d["shape"]
    return (int(s[0]), int(s[1]), int(s[2])), AffineMatrix(np.asarray(d["affine"], dtype=np.float64))


def _resolve_target(target, batch, shape, affine):
    """User-facing ``target`` -> ``(shape, affine)`` or None (spatial.py:1392-1422): an Image, a
    ``(shape, affine)`` pair, the name of an image of the subject, or a spacing specification
    (scalar, 3 values, or anything `_ParameterRange` samples: ranges, Choice, Distribution — drawn
    here, after the geometry, as upstream)."""
    if target is None:
        return None
    if isinstance(target, Image):
        return tuple(target.spatial_shape), target.affine.clone()
    if isinstance(target, (str, Path)):
        if isinstance(target, str) and target in batch.images:
            reference = batch.images[target]
            return _shape_of(reference), reference.affines[0].clone()
        if Path(target).is_file():
            raise NotImplementedError("torchio_b200 reads no image files: pass the target Image or (shape, affine)")
        raise ValueError(f'Unknown target "{target}". Pass a file path, an image name in the'
                         " subject, an Image, or a spacing specification")
    if isinstance(target, tuple) and len(target) == 2 and not isinstance(target[0], Number):
        s, a = target
        if len(s) != 3:
            raise ValueError(f"Target shape must have length 3, got {len(s)}")
        return (int(s[0]), int(s[1]), int(s[2])), AffineMatrix(a)
    if not isinstance(target, (int, float, tuple, list, np.ndarray, Choice, Distribution)):
        raise ValueError(f'Target not understood: "{target}"')
    return _space_for_spacing(shape, affine, _resolve_target_spacing(target))


def _parse_spacing(value) -> tuple[float, float, float]:
    """Strictly positive 3-tuple (spatial.py:2566-2587)."""
    if isinstance(value, (int, float)):
        spacing = (float(value),) * 3
    else:
        flat = [float(v) for v in (value.flat if isinstance(value, np.ndarray) else value)]
        if len(flat) != 3:
            kind = "Spacing array" if isinstance(value, np.ndarray) else "Spacing"
            raise ValueError(f"{kind} must have 3 values, got {len(flat)}")
        spacing = (flat[0], flat[1], flat[2])
    if any(v <= 0 for v in spacing):
        raise ValueError(f"Spacing must be strictly positive, got {spacing}")
    return spacing


def _resolve_target_spacing(value) -> tuple[float, float, float]:
    """spatial.py:1445-1469: deterministic for scalars / arrays, else one `_ParameterRange` draw."""
    if isinstance(value, np.ndarray):
        return _parse_spacing(value)
    if isinstance(value, (int, float)):
        return _parse_spacing(float(value))
    spec = tuple(value) if isinstance(value, list) else value
    return _parse_spacing(to_range(spec).sample())


def _space_for_spacing(shape, affine: AffineMatrix, spacing):
    """Output grid of a new voxel spacing: same physical centre, ``floor(shape * old / new)``
    voxels, singleton axes kept (spatial.py:1472-1501)."""
    old_spacing = np.asarray(affine.spacing, dtype=np.float64)
    new_spacing = np.asarray(spacing, dtype=np.float64)
    old_shape = np.asarray(shape, dtype=np.float64)
    new_shape = np.floor(old_shape * old_spacing / new_spacing)
    new_shape[old_shape == 1] = 1
    rotation = np.asarray(affine.direction, dtype=np.float64)
    old_center = np.asarray(affine.origin, dtype=np.float64) + rotation @ (((old_shape - 1) / 2) * old_spacing)
    new_origin = old_center - rotation @ (((new_shape - 1) / 2) * new_spacing)
    matrix = np.eye(4, dtype=np.float64)
    matrix[:3, :3] = rotation * new_spacing
    matrix[:3, 3] = new_origin
    return (int(new_shape[0]), int(new_shape[1]), int(new_shape[2])), AffineMatrix(matrix)


def _antialias_sigmas(factors, spacing) -> np.ndarray:
    """Per-axis sigma in voxels for the axes that are downsampled (Cardoso et al., MICCAI 2015;
    spatial.py:1951-1978, same float64 operation order)."""
    sigmas = np.zeros(3, dtype=np.float64)
    for axis in range(3):
        k = factors[axis]
        if k <= 1.0:
            continue
        variance = (k**2 - 1) * (2 * np.sqrt(2 * np.log(2))) ** (-2)
        sigma_mm = spacing[axis] * np.sqrt(variance)
        sigmas[axis] = sigma_mm / spacing[axis]
    return sigmas


def _antialias(data, a_in: AffineMatrix, a_out: AffineMatrix):
    """Gaussian pre-filter of `_antialias_batch` (spatial.py:1921-1948): one shared set of taps,
    replicate padding, through the blur kernels of the intensity path (K3)."""
    input_spacing = np.asarray(a_in.spacing, dtype=np.float64)
    factors = np.asarray(a_out.spacing, dtype=np.float64) / input_spacing
    sigmas = _antialias_sigmas(factors, input_spacing)
    if np.all(sigmas == 0):
        return data
    t = tables.blur_tables([float(v) for v in sigmas], data.shape[0])
    taps, radius = ops.upload(data.device, t.taps, t.radius)
    native = data if data.dtype == torch.float32 else data.float()
    out = ops.blur(native, taps, radius, t.big_r, t.axes_mask, None)
    return out if out.dtype == data.dtype else out.to(data.dtype)


# ---- the transform -----------------------------------------------------------


class Spatial(SpatialTransform):
    """Resample + affine + elastic in one fused pass (spatial.py:158-369)."""

    differentiable = True  # orders 0-1 without antialias: autograd.resample

    def __init__(self, *, target=None, scales=1.0, degrees=0.0, translation=0.0,
                 isotropic: bool = False, center: str = "image", control_points=None,
                 num_control_points=7, max_displacement=0.0, locked_borders: int = 2,
                 affine_first: bool = True, image_interpolation="linear",
                 label_interpolation="nearest", one_hot_label_interpolation="linear",
                 antialias: bool = False, default_pad_value="minimum",
                 default_pad_label=0, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        self.target = target
        if isotropic and not isinstance(scales, Distribution):
            if isinstance(scales, tuple) and len(scales) in (3, 6):
                raise ValueError(
                    "If isotropic=True, scales must be a single value or a 2-value range"
                )
        self.scales = _positive_range(scales)
        self.degrees = _range(degrees)
        self.translation = _range(translation)
        self.isotropic = isotropic
        if center not in ("image", "origin"):
            raise ValueError(f'center must be "image" or "origin", got "{center}"')
        self.center = center
        self.control_points = None if control_points is None else _control_points(control_points)
        ncp = (num_control_points,) * 3 if isinstance(num_control_points, int) else num_control_points
        for axis, number in enumerate(ncp):
            if not isinstance(number, int) or number < 4:
                raise ValueError(
                    "Each num_control_points value must be an integer greater than 3;"
                    f" axis {axis} got {number}"
                )
        self.num_control_points = tuple(ncp)
        self.max_displacement = _nonnegative_range(max_displacement)
        if locked_borders not in (0, 1, 2):
            raise ValueError(f"locked_borders must be 0, 1, or 2, got {locked_borders}")
        self.locked_borders = locked_borders
        if self.locked_borders == 2 and 4 in self.num_control_points:
            raise ValueError(
                "locked_borders=2 with 4 control points along any axis yields an"
                " identity elastic field"
            )
        self.affine_first = affine_first
        image_interpolation = _interpolation(image_interpolation)
        if image_interpolation == LABEL_INTERPOLATION:
            raise ValueError(
                f'image_interpolation cannot be "{LABEL_INTERPOLATION}"; that mode'
                " is only valid for label_interpolation"
            )
        self.image_interpolation = image_interpolation
        self.label_interpolation = _interpolation(label_interpolation)
        one_hot = _interpolation(one_hot_label_interpolation)
        if one_hot == LABEL_INTERPOLATION:
            raise ValueError(
                f'one_hot_label_interpolation cannot be "{LABEL_INTERPOLATION}"; choose'
                ' an interpolation for the one-hot channels (e.g. "linear")'
            )
        self.one_hot_label_interpolation = one_hot
        self.antialias = antialias
        if isinstance(default_pad_value, Number):
            default_pad_value = float(default_pad_value)
        elif default_pad_value not in _PAD_MODES:
            raise ValueError(
                'default_pad_value must be "minimum", "mean", "otsu", or a numeric value'
            )
        self.default_pad_value = default_pad_value
        if not isinstance(default_pad_label, Number):
            raise TypeError(f"default_pad_label must be numeric, got {type(default_pad_label)}")
        self.default_pad_label = float(default_pad_label)

    @property
    def supports_per_instance_params(self) -> bool:
        return True

    @property
    def supports_per_instance_p(self) -> bool:
        return self.target is None

    # -- sampling (RNG order: SURVEY.md Appendix B) ---------------------------

    def _sample_one(self, shape, affine: AffineMatrix):
        if self.isotropic:
            v = self.scales.sample_1d()
            scales = (v, v, v)
        else:
            scales = self.scales.sample()
        degrees = self.degrees.sample()
        translation = self.translation.sample()
        has_affine = not (
            _close3(scales, 1.0) and _close3(degrees, 0.0) and _close3(translation, 0.0)
        )
        if self.control_points is not None:
            cp, max_disp = self.control_points.clone(), _max_abs(self.control_points)
        else:
            max_disp = self.max_displacement.sample()
            if all(v == 0.0 for v in max_disp):
                cp, max_disp = None, None
            else:
                cp = _sample_control_points(self.num_control_points, max_disp, self.locked_borders)
        forward = None
        if has_affine:
            forward = build_forward_affine(scales, degrees, translation, self.center, shape, affine)
        return forward, cp, max_disp

    # -- vectorised per-instance sampling (same RNG stream, one draw) ----------

    def _draw_plan(self):
        """[(lo, hi) | constant] in the order `_sample_one` consumes the stream, or
        None when a spec is not a plain number / (lo, hi) range."""
        if self.control_points is not None:
            return None
        plan = []
        groups = [self.scales._axes[:1] if self.isotropic else self.scales._axes,
                  self.degrees._axes, self.translation._axes, self.max_displacement._axes]
        for axes in groups:
            for spec in axes:
                if isinstance(spec, (int, float)):
                    plan.append(float(spec))
                elif isinstance(spec, tuple):
                    plan.append(float(spec[0]) if spec[0] == spec[1] else (float(spec[0]), float(spec[1])))
                else:
                    return None
        return plan

    def _sample_batch_fast(self, n, keep, shape, affine):
        """All kept elements from ONE `torch.rand` call that consumes exactly the
        numbers the per-element loop would (uniform_ == fma(u, hi-lo, lo); a
        block `torch.rand(m)` == m consecutive draws).  Returns None (RNG
        untouched) when the fast plan does not apply."""
        plan = self._draw_plan()
        if plan is None:
            return None
        kept = [i for i in range(n) if keep is None or bool(keep[i])]
        n_scalar = sum(isinstance(p, tuple) for p in plan)
        disp_specs = plan[-3:]
        elastic = not all(not isinstance(p, tuple) and p == 0.0 for p in disp_specs)
        n_cp = int(np.prod(self.num_control_points)) * 3 if elastic else 0
        per = n_scalar + n_cp
        state = torch.get_rng_state() if (elastic and per) else None
        u = torch.rand(len(kept) * per).numpy().reshape(len(kept), per) if per else None
        cols, col = [], 0
        for p in plan:
            if isinstance(p, tuple):
                cols.append(uniform_from_unit(u[:, col], *p).astype(np.float64))
                col += 1
            else:
                cols.append(np.full(len(kept), p, dtype=np.float64))
        values = np.stack(cols, axis=1) if cols else np.zeros((len(kept), 0))
        ns = 1 if self.isotropic else 3
        scales = np.repeat(values[:, :1], 3, axis=1) if self.isotropic else values[:, :3]
        degrees, translation = values[:, ns:ns + 3], values[:, ns + 3:ns + 6]
        max_disp = values[:, ns + 6:ns + 9]
        if elastic and bool(np.any(np.all(max_disp == 0.0, axis=1))):
            torch.set_rng_state(state)  # an all-zero draw skips the grid: replay the slow way
            return None
        forwards, cps, disps = [None] * n, [None] * n, [None] * n
        tol1, tol0 = 1e-8 + 1e-5, 1e-8
        has_affine = ~(np.all(np.abs(scales - 1.0) <= tol1, axis=1)
                       & np.all(np.abs(degrees) <= tol0, axis=1)
                       & np.all(np.abs(translation) <= tol0, axis=1))
        fields = None
        if elastic:
            ni, nj, nk = self.num_control_points
            fields = u[:, n_scalar:].reshape(len(kept), ni, nj, nk, 3).copy()
            fields -= np.float32(0.5)
            fields *= np.float32(2)
            fields *= max_disp.astype(np.float32)[:, None, None, None, :]
            for border in range(self.locked_borders):
                fields[:, border] = 0; fields[:, -1 - border] = 0
                fields[:, :, border] = 0; fields[:, :, -1 - border] = 0
                fields[:, :, :, border] = 0; fields[:, :, :, -1 - border] = 0
        if has_affine.any():
            rows = np.nonzero(has_affine)[0]
            mats = build_forward_affines(scales[rows], degrees[rows], translation[rows],
                                         self.center, shape, affine)
            for row, mat in zip(rows, mats):
                forwards[kept[row]] = mat
        for row, index in enumerate(kept):
            if elastic:
                cps[index] = fields[row]
                disps[index] = [float(v) for v in max_disp[row]]
        return forwards, cps, disps

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        images = self._get_images(batch)
        if not images:
            return {"selected_images": []}
        first = next(iter(images.values()))
        shape, affine = _shape_of(first), first.affines[0]
        params = LazyParams({
            "selected_images": list(images),
            "original": _space_to_json((shape, affine)),
            "affine_first": self.affine_first,
            "image_interpolation": self.image_interpolation,
            "label_interpolation": self.label_interpolation,
            "one_hot_label_interpolation": self.one_hot_label_interpolation,
            "antialias": self.antialias,
            "default_pad_value": self.default_pad_value,
            "default_pad_label": self.default_pad_label,
        })
        n = self._resolve_n(batch)
        if n is None:
            forward, cp, max_disp = self._sample_one(shape, affine)
            if forward is not None or cp is not None:
                _check_shared_space(images, shape, affine)
            params["target"] = _space_to_json(_resolve_target(self.target, batch, shape, affine))
            params["affine_matrix"] = None if forward is None else forward.tolist()
            params["control_points"] = None if cp is None else cp.tolist()
            params["max_displacement"] = list(max_disp) if max_disp else None
            params._packed = ([forward], [None if cp is None else cp.numpy()], False)
            return params
        keep = self._keep_mask(batch, n)
        sampled = self._sample_batch_fast(n, keep, shape, affine)
        if sampled is None:
            forwards, cps, disps = [], [], []
            for index in range(n):
                if keep is not None and not bool(keep[index]):
                    forwards.append(None); cps.append(None); disps.append(None)
                    continue
                forward, cp, max_disp = self._sample_one(shape, affine)
                forwards.append(forward)
                cps.append(None if cp is None else cp.numpy())
                disps.append(list(max_disp) if max_disp else None)
        else:
            forwards, cps, disps = sampled
        if any(f is not None for f in forwards) or any(c is not None for c in cps):
            _check_shared_space(images, shape, affine)
        params["target"] = _space_to_json(_resolve_target(self.target, batch, shape, affine))
        params.set_lazy("affine_matrix",
                        lambda: [None if f is None else f.tolist() for f in forwards])
        params.set_lazy("control_points",
                        lambda: [None if c is None else c.tolist() for c in cps])
        params["max_displacement"] = disps
        self._tag_batched(params, batch, n, keep,
                          ["affine_matrix", "control_points", "max_displacement"])
        params._packed = (forwards, cps, True)
        return params

    def supports_chunks(self, batch: SubjectsBatch) -> bool:
        # a target space changes shape/affine, which later children's make_params read;
        # streamed execution samples every child on the batch as it enters the pipeline
        return self.target is None

    def plan_checks(self, batch: SubjectsBatch, params: dict[str, Any]) -> None:
        """Whole-batch host checks of `apply_transform`, run once when the batch is
        streamed in slices (each slice then skips them)."""
        names = params.get("selected_images", [])
        if not names:
            return
        mats, cps, per_instance = _unpack_geometry(params)
        first = batch.images[names[0]]
        target = _space_from_json(params["target"])
        out_shape, a_out = (_shape_of(first), first.affines[0]) if target is None else target
        no_geometry = all(m is None for m in mats) and all(c is None for c in cps)
        if no_geometry and target is None:
            return
        disps = params["max_displacement"]
        _folding_warning(cps, disps if per_instance else [disps], out_shape, a_out)

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        names = params.get("selected_images", [])
        if not names:
            return batch
        geometry = _unpack_geometry(params)
        disps = params["max_displacement"]
        if not geometry[2]:
            disps = [disps]
        _apply_spatial(
            batch, names, _space_from_json(params["target"]), geometry, max_displacements=disps,
            affine_first=params["affine_first"],
            image_interpolation=params["image_interpolation"],
            label_interpolation=params["label_interpolation"],
            antialias=params.get("antialias", False),
            one_hot_label_interpolation=params.get("one_hot_label_interpolation", "linear"),
            default_pad_value=params["default_pad_value"],
            default_pad_label=float(params["default_pad_label"]), transform=type(self).__name__,
        )
        return batch

    @property
    def invertible(self) -> bool:
        return True

    def inverse(self, params: dict[str, Any]) -> _SpatialInverse:
        """Exact inverse affine, negated elastic field, flipped order, original
        grid as target (spatial.py:617-676, 925-959)."""
        original = _space_from_json(params["original"])
        if original is None:
            raise RuntimeError("Spatial inverse needs the original output space")
        mats, cps, per_instance = _unpack_geometry(params)
        inv_mats = [None if m is None else np.linalg.inv(np.asarray(m, dtype=np.float64))
                    for m in mats]
        inv_cps = [None if c is None else -np.asarray(c, dtype=np.float32) for c in cps]
        return _SpatialInverse(
            target=original, geometry=(inv_mats, inv_cps, per_instance),
            affine_first=not params["affine_first"],
            image_interpolation=params["image_interpolation"],
            label_interpolation=params["label_interpolation"],
            one_hot_label_interpolation=params.get("one_hot_label_interpolation", "linear"),
            default_pad_value=params["default_pad_value"],
            default_pad_label=float(params["default_pad_label"]),
            copy=False, include=params["selected_images"],
        )


def _unpack_geometry(params):
    """(affine matrices, control grids, per_instance) as numpy, reusing the
    arrays make_params just produced when ``params`` is that very dict."""
    packed = getattr(params, "_packed", None)
    if packed is not None:
        return packed
    per_instance = "affine_matrix" in (params.get("_batched_keys") or [])
    mats, cps = params["affine_matrix"], params["control_points"]
    if not per_instance:
        mats, cps = [mats], [cps]
    mats = [None if m is None else np.asarray(m, dtype=np.float64) for m in mats]
    cps = [None if c is None else np.asarray(c, dtype=np.float32) for c in cps]
    return mats, cps, per_instance


class _SpatialInverse(SpatialTransform):
    """Concrete inverse used by history replay (spatial.py:679-756)."""

    differentiable = True

    def __init__(self, *, target, geometry, affine_first, image_interpolation,
                 label_interpolation, default_pad_value, default_pad_label,
                 one_hot_label_interpolation="linear", **kwargs: Any):
        super().__init__(**kwargs)
        self.one_hot_label_interpolation = one_hot_label_interpolation
        self.target = target
        self.geometry = geometry
        self.affine_first = affine_first
        self.image_interpolation = image_interpolation
        self.label_interpolation = label_interpolation
        self.default_pad_value = default_pad_value
        self.default_pad_label = float(default_pad_label)

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        _apply_spatial(
            batch, list(self._get_images(batch)), self.target, self.geometry,
            affine_first=self.affine_first, image_interpolation=self.image_interpolation,
            label_interpolation=self.label_interpolation, antialias=False,
            one_hot_label_interpolation=self.one_hot_label_interpolation,
            default_pad_value=self.default_pad_value, default_pad_label=self.default_pad_label,
            transform=type(self).__name__,
        )
        return batch


def _border_faces(data: Tensor) -> Tensor:
    """(C, n) values of the six boundary faces of sample 0, in the reference's order (edges and
    corners counted once per face they belong to, spatial.py:2115-2124)."""
    x = data[0]
    c = x.shape[0]
    faces = [x[:, 0], x[:, -1], x[:, :, 0], x[:, :, -1], x[:, :, :, 0], x[:, :, :, -1]]
    return torch.cat([f.reshape(c, -1) for f in faces], dim=1)


def _otsu_border_mean(borders: np.ndarray) -> float:
    """`_border_mean(filter_otsu=True)` of one channel (spatial.py:2105-2168).  The reference sweeps
    the sorted values in a Python loop with float64 running sums; cumsum is the same left-to-right
    accumulation, so threshold and mean are the reference's bit for bit (fp32 mean included)."""
    values = np.sort(borders.astype(np.float32), kind="stable")
    n = values.size
    if n == 0:
        return 0.0
    as64 = values.astype(np.float64)
    total = float(torch.from_numpy(values).sum().item())  # sorted_values.sum(): torch's fp32 reduction
    threshold = float(values[0])
    if n > 1:
        counts = np.arange(1, n, dtype=np.float64)
        background = np.cumsum(as64[:-1])
        mean_b = background / counts
        mean_f = (total - background) / (n - counts)
        variance = (counts / n) * ((n - counts) / n) * (mean_b - mean_f) ** 2
        best = int(np.argmax(variance))  # first maximum, like the strict `>` of the sweep
        if variance[best] > 0.0:
            threshold = float(values[best])
    below = torch.from_numpy(borders.astype(np.float32))
    below = below[below < threshold]
    if below.numel() > 0:
        return float(below.mean().item())
    return float(torch.from_numpy(borders.astype(np.float32)).mean().item())


def _fill_tensor(data: Tensor, is_label: bool, pad_value, pad_label):
    """Device (C,) fill or None (= skip the mask step, only for a python-float
    0.0; spatial.py:2034-2086)."""
    c = data.shape[1]
    if is_label:
        value = float(pad_label)
    elif isinstance(pad_value, Number):
        value = float(pad_value)
    elif pad_value == "minimum":  # sample 0, per channel, no host sync
        first = data[:1]
        return ops.min_sample0(first if first.dtype == torch.float32 else first.float())
    elif pad_value == "mean":  # mean of the six border faces of sample 0
        return _border_faces(data).float().mean(dim=1)
    else:  # "otsu": mean of the border voxels below their Otsu threshold (spatial.py:2105-2168)
        borders = _border_faces(data).float().cpu().numpy()  # C x 6 faces: ~1.5 MB at 256^3
        return torch.tensor([_otsu_border_mean(row) for row in borders], dtype=torch.float32, device=data.device)
    if value == 0.0:
        return None
    return torch.full((c,), value, dtype=torch.float32, device=data.device)


def _resample_label_pv(data, resample, spline, *, antialias, a_in, a_out, one_hot_interpolation, pad_label):
    """``label_interpolation="label"`` (spatial.py:1275-1389).  ``resample(tensor, mode, fill, exact)``
    runs K1 with the call's geometry, ``spline(tensor, order, in_place)`` the B-spline pull of order
    2-7 (`_spline`).

    C == 1, linear, no anti-aliasing: the fused TIO_LABEL_PV mode (no one-hot channels in HBM).
    C == 1 otherwise: one-hot channels -> [blur] -> K1 with the reference's exact coordinate chain
    (argmax ties and the 0.5 threshold are decided by the last bit), or the B-spline prefilter in
    place and pull -> argmax / pad label.
    C > 1: the channels are sampled as they are, zero padding, floating-point result."""
    order = _ORDERS[one_hot_interpolation]
    mode = ops.NEAREST if order == 0 else ops.LINEAR
    if data.shape[1] > 1:
        smoothed = data if data.dtype == torch.float32 else data.float()
        if antialias:
            smoothed = _antialias(smoothed, a_in, a_out)
        if order >= 2:  # in place only on a tensor made here
            sampled = spline(smoothed, order, smoothed is not data)
        else:
            sampled = resample(smoothed, mode, None, True)
        return sampled.to(data.dtype) if data.dtype.is_floating_point else sampled
    native = data if data.dtype in ops.DTYPE_CODES else data.float()
    if not antialias and order == 1:
        pad = torch.full((1,), float(pad_label), dtype=torch.float32, device=data.device)
        out = resample(native, ops.LABEL_PV, pad, True)
    else:
        labels = torch.unique(native)  # ascending: the channel order of the reference
        one_hot = ops.onehot(native, labels)
        if antialias:
            one_hot = _antialias(one_hot, a_in, a_out)
        if order >= 2:
            sampled = spline(one_hot, order, True)
        else:
            sampled = resample(one_hot, mode, None, True)
        out = ops.label_argmax(sampled, labels, float(pad_label), native.dtype)
    return out if out.dtype == data.dtype else out.to(data.dtype)


def _apply_spatial(batch, names, target_space, geometry, *, affine_first, image_interpolation,
                   label_interpolation, antialias, default_pad_value, default_pad_label,
                   one_hot_label_interpolation="linear", max_displacements=None,
                   transform: str = "Spatial") -> None:
    if not names:
        return
    mats, cps, per_instance = geometry
    first = batch.images[names[0]]
    in_shape, a_in = _shape_of(first), first.affines[0]
    out_shape, a_out = (in_shape, a_in) if target_space is None else target_space
    b = first.batch_size
    packed = tables.spatial_tables(
        mats if per_instance else mats[0], cps if per_instance else cps[0], b,
        a_in.numpy(), a_out.numpy(), per_instance=per_instance,
        has_target=target_space is not None,
    )
    info = chunk_info()
    if info is not None and info.b0 == 0:
        # "minimum"/"mean" read batch element 0, which only the first slice of a streamed batch
        # holds: derive the fills now, even if every element of this slice is gated out
        for name in names:
            ib = batch.images[name]
            is_label = issubclass(ib._image_class, LabelMap)
            interp = label_interpolation if is_label else image_interpolation
            if interp == LABEL_INTERPOLATION or _ORDERS[interp] >= 2:  # no fill
                continue
            native = ib.data if ib.data.dtype in ops.DTYPE_CODES else ib.data.float()
            info.cache[("fill", info.step, name)] = _fill_tensor(native, is_label, default_pad_value,
                                                                 default_pad_label)
    if packed is None:  # exact no-op: data and affines untouched (spatial.py:579-590)
        return
    if info is None:  # streamed batches: checked once on the whole batch (Spatial.plan_checks)
        _folding_warning(cps, max_displacements, out_shape, a_out)
    device = first.data.device
    box_hint = _box_hint(packed, a_in.spacing, a_out.spacing, out_shape)
    order, runs = _box_tiers(packed, box_hint, out_shape)
    mat_d, cp_d, flags_d, order_d = ops.upload(device, packed.mat, packed.cp, packed.flags, order)
    tiers = None if order is None else (order_d, runs)
    target_shape = None if target_space is None else out_shape

    def spline(tensor, order, in_place, source=None):
        """B-spline of ``order`` through the call's geometry: coefficients of ``tensor`` (over it
        when ``in_place``), passthrough elements copied from ``source`` (default ``tensor``, whose
        passthrough elements the prefilter leaves as they are)."""
        coeff = ops.bspline_prefilter(tensor, order, flags_d, in_place=in_place)
        return ops.bspline_resample(
            coeff, tensor if source is None else source, mat_d, cp_d, flags_d, a_in.spacing, a_out.spacing,
            affine_first=affine_first, order=order, out_shape=target_shape)

    keep_original = set(packed.passthrough)
    for name in names:
        ib = batch.images[name]
        is_label = issubclass(ib._image_class, LabelMap)
        interp = label_interpolation if is_label else image_interpolation
        data = ib.data
        graph = autograd.records_graph(data)
        if graph:
            if is_label:
                autograd.refuse(transform, f'label map "{name}"')
            if interp == LABEL_INTERPOLATION or _ORDERS[interp] >= 2:
                autograd.refuse(transform, f'interpolation "{interp}"')
            if antialias:
                autograd.refuse(transform, "antialias")
        elif data.requires_grad and ops.differentiable_default():
            data = data.detach()  # grad mode is off: no graph to record, the usual kernels run
        if is_label and interp == LABEL_INTERPOLATION:
            def run(tensor, mode, fill, exact):
                return ops.resample(
                    tensor, mat_d, cp_d, flags_d, a_in.spacing, a_out.spacing, affine_first=affine_first,
                    mode=mode, fill=fill, out_shape=target_shape, box_hint=box_hint, exact_coords=exact)
            ib.data = _resample_label_pv(
                data, run, spline, antialias=antialias, a_in=a_in, a_out=a_out,
                one_hot_interpolation=one_hot_label_interpolation, pad_label=default_pad_label)
            ib.affines[:] = [ib.affines[i] if i in keep_original else a_out.clone() for i in range(b)]
            continue
        native = data if data.dtype in ops.DTYPE_CODES else data.float()
        order = _ORDERS[interp]
        if order >= 2:  # data.float() -> [blur] -> grid_pull -> .to(dtype); no fill (spatial.py:1734-1761)
            smoothed = _antialias(native, a_in, a_out) if antialias and not is_label else native
            out = spline(smoothed, order, False, native)
            out = out if out.dtype == data.dtype else out.to(data.dtype)
            if keep_original and data.dtype not in ops.DTYPE_CODES:  # native rounded them to fp32
                rows = torch.tensor(sorted(keep_original), device=device)
                out[rows] = data[rows]
            ib.data = out
            ib.affines[:] = [ib.affines[i] if i in keep_original else a_out.clone() for i in range(b)]
            continue
        if info is None:  # fill statistics are constants of the graph (the reference takes .item())
            fill = _fill_tensor(native.detach() if graph else native, is_label, default_pad_value,
                                default_pad_label)
        else:  # streamed: derived from batch element 0 when the first slice came through
            fill = info.cache[("fill", info.step, name)]
        if antialias and not is_label:  # after the fill value (spatial.py:1249-1257): blur what is downsampled
            native = _antialias(native, a_in, a_out)
        mode = ops.NEAREST if interp == "nearest" else ops.LINEAR
        tiered = mode == ops.LINEAR and native.dtype == torch.float32 and not ops.exact_coords_default()
        resample = autograd.resample if graph else ops.resample
        out = resample(
            native, mat=mat_d, cp=cp_d, flags=flags_d, spacing_in=a_in.spacing, spacing_out=a_out.spacing,
            affine_first=affine_first, mode=mode, fill=fill, out_shape=target_shape,
            box_hint=box_hint, tiers=tiers if tiered else None,
        )
        ib.data = out if out.dtype == data.dtype else out.to(data.dtype)
        ib.affines[:] = [
            ib.affines[i] if i in keep_original else a_out.clone() for i in range(b)
        ]


def _box_hint(packed, sp_in, sp_out, out_shape) -> int:
    """Edge (20/22/24/28/32) of the input box covering the pre-image of a 16^3 output
    tile for every element: sum_b |M_ab| * 15 voxels + 2 taps, plus the largest
    change an elastic field can make across the tile (adjacent control-point
    deltas x control cells per voxel).  Tiles that still do not fit fall back to
    the general path inside the kernel, so this only steers occupancy."""
    m = np.abs(packed.mat.reshape(-1, 3, 4)[:, :, :3])
    extent = (m.sum(axis=2) * 15.0).max(axis=0) + 2.0  # per input axis
    if packed.cp is not None:
        cp = packed.cp
        spacing = np.minimum(np.asarray(sp_in, dtype=np.float64), np.asarray(sp_out))
        variation = np.zeros(3)
        # adjacent control points differ by at most twice the largest magnitude
        delta = 2.0 * np.abs(cp).reshape(-1, 3).max(axis=0)
        for axis in range(3):
            n_cp, n_out = cp.shape[1 + axis], out_shape[axis]
            if n_cp > 1 and n_out > 1:
                variation += delta * ((n_cp - 1) / (n_out - 1)) * 15.0
        # all three partial derivatives peaking together is the rare case: budget a
        # third of the worst case, outlier tiles take the in-kernel fallback
        extent = extent + variation / spacing / 3.0
    worst = float(np.max(extent))
    for edge in (20, 22, 24, 28):
        if worst <= edge:
            return edge
    return 32


_BOX_EDGES = (20, 22, 24, 28, 32)


def _box_tiers(packed, cap: int, out_shape):
    """Box edge per element for the affine-only fp32 trilinear launches: (elements ordered by
    edge as int32, [(count, edge), ...] ascending), or (None, None) when every element needs the
    launch's own box ``cap`` (or the call has a control grid: elastic launches keep one box).
    A smaller box leaves more shared memory and registers per SM: boxes of 20 and 22 run four
    CTAs per SM, 24 three."""
    if packed.cp is not None:
        return None, None
    edges = _affine_box_edges(packed.mat, cap, out_shape)
    if (edges == cap).all():
        return None, None
    order = np.argsort(edges, kind="stable").astype(np.int32)
    values, counts = np.unique(edges, return_counts=True)
    return order, [(int(n), int(e)) for e, n in zip(values, counts)]


def _affine_box_edges(mat, cap: int, out_shape) -> np.ndarray:
    """Per element of an affine-only launch: the smallest box edge (of `_BOX_EDGES`, at most
    ``cap``, the launch's own box) whose edge x edge x box_k_extent(edge) box holds the pre-image
    of every 16^3 output tile, as `tile_bounds_kernel` measures it; ``cap`` where none does.

    The pre-pass takes, per input axis, q in [qlo, qhi] with qhi - qlo <= 15 * sum_b |M_ab| widened
    by its margin 0.02 + 1e-5 |q| on each side, then lo = floor(qlo), hi = floor(qhi) + 1, so a tile
    needs at most floor(width) + 3 planes, and K three more for rounding lo down to 16 bytes.
    The 1e-3 covers the pre-pass's fp32 rounding.  Since no tile needs more than its element's
    edge, and a tile that does not fit ``cap`` is never moved below it, every tile takes the same
    path (staged box or fallback) as in a launch of ``cap`` for all."""
    m = np.asarray(mat, dtype=np.float64).reshape(-1, 3, 4)
    lin = np.abs(m[:, :, :3])
    span = np.maximum(np.asarray(out_shape, dtype=np.float64) - 1.0, 0.0)
    q_max = np.abs(m[:, :, 3]) + lin @ span  # bound of |q| over the whole output
    width = lin.sum(axis=2) * 15.0 + 2.0 * (0.02 + 1e-5 * q_max) + 1e-3
    with np.errstate(invalid="ignore"):
        need = np.floor(width) + 3.0
        need[:, 2] += 3.0
        need[~np.isfinite(need)] = np.inf
        edges = np.full(len(m), cap, dtype=np.int32)
        for edge in reversed([e for e in _BOX_EDGES if e < cap]):
            fits = (need[:, 0] <= edge) & (need[:, 1] <= edge) & (need[:, 2] <= (edge + 7) // 4 * 4)
            edges[fits] = edge
    return edges


class Resample(Spatial):
    """Resampling-only wrapper: ``Resample(2)`` = 2 mm isotropic, ``Resample("t1")`` = the space of
    that image, ``Resample((1, 1, 3))`` (spatial.py:759-803)."""

    def __init__(self, target=1, image_interpolation="linear", label_interpolation="nearest",
                 one_hot_label_interpolation="linear", antialias: bool = False, **kwargs: Any) -> None:
        super().__init__(target=target, image_interpolation=image_interpolation,
                         label_interpolation=label_interpolation,
                         one_hot_label_interpolation=one_hot_label_interpolation, antialias=antialias, **kwargs)


class Affine(Spatial):
    """Affine-only wrapper (spatial.py:806-869)."""

    def __init__(self, *, scales=1.0, degrees=0.0, translation=0.0, isotropic: bool = False,
                 center: str = "image", default_pad_value="minimum", default_pad_label=0,
                 image_interpolation="linear", label_interpolation="nearest",
                 one_hot_label_interpolation="linear", **kwargs: Any) -> None:
        super().__init__(
            scales=scales, degrees=degrees, translation=translation, isotropic=isotropic,
            center=center, default_pad_value=default_pad_value,
            default_pad_label=default_pad_label, image_interpolation=image_interpolation,
            label_interpolation=label_interpolation,
            one_hot_label_interpolation=one_hot_label_interpolation, **kwargs,
        )
        self._warn_if_noop(
            is_noop=self.scales.is_constant(1.0) and self.degrees.is_constant(0.0)
            and self.translation.is_constant(0.0),
            hint="degrees=(-15, 15)",
        )


class ElasticDeformation(Spatial):
    """Elastic-only wrapper (spatial.py:872-922)."""

    def __init__(self, *, control_points=None, num_control_points=7, max_displacement=7.5,
                 locked_borders: int = 2, image_interpolation="linear",
                 label_interpolation="nearest", one_hot_label_interpolation="linear",
                 **kwargs: Any) -> None:
        super().__init__(
            control_points=control_points, num_control_points=num_control_points,
            max_displacement=max_displacement, locked_borders=locked_borders,
            image_interpolation=image_interpolation, label_interpolation=label_interpolation,
            one_hot_label_interpolation=one_hot_label_interpolation, **kwargs,
        )
