"""Motion test infrastructure: the fixture cases, their seeded inputs, the reference's op sequence
(transforms/intensity/motion.py:140-561 of TorchIO 2.0.0a2) restated on torch ops, runnable on CPU
and CUDA tensors, and a float64 oracle of the one-axis identity the kernel computes.
``tests/golden/generate_motion.py`` runs the reference's class on these cases; nothing here is
imported by the product."""

from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from ghosting_cases import random_values
from spike_cases import (BF16, DTYPES, F16, F32, F64, GOLDEN, I8, I16, I32, I64, SHORT, U8,  # noqa: F401
                         as_float64, as_stored, load_fixture)

# Inputs as in ghosting_cases: "t1" (B, C, *shape) of `dtype`, C = 2 unless the case says otherwise,
# kind "nonneg", "signed" or "nonfinite".  With `seg`, an int16 LabelMap "seg" that must stay
# untouched.  With `compose`, the reference's Compose([Motion(**kwargs), Ghosting(**ghosting),
# BiasField(**bias)]).  Cases named "*_error_*" raise: in the constructor, or (segments) in the call.
SMALL = (12, 10, 9)
RANGES = dict(degrees=(-10, 10), translation=(-3, 3))
CASES_LIST = [
    dict(name="motion_b1_default", batch=1, channels=1, shape=(20, 16, 14), dtype=F32, kind="signed", kwargs=dict()),
    dict(name="motion_b3_f32", batch=3, shape=SMALL, dtype=F32, kind="signed", kwargs=dict(RANGES)),
    dict(name="motion_b3_shared_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(RANGES, per_instance=False)),
    dict(name="motion_b3_p05_f32", batch=3, shape=SMALL, dtype=F32, kind="signed", kwargs=dict(RANGES, p=0.5)),
    dict(name="motion_b3_n1_f32", batch=3, shape=SMALL, dtype=F32, kind="signed", kwargs=dict(RANGES, num_transforms=1)),
    dict(name="motion_b3_n4_f32", batch=3, shape=SMALL, dtype=F32, kind="signed", kwargs=dict(RANGES, num_transforms=4)),
    dict(name="motion_b3_rows1_f32", batch=3, shape=(3, 10, 9), dtype=F32, kind="signed", kwargs=dict(RANGES)),
    dict(name="motion_b3_ragged_f32", batch=3, shape=(11, 10, 9), dtype=F32, kind="signed", kwargs=dict(RANGES)),
    dict(name="motion_b1_prime_f32", batch=1, channels=1, shape=(37, 29, 23), dtype=F32, kind="signed",
         kwargs=dict(degrees=(-8, 8), translation=(-4, 4), num_transforms=3)),
    dict(name="motion_b3_j1_f32", batch=3, shape=(12, 1, 10), dtype=F32, kind="signed", kwargs=dict(RANGES)),
    dict(name="motion_b3_k1_f32", batch=3, shape=(12, 10, 1), dtype=F32, kind="signed", kwargs=dict(RANGES)),
    dict(name="motion_b3_axes_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(degrees=(-5, 5, 0, 0, -15, 15), translation=(-2, 2, -1, 1, 0, 3))),
    dict(name="motion_b3_outside_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(degrees=(-20, 20), translation=(6, 12))),
    dict(name="motion_b3_bool_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(RANGES, num_transforms=True)),
    dict(name="motion_b3_seg_f32", batch=3, shape=SMALL, dtype=F32, kind="signed", seg=True, kwargs=dict(RANGES)),
    dict(name="motion_b3_nonfinite_f32", batch=3, shape=SMALL, dtype=F32, kind="nonfinite", kwargs=dict(RANGES)),
    dict(name="motion_compose_f32", batch=3, shape=SMALL, dtype=F32, kind="nonneg", compose=True,
         ghosting=dict(num_ghosts=(2, 6), intensity=(0.5, 1)), bias=dict(std=0.3), kwargs=dict(RANGES)),
    dict(name="motion_error_segments", batch=3, shape=(2, 8, 8), dtype=F32, kind="signed", kwargs=dict(RANGES)),
    dict(name="motion_error_num_transforms", batch=1, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_transforms=0)),
    dict(name="motion_error_float_transforms", batch=1, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_transforms=2.0)),
    *[dict(name=f"motion_b3_{SHORT[d]}", batch=3, shape=(10, 8, 7), dtype=d,
           kind="nonneg" if d == U8 else "signed", kwargs=dict(RANGES))
      for d in DTYPES],
]
CASES = {c["name"]: c for c in CASES_LIST}


def seed(case) -> int:
    return 1400 + sorted(CASES).index(case["name"])


def scalar_image(case) -> torch.Tensor:
    rng = np.random.default_rng(seed(case))
    return random_values(rng, (case["batch"], case.get("channels", 2), *case["shape"]), case["dtype"], case["kind"])


def label_map(case) -> torch.Tensor | None:
    if not case.get("seg"):
        return None
    rng = np.random.default_rng(seed(case) + 1000)
    return torch.as_tensor(rng.integers(0, 4, (case["batch"], 1, *case["shape"])), dtype=torch.int16)


def per_element(params: dict, batch: int) -> list[list[dict]]:
    """Each element's list of rigid transforms from recorded params (shared or per instance); an
    empty list marks a gated-out element."""
    if "_batched_keys" in params:
        return params["transforms"]
    return [params["transforms"]] * batch


# ---- the reference's op sequence on torch tensors -----------------------------------------------

_IDENTITY = {"degrees": (0.0, 0.0, 0.0), "translation": (0.0, 0.0, 0.0)}


def _axis_rotation(angles: torch.Tensor, axis: int) -> torch.Tensor:
    cos, sin = torch.cos(angles), torch.sin(angles)
    m = torch.zeros(angles.shape[0], 3, 3, dtype=angles.dtype, device=angles.device)
    if axis == 0:
        m[:, 0, 0] = 1
        m[:, 1, 1], m[:, 1, 2], m[:, 2, 1], m[:, 2, 2] = cos, -sin, sin, cos
    elif axis == 1:
        m[:, 0, 0], m[:, 0, 2], m[:, 2, 0], m[:, 2, 2] = cos, sin, -sin, cos
        m[:, 1, 1] = 1
    else:
        m[:, 0, 0], m[:, 0, 1], m[:, 1, 0], m[:, 1, 1] = cos, -sin, sin, cos
        m[:, 2, 2] = 1
    return m


def affine_matrices(degrees: torch.Tensor, translation: torch.Tensor, shape) -> torch.Tensor:
    """motion.py:452-561: (B, 3, 4) from (B, 3) degrees and translations of one segment."""
    theta = torch.zeros(degrees.shape[0], 3, 4, dtype=degrees.dtype, device=degrees.device)
    rx, ry, rz = torch.deg2rad(degrees).unbind(dim=-1)
    theta[:, :3, :3] = _axis_rotation(rz, 2) @ _axis_rotation(ry, 1) @ _axis_rotation(rx, 0)
    size = torch.as_tensor(list(shape), dtype=translation.dtype, device=translation.device)
    theta[:, :3, 3] = translation / (size / 2)
    return theta


def segment_tensors(transforms: list[list[dict]], s: int, device=None) -> tuple[torch.Tensor, torch.Tensor]:
    """motion.py:279-309: segment s's fp32 (B, 3) degrees and translations (identity when gated out)."""
    chosen = [t[s] if t else _IDENTITY for t in transforms]
    return (torch.as_tensor(tuple(t["degrees"] for t in chosen), dtype=torch.float32, device=device),
            torch.as_tensor(tuple(t["translation"] for t in chosen), dtype=torch.float32, device=device))


def moved(x: torch.Tensor, theta: torch.Tensor) -> torch.Tensor:
    """motion.py:416-449: every channel of element b resampled with element b's grid."""
    b, c, *shape = x.shape
    grid = F.affine_grid(theta, [b, 1, *shape], align_corners=True)
    out = F.grid_sample(x.reshape(b * c, 1, *shape), grid.repeat_interleave(c, dim=0), mode="bilinear",
                        padding_mode="zeros", align_corners=True)
    return out.reshape(b, c, *shape)


def bounds(s: int, segments: int, first: int) -> tuple[int, int]:
    size = first // segments
    return s * size, first if s == segments - 1 else (s + 1) * size


def reference_ops(data: torch.Tensor, params: dict) -> torch.Tensor:
    """motion.py:140-414 on ``data`` (any device): the per-element path returns ``data`` when no
    element is active and keeps gated-out elements through ``torch.where``."""
    transforms = per_element(params, data.shape[0])
    active = torch.as_tensor([bool(t) for t in transforms], device=data.device)
    if not bool(active.any()):
        return data
    n = max(len(t) for t in transforms)
    result = data.float()
    shape = result.shape[-3:]
    dims = (-3, -2, -1)
    spectrum = torch.fft.fftn(result, dim=dims)
    for s in range(1, n + 1):
        degrees, translation = segment_tensors(transforms, s - 1, data.device)
        moved_spectrum = torch.fft.fftn(moved(result, affine_matrices(degrees, translation, shape)), dim=dims)
        start, end = bounds(s, n + 1, shape[0])
        spectrum[:, :, start:end] = moved_spectrum[:, :, start:end]
    out = torch.fft.ifftn(spectrum, dim=dims).real.to(data.dtype)
    if "_batched_keys" in params:
        out = torch.where(active.view(-1, 1, 1, 1, 1), out, data)
    return out


# ---- float64 oracle of the one-axis identity ----------------------------------------------------

def thetas(transforms: list[list[dict]], shape, device=None) -> list[torch.Tensor]:
    """The reference's fp32 (B, 3, 4) matrices of every segment s = 1..N."""
    n = max(len(t) for t in transforms)
    return [affine_matrices(*segment_tensors(transforms, s, device), shape) for s in range(n)]


def one_axis(x: torch.Tensor, params: dict) -> torch.Tensor:
    """The identity the kernel computes, in float64, for float64 ``x`` (B, C, I, J, K) on any device:
    each line along I becomes ifft_I(sum_s Hs_s fft_I(x_s)), with x_s = grid_sample in float64 on
    the reference's fp32 matrices.  Gated-out elements keep x; a (b, c) with a non-finite voxel
    becomes NaN."""
    transforms = per_element(params, x.shape[0])
    active = [bool(t) for t in transforms]
    out = x.clone()
    if not any(active):
        return out
    first = x.shape[2]
    copies = [torch.nan_to_num(x, nan=0.0, posinf=0.0, neginf=0.0)]
    copies += [moved(copies[0], theta.double()) for theta in thetas(transforms, x.shape[2:], x.device)]
    segments = len(copies)
    total = torch.zeros(x.shape, dtype=torch.complex128, device=x.device)
    for s, xs in enumerate(copies):
        start, end = bounds(s, segments, first)
        p = torch.zeros(first, dtype=torch.float64, device=x.device)
        p[start:end] = 1
        hs = (p + torch.roll(p.flip(0), 1)) / 2  # (P(f) + P(-f mod I)) / 2
        total += hs.view(-1, 1, 1) * torch.fft.fft(xs, dim=2)
    y = torch.fft.ifft(total, dim=2).real
    y[~torch.isfinite(x).flatten(2).all(dim=2)] = float("nan")
    for b, on in enumerate(active):
        if on:
            out[b] = y[b]
    return out


def check_against_oracle(got: np.ndarray, x: np.ndarray, params: dict, dtype: torch.dtype, rel: float = 1e-5) -> None:
    """Assert ``got`` (float64 values of an output of ``dtype``) is `one_axis` within rel * max|x|
    of the (b, c) row plus the output format's rounding (floats), or within 1 where the float64
    value lies inside the dtype's range (integers); NaN positions equal."""
    want = one_axis(torch.from_numpy(x), params).numpy()
    finite_x = np.where(np.isfinite(x), np.abs(x), 0.0)
    tol = rel * finite_x.max(axis=(2, 3, 4), keepdims=True)
    assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN positions differ"
    ok = ~np.isnan(want)
    g, w, t = got[ok], want[ok], np.broadcast_to(tol, want.shape)[ok]
    if dtype.is_floating_point:
        ulp = {F16: 2.0**-10, BF16: 2.0**-7}.get(dtype, 0.0)
        bad = np.abs(g - w) > t + ulp * np.abs(w)
        assert not bad.any(), f"max |diff| {np.abs(g - w).max()}, tolerance {t.min()}"
        return
    info = torch.iinfo(dtype)
    inside = (w > info.min - 1) & (w < info.max + 1)
    assert np.all(np.abs(g[inside] - np.trunc(w[inside])) <= 1), f"max |diff| {np.abs(g - np.trunc(w)).max()}"


def error_bound(x: torch.Tensor, params: dict) -> torch.Tensor:
    """Per-voxel bound on |kernel - one_axis| for fp32 arithmetic (u = 2^-24) on float64 ``x``:
    per line along I and per segment s,
    - Ghosting's FFT bound 16 ceil(log2 I) u ||x_s line||_2 (|Hs_s| <= 1), summed over segments;
    - the fp32 sample coordinates: each of the three is off by at most
      delta_s = 8 u (1 + max row sum |theta_s|) (max(I, J, K) - 1) / 2 voxels, and a trilinear
      sample moves by at most 2 max|x| per voxel along each axis, plus 16 u max|x| for the sample's
      own rounding; over a line in L2: sqrt(I) (6 delta_s + 16 u) max|x| of the (b, c) row.
    The filter does not increase the L2 norm of a line's error, and a voxel's error is at most
    its line's L2 norm."""
    u = 2.0**-24
    transforms = per_element(params, x.shape[0])
    bound = torch.zeros_like(x)
    if not any(bool(t) for t in transforms):
        return bound
    first = x.shape[2]
    xf = torch.nan_to_num(x, nan=0.0, posinf=0.0, neginf=0.0)
    peak = xf.abs().amax(dim=(2, 3, 4), keepdim=True)
    fft_factor = 16 * max(1, math.ceil(math.log2(first))) * u
    bound += fft_factor * torch.linalg.vector_norm(xf, dim=2, keepdim=True)
    longest = max(x.shape[2:]) - 1
    for theta in thetas(transforms, x.shape[2:], x.device):
        xs = moved(xf, theta.double())
        delta = 8 * u * (1 + theta.double().abs().sum(dim=2).amax(dim=1)) * longest / 2  # (B,)
        bound += fft_factor * torch.linalg.vector_norm(xs, dim=2, keepdim=True)
        bound += math.sqrt(first) * (6 * delta.view(-1, 1, 1, 1, 1) + 16 * u) * peak
    return bound
