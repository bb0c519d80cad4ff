"""Host-side parameter tables: reference ``params`` dicts -> kernel inputs.

Everything here is tiny float64/fp32 host math (no voxels).  It follows the
reference's own host code so the device kernels start from bit-identical
numbers (TorchIO 2.0.0a2, paths relative to src/torchio/transforms/):
  output->input matrix   spatial/spatial.py:1582-1601
  Gaussian taps          intensity/blur.py:179-183 (shared), :292-328 (per element)
  coarse bias fields     intensity/bias_field.py:258-293, 316-329
  gamma = exp(log_gamma) intensity/gamma.py:103-120
"""

from __future__ import annotations

import functools
import math
from dataclasses import dataclass

import numpy as np
import torch

FLAG_PASSTHROUGH, FLAG_ELASTIC = 1, 2


# ---- spatial ---------------------------------------------------------------


def voxel_matrix(a_in: np.ndarray, a_out: np.ndarray, world) -> np.ndarray:
    """fp32 rows 0..2 of inv(A_in) @ inv(T) @ A_out (12 floats)."""
    inv_t = np.eye(4) if world is None else np.linalg.inv(np.asarray(world, dtype=np.float64))
    m = np.linalg.inv(a_in) @ inv_t @ a_out
    return m.astype(np.float32)[:3].reshape(12)


@dataclass
class SpatialTables:
    mat: np.ndarray            # (B, 12) fp32
    cp: np.ndarray | None      # (B, ni, nj, nk, 3) fp32
    flags: np.ndarray          # (B,) uint8
    passthrough: list[int]


def spatial_tables(affine_matrices, control_points, batch_size: int, a_in: np.ndarray,
                   a_out: np.ndarray, *, per_instance: bool, has_target: bool):
    """Pack per-element geometry.  ``affine_matrices``/``control_points`` are
    lists (per element) when ``per_instance`` else single values; entries may
    be None (identity).  Returns None for a complete no-op."""
    if not per_instance:
        affine_matrices = [affine_matrices] * batch_size
        control_points = [control_points] * batch_size
    if len(affine_matrices) != batch_size:
        raise RuntimeError(
            "Per-instance spatial parameters were recorded for"
            f" {len(affine_matrices)} elements but the batch has {batch_size}"
        )
    no_geometry = all(m is None for m in affine_matrices) and all(
        c is None for c in control_points
    )
    if no_geometry and not has_target:
        return None
    mat = np.empty((batch_size, 12), dtype=np.float32)
    flags = np.zeros(batch_size, dtype=np.uint8)
    rows = [b for b, w in enumerate(affine_matrices) if w is not None]
    if len(rows) < batch_size:
        identity = voxel_matrix(a_in, a_out, None)
        for b, w in enumerate(affine_matrices):
            if w is None:
                mat[b] = identity
    if rows:
        # stacked inv/matmul == per-element calls bit for bit (same LAPACK/BLAS kernels)
        worlds = np.stack([np.asarray(affine_matrices[b], dtype=np.float64) for b in rows])
        m = np.linalg.inv(a_in) @ np.linalg.inv(worlds) @ a_out
        mat[rows] = m.astype(np.float32)[:, :3].reshape(len(rows), 12)
    cp = None
    grids = [None if c is None else np.asarray(c, dtype=np.float32) for c in control_points]
    shapes = {g.shape for g in grids if g is not None}
    if shapes:
        if len(shapes) != 1:
            raise RuntimeError("control-point grids of one batch must share a shape")
        cp = np.zeros((batch_size, *shapes.pop()), dtype=np.float32)
        for b, g in enumerate(grids):
            if g is not None:
                cp[b] = g
                flags[b] |= FLAG_ELASTIC
    passthrough = []
    if per_instance and not has_target:
        for b in range(batch_size):
            if affine_matrices[b] is None and control_points[b] is None:
                flags[b] |= FLAG_PASSTHROUGH
                passthrough.append(b)
    return SpatialTables(mat, cp, flags, passthrough)


# ---- bias field --------------------------------------------------------------


def coarse_shape(spatial_shape, scale: float) -> list[int]:
    return [max(round(s * scale), 4) for s in spatial_shape]


def coarse_bias_fields(shape, std, seed, scale: float) -> torch.Tensor:
    """Host torch.normal draws from the recorded CPU-generator seeds."""
    b, c = int(shape[0]), int(shape[1])
    small = coarse_shape(shape[2:], scale)
    if isinstance(std, list):
        out = torch.empty((b, c, *small), dtype=torch.float32)
        for row, (s, sd) in enumerate(zip(std, seed, strict=True)):
            g = torch.Generator(device="cpu")
            g.manual_seed(int(sd))
            out[row] = torch.normal(mean=0.0, std=float(s), size=(1, c, *small), generator=g)[0]
        return out
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    return torch.normal(mean=0.0, std=float(std), size=(b, c, *small), generator=g)


# ---- blur ---------------------------------------------------------------------


@dataclass
class BlurTables:
    taps: torch.Tensor       # (3, B, 2R+1) fp32
    radius: torch.Tensor     # (3, B) int32
    big_r: int
    axes_mask: int
    identity: torch.Tensor   # (B,) uint8


def _taps_shared(sigma: float) -> torch.Tensor:
    radius = max(int(np.ceil(3 * sigma)), 1)
    x = torch.arange(2 * radius + 1, dtype=torch.float32) - radius
    k = torch.exp(-0.5 * (x / sigma) ** 2)
    return k / k.sum()


def _taps_stacked(sigmas: np.ndarray) -> tuple[torch.Tensor, np.ndarray]:
    radii = np.zeros(len(sigmas), dtype=np.int64)
    pos = sigmas > 0
    radii[pos] = np.maximum(np.ceil(3 * sigmas[pos]).astype(np.int64), 1)
    rmax = int(radii.max())
    offs = (torch.arange(2 * rmax + 1, dtype=torch.float32) - rmax)[None]
    sig = torch.as_tensor(sigmas, dtype=torch.float32)[:, None]
    safe = torch.where(sig > 0, sig, torch.ones_like(sig))
    k = torch.exp(-0.5 * (offs / safe) ** 2)
    k = torch.where(offs.abs() <= torch.as_tensor(radii)[:, None], k, torch.zeros_like(k))
    delta = torch.zeros_like(k)
    delta[:, rmax] = 1.0
    k = torch.where(sig > 0, k, delta)
    return k / k.sum(dim=1, keepdim=True), radii


def blur_tables(sigmas_vox, batch_size: int) -> BlurTables | None:
    """Dispatch of _gaussian_smooth (blur.py:143-154): None = return input
    unchanged; 1-D or all-equal rows = shared taps; else per-element taps."""
    sig = np.asarray(sigmas_vox, dtype=np.float64)
    if np.all(sig <= 0):
        return None
    if sig.ndim == 2 and np.all(sig == sig[0]):
        sig = sig[0]
    rows: list[torch.Tensor | None] = []
    radius = torch.zeros((3, batch_size), dtype=torch.int32)
    if sig.ndim == 1:
        for axis in range(3):
            s = float(sig[axis])
            if s <= 0:
                rows.append(None)
                continue
            t = _taps_shared(s)
            radius[axis, :] = (t.numel() - 1) // 2
            rows.append(t[None].expand(batch_size, -1))
        identity = torch.zeros(batch_size, dtype=torch.uint8)
    else:
        if sig.shape[0] != batch_size:
            raise RuntimeError(
                f"Per-instance blur sigmas were recorded for {sig.shape[0]} elements"
                f" but the batch has {batch_size}"
            )
        for axis in range(3):
            col = sig[:, axis]
            if np.all(col <= 0):
                rows.append(None)
                continue
            t, radii = _taps_stacked(col)
            radius[axis] = torch.as_tensor(radii, dtype=torch.int32)
            rows.append(t)
        identity = torch.as_tensor(np.all(sig <= 0, axis=1)).to(torch.uint8)
    big_r = max((t.shape[1] - 1) // 2 for t in rows if t is not None)
    taps = torch.zeros((3, batch_size, 2 * big_r + 1), dtype=torch.float32)
    mask = 0
    for axis, t in enumerate(rows):
        if t is None:
            continue
        r = (t.shape[1] - 1) // 2
        taps[axis, :, big_r - r: big_r + r + 1] = t
        mask |= 1 << axis
    return BlurTables(taps, radius, big_r, mask, identity)


# ---- noise / gamma ---------------------------------------------------------


def per_element_vector(value, batch_size: int) -> np.ndarray:
    if isinstance(value, list):
        if len(value) != batch_size:
            raise RuntimeError(
                f"Per-instance parameters were recorded for {len(value)} elements"
                f" but the batch has {batch_size}"
            )
        return np.asarray(value, dtype=np.float32)
    return np.full(batch_size, value, dtype=np.float32)


def gamma_values(log_gamma, batch_size: int) -> np.ndarray:
    """exp(log_gamma): fp32 torch.exp per element, float64 math.exp when shared
    (gamma.py:117-120)."""
    if isinstance(log_gamma, list):
        if len(log_gamma) != batch_size:
            raise RuntimeError(
                f"Per-instance parameters were recorded for {len(log_gamma)} elements"
                f" but the batch has {batch_size}"
            )
        return torch.exp(torch.tensor(log_gamma, dtype=torch.float32)).numpy()
    return np.full(batch_size, math.exp(log_gamma), dtype=np.float32)


# ---- labels to image -----------------------------------------------------------

#: Largest draw ATen's CUDA normal kernel runs as a single launch: TensorIterator's
#: can_use_32bit_indexing needs the last fp32 byte offset to fit in int32, i.e. numel <= 2**29.
#: Larger draws are split into sub-launches, each with an offset of its own.
RANDN_MAX_NUMEL = 1 << 29


def check_randn_numel(numel: int) -> None:
    if numel > RANDN_MAX_NUMEL:
        raise NotImplementedError(
            f"a draw of {numel} values exceeds 2**29; ATen splits it into 32-bit-indexed"
            " sub-launches, whose stream is not reproduced")


def randn_cuda_layout(numel: int, sm_count: int, max_threads_per_sm: int) -> tuple[int, int]:
    """(grid_x, counter_offset) of ATen's launch of ``normal_`` on ``numel`` fp32 CUDA values
    (calc_execution_policy, ATen/native/cuda/DistributionTemplates.h: 256-thread blocks, 4 values
    per curand_normal4).  ``counter_offset`` is how far the draw advances the generator's offset."""
    if numel < 1:
        raise ValueError(f"randn_cuda_layout: numel must be positive, got {numel}")
    check_randn_numel(numel)
    block = 256
    grid_x = min(sm_count * (max_threads_per_sm // block), (numel + block - 1) // block)
    counter_offset = ((numel - 1) // (block * grid_x * 4) + 1) * 4
    return grid_x, counter_offset


def label_synthesis_tables(means, stds, batch_size: int):
    """LabelsToImage params -> (label values (n,) int64 ascending, draw index (n,) int64 with -1 for
    a label that is not drawn, mean (B, n) fp32, std (B, n) fp32).

    Draw order is the reference's: the ``means`` dict's order for shared params
    (labels_to_image.py:282-285), the sorted union of the per-element dicts otherwise (:201-213).
    A label draws nothing when its mean and std are all zero (:212, :284).  Keys may be ints or,
    for params read back from JSON, their strings."""
    per_element = isinstance(means, list)
    if per_element:
        if len(means) != batch_size or len(stds) != batch_size:
            raise RuntimeError(f"Per-instance parameters were recorded for {len(means)} elements"
                               f" but the batch has {batch_size}")
        m_rows = [{int(k): float(v) for k, v in m.items()} for m in means]
        s_rows = [{int(k): float(v) for k, v in s.items()} for s in stds]
        order = sorted(set().union(*(m.keys() for m in m_rows)))
    else:
        m_rows = [{int(k): float(v) for k, v in means.items()}] * batch_size
        s_rows = [{int(k): float(v) for k, v in stds.items()}] * batch_size
        order = list(m_rows[0])
    values = np.asarray(sorted(order), dtype=np.int64)
    column = {int(v): i for i, v in enumerate(values)}
    mean = np.zeros((batch_size, len(values)), dtype=np.float32)
    std = np.zeros_like(mean)
    for b in range(batch_size):
        for label in order:
            mean[b, column[label]] = m_rows[b].get(label, 0.0)
            std[b, column[label]] = s_rows[b].get(label, 0.0)
    draw = np.full(len(values), -1, dtype=np.int64)
    drawn = 0
    for label in order:
        c = column[label]
        if per_element:  # count_nonzero of the fp32 (B,) tensors
            active = np.any(mean[:, c] != 0) or np.any(std[:, c] != 0)
        else:  # python floats
            active = m_rows[0][label] != 0.0 or s_rows[0].get(label, 0.0) != 0.0
        if active:
            draw[c] = drawn
            drawn += 1
    return values, draw, mean, std


# ---- label-map lookup tables (label/remap_labels.py:50-58, sequential_labels.py:53-61) ----------

_NUMPY_DTYPES = {torch.float32: np.float32, torch.uint8: np.uint8, torch.int8: np.int8,
                 torch.int16: np.int16, torch.int32: np.int32, torch.int64: np.int64}


def label_lut(pairs, dtype: torch.dtype, device) -> tuple[np.ndarray, np.ndarray]:
    """(keys, values) of what ``for old, new in pairs: data[src == old] = new`` does to a map of
    ``dtype``, every mask taken on the unmodified ``src``.  keys: ascending stored values that
    match some ``old`` (int64, or fp32 for fp32 maps); values: the stored ``new`` (numpy ``dtype``).

    The comparison and assignment rules of a Python scalar against a tensor depend on the dtype
    (u8 == 257 matches 1, fp32 == 2**24 + 1 matches 2**24, u8[mask] = -1 stores 255, i16[mask] =
    70000 raises), so torch decides each one, on a one-element tensor of ``dtype`` on ``device``:
    the candidate for ``old`` is ``old`` converted to ``dtype`` and is kept when it compares equal
    to ``old``; the stored value is what ``t[mask] = new`` leaves (or raises).  A later pair whose
    candidate equals an earlier one's overrides it, as its index_put runs later."""
    pairs = [(old, new) for old, new in pairs]
    return _label_lut(tuple((type(o), o, type(n), n) for o, n in pairs), dtype, torch.device(device))


@functools.lru_cache(maxsize=256)
def _label_lut(items, dtype, device):
    mask = torch.ones(1, dtype=torch.bool, device=device)
    candidates, matches, stored = [], [], []
    for _, old, _, new in items:
        source = torch.tensor([old], dtype=torch.float64 if isinstance(old, float) else torch.int64)
        candidate = source.to(device).to(dtype)
        candidates.append(candidate)
        matches.append(candidate == old)
        t = torch.zeros(1, dtype=dtype, device=device)
        t[mask] = new
        stored.append(t)
    if not items:
        key_dtype = np.float32 if dtype == torch.float32 else np.int64
        return np.zeros(0, dtype=key_dtype), np.zeros(0, dtype=_NUMPY_DTYPES[dtype])
    candidates = torch.cat(candidates).tolist()
    matches = torch.cat(matches).tolist()
    stored = torch.cat(stored).cpu().numpy()
    table = {}
    for candidate, match, value in zip(candidates, matches, stored):
        if match:
            table[candidate + 0.0 if dtype == torch.float32 else candidate] = value  # -0.0 -> +0.0
    keys = sorted(table)
    key_dtype = np.float32 if dtype == torch.float32 else np.int64
    return (np.asarray(keys, dtype=key_dtype),
            np.asarray([table[k] for k in keys], dtype=_NUMPY_DTYPES[dtype]).reshape(len(keys)))


# ---- Resize / Anisotropy index tables (spatial/resize.py, spatial/anisotropy.py) ---------------
#
# ATen's CUDA upsample (ATen/native/cuda/UpSample.cuh, restated in fp32 with numpy's
# round-to-nearest scalar ops):
#   linear, align_corners=True: scale = float(in - 1) / float(out - 1) (0 when out == 1),
#     pos = scale * float(o), i0 = int(pos), i1 = i0 + (i0 < in - 1), l1 = pos - float(i0), l0 = 1 - l1
#   nearest: scale = float(in) / float(out), i = min(floorf(float(o) * scale), in - 1)


@functools.lru_cache(maxsize=1024)
def aten_linear_axis(n_in: int, n_out: int) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
    """(i0, i1, l0, l1) of ATen's align_corners=True linear upsample of one axis, n_in -> n_out."""
    scale = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0.0)
    pos = np.arange(n_out, dtype=np.float32) * scale
    i0 = pos.astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)
    l1 = pos - i0.astype(np.float32)
    l0 = np.float32(1.0) - l1
    return i0, i1, l0, l1


@functools.lru_cache(maxsize=1024)
def aten_nearest_axis(n_in: int, n_out: int) -> np.ndarray:
    """Source index of each output index of ATen's nearest resize of one axis, n_in -> n_out."""
    scale = np.float32(n_in) / np.float32(n_out)
    pos = np.arange(n_out, dtype=np.float32) * scale
    return np.minimum(np.floor(pos).astype(np.int64), n_in - 1)


def _pack_axes(axes) -> tuple[np.ndarray, np.ndarray | None]:
    """[(i0, i1, l0, l1) or i0 per axis] -> the (idx, lam) tables of tio_interpolate."""
    if all(isinstance(a, np.ndarray) for a in axes):
        idx = np.concatenate([np.concatenate([a, a]) for a in axes]).astype(np.int32)
        return idx, None
    idx = np.concatenate([np.concatenate([a[0], a[1]]) for a in axes]).astype(np.int32)
    lam = np.concatenate([np.concatenate([a[2], a[3]]) for a in axes]).astype(np.float32)
    return idx, lam


# One axis of a tio_interpolate pass is named by (n_in, n_out, linear, down): ATen's resize of
# n_in -> n_out, or with ``down`` > 0 Anisotropy's degraded axis (n_in = n_out = L, nearest down to
# ``down``, back up with the composed up table).  The forward and adjoint tables of each axis are
# cached per name.

def _resize_axes(in_shape, out_shape, linear: bool) -> list[tuple[int, int, bool, int]]:
    in_shape, out_shape = tuple(int(s) for s in in_shape), tuple(int(s) for s in out_shape)
    linear = linear and in_shape != out_shape  # ATen's trilinear copies: identity nearest tables
    return [(i, o, linear, 0) for i, o in zip(in_shape, out_shape)]


def _anisotropy_shared_axes(shape, axis: int, factor: float, linear: bool) -> list[tuple[int, int, bool, int]]:
    shape = [int(s) for s in shape]
    length = shape[axis]
    down = max(1, round(length / factor))
    linear = linear and down != length  # D == L: ATen's trilinear pass is a copy
    axes = [(n, n, linear, 0) for n in shape]
    axes[range(3)[axis]] = (length, length, linear, down)
    return axes


@functools.lru_cache(maxsize=1024)
def _forward_axis(n_in: int, n_out: int, linear: bool, down: int):
    """(i0, i1, l0, l1) (linear) or i0 (nearest) of one named axis."""
    if not down:
        return aten_linear_axis(n_in, n_out) if linear else aten_nearest_axis(n_in, n_out)
    down_map = aten_nearest_axis(n_in, down)
    if linear:
        i0, i1, l0, l1 = aten_linear_axis(down, n_out)
        return down_map[i0], down_map[i1], l0, l1
    return down_map[aten_nearest_axis(down, n_out)]


def resize_tables(in_shape, out_shape, linear: bool) -> tuple[np.ndarray, np.ndarray | None]:
    """(idx, lam) of ``F.interpolate(size=out_shape, mode="trilinear", align_corners=True)``
    (``linear``) or ``mode="nearest"`` on CUDA; lam is None for a nearest pass.  ATen's trilinear
    copies when the shapes are equal, which the identity nearest tables reproduce."""
    return _pack_axes([_forward_axis(*a) for a in _resize_axes(in_shape, out_shape, linear)])


def anisotropy_shared_tables(shape, axis: int, factor: float, linear: bool):
    """(idx, lam) of _simulate_anisotropy (anisotropy.py:353-392) as ONE tio_interpolate pass:
    nearest down to D = max(1, round(L / factor)) along ``axis``, then trilinear
    (align_corners=True) or nearest back to L.  The up table's source indices along ``axis`` are
    composed with the down map; the other axes keep their size in both passes, so their up tables
    are ATen's L -> L ones (trilinear: weight 1 on the voxel, 0 on its neighbour, both read).
    D == L makes the trilinear pass a copy in ATen."""
    return _pack_axes([_forward_axis(*a) for a in _anisotropy_shared_axes(shape, axis, factor, linear)])


# ---- adjoint tables: the forward taps inverted per input index (tio_*_backward) ----------------


def invert_taps(src: np.ndarray, out: np.ndarray, n_in: int) -> tuple[np.ndarray, np.ndarray]:
    """CSR inverse of a list of taps: tap t reads input ``src[t]`` for output ``out[t]``.  Returns
    (ptr [n_in + 1], order) with ``order`` the tap numbers sorted stably by (input, output): the
    taps of input x are order[ptr[x]:ptr[x + 1]], in ascending output, and two taps of one output
    on one input (the pair that collapses onto the last plane) in the order they are listed.  No
    monotonicity of ``src`` is assumed.  Every tap is kept, zero weights included."""
    src = np.asarray(src, dtype=np.int64)
    order = np.lexsort((np.asarray(out, dtype=np.int64), src))
    ptr = np.zeros(n_in + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n_in), out=ptr[1:])
    return ptr, order


@functools.lru_cache(maxsize=1024)
def _adjoint_axis(n_in: int, n_out: int, linear: bool, down: int):
    """(ptr [n_in + 1], output index, weight) of one named axis: the taps of input x, lower taps
    listed before upper ones, are entries ptr[x]:ptr[x + 1]."""
    taps = _forward_axis(n_in, n_out, linear, down)
    o = np.arange(n_out, dtype=np.int64)
    if linear:
        src, out, w = np.concatenate(taps[:2]), np.concatenate([o, o]), np.concatenate(taps[2:])
    else:
        src, out, w = taps, o, np.ones(n_out, dtype=np.float32)
    ptr, order = invert_taps(src, out, n_in)
    return ptr, out[order], w[order].astype(np.float32)


def _pack_adjoint(axes) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """[(ptr, out, w) per axis] -> the (ptr, ent, wt) tables of tio_interpolate_backward: one entry
    list for the three axes, each axis's row starts offset into it."""
    ptrs, base = [], 0
    for ptr, out, _ in axes:
        ptrs.append(ptr + base)
        base += len(out)
    return (np.concatenate(ptrs).astype(np.int32), np.concatenate([a[1] for a in axes]).astype(np.int32),
            np.concatenate([a[2] for a in axes]).astype(np.float32))


def resize_adjoint_tables(in_shape, out_shape, linear: bool) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(ptr, ent, wt) of the transpose of the `resize_tables` pass (tio_interpolate_backward)."""
    return _pack_adjoint([_adjoint_axis(*a) for a in _resize_axes(in_shape, out_shape, linear)])


def anisotropy_shared_adjoint_tables(shape, axis: int, factor: float, linear: bool):
    """(ptr, ent, wt) of the transpose of the `anisotropy_shared_tables` pass."""
    return _pack_adjoint([_adjoint_axis(*a) for a in _anisotropy_shared_axes(shape, axis, factor, linear)])


@functools.lru_cache(maxsize=1024)
def _instance_axis(length: int, down: int, linear: bool):
    """(lo, hi, w) source indices along the axis of one element (anisotropy.py:238-331), as the
    reference computes them on a CUDA batch."""
    def source(lowres):  # _downsample_source_indices: floor(m * L / D) in int64, clamped
        return np.minimum(lowres * length // down, length - 1)

    if not linear:  # _nearest_source_indices
        lo = source(np.arange(length, dtype=np.int64) * down // length)
        return lo, lo, np.zeros(length, dtype=np.float32)
    if length == 1:
        pos = np.zeros(1, dtype=np.float32)
    else:
        # `(D - 1.0) / (length - 1)` on a CUDA tensor: ATen divides by a Python scalar as a multiply
        # by its fp32 reciprocal (div_true_kernel_cuda), which the CPU's true division does not
        scale = (np.float32(down) - np.float32(1.0)) * (np.float32(1.0) / np.float32(length - 1))
        pos = np.arange(length, dtype=np.float32) * scale
    lower = np.floor(pos).astype(np.int64)
    upper = np.minimum(lower + 1, down - 1)
    return source(lower), source(upper), pos - lower.astype(np.float32)


def anisotropy_down_size(length: int, factor: float) -> int:
    """``torch.round(length / factors)`` of _downsample_sizes (anisotropy.py:219-235), at least 1.
    ``int / Tensor`` is ``Tensor.__rtruediv__``, which torch runs as ``reciprocal() * int`` in
    float64, not as a true division: the two round to different sizes near .5 (L = 33, factor 4.4:
    8 here, 7 by true division).  Half to even, as torch.round."""
    return max(1, int(np.round(np.float64(length) * (np.float64(1.0) / np.float64(factor)))))


def anisotropy_instance_tables(shape, axes, factors, linear: bool):
    """(axis [B] int32, lo, hi [B, L] int32, w [B, L] fp32) of
    _simulate_anisotropy_per_instance for tio_axis_resample, L = max(shape); an element with
    factor <= 1 gets axis -1 (copied).  The caller has checked the active axes are 0, 1 or 2."""
    shape = [int(s) for s in shape]
    width = max(shape)
    n = len(axes)
    axis = np.full(n, -1, dtype=np.int32)
    lo = np.zeros((n, width), dtype=np.int32)
    hi = np.zeros((n, width), dtype=np.int32)
    w = np.zeros((n, width), dtype=np.float32)
    for b, (a, f) in enumerate(zip(axes, factors)):
        if not f > 1.0:
            continue
        length = shape[a]
        rows = _instance_axis(length, anisotropy_down_size(length, f), linear)
        axis[b] = a
        lo[b, :length], hi[b, :length], w[b, :length] = rows
    return axis, lo, hi, w


@functools.lru_cache(maxsize=1024)
def _instance_adjoint_axis(length: int, down: int, linear: bool) -> tuple[np.ndarray, np.ndarray]:
    """(ptr [length + 1], entries) of one element's axis: the entries of input plane p are
    2*o (lo[o] = p) and 2*o + 1 (hi[o] = p, linear only), ascending o, lo before hi."""
    lo, hi, _ = _instance_axis(length, down, linear)
    o = np.arange(length, dtype=np.int64)
    if linear:
        src, code = np.concatenate([lo, hi]), np.concatenate([2 * o, 2 * o + 1])
    else:
        src, code = lo, 2 * o
    ptr, order = invert_taps(src, code, length)
    return ptr, code[order]


def anisotropy_instance_adjoint_tables(shape, axes, factors, linear: bool) -> tuple[np.ndarray, np.ndarray]:
    """(ptr [B, L + 1], ent [B, 2L]) int32 of tio_axis_resample_backward for the
    `anisotropy_instance_tables` of the same arguments, L = max(shape).  An element with axis -1
    has empty rows; past the axis's length, rows repeat the last start (empty)."""
    shape = [int(s) for s in shape]
    width = max(shape)
    n = len(axes)
    ptr = np.zeros((n, width + 1), dtype=np.int32)
    ent = np.zeros((n, 2 * width), dtype=np.int32)
    for b, (a, f) in enumerate(zip(axes, factors)):
        if not f > 1.0:
            continue
        length = shape[a]
        p, e = _instance_adjoint_axis(length, anisotropy_down_size(length, f), linear)
        ptr[b, :length + 1], ptr[b, length + 1:] = p, p[-1]
        ent[b, :len(e)] = e
    return ptr, ent
