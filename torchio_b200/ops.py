"""Functional, tensor-level API over the C-ABI kernels.

Each function is the plain-tensor replacement of one reference helper
(cited per function; TorchIO 2.0.0a2, paths relative to
src/torchio/transforms/).  Inputs are CUDA tensors; parameter tables are
uploaded with one pinned staging copy per call (`upload`).  Launches go to the
caller's current CUDA stream on the tensor's device.  No CPU fallback.
"""

from __future__ import annotations

import os
import threading

import numpy as np
import torch
from torch import Tensor

from . import _native, tables

DTYPE_CODES = {
    torch.float32: 0, torch.uint8: 1, torch.int8: 2,
    torch.int16: 3, torch.int32: 4, torch.int64: 5,
}
NEAREST, LINEAR, LABEL_PV = 0, 1, 2
FLAG_PASSTHROUGH, FLAG_ELASTIC = 1, 2

_counter = threading.local()


def launches() -> int:
    """Number of kernels this thread has launched through the library."""
    return getattr(_counter, "n", 0)


def _count(n: int) -> None:
    _counter.n = getattr(_counter, "n", 0) + n


def _stream(t: Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _ptr(t: Tensor | None):
    return None if t is None else t.data_ptr()


def _require_cuda(t: Tensor, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(
            f"torchio_b200.ops.{name}: expected a CUDA tensor (got {t.device});"
            " the kernels have no CPU fallback"
        )
    if t.requires_grad:
        raise NotImplementedError(
            f"torchio_b200.ops.{name}: kernels are forward-only; detach() the input"
        )


class _StagingRing:
    """Fixed ring of pinned staging buffers for the per-call parameter tables.

    Allocating pinned memory per call (``torch.empty(pin_memory=True)``) looked
    free but is not: while the host runs ahead of the GPU the caching host
    allocator cannot recycle blocks whose copies are still queued, so every call
    ends in ``cudaHostAlloc``, which stalls the GPU.  The ring allocates once; a
    slot is reused only after the event
    recorded behind its last copy has completed."""

    SLOTS = 64
    SLOT_BYTES = 1 << 20

    def __init__(self) -> None:
        self.buffers = [torch.empty(self.SLOT_BYTES, dtype=torch.uint8, pin_memory=True)
                        for _ in range(self.SLOTS)]
        self.events: list = [None] * self.SLOTS
        self.index = 0
        self.lock = threading.Lock()

    def take(self):
        with self.lock:
            i = self.index
            self.index = (i + 1) % self.SLOTS
            pending, self.events[i] = self.events[i], None
        if pending is not None:  # the copy queued behind this slot's previous use
            pending.synchronize()
        return i, self.buffers[i]

    def release(self, i: int, device: torch.device) -> None:
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        with self.lock:
            self.events[i] = ev


_ring: _StagingRing | None = None
_init_lock = threading.Lock()


def upload(device: torch.device, *arrays):
    """Pack host arrays into one pinned buffer, copy once, return device views.

    Each array is a numpy array or CPU tensor (or None -> None).  16-byte
    aligned segments so float4/TMA consumers can read them directly.
    """
    global _ring
    specs, offset = [], 0
    for a in arrays:
        if a is None:
            specs.append(None)
            continue
        t = torch.as_tensor(a)
        t = t.contiguous()
        nbytes = t.numel() * t.element_size()
        specs.append((t, offset, nbytes))
        offset += (nbytes + 15) // 16 * 16
    if offset == 0:
        return [None] * len(arrays)
    slot = None
    if torch.cuda.is_available() and offset <= _StagingRing.SLOT_BYTES:
        if _ring is None:
            with _init_lock:
                if _ring is None:
                    _ring = _StagingRing()
        slot, stage = _ring.take()
        stage = stage[:offset]
    else:
        stage = torch.empty(offset, dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    # plain memcpy through numpy views: torch's CPU copy_ fans tensors above 32 KiB out to
    # the intra-op thread pool, and waking a large OpenMP pool on a busy host stalls this
    # call (tools/host_stalls3.py finds such stalls)
    stage_np = stage.numpy()
    for s in specs:
        if s is None:
            continue
        t, off, nbytes = s
        stage_np[off:off + nbytes] = t.reshape(-1).numpy().view(np.uint8)
    if slot is not None:
        # SM copy kernel instead of cudaMemcpyAsync: see tio_upload in include/tio_b200.h
        dev = torch.empty(offset, dtype=torch.uint8, device=device)
        _native.call("tio_upload", stage.data_ptr(), dev.data_ptr(), offset,
                     torch.cuda.current_stream(dev.device).cuda_stream)
        _count(1)
        _ring.release(slot, torch.device(device))
    else:
        dev = stage.to(device, non_blocking=True)
    out = []
    for s in specs:
        if s is None:
            out.append(None)
            continue
        t, off, nbytes = s
        out.append(dev[off:off + nbytes].view(t.dtype).reshape(t.shape))
    return out


EXACT_COORDS = 0x100  # TIO_EXACT_COORDS
_exact_default = os.environ.get("TIO_B200_EXACT_COORDS", "0") not in ("", "0")


def set_exact_coords(enabled: bool) -> bool:
    """Process-wide default of ``resample(exact_coords=None)``; returns the previous value.
    Also settable with ``TIO_B200_EXACT_COORDS=1`` before import."""
    global _exact_default
    previous, _exact_default = _exact_default, bool(enabled)
    return previous


def exact_coords_default() -> bool:
    return _exact_default


def resample(
    src: Tensor, mat: Tensor, cp: Tensor | None, flags: Tensor | None,
    spacing_in, spacing_out, *, affine_first: bool, mode: int,
    fill: Tensor | None, out_shape=None, box_hint: int = 0, exact_coords: bool | None = None,
) -> Tensor:
    """K1.  Replaces _build_sampling_grid + _sample_batch[_per_sample]
    (spatial/spatial.py:1504-1579,1651-1857).

    src (B,C,I,J,K) fp32 or integer label dtype; mat (B,12) fp32 cuda;
    cp (B,ni,nj,nk,3) fp32 cuda or None; flags (B,) uint8 cuda or None;
    fill (C,) fp32 cuda or None (= no mask step).

    exact_coords: keep the reference's fp32 rounding sequence of the sampling coordinates on
    every voxel (TIO_EXACT_COORDS).  Default (None -> ``exact_coords_default()``): fp32
    trilinear voxels whose taps all lie inside the volume use one fma per axis, which differs
    from the reference by its own coordinate noise (<= ~2e-5 voxel); label maps, padding and
    fill decisions are exact either way.
    """
    _require_cuda(src, "resample")
    if src.dtype not in DTYPE_CODES:
        raise TypeError(f"resample: unsupported dtype {src.dtype}")
    src = src.contiguous()
    b, c, i, j, k = src.shape
    oi, oj, ok = (i, j, k) if out_shape is None else out_shape
    dst = torch.empty((b, c, oi, oj, ok), dtype=src.dtype, device=src.device)
    ni = nj = nk = 0
    if cp is not None:
        ni, nj, nk = cp.shape[1:4]
    sp_in = np.asarray(spacing_in, dtype=np.float32)
    sp_out = np.asarray(spacing_out, dtype=np.float32)
    workspace, ws_bytes = None, 0
    tiled = (src.dtype == torch.float32 and mode == LINEAR) or (
        mode in (NEAREST, LABEL_PV) and src.dtype in (torch.uint8, torch.int16, torch.int32))
    if box_hint >= 0 and tiled:
        ws_bytes = _native.lib().tio_resample_workspace_bytes(b, oi, oj, ok)
        workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=src.device)
    with torch.cuda.device(src.device):
        _native.call(
            "tio_resample", _ptr(src), _ptr(dst), DTYPE_CODES[src.dtype],
            b, c, i, j, k, oi, oj, ok, _ptr(mat), _ptr(cp), _ptr(flags), ni, nj, nk,
            sp_in.ctypes.data, sp_out.ctypes.data, int(bool(affine_first)),
            int(mode) | (EXACT_COORDS if (_exact_default if exact_coords is None else exact_coords) else 0),
            _ptr(fill), int(box_hint), _ptr(workspace), ws_bytes, _stream(src),
        )
    _count(2 if workspace is not None else 1)
    return dst


def _label_table(labels: Tensor, dtype: torch.dtype) -> Tensor:
    return labels.to(torch.float32 if dtype == torch.float32 else torch.int64).contiguous()


def onehot(src: Tensor, labels: Tensor) -> Tensor:
    """(B,1,I,J,K) label batch -> (B,n,I,J,K) fp32 one-hot channels, ``labels`` = the distinct
    values in ascending order (spatial/spatial.py:1362-1365)."""
    _require_cuda(src, "onehot")
    if src.dtype not in DTYPE_CODES:
        raise TypeError(f"onehot: unsupported dtype {src.dtype}")
    src = src.contiguous()
    b, n = src.shape[0], int(labels.numel())
    vox = src[0].numel()
    table = _label_table(labels, src.dtype)
    dst = torch.empty((b, n, *src.shape[2:]), dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        _native.call("tio_onehot", _ptr(src), DTYPE_CODES[src.dtype], b, vox, _ptr(table), n, _ptr(dst),
                     _stream(src))
    _count(1)
    return dst


def label_argmax(sampled: Tensor, labels: Tensor, pad_label: float, dtype: torch.dtype) -> Tensor:
    """(B,n,I,J,K) sampled one-hot channels -> (B,1,I,J,K) labels of ``dtype``: first maximum over
    the channels, ``pad_label`` where their sum is not > 0.5 (spatial/spatial.py:1378-1389)."""
    _require_cuda(sampled, "label_argmax")
    if dtype not in DTYPE_CODES:
        raise TypeError(f"label_argmax: unsupported dtype {dtype}")
    sampled = sampled.contiguous()
    b, n = sampled.shape[:2]
    vox = sampled[0, 0].numel()
    table = _label_table(labels, dtype)
    dst = torch.empty((b, 1, *sampled.shape[2:]), dtype=dtype, device=sampled.device)
    with torch.cuda.device(sampled.device):
        _native.call("tio_label_argmax", _ptr(sampled), b, n, vox, _ptr(table), float(pad_label), _ptr(dst),
                     DTYPE_CODES[dtype], _stream(sampled))
    _count(1)
    return dst


def min_sample0(src: Tensor) -> Tensor:
    """Per-channel min of batch element 0, on device, no sync
    (spatial/spatial.py:2054-2060,2094-2095)."""
    _require_cuda(src, "min_sample0")
    src = src.contiguous()
    c = src.shape[1]
    n = src[0, 0].numel()
    fill = torch.empty(c, dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        _native.call("tio_min_sample0", _ptr(src), c, n, _ptr(fill), _stream(src))
    _count(2)
    return fill


def crop_patches(volume: Tensor, corners, size, out: Tensor | None = None) -> Tensor:
    """Gather ``n`` patches of ``size`` at voxel ``corners`` (n,3) from one volume
    (C,I,J,K) into a dense (n,C,*size) block in a single launch
    (data/sampler.py:54-67 + loader.py:15-24).  ``out``: a contiguous (n,C,*size) block to
    write into (e.g. consecutive slots of a patch ring) instead of a fresh tensor."""
    _require_cuda(volume, "crop_patches")
    if volume.ndim != 4:
        raise ValueError(f"crop_patches expects a (C, I, J, K) volume, got {tuple(volume.shape)}")
    volume = volume.contiguous()
    corners = np.ascontiguousarray(np.asarray(corners, dtype=np.int32).reshape(-1, 3))
    n = corners.shape[0]
    c, i, j, k = (int(v) for v in volume.shape)
    pi, pj, pk = (int(v) for v in size)
    if n == 0:
        return volume.new_empty((0, c, pi, pj, pk))
    if corners.min() < 0 or np.any(corners + np.asarray([pi, pj, pk]) > np.asarray([i, j, k])):
        raise ValueError("crop_patches: a patch extends beyond the volume")
    (corners_d,) = upload(volume.device, corners)
    if out is None:
        dst = torch.empty((n, c, pi, pj, pk), dtype=volume.dtype, device=volume.device)
    else:
        dst = out
        if (tuple(dst.shape) != (n, c, pi, pj, pk) or dst.dtype != volume.dtype or dst.device != volume.device
                or not dst.is_contiguous()):
            raise ValueError("crop_patches: `out` must be a contiguous (n, C, *size) block of the volume's dtype/device")
    with torch.cuda.device(volume.device):
        _native.call(
            "tio_crop_patches", _ptr(volume), _ptr(dst), volume.element_size(), c, i, j, k, n,
            _ptr(corners_d), pi, pj, pk, _stream(volume),
        )
    _count(1)
    return dst


PAD_MODES = {"constant": 0, "replicate": 1, "reflect": 2, "circular": 3}


def remap(src: Tensor, out_shape, offsets, *, mode: str = "constant", fill=0, flip: Tensor | None = None,
          out: Tensor | None = None) -> Tensor:
    """Flip / Crop / Pad in one pass: ``out[..., o] = src[..., o - offset]`` per spatial
    axis with F.pad's out-of-range rules, then per-element axis reversal (``flip``: (B,)
    uint8 cuda, bit 0 I, 1 J, 2 K).  flip.py:233-263, crop.py:84-101, _padding.py:73-104."""
    _require_cuda(src, "remap")
    if src.ndim != 5:
        raise ValueError(f"remap expects (B, C, I, J, K), got {tuple(src.shape)}")
    src = src.contiguous()
    b, c, i, j, k = (int(v) for v in src.shape)
    oi, oj, ok = (int(v) for v in out_shape)
    if out is None:
        dst = torch.empty((b, c, oi, oj, ok), dtype=src.dtype, device=src.device)
    else:
        dst = out
        if (tuple(dst.shape) != (b, c, oi, oj, ok) or dst.dtype != src.dtype or dst.device != src.device
                or not dst.is_contiguous()):
            raise ValueError("remap: `out` must be a contiguous (B, C, *out_shape) block of the source's dtype/device")
    fill_host = torch.tensor([fill]).to(src.dtype)  # F.pad casts the value to the tensor's dtype
    with torch.cuda.device(src.device):
        _native.call(
            "tio_remap", _ptr(src), _ptr(dst), src.element_size(), b, c, i, j, k, oi, oj, ok,
            int(offsets[0]), int(offsets[1]), int(offsets[2]), PAD_MODES[mode],
            fill_host.data_ptr(), _ptr(flip), _stream(src),
        )
    _count(1)
    return dst


def blur(src: Tensor, taps: Tensor, radius: Tensor, big_r: int, axes_mask: int,
         identity: Tensor | None) -> Tensor:
    """K3 (intensity/blur.py:129-252)."""
    _require_cuda(src, "blur")
    src = src.contiguous()
    b, c, i, j, k = src.shape
    dst = torch.empty_like(src)
    scratch = torch.empty_like(src) if (axes_mask & 6) else None
    with torch.cuda.device(src.device):
        _native.call(
            "tio_blur", _ptr(src), _ptr(dst), _ptr(scratch), b, c, i, j, k, _ptr(taps),
            _ptr(radius), int(big_r), int(axes_mask), _ptr(identity), _stream(src),
        )
    _count(_fused_launches(axes_mask, False))
    return dst


def _fused_launches(axes_mask: int, has_bias: bool) -> int:
    jk = bool(axes_mask & 6)
    march = (not jk) or bool(axes_mask & 1) or has_bias
    return int(jk) + int(march)


def moments(values: Tensor, mask: Tensor | None = None) -> tuple[float, float, float]:
    """(sum, sum of squares, count) of the selected values of a contiguous fp32 CUDA tensor, fp64
    accumulation on the device, one small D2H read (the reference calls ``.item()`` here too:
    standardize.py:76-77)."""
    _require_cuda(values, "moments")
    values = values.contiguous()
    m8 = None if mask is None else mask.expand_as(values).contiguous().to(torch.uint8)
    out = torch.empty(3, dtype=torch.float64, device=values.device)
    with torch.cuda.device(values.device):
        _native.call("tio_moments", _ptr(values), _ptr(m8), values.numel(), _ptr(out), _stream(values))
    _count(1)
    s, ss, n = out.tolist()
    return s, ss, n


def quantile_neighbours(values: Tensor, qs, mask: Tensor | None = None):
    """For each q in ``qs`` (at most two): the order statistics torch.kthvalue(lower + 1) and
    kthvalue(lower + 2) return, and ``index - lower`` (transforms/_statistics.py:37-45), found by
    an exact radix select on the device.  Returns (values[2m], weights[m], count)."""
    _require_cuda(values, "quantile_neighbours")
    values = values.contiguous()
    m8 = None if mask is None else mask.expand_as(values).contiguous().to(torch.uint8)
    qs = np.ascontiguousarray(np.asarray(qs, dtype=np.float64).reshape(-1))
    m = int(qs.shape[0])
    dev = values.device
    vals = torch.empty(2 * m, dtype=torch.float32, device=dev)
    out = torch.empty(m + 1, dtype=torch.float64, device=dev)
    ws_bytes = _native.lib().tio_quantiles_workspace_bytes()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _native.call("tio_quantiles", _ptr(values), _ptr(m8), values.numel(), qs.ctypes.data, m, _ptr(vals),
                     _ptr(out), out[m:].data_ptr(), _ptr(ws), ws_bytes, _stream(values))
    _count(7)
    host = out.tolist()
    return vals.tolist(), host[:m], int(host[m])


def quantiles_batched(values: Tensor, qs, mask: Tensor | None = None):
    """`quantile_neighbours` for every element of a (B, ...) CUDA tensor of any image dtype (values
    taken as ``.float()`` gives them), with any number of quantiles, left on the device: returns
    (values (B, 2m) fp32, weights (B, m) fp64, count (B,) fp64, has_nan (B,) uint8) without a
    host sync (histogram_standardization.py:100-108,279)."""
    _require_cuda(values, "quantiles_batched")
    if values.dtype not in RESOLUTION_DTYPE_CODES:
        raise TypeError(f"quantiles_batched: unsupported dtype {values.dtype}")
    values = values.contiguous()
    b = values.shape[0]
    per_elem = values[0].numel()
    m8 = None if mask is None else mask.expand_as(values).contiguous().to(torch.uint8)
    qs = np.ascontiguousarray(np.asarray(qs, dtype=np.float64).reshape(-1))
    m = int(qs.shape[0])
    dev = values.device
    vals = torch.empty((b, 2 * m), dtype=torch.float32, device=dev)
    weights = torch.empty((b, m), dtype=torch.float64, device=dev)
    count = torch.empty(b, dtype=torch.float64, device=dev)
    has_nan = torch.empty(b, dtype=torch.uint8, device=dev)
    ws_bytes = _native.lib().tio_quantiles_batched_workspace_bytes(b, m)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _native.call("tio_quantiles_batched", _ptr(values), RESOLUTION_DTYPE_CODES[values.dtype], _ptr(m8), b,
                     per_elem, qs.ctypes.data, m, _ptr(vals), _ptr(weights), _ptr(count), _ptr(has_nan), _ptr(ws),
                     ws_bytes, _stream(values))
    _count(2 + 5 * ((m + 12) // 13))
    return vals, weights, count, has_nan


def histogram_tables(values: Tensor, weights: Tensor, has_nan: Tensor, landmarks: Tensor) -> Tensor:
    """(B, 3 (m - 1)) fp32 device tables {slopes, intercepts, edges} of
    _apply_histogram_standardization (histogram_standardization.py:279-300) from the output of
    `quantiles_batched` and the m fp32 landmarks, built on the device."""
    b, m = weights.shape
    landmarks = landmarks.to(device=values.device, dtype=torch.float32).contiguous()
    tables = torch.empty((b, 3 * (m - 1)), dtype=torch.float32, device=values.device)
    with torch.cuda.device(values.device):
        _native.call("tio_histogram_tables", _ptr(values), _ptr(weights), _ptr(has_nan), _ptr(landmarks), b, m,
                     _ptr(tables), _stream(values))
    _count(1)
    return tables


def histogram_map(data: Tensor, tables: Tensor, m: int) -> None:
    """In place: each element of the contiguous (B, ...) CUDA tensor ``data`` through its
    piecewise-linear map ``slopes[bin] * x + intercepts[bin]``, bin = torch.bucketize(x, edges),
    computed in fp32 and stored in data's dtype (histogram_standardization.py:302-303)."""
    _require_cuda(data, "histogram_map")
    if data.dtype not in RESOLUTION_DTYPE_CODES:
        raise TypeError(f"histogram_map: unsupported dtype {data.dtype}")
    if not data.is_contiguous():
        raise ValueError("histogram_map: data must be contiguous")
    if data.numel() == 0:
        return
    with torch.cuda.device(data.device):
        _native.call("tio_histogram_map", _ptr(data), _ptr(data), RESOLUTION_DTYPE_CODES[data.dtype], data.shape[0],
                     data[0].numel(), _ptr(tables), int(m), _stream(data))
    _count(1)


def rescale(src: Tensor, *, lo: float | None = None, hi: float | None = None, sub=None, div=None, mul=None,
            add=None, keep=None) -> Tensor:
    """``((clamp(src, lo, hi) - sub[b]) / div[b]) * mul[b] + add[b]`` over a (B, ...) fp32 batch, each
    step rounded like the reference's separate elementwise ops; omitted steps are skipped.
    ``sub/div/mul/add``: scalars or length-B sequences; ``keep``: length-B, 0 = copy the row."""
    _require_cuda(src, "rescale")
    src = src.contiguous()
    b = src.shape[0]
    flags = (1 if lo is not None else 0)
    tabs = []
    for bit, table in ((2, sub), (4, div), (8, mul), (16, add)):
        if table is None:
            tabs.append(None)
            continue
        flags |= bit
        arr = np.asarray(table, dtype=np.float32).reshape(-1)
        tabs.append(np.ascontiguousarray(np.broadcast_to(arr, (b,)) if arr.size == 1 else arr))
    keep_np = None if keep is None else np.ascontiguousarray(np.asarray(keep, dtype=np.uint8))
    sub_d, div_d, mul_d, add_d, keep_d = upload(src.device, *tabs, keep_np)
    dst = torch.empty_like(src)
    with torch.cuda.device(src.device):
        _native.call("tio_rescale", _ptr(src), _ptr(dst), b, src[0].numel(),
                     float(lo if lo is not None else 0.0), float(hi if hi is not None else 0.0),
                     _ptr(sub_d), _ptr(div_d), _ptr(mul_d), _ptr(add_d), _ptr(keep_d), flags, _stream(src))
    _count(2)
    return dst


def intensity_fused(
    src: Tensor, *, coarse: Tensor | None = None, bias_identity: Tensor | None = None,
    bias_divide: bool = False, taps: Tensor | None = None, radius: Tensor | None = None,
    big_r: int = 0, axes_mask: int = 0, mean: Tensor | None = None, std: Tensor | None = None,
    keep: Tensor | None = None, z: Tensor | None = None, z2: Tensor | None = None,
    philox_seed: int = 0, noise_mode: int = 0, rician: bool = False,
    gamma: Tensor | None = None,
) -> Tensor:
    """Fused bias -> blur -> noise -> gamma (two HBM passes); any stage optional.

    Compose-level fusion of consecutive intensity transforms; a single transform
    is a call with only its own stage set.
    """
    _require_cuda(src, "intensity_fused")
    src = src.contiguous()
    b, c, i, j, k = src.shape
    dst = torch.empty_like(src)
    jk = taps is not None and (axes_mask & 6)
    scratch = torch.empty_like(src) if jk else None
    si = sj = sk = 0
    if coarse is not None:
        si, sj, sk = coarse.shape[2:]
    with torch.cuda.device(src.device):
        _native.call(
            "tio_intensity_fused", _ptr(src), _ptr(dst), _ptr(scratch), b, c, i, j, k,
            _ptr(coarse), si, sj, sk, _ptr(bias_identity), int(bool(bias_divide)),
            _ptr(taps), _ptr(radius), int(big_r), int(axes_mask),
            _ptr(mean), _ptr(std), _ptr(keep), _ptr(z), _ptr(z2),
            int(philox_seed) & (2**64 - 1), int(noise_mode), int(bool(rician)),
            _ptr(gamma), _stream(src),
        )
    _count(_fused_launches(axes_mask if taps is not None else 0, coarse is not None))
    return dst


# ---- exact replay of torch's CPU randn stream (K4a) ---------------------------

_MT_TABLE_FILE = _native.LIB_PATH.parent / "mt19937_jump.bin"
_mt_host_table: Tensor | None = None
_mt_device_tables: dict = {}
_mt_lock = threading.Lock()
MT_MAX_WORDS = 1 << 31  # stream positions the two-level jump table reaches
# uint32 header of the table the library builds (csrc/mt19937_layout.h): magic "MTJ1",
# log2(segment length), S2, S1, polynomials, stride.  Tables for another segment length
# have the same size, so a cached file is only used when its header matches.
MT_TABLE_HEADER = (0x4D544A31, 21, 16, 64, 78, 10496)


def mt19937_host_table() -> Tensor:
    """Jump-ahead table (constants of MT19937): loaded from the file written at
    build time if its size and header match, else computed on the host (~2 s) and cached."""
    global _mt_host_table
    with _mt_lock:
        if _mt_host_table is None:
            lib = _native.lib()
            nbytes = lib.tio_mt19937_table_bytes()
            blob = None
            if _MT_TABLE_FILE.exists() and _MT_TABLE_FILE.stat().st_size == nbytes:
                cached = np.fromfile(_MT_TABLE_FILE, dtype=np.uint8)
                if tuple(int(v) for v in cached[:24].view(np.uint32)) == MT_TABLE_HEADER:
                    blob = torch.from_numpy(cached)
            if blob is None:
                blob = torch.zeros(nbytes, dtype=torch.uint8)
                _native.call("tio_mt19937_build_table", blob.data_ptr(), nbytes)
                try:
                    blob.numpy().tofile(_MT_TABLE_FILE)
                except OSError:
                    pass
            _mt_host_table = blob
        return _mt_host_table


def _mt_table(device: torch.device) -> Tensor:
    key = (device.type, device.index)
    table = _mt_device_tables.get(key)
    if table is None:
        with _init_lock:
            table = _mt_device_tables.get(key)
            if table is None:
                table = mt19937_host_table().to(device)
                torch.cuda.synchronize(device)  # other threads' streams may read it right away
                _mt_device_tables[key] = table
    return table


def randn_mt19937(seed: int, offset: int, n: int, device, out: Tensor | None = None) -> Tensor:
    """Elements [offset, offset+n) of ``torch.randn(N, generator=CPU mt19937(seed))``
    computed on ``device`` (to ~1 ulp of the host's libm).  Needs offset, n
    multiples of 16 and offset + n <= 2**31; callers keep ragged tails on the host."""
    device = torch.device(device)
    if n < 16 or n % 16 or offset % 16 or offset + n > MT_MAX_WORDS:
        raise ValueError("randn_mt19937: offset and n must be multiples of 16, n >= 16,"
                         " offset + n <= 2**31")
    z = torch.empty(n, dtype=torch.float32, device=device) if out is None else out
    lib = _native.lib()
    ws_bytes = lib.tio_randn_mt19937_workspace_bytes(offset, n)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    table = _mt_table(device)
    with torch.cuda.device(device):
        _native.call("tio_randn_mt19937", int(seed) & 0xFFFFFFFF, offset, n, _ptr(z), _ptr(table),
                     _ptr(workspace), ws_bytes, torch.cuda.current_stream(device).cuda_stream)
    _count(4)
    return z


# ---- LabelsToImage: the reference's CUDA randn_like draws, recomputed per voxel --------

_cuda_rng_lock = threading.Lock()


def labels_to_image(labels: Tensor, label_values, means, stds, draw=None) -> Tensor:
    """(B, C, I, J, K) label batch -> (B, 1, I, J, K) fp32 synthetic image, bit-identical to
    _generate_from_labels / _generate_per_element (intensity/labels_to_image.py:182-290) run on
    the same CUDA tensors from the same CUDA generator state, which it advances by as much.

    ``label_values``: ascending distinct labels; ``means`` / ``stds``: (B, n) or (n,) values per
    label; ``draw``: (n,) position of each label in the reference's draw order, -1 = no draw
    (default: ascending order, skipping labels whose means and stds are all zero).  Channel 0 is
    read.  One draw of B*I*J*K normals per drawn label is reserved on the device's default CUDA
    generator, as ATen's ``philox_cuda_state`` would hand them out."""
    if labels.dtype not in DTYPE_CODES:
        raise TypeError(f"labels_to_image: unsupported label dtype {labels.dtype}")
    if labels.ndim != 5:
        raise ValueError(f"labels_to_image expects (B, C, I, J, K), got {tuple(labels.shape)}")
    b, c = int(labels.shape[0]), int(labels.shape[1])
    vox = int(np.prod(labels.shape[2:]))
    numel = b * vox
    tables.check_randn_numel(numel)
    _require_cuda(labels, "labels_to_image")
    if torch.cuda.is_current_stream_capturing():
        raise RuntimeError("labels_to_image: CUDA-graph capture is not supported (the generator offsets are"
                           " reserved on the host)")
    values = np.ascontiguousarray(np.asarray(label_values, dtype=np.int64).reshape(-1))
    n = int(values.shape[0])
    if n and np.any(np.diff(values) <= 0):
        raise ValueError("labels_to_image: label_values must be strictly ascending")
    mean = np.array(np.broadcast_to(np.asarray(means, dtype=np.float32).reshape(-1, n), (b, n)))
    std = np.array(np.broadcast_to(np.asarray(stds, dtype=np.float32).reshape(-1, n), (b, n)))
    if draw is None:
        active = np.any(mean != 0, axis=0) | np.any(std != 0, axis=0)
        draw = np.where(active, np.cumsum(active) - 1, -1)
    draw = np.asarray(draw, dtype=np.int64).reshape(n)
    n_draws = int((draw >= 0).sum())
    out = torch.empty((b, 1, *labels.shape[2:]), dtype=torch.float32, device=labels.device)
    if numel == 0:
        return out  # randn_like of an empty tensor consumes nothing
    device = labels.device
    props = torch.cuda.get_device_properties(device)
    grid_x, counter_offset = tables.randn_cuda_layout(numel, props.multi_processor_count,
                                                      props.max_threads_per_multi_processor)
    gen = torch.cuda.default_generators[device.index]
    with _cuda_rng_lock:
        seed = int(gen.initial_seed())
        base = int(gen.get_offset())
        if n_draws:
            gen.set_offset(base + n_draws * counter_offset)
    # draw k starts where the k previous draws left the offset; -1 (all bits set) = not drawn
    offsets = np.where(draw >= 0, base + draw * counter_offset, -1).astype(np.int64)
    labels = labels.contiguous()
    values_d, mean_d, std_d, offsets_d = upload(device, values, mean, std, offsets) if n else (None,) * 4
    with torch.cuda.device(device):
        _native.call("tio_labels_to_image", _ptr(labels), DTYPE_CODES[labels.dtype], c, b, vox, _ptr(values_d), n,
                     _ptr(mean_d), _ptr(std_d), _ptr(offsets_d), seed & (2**64 - 1), grid_x, _ptr(out),
                     _stream(labels))
    _count(2 if n else 1)
    return out


# ---- label-map utilities (transforms/label/) ----------------------------------------------------


def _label_map(src: Tensor, name: str) -> Tensor:
    _require_cuda(src, name)
    if src.dtype not in DTYPE_CODES:
        raise TypeError(f"{name}: unsupported label dtype {src.dtype}")
    if src.ndim != 5:
        raise ValueError(f"{name} expects (B, C, I, J, K), got {tuple(src.shape)}")
    return src.contiguous()


def label_lut(src: Tensor, keys: np.ndarray, values: np.ndarray, *, identity: bool) -> Tensor:
    """``src`` with every element equal to ``keys[i]`` replaced by ``values[i]`` (tables from
    `tables.label_lut`), and every other element kept (``identity``) or set to 0 — the result of
    RemapLabels / RemoveLabels (``clone``) or SequentialLabels (``zeros_like``), one pass."""
    src = _label_map(src, "label_lut")
    dst = torch.empty_like(src)
    n = int(keys.shape[0])
    keys_d, values_d = upload(src.device, keys, values) if n else (None, None)
    with torch.cuda.device(src.device):
        _native.call("tio_label_lut", _ptr(src), _ptr(dst), DTYPE_CODES[src.dtype], src.numel(), _ptr(keys_d),
                     _ptr(values_d), n, int(bool(identity)), _stream(src))
    _count(2 if n else 1)
    return dst


def label_contour(src: Tensor) -> Tensor:
    """(B, C, I, J, K) labels -> fp32 1 where the 3x3x3 minimum of float(v) (-1 outside the volume)
    differs from float(v), else 0 (label/contour.py:52-71)."""
    src = _label_map(src, "label_contour")
    dst = torch.empty(src.shape, dtype=torch.float32, device=src.device)
    if src.numel():
        b, c, i, j, k = src.shape
        with torch.cuda.device(src.device):
            _native.call("tio_label_contour", _ptr(src), DTYPE_CODES[src.dtype], b * c, i, j, k, _ptr(dst),
                         _stream(src))
        _count(1)
    return dst


def label_range(src: Tensor) -> tuple[int, int]:
    """(min, max) of ``long(v)`` over channel 0 of a non-empty (B, C, I, J, K) batch: one small
    device-to-host read."""
    src = _label_map(src, "label_range")
    b, c = src.shape[:2]
    out = torch.empty(2, dtype=torch.int64, device=src.device)
    with torch.cuda.device(src.device):
        _native.call("tio_label_range", _ptr(src), DTYPE_CODES[src.dtype], b, c, src[0, 0].numel(), _ptr(out),
                     _stream(src))
    _count(2)
    lo, hi = out.tolist()
    return lo, hi


def onehot_classes(src: Tensor, num_classes: int) -> Tensor:
    """(B, C, I, J, K) labels -> (B, num_classes, I, J, K) fp32: channel c is ``long(v) == c`` on
    channel 0 of the map (label/one_hot.py:64-68).  The caller checks the classes' range first."""
    src = _label_map(src, "onehot_classes")
    b, c = src.shape[:2]
    dst = torch.empty((b, num_classes, *src.shape[2:]), dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        _native.call("tio_onehot_classes", _ptr(src), DTYPE_CODES[src.dtype], b, c, src[0, 0].numel(),
                     int(num_classes), _ptr(dst), _stream(src))
    _count(1)
    return dst


def channel_argmax(src: Tensor) -> Tensor:
    """(B, C, I, J, K) -> (B, 1, I, J, K) fp32 ``argmax(dim=1, keepdim=True).float()``: the first
    maximum, a NaN counting as the maximum (label/one_hot.py:95-96)."""
    src = _label_map(src, "channel_argmax")
    b, c = src.shape[:2]
    dst = torch.empty((b, 1, *src.shape[2:]), dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        _native.call("tio_channel_argmax", _ptr(src), DTYPE_CODES[src.dtype], b, c, src[0, 0].numel(), _ptr(dst),
                     _stream(src))
    _count(1)
    return dst


# ---- resolution changes (spatial/resize.py, spatial/anisotropy.py) ------------------------------

# every label dtype, and fp16 / bf16 / fp64 images, which the kernels compute in fp32 and cast back
# as the reference's data.float() ... .to(dtype) do (tio_dtype TIO_F16 / TIO_BF16 / TIO_F64)
RESOLUTION_DTYPE_CODES = {**DTYPE_CODES, torch.float16: 6, torch.bfloat16: 7, torch.float64: 8}


def _volume_batch(src: Tensor, name: str) -> Tensor:
    _require_cuda(src, name)
    if src.dtype not in RESOLUTION_DTYPE_CODES:
        raise TypeError(f"{name}: unsupported dtype {src.dtype}")
    if src.ndim != 5:
        raise ValueError(f"{name} expects (B, C, I, J, K), got {tuple(src.shape)}")
    return src.contiguous()


def interpolate(src: Tensor, out_shape, idx: np.ndarray, lam: np.ndarray | None) -> Tensor:
    """(B, C, I, J, K) -> (B, C, *out_shape) of src's dtype: ATen's CUDA trilinear
    (align_corners=True; ``lam`` given) or nearest resize of ``src.float()``, cast back, from the
    per-axis tables of `tables.resize_tables` / `tables.anisotropy_shared_tables`, one pass."""
    src = _volume_batch(src, "interpolate")
    b, c, i, j, k = src.shape
    oi, oj, ok = (int(s) for s in out_shape)
    dst = torch.empty((b, c, oi, oj, ok), dtype=src.dtype, device=src.device)
    if src.numel() and dst.numel():
        idx_d, lam_d = upload(src.device, idx, lam)
        with torch.cuda.device(src.device):
            _native.call("tio_interpolate", _ptr(src), _ptr(dst), RESOLUTION_DTYPE_CODES[src.dtype], b * c, i, j, k, oi, oj,
                         ok, _ptr(idx_d), _ptr(lam_d), int(lam is not None), _stream(src))
        _count(1)
    return dst


def axis_resample(src: Tensor, axis: np.ndarray, lo: np.ndarray, hi: np.ndarray, w: np.ndarray, *,
                  linear: bool) -> Tensor:
    """Anisotropy's per-instance degradation of a (B, C, I, J, K) batch, one pass: element b is
    resampled along ``axis[b]`` from the (lo, hi, w) rows of `tables.anisotropy_instance_tables`
    (nearest: lo only), or copied when ``axis[b]`` is -1 (anisotropy.py:132-214)."""
    src = _volume_batch(src, "axis_resample")
    b, c, i, j, k = src.shape
    dst = torch.empty_like(src)
    if src.numel():
        if linear:
            axis_d, lo_d, hi_d, w_d = upload(src.device, axis, lo, hi, w)
        else:
            (axis_d, lo_d), hi_d, w_d = upload(src.device, axis, lo), None, None
        with torch.cuda.device(src.device):
            _native.call("tio_axis_resample", _ptr(src), _ptr(dst), RESOLUTION_DTYPE_CODES[src.dtype], b, c, i, j, k,
                         _ptr(axis_d), _ptr(lo_d), _ptr(hi_d), _ptr(w_d), int(lo.shape[1]), int(bool(linear)),
                         _stream(src))
        _count(1)
    return dst
