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
# every label dtype, and fp16 / bf16 / fp64 images, which the kernels compute in fp32 and cast back
# as the reference's data.float() ... .to(dtype) do (tio_dtype TIO_F16 / TIO_BF16 / TIO_F64)
IMAGE_DTYPE_CODES = {**DTYPE_CODES, torch.float16: 6, torch.bfloat16: 7, torch.float64: 8}
NEAREST, LINEAR, LABEL_PV = 0, 1, 2
FLAG_PASSTHROUGH, FLAG_ELASTIC = 1, 2

def launches() -> int:
    """Number of kernels this thread has launched through the library, counted by the library at
    each launch (`tio_launch_count`)."""
    return _native.lib().tio_launch_count()


def _launch(name: str, device, *args) -> None:
    """Call the stream-taking entry point ``name`` with ``args`` and the current stream of
    ``device``, with ``device`` current: CUDA refuses a launch into another device's stream."""
    with torch.cuda.device(device):
        _native.call(name, *args, torch.cuda.current_stream(device).cuda_stream)


def _ptr(t: Tensor | None):
    return None if t is None else t.data_ptr()


def _check(t: Tensor, name: str, *, dtypes=None, ndim: int | None = 5) -> None:
    """Refuse ``t`` as an input of ops.``name`` unless it is a CUDA tensor that does not require
    grad, of a dtype in ``dtypes`` (None: any) with ``ndim`` dimensions (None: any)."""
    if not t.is_cuda:
        raise RuntimeError(
            f"torchio_b200.ops.{name}: expected a CUDA tensor (got {t.device});"
            " the kernels have no CPU fallback"
        )
    if t.requires_grad:
        raise NotImplementedError(
            f"torchio_b200.ops.{name}: kernels are forward-only; detach() the input"
        )
    if dtypes is not None and t.dtype not in dtypes:
        raise TypeError(f"{name}: unsupported dtype {t.dtype}")
    if ndim is not None and t.ndim != ndim:
        raise ValueError(f"{name} expects a {ndim}-D tensor, got {tuple(t.shape)}")


def _batch(t: Tensor, name: str, *, dtypes=None, ndim: int | None = 5, in_place: bool = False) -> Tensor:
    """``t`` checked by `_check` and returned contiguous: a non-contiguous ``t`` is copied, or
    refused when ``in_place`` (the op uses ``t`` itself)."""
    _check(t, name, dtypes=dtypes, ndim=ndim)
    if not in_place:
        return t.contiguous()
    if not t.is_contiguous():
        raise ValueError(f"{name} expects a contiguous tensor, got strides {t.stride()}")
    return t


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
        _launch("tio_upload", dev.device, stage.data_ptr(), dev.data_ptr(), offset)
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


_differentiable = False


def set_differentiable(enabled: bool) -> bool:
    """Process-wide switch of the transforms' differentiable path; returns the previous value.

    Off (the default), a transform refuses an image that requires grad.  On, a transform of the
    differentiable set (see `torchio_b200.autograd`) records a graph node when
    ``torch.is_grad_enabled()`` and an image it modifies requires grad, and any other transform
    that would modify such an image raises NotImplementedError naming itself.  The ``ops``
    functions themselves stay forward-only either way."""
    global _differentiable
    previous, _differentiable = _differentiable, bool(enabled)
    return previous


def differentiable_default() -> bool:
    return _differentiable


def resample(
    src: Tensor, mat: Tensor, cp: Tensor | None, flags: Tensor | None,
    spacing_in, spacing_out, *, affine_first: bool, mode: int,
    fill: Tensor | None, out_shape=None, box_hint: int = 0, exact_coords: bool | None = None,
    tiers=None,
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

    tiers: ``(elems, runs)`` for a box edge per element (`tio_resample_tiered`): ``elems`` an
    int32 (B,) cuda permutation of the batch, ``runs`` ``[(count, edge), ...]`` over it in
    ascending edges.  fp32 trilinear without exact coordinates only; same output as without.
    """
    src = _batch(src, "resample", dtypes=DTYPE_CODES)
    exact = _exact_default if exact_coords is None else exact_coords
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
    args = (_ptr(src), _ptr(dst), DTYPE_CODES[src.dtype],
            b, c, i, j, k, oi, oj, ok, _ptr(mat), _ptr(cp), _ptr(flags), ni, nj, nk,
            sp_in.ctypes.data, sp_out.ctypes.data, int(bool(affine_first)),
            int(mode) | (EXACT_COORDS if exact else 0), _ptr(fill), int(box_hint))
    if tiers is None:
        _launch("tio_resample", src.device, *args, _ptr(workspace), ws_bytes)
        return dst
    elems, runs = tiers
    if elems.dtype != torch.int32 or elems.shape != (b,) or not elems.is_cuda:
        raise ValueError(f"resample: tiers needs an int32 ({b},) cuda element list")
    runs = np.asarray(runs, dtype=np.int32).reshape(-1, 2)
    _launch("tio_resample_tiered", src.device, *args, _ptr(elems), runs.ctypes.data, len(runs),
            _ptr(workspace), ws_bytes)
    return dst


def resample_backward(
    grad_out: Tensor, in_shape, mat: Tensor, cp: Tensor | None, flags: Tensor | None,
    spacing_in, spacing_out, *, affine_first: bool, mode: int, fill: Tensor | None, box_hint: int = 0,
) -> Tensor:
    """K1ᵀ (`tio_resample_backward`): the fp32 (B, C, *in_shape) gradient of `resample`'s input for
    the fp32 (B, C, OI, OJ, OK) gradient ``grad_out`` of its output, same geometry arguments, modes
    NEAREST and LINEAR.  Not deterministic: the taps are added with atomics."""
    grad_out = _batch(grad_out, "resample_backward", dtypes=(torch.float32,))
    b, c, oi, oj, ok = grad_out.shape
    i, j, k = (int(v) for v in in_shape)
    if mode not in (NEAREST, LINEAR):
        raise ValueError(f"resample_backward: mode {mode} has no adjoint kernel")
    grad_in = torch.empty((b, c, i, j, k), dtype=torch.float32, device=grad_out.device)
    ni = nj = nk = 0
    if cp is not None:
        ni, nj, nk = cp.shape[1:4]
    sp_in = np.asarray(spacing_in, dtype=np.float32)
    sp_out = np.asarray(spacing_out, dtype=np.float32)
    ws_bytes = _native.lib().tio_resample_workspace_bytes(b, oi, oj, ok)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=grad_out.device)
    _launch("tio_resample_backward", grad_out.device, _ptr(grad_out), _ptr(grad_in), b, c, i, j, k, oi, oj, ok,
            _ptr(mat), _ptr(cp), _ptr(flags), ni, nj, nk, sp_in.ctypes.data, sp_out.ctypes.data,
            int(bool(affine_first)), int(mode), _ptr(fill), int(box_hint), _ptr(workspace), ws_bytes)
    return grad_in


def bspline_prefilter(src: Tensor, order: int, flags: Tensor | None = None, *, in_place: bool = False) -> Tensor:
    """(B,C,I,J,K) -> fp32 interpolating B-spline coefficients of ``order`` (2-7) under the dct2
    boundary, the prefilter of ``interpol.grid_pull(..., bound="dct2", prefilter=True)``
    (spatial/spatial.py:1734-1761, 1860-1878).  ``in_place`` (fp32 ``src`` only) overwrites ``src``
    with them.  Elements flagged passthrough are left as they are."""
    src = _batch(src, "bspline_prefilter", dtypes=DTYPE_CODES, in_place=in_place)
    if in_place and src.dtype != torch.float32:
        raise TypeError(f"bspline_prefilter: in_place needs a float32 tensor, got {src.dtype}")
    coeff = src if in_place else torch.empty(src.shape, dtype=torch.float32, device=src.device)
    _launch("tio_bspline_prefilter", src.device, _ptr(src), DTYPE_CODES[src.dtype], _ptr(coeff), _ptr(flags),
            *src.shape, int(order))
    return coeff


def bspline_resample(
    coeff: Tensor, src: Tensor, mat: Tensor, cp: Tensor | None, flags: Tensor | None,
    spacing_in, spacing_out, *, affine_first: bool, order: int, out_shape=None,
) -> Tensor:
    """The B-spline of ``coeff`` (from `bspline_prefilter`) at K1's sampling coordinates, 0 outside
    (-0.05, n - 1 + 0.05), cast to ``src.dtype``; passthrough elements copy ``src``.  Geometry
    arguments as `resample`."""
    src = _batch(src, "bspline_resample", dtypes=DTYPE_CODES)
    _check(coeff, "bspline_resample", dtypes=(torch.float32,))
    if coeff.shape != src.shape or not coeff.is_contiguous():
        raise ValueError(f"bspline_resample: coeff must be contiguous of shape {tuple(src.shape)}")
    b, c, i, j, k = src.shape
    oi, oj, ok = (i, j, k) if out_shape is None else out_shape
    dst = torch.empty((b, c, oi, oj, ok), dtype=src.dtype, device=src.device)
    ni = nj = nk = 0
    if cp is not None:
        ni, nj, nk = cp.shape[1:4]
    sp_in = np.asarray(spacing_in, dtype=np.float32)
    sp_out = np.asarray(spacing_out, dtype=np.float32)
    _launch("tio_bspline_resample", src.device, _ptr(coeff), _ptr(src), _ptr(dst), DTYPE_CODES[src.dtype],
            b, c, i, j, k, oi, oj, ok, _ptr(mat), _ptr(cp), _ptr(flags), ni, nj, nk,
            sp_in.ctypes.data, sp_out.ctypes.data, int(bool(affine_first)), int(order))
    return dst


def _label_table(labels: Tensor, dtype: torch.dtype, device: torch.device) -> Tensor:
    return labels.to(device=device, dtype=torch.float32 if dtype == torch.float32 else torch.int64).contiguous()


def onehot(src: Tensor, labels: Tensor) -> Tensor:
    """(B,1,I,J,K) label batch -> (B,n,I,J,K) fp32 one-hot channels, ``labels`` = the distinct
    values in ascending order (spatial/spatial.py:1362-1365)."""
    src = _batch(src, "onehot", dtypes=DTYPE_CODES, ndim=None)
    b, n = src.shape[0], int(labels.numel())
    vox = src[0].numel()
    table = _label_table(labels, src.dtype, src.device)
    dst = torch.empty((b, n, *src.shape[2:]), dtype=torch.float32, device=src.device)
    _launch("tio_onehot", src.device, _ptr(src), DTYPE_CODES[src.dtype], b, vox, _ptr(table), n, _ptr(dst))
    return dst


def label_argmax(sampled: Tensor, labels: Tensor, pad_label: float, dtype: torch.dtype) -> Tensor:
    """(B,n,I,J,K) sampled one-hot channels -> (B,1,I,J,K) labels of ``dtype``: first maximum over
    the channels, ``pad_label`` where their sum is not > 0.5 (spatial/spatial.py:1378-1389)."""
    sampled = _batch(sampled, "label_argmax", ndim=None)
    if dtype not in DTYPE_CODES:
        raise TypeError(f"label_argmax: unsupported dtype {dtype}")
    b, n = sampled.shape[:2]
    vox = sampled[0, 0].numel()
    table = _label_table(labels, dtype, sampled.device)
    dst = torch.empty((b, 1, *sampled.shape[2:]), dtype=dtype, device=sampled.device)
    _launch("tio_label_argmax", sampled.device, _ptr(sampled), b, n, vox, _ptr(table), float(pad_label), _ptr(dst),
            DTYPE_CODES[dtype])
    return dst


def min_sample0(src: Tensor) -> Tensor:
    """Per-channel min of batch element 0, on device, no sync
    (spatial/spatial.py:2054-2060,2094-2095)."""
    src = _batch(src, "min_sample0", ndim=None)
    c = src.shape[1]
    n = src[0, 0].numel()
    fill = torch.empty(c, dtype=torch.float32, device=src.device)
    _launch("tio_min_sample0", src.device, _ptr(src), c, n, _ptr(fill))
    return fill


def crop_patches(volume: Tensor, corners, size, out: Tensor | None = None) -> Tensor:
    """Gather ``n`` patches of ``size`` at voxel ``corners`` (n,3) from one volume
    (C,I,J,K) into a dense (n,C,*size) block in a single launch
    (data/sampler.py:54-67 + loader.py:15-24).  ``out``: a contiguous (n,C,*size) block to
    write into (e.g. consecutive slots of a patch ring) instead of a fresh tensor."""
    volume = _batch(volume, "crop_patches", ndim=4)
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
    _launch("tio_crop_patches", volume.device, _ptr(volume), _ptr(dst), volume.element_size(), c, i, j, k, n,
            _ptr(corners_d), pi, pj, pk)
    return dst


AGGREGATE_MODES = {"crop": 0, "average": 1, "hann": 2}


def aggregate_patches(patches: Tensor, out: Tensor, counts: Tensor | None, boxes: np.ndarray, mode: str,
                      window: np.ndarray | None = None) -> None:
    """In place: add the patches of a batch (B, C, pi, pj, pk) into the PatchAggregator buffer ``out``
    (C, I, J, K) of the same dtype and device, in the order of ``boxes``, as the reference's
    `_add_crop` / `_add_average` / `_add_hann` do one patch at a time (data/aggregator.py:143-237).
    ``counts``: the (1, I, J, K) count buffer of "average" and "hann", None for "crop".
    ``boxes``: int32 (n, 10) rows ``dst lo (3), dst hi (3), src lo (3), patch row``.  ``window``: fp32
    (pi + pj + pk,), the three 1-D Hann windows of the patch, for "hann" only.  One launch, no host
    sync."""
    _check(patches, "aggregate_patches")
    out = _batch(out, "aggregate_patches", ndim=4, in_place=True)
    if mode not in AGGREGATE_MODES:
        raise ValueError(f"aggregate_patches: mode {mode!r} not in {tuple(AGGREGATE_MODES)}")
    if patches.dtype != out.dtype or (counts is not None and counts.dtype != out.dtype):
        raise TypeError(f"aggregate_patches: patches {patches.dtype} and buffers {out.dtype} differ")
    dtype = torch.uint8 if out.dtype == torch.bool and mode == "crop" else out.dtype
    if dtype not in IMAGE_DTYPE_CODES:
        raise TypeError(f"aggregate_patches: unsupported dtype {out.dtype} in {mode} mode")
    if patches.device != out.device:
        raise ValueError(f"aggregate_patches: patches on {patches.device}, buffer on {out.device}")
    if counts is not None and (tuple(counts.shape) != (1, *out.shape[1:]) or not counts.is_contiguous()
                               or counts.device != out.device):
        raise ValueError(f"aggregate_patches: counts {tuple(counts.shape)} for a buffer {tuple(out.shape)}")
    boxes = np.ascontiguousarray(boxes, dtype=np.int32).reshape(-1, 10)
    if boxes.shape[0] == 0:
        return
    if window is not None:
        window = np.ascontiguousarray(window, dtype=np.float32)
    patches = patches.contiguous()
    b, c, pi, pj, pk = (int(s) for s in patches.shape)
    boxes_d, window_d = upload(out.device, boxes, window)
    _launch("tio_aggregate_patches", out.device, _ptr(patches), _ptr(out), _ptr(counts), IMAGE_DTYPE_CODES[dtype],
            AGGREGATE_MODES[mode], *(int(s) for s in out.shape), b, pi, pj, pk, int(boxes.shape[0]),
            boxes.ctypes.data, _ptr(boxes_d), _ptr(window_d))


def aggregate_finish(out: Tensor, counts: Tensor) -> Tensor:
    """A new tensor ``out / counts.clamp(min=1)`` (data/aggregator.py:117-120) for a PatchAggregator
    buffer (C, I, J, K) and its (1, I, J, K) count: the buffer's dtype, fp32 for integers.  One launch."""
    out = _batch(out, "aggregate_finish", dtypes=IMAGE_DTYPE_CODES, ndim=4, in_place=True)
    if counts.dtype != out.dtype:
        raise TypeError(f"aggregate_finish: unsupported dtypes {out.dtype} / {counts.dtype}")
    if tuple(counts.shape) != (1, *out.shape[1:]) or not counts.is_contiguous() or counts.device != out.device:
        raise ValueError(f"aggregate_finish: buffer {tuple(out.shape)} and counts {tuple(counts.shape)}")
    floating = out.dtype.is_floating_point
    dst = torch.empty(out.shape, dtype=out.dtype if floating else torch.float32, device=out.device)
    if out.numel() == 0:
        return dst
    _launch("tio_aggregate_finish", out.device, _ptr(out), _ptr(counts), _ptr(dst), IMAGE_DTYPE_CODES[out.dtype],
            int(out.shape[0]), out[0].numel())
    return dst


PAD_MODES = {"constant": 0, "replicate": 1, "reflect": 2, "circular": 3}


def remap(src: Tensor, out_shape, offsets, *, mode: str = "constant", fill=0, flip: Tensor | None = None,
          out: Tensor | None = None) -> Tensor:
    """Flip / Crop / Pad in one pass: ``out[..., o] = src[..., o - offset]`` per spatial
    axis with F.pad's out-of-range rules, then per-element axis reversal (``flip``: (B,)
    uint8 cuda, bit 0 I, 1 J, 2 K).  flip.py:233-263, crop.py:84-101, _padding.py:73-104."""
    src = _batch(src, "remap")
    b, c, i, j, k = (int(v) for v in src.shape)
    oi, oj, ok = (int(v) for v in out_shape)
    if out is None:
        dst = torch.empty((b, c, oi, oj, ok), dtype=src.dtype, device=src.device)
    else:
        dst = out
        if (tuple(dst.shape) != (b, c, oi, oj, ok) or dst.dtype != src.dtype or dst.device != src.device
                or not dst.is_contiguous()):
            raise ValueError("remap: `out` must be a contiguous (B, C, *out_shape) block of the source's dtype/device")
    # F.pad casts the value (a double) to the tensor's dtype: an fp64 tensor keeps all of it
    fill_host = torch.tensor([fill], dtype=torch.float64 if isinstance(fill, float) else None).to(src.dtype)
    _launch("tio_remap", src.device, _ptr(src), _ptr(dst), src.element_size(), b, c, i, j, k, oi, oj, ok,
            int(offsets[0]), int(offsets[1]), int(offsets[2]), PAD_MODES[mode], fill_host.data_ptr(), _ptr(flip))
    return dst


def permute(src: Tensor, perm, flip_bits: int = 0) -> Tensor:
    """Spatial axis permutation with flips of a (B, C, I, J, K) batch in one pass: output axis d is
    input axis ``perm[d]``, reversed when bit ``perm[d]`` of ``flip_bits`` is set (flips indexed by
    input axis, applied before the transpose).  The identity permutation flips through `remap`
    with the same bits for every element, or returns ``src`` itself when nothing flips, as the
    reference does.  reorient.py:63-91, transpose.py:36-50."""
    _check(src, "permute")
    perm = tuple(int(p) for p in perm)
    if sorted(perm) != [0, 1, 2]:
        raise ValueError(f"permute: {perm} is not a permutation of (0, 1, 2)")
    flip_bits = int(flip_bits)
    if perm == (0, 1, 2):
        if flip_bits == 0:
            return src
        (flags,) = upload(src.device, np.full(src.shape[0], flip_bits, dtype=np.uint8))
        return remap(src, src.shape[2:], (0, 0, 0), flip=flags)
    src = src.contiguous()
    b, c, i, j, k = (int(v) for v in src.shape)
    n = (i, j, k)
    dst = torch.empty((b, c, *(n[p] for p in perm)), dtype=src.dtype, device=src.device)
    _launch("tio_permute", src.device, _ptr(src), _ptr(dst), src.element_size(), b, c, i, j, k, *perm, flip_bits)
    return dst


def blur(src: Tensor, taps: Tensor, radius: Tensor, big_r: int, axes_mask: int,
         identity: Tensor | None) -> Tensor:
    """K3 (intensity/blur.py:129-252)."""
    src = _batch(src, "blur")
    b, c, i, j, k = src.shape
    dst = torch.empty_like(src)
    scratch = torch.empty_like(src) if (axes_mask & 6) or big_r > WIDE_R else None
    _launch("tio_blur", src.device, _ptr(src), _ptr(dst), _ptr(scratch), b, c, i, j, k, _ptr(taps),
            _ptr(radius), int(big_r), int(axes_mask), _ptr(identity))
    return dst


#: Tables with a larger radius run one launch per blurred axis (after the bias pass), through
#: a scratch buffer whatever the axes.
WIDE_R = 16


def moments(values: Tensor, mask: Tensor | None = None) -> tuple[float, float, float]:
    """(sum, sum of squared deviations from the mean, count) of the selected values of a contiguous
    fp32 CUDA tensor, fp64 accumulation on the device, one small D2H read (the reference calls
    ``.item()`` here too: standardize.py:76-77)."""
    values = _batch(values, "moments", ndim=None)
    m8 = None if mask is None else mask.expand_as(values).contiguous().to(torch.uint8)
    out = torch.empty(3, dtype=torch.float64, device=values.device)
    _launch("tio_moments", values.device, _ptr(values), _ptr(m8), values.numel(), _ptr(out))
    s, ss, n = out.tolist()
    return s, ss, n


def quantile_neighbours(values: Tensor, qs, mask: Tensor | None = None):
    """For each q in ``qs`` (at most two): the order statistics torch.kthvalue(lower + 1) and
    kthvalue(lower + 2) return, and ``index - lower`` (transforms/_statistics.py:37-45), found by
    an exact radix select on the device.  Returns (values[2m], weights[m], count)."""
    values = _batch(values, "quantile_neighbours", ndim=None)
    m8 = None if mask is None else mask.expand_as(values).contiguous().to(torch.uint8)
    qs = np.ascontiguousarray(np.asarray(qs, dtype=np.float64).reshape(-1))
    m = int(qs.shape[0])
    dev = values.device
    vals = torch.empty(2 * m, dtype=torch.float32, device=dev)
    out = torch.empty(m + 1, dtype=torch.float64, device=dev)
    ws_bytes = _native.lib().tio_quantiles_workspace_bytes()
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _launch("tio_quantiles", dev, _ptr(values), _ptr(m8), values.numel(), qs.ctypes.data, m, _ptr(vals),
            _ptr(out), out[m:].data_ptr(), _ptr(ws), ws_bytes)
    host = out.tolist()
    return vals.tolist(), host[:m], int(host[m])


def quantiles_batched(values: Tensor, qs, mask: Tensor | None = None):
    """`quantile_neighbours` for every element of a (B, ...) CUDA tensor of any image dtype (values
    taken as ``.float()`` gives them), with any number of quantiles, left on the device: returns
    (values (B, 2m) fp32, weights (B, m) fp64, count (B,) fp64, has_nan (B,) uint8) without a
    host sync (histogram_standardization.py:100-108,279)."""
    values = _batch(values, "quantiles_batched", dtypes=IMAGE_DTYPE_CODES, ndim=None)
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
    _launch("tio_quantiles_batched", dev, _ptr(values), IMAGE_DTYPE_CODES[values.dtype], _ptr(m8), b, per_elem,
            qs.ctypes.data, m, _ptr(vals), _ptr(weights), _ptr(count), _ptr(has_nan), _ptr(ws), ws_bytes)
    return vals, weights, count, has_nan


def histogram_tables(values: Tensor, weights: Tensor, has_nan: Tensor, landmarks: Tensor) -> Tensor:
    """(B, 3 (m - 1)) fp32 device tables {slopes, intercepts, edges} of
    _apply_histogram_standardization (histogram_standardization.py:279-300) from the output of
    `quantiles_batched` and the m fp32 landmarks, built on the device."""
    b, m = weights.shape
    landmarks = landmarks.to(device=values.device, dtype=torch.float32).contiguous()
    tables = torch.empty((b, 3 * (m - 1)), dtype=torch.float32, device=values.device)
    _launch("tio_histogram_tables", values.device, _ptr(values), _ptr(weights), _ptr(has_nan), _ptr(landmarks), b,
            m, _ptr(tables))
    return tables


def histogram_map(data: Tensor, tables: Tensor, m: int) -> None:
    """In place: each element of the contiguous (B, ...) CUDA tensor ``data`` through its
    piecewise-linear map ``slopes[bin] * x + intercepts[bin]``, bin = torch.bucketize(x, edges),
    computed in fp32 and stored in data's dtype (histogram_standardization.py:302-303)."""
    data = _batch(data, "histogram_map", dtypes=IMAGE_DTYPE_CODES, ndim=None, in_place=True)
    if data.numel() == 0:
        return
    _launch("tio_histogram_map", data.device, _ptr(data), _ptr(data), IMAGE_DTYPE_CODES[data.dtype], data.shape[0],
            data[0].numel(), _ptr(tables), int(m))


def rescale(src: Tensor, *, lo: float | None = None, hi: float | None = None, sub=None, div=None, mul=None,
            add=None, keep=None) -> Tensor:
    """``((clamp(src, lo, hi) - sub[b]) / div[b]) * mul[b] + add[b]`` over a (B, ...) fp32 batch, each
    step rounded like the reference's separate elementwise ops; omitted steps are skipped.
    ``sub/div/mul/add``: scalars or length-B sequences; ``keep``: length-B, 0 = copy the row."""
    src = _batch(src, "rescale", ndim=None)
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
    _launch("tio_rescale", src.device, _ptr(src), _ptr(dst), b, src[0].numel(),
            float(lo if lo is not None else 0.0), float(hi if hi is not None else 0.0),
            _ptr(sub_d), _ptr(div_d), _ptr(mul_d), _ptr(add_d), _ptr(keep_d), flags)
    return dst


def intensity_fused(
    src: Tensor, *, coarse: Tensor | None = None, bias_identity: Tensor | None = None,
    bias_divide: bool = False, taps: Tensor | None = None, radius: Tensor | None = None,
    big_r: int = 0, axes_mask: int = 0, mean: Tensor | None = None, std: Tensor | None = None,
    keep: Tensor | None = None, z: Tensor | None = None, z2: Tensor | None = None,
    philox_seed: int = 0, noise_mode: int = 0, rician: bool = False,
    gamma: Tensor | None = None, z_replay: tuple[int, ...] | None = None,
) -> Tensor:
    """Fused bias -> blur -> noise -> gamma (two HBM passes); any stage optional.

    Compose-level fusion of consecutive intensity transforms; a single transform
    is a call with only its own stage set.

    ``z_replay`` instead of ``z``: (seed, offset) for the normals of `randn_mt19937(seed, offset,
    src.numel())`, or (seed, offset, n, lo) for outputs [lo, lo + src.numel()) of the draw of n
    normals at stream word ``offset`` (a slice of the batch a draw was made for).  When the
    normals are a draw of their own on 16-word boundaries and the chain has a first pass and a
    J/K pass of table radius <= 6 on 16-byte aligned rows, they are generated inside the first
    pass (`tio_intensity_pass1_with_normals`) instead of before it; the result is the same bit
    for bit.
    """
    src = _batch(src, "intensity_fused")
    b, c, i, j, k = src.shape
    if z_replay is not None:
        seed, offset, n, lo = z_replay if len(z_replay) == 4 else (*z_replay, src.numel(), 0)
        hi = lo + src.numel()
        aligned = _mt_aligned_draw(offset, n, lo, hi)
        blur_jk = taps is not None and bool(axes_mask & 6) and big_r <= 6
        first_pass = coarse is not None or (taps is not None and bool(axes_mask & 1))
        if (aligned is not None and blur_jk and first_pass and noise_mode == 1 and not rician
                and k % 4 == 0 and src.data_ptr() % 16 == 0):
            return _intensity_fused_pass1_normals(
                src, coarse, bias_identity, bias_divide, taps, radius, big_r, axes_mask, mean, std,
                keep, gamma, seed, aligned)
        z = randn_mt19937(seed, offset, n, src.device, lo=lo, hi=hi).view(src.shape)
    dst = torch.empty_like(src)
    # the J/K pass alone reads src directly; after a first pass it reads the scratch buffer
    two_pass = taps is not None and axes_mask & 6 and (coarse is not None or axes_mask & 1)
    wide = taps is not None and axes_mask & 7 and big_r > WIDE_R
    scratch = torch.empty_like(src) if two_pass or wide else None
    si = sj = sk = 0
    if coarse is not None:
        si, sj, sk = coarse.shape[2:]
    _launch(
        "tio_intensity_fused", src.device, _ptr(src), _ptr(dst), _ptr(scratch), b, c, i, j, k,
        _ptr(coarse), si, sj, sk, _ptr(bias_identity), int(bool(bias_divide)),
        _ptr(taps), _ptr(radius), int(big_r), int(axes_mask),
        _ptr(mean), _ptr(std), _ptr(keep), _ptr(z), _ptr(z2),
        int(philox_seed) & (2**64 - 1), int(noise_mode), int(bool(rician)), _ptr(gamma),
    )
    return dst


def intensity_pass1_with_normals(
    src: Tensor, seed: int, offset: int, *, coarse: Tensor | None = None,
    bias_identity: Tensor | None = None, bias_divide: bool = False, taps: Tensor | None = None,
    radius: Tensor | None = None, big_r: int = 0, axes_mask: int = 0,
) -> tuple[Tensor, Tensor]:
    """(first pass of `intensity_fused` on ``src``: bias and the I axis of the blur,
    elements [offset, offset + src.numel()) of `randn_mt19937(seed)` shaped like ``src``), from one
    kernel in which the two run side by side on every SM.  Needs table radius <= 6, K % 4 == 0 and
    16-byte aligned data; the library refuses anything else."""
    src = _batch(src, "intensity_pass1_with_normals")
    b, c, i, j, k = src.shape
    n = src.numel()
    if n < 16 or n % 16 or offset % 16 or offset + n > MT_MAX_WORDS:
        raise ValueError("intensity_pass1_with_normals: offset and numel must be multiples of 16,"
                         " numel >= 16, offset + numel <= 2**31")
    dst = torch.empty_like(src)
    z = torch.empty_like(src)
    ws_bytes = _native.lib().tio_intensity_pass1_with_normals_workspace_bytes(offset, n)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=src.device)
    table = _mt_table(src.device)
    si = sj = sk = 0
    if coarse is not None:
        si, sj, sk = coarse.shape[2:]
    _launch(
        "tio_intensity_pass1_with_normals", src.device, _ptr(src), _ptr(dst), b, c, i, j, k,
        _ptr(coarse), si, sj, sk, _ptr(bias_identity), int(bool(bias_divide)),
        _ptr(taps), _ptr(radius), int(big_r), int(axes_mask),
        int(seed) & 0xFFFFFFFF, offset, n, _ptr(z), _ptr(table), _ptr(workspace), ws_bytes,
    )
    return dst, z


def _intensity_fused_pass1_normals(src, coarse, bias_identity, bias_divide, taps, radius, big_r,
                                   axes_mask, mean, std, keep, gamma, seed, offset) -> Tensor:
    """`intensity_fused` with the exact-noise normals generated under its first pass: that pass
    and the normals in one launch, then the J/K pass with noise and gamma at the store."""
    first, z = intensity_pass1_with_normals(
        src, seed, offset, coarse=coarse, bias_identity=bias_identity, bias_divide=bias_divide,
        taps=taps, radius=radius, big_r=big_r, axes_mask=axes_mask)
    return intensity_fused(first, taps=taps, radius=radius, big_r=big_r, axes_mask=axes_mask & 6,
                           mean=mean, std=std, keep=keep, z=z, noise_mode=1, gamma=gamma)


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
    """The jump-ahead table on ``device``, copied there once.  Cached by device index: a device
    without one ("cuda") is the current device, whose table the kernel must read."""
    index = torch.cuda.current_device() if device.index is None else device.index
    table = _mt_device_tables.get(index)
    if table is None:
        with _init_lock:
            table = _mt_device_tables.get(index)
            if table is None:
                table = mt19937_host_table().to(torch.device("cuda", index))
                torch.cuda.synchronize(index)  # other threads' streams may read it right away
                _mt_device_tables[index] = table
    return table


def mt_draw_words(n: int) -> int:
    """Words of the CPU generator's stream that ``torch.randn(n)`` takes, n >= 16: the n
    uniforms, then 16 more when n % 16 != 0 (normal_fill recomputes its last 16 outputs)."""
    return n + (16 if n % 16 else 0)


def _mt_aligned_draw(offset: int, n: int, lo: int, hi: int) -> int | None:
    """Outputs [lo, hi) of the draw of n at ``offset`` are the draw of hi - lo at the returned
    offset when all four are multiples of 16 (whole 16-groups of an aligned draw); else None."""
    return offset + lo if offset % 16 == 0 and n % 16 == 0 and lo % 16 == 0 and hi % 16 == 0 else None


def randn_mt19937(seed: int, offset: int, n: int, device, out: Tensor | None = None, *,
                  lo: int = 0, hi: int | None = None) -> Tensor:
    """Outputs [lo, hi) (default: all n) of ``torch.randn(n, generator=g)`` for a CPU mt19937
    generator ``g`` seeded with ``seed`` that has already used ``offset`` words of its stream
    (for an aligned ``offset``: elements [offset, offset+n) of ``torch.randn(N, generator=CPU
    mt19937(seed))``), computed on ``device`` to ~1 ulp of the host's libm.  Any offset, n >= 16,
    0 <= lo < hi <= n, and the draw must end within the jump table's reach:
    offset + `mt_draw_words`(n) <= 2**31."""
    device = torch.device(device)
    hi = n if hi is None else hi
    if n < 16 or offset < 0 or not 0 <= lo < hi <= n:
        raise ValueError(f"randn_mt19937: needs n >= 16, offset >= 0 and 0 <= lo < hi <= n,"
                         f" got offset={offset} n={n} lo={lo} hi={hi}")
    if offset + mt_draw_words(n) > MT_MAX_WORDS:
        raise ValueError(f"randn_mt19937: the draw of {n} at stream word {offset} ends beyond 2**31")
    z = torch.empty(hi - lo, dtype=torch.float32, device=device) if out is None else out
    lib = _native.lib()
    table = _mt_table(device)
    aligned = _mt_aligned_draw(offset, n, lo, hi)
    if aligned is not None:
        ws_bytes = lib.tio_randn_mt19937_workspace_bytes(aligned, hi - lo)
        workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
        _launch("tio_randn_mt19937", device, int(seed) & 0xFFFFFFFF, aligned, hi - lo, _ptr(z), _ptr(table),
                _ptr(workspace), ws_bytes)
        return z
    ws_bytes = lib.tio_randn_mt19937_window_workspace_bytes(offset, n)
    workspace = torch.empty(ws_bytes, dtype=torch.uint8, device=device)
    _launch("tio_randn_mt19937_window", device, int(seed) & 0xFFFFFFFF, offset, n, lo, hi, _ptr(z),
            _ptr(table), _ptr(workspace), ws_bytes)
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
    # dtype, shape and size are refused before the device is looked at, on any device
    if labels.dtype not in DTYPE_CODES:
        raise TypeError(f"labels_to_image: unsupported label dtype {labels.dtype}")
    if labels.ndim != 5:
        raise ValueError(f"labels_to_image expects (B, C, I, J, K), got {tuple(labels.shape)}")
    b, c = int(labels.shape[0]), int(labels.shape[1])
    vox = int(np.prod(labels.shape[2:]))
    numel = b * vox
    tables.check_randn_numel(numel)
    labels = _batch(labels, "labels_to_image")
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
    values_d, mean_d, std_d, offsets_d = upload(device, values, mean, std, offsets) if n else (None,) * 4
    _launch("tio_labels_to_image", device, _ptr(labels), DTYPE_CODES[labels.dtype], c, b, vox, _ptr(values_d), n,
            _ptr(mean_d), _ptr(std_d), _ptr(offsets_d), seed & (2**64 - 1), grid_x, _ptr(out))
    return out


# ---- label-map utilities (transforms/label/) ----------------------------------------------------


def label_lut(src: Tensor, keys: np.ndarray, values: np.ndarray, *, identity: bool) -> Tensor:
    """``src`` with every element equal to ``keys[i]`` replaced by ``values[i]`` (tables from
    `tables.label_lut`), and every other element kept (``identity``) or set to 0 — the result of
    RemapLabels / RemoveLabels (``clone``) or SequentialLabels (``zeros_like``), one pass."""
    src = _batch(src, "label_lut", dtypes=DTYPE_CODES)
    dst = torch.empty_like(src)
    n = int(keys.shape[0])
    keys_d, values_d = upload(src.device, keys, values) if n else (None, None)
    _launch("tio_label_lut", src.device, _ptr(src), _ptr(dst), DTYPE_CODES[src.dtype], src.numel(), _ptr(keys_d),
            _ptr(values_d), n, int(bool(identity)))
    return dst


def label_contour(src: Tensor) -> Tensor:
    """(B, C, I, J, K) labels -> fp32 1 where the 3x3x3 minimum of float(v) (-1 outside the volume)
    differs from float(v), else 0 (label/contour.py:52-71)."""
    src = _batch(src, "label_contour", dtypes=DTYPE_CODES)
    dst = torch.empty(src.shape, dtype=torch.float32, device=src.device)
    if src.numel():
        b, c, i, j, k = src.shape
        _launch("tio_label_contour", src.device, _ptr(src), DTYPE_CODES[src.dtype], b * c, i, j, k, _ptr(dst))
    return dst


def label_range(src: Tensor) -> tuple[int, int]:
    """(min, max) of ``long(v)`` over channel 0 of a non-empty (B, C, I, J, K) batch: one small
    device-to-host read."""
    src = _batch(src, "label_range", dtypes=DTYPE_CODES)
    b, c = src.shape[:2]
    out = torch.empty(2, dtype=torch.int64, device=src.device)
    _launch("tio_label_range", src.device, _ptr(src), DTYPE_CODES[src.dtype], b, c, src[0, 0].numel(), _ptr(out))
    lo, hi = out.tolist()
    return lo, hi


def onehot_classes(src: Tensor, num_classes: int) -> Tensor:
    """(B, C, I, J, K) labels -> (B, num_classes, I, J, K) fp32: channel c is ``long(v) == c`` on
    channel 0 of the map (label/one_hot.py:64-68).  The caller checks the classes' range first."""
    src = _batch(src, "onehot_classes", dtypes=DTYPE_CODES)
    b, c = src.shape[:2]
    dst = torch.empty((b, num_classes, *src.shape[2:]), dtype=torch.float32, device=src.device)
    _launch("tio_onehot_classes", src.device, _ptr(src), DTYPE_CODES[src.dtype], b, c, src[0, 0].numel(),
            int(num_classes), _ptr(dst))
    return dst


def channel_argmax(src: Tensor) -> Tensor:
    """(B, C, I, J, K) -> (B, 1, I, J, K) fp32 ``argmax(dim=1, keepdim=True).float()``: the first
    maximum, a NaN counting as the maximum (label/one_hot.py:95-96)."""
    src = _batch(src, "channel_argmax", dtypes=DTYPE_CODES)
    b, c = src.shape[:2]
    dst = torch.empty((b, 1, *src.shape[2:]), dtype=torch.float32, device=src.device)
    _launch("tio_channel_argmax", src.device, _ptr(src), DTYPE_CODES[src.dtype], b, c, src[0, 0].numel(), _ptr(dst))
    return dst


# ---- resolution changes (spatial/resize.py, spatial/anisotropy.py) ------------------------------

def interpolate(src: Tensor, out_shape, idx: np.ndarray, lam: np.ndarray | None) -> Tensor:
    """(B, C, I, J, K) -> (B, C, *out_shape) of src's dtype: ATen's CUDA trilinear
    (align_corners=True; ``lam`` given) or nearest resize of ``src.float()``, cast back, from the
    per-axis tables of `tables.resize_tables` / `tables.anisotropy_shared_tables`, one pass."""
    src = _batch(src, "interpolate", dtypes=IMAGE_DTYPE_CODES)
    b, c, i, j, k = src.shape
    oi, oj, ok = (int(s) for s in out_shape)
    dst = torch.empty((b, c, oi, oj, ok), dtype=src.dtype, device=src.device)
    if src.numel() and dst.numel():
        idx_d, lam_d = upload(src.device, idx, lam)
        _launch("tio_interpolate", src.device, _ptr(src), _ptr(dst), IMAGE_DTYPE_CODES[src.dtype], b * c, i, j, k,
                oi, oj, ok, _ptr(idx_d), _ptr(lam_d), int(lam is not None))
    return dst


def axis_resample(src: Tensor, axis: np.ndarray, lo: np.ndarray, hi: np.ndarray, w: np.ndarray, *,
                  linear: bool) -> Tensor:
    """Anisotropy's per-instance degradation of a (B, C, I, J, K) batch, one pass: element b is
    resampled along ``axis[b]`` from the (lo, hi, w) rows of `tables.anisotropy_instance_tables`
    (nearest: lo only), or copied when ``axis[b]`` is -1 (anisotropy.py:132-214)."""
    src = _batch(src, "axis_resample", dtypes=IMAGE_DTYPE_CODES)
    b, c, i, j, k = src.shape
    dst = torch.empty_like(src)
    if src.numel():
        if linear:
            axis_d, lo_d, hi_d, w_d = upload(src.device, axis, lo, hi, w)
        else:
            (axis_d, lo_d), hi_d, w_d = upload(src.device, axis, lo), None, None
        _launch("tio_axis_resample", src.device, _ptr(src), _ptr(dst), IMAGE_DTYPE_CODES[src.dtype], b, c, i, j, k,
                _ptr(axis_d), _ptr(lo_d), _ptr(hi_d), _ptr(w_d), int(lo.shape[1]), int(bool(linear)))
    return dst


def interpolate_backward(grad_out: Tensor, in_shape, ptr: np.ndarray, ent: np.ndarray, wt: np.ndarray) -> Tensor:
    """The fp32 (B, C, *in_shape) gradient of `interpolate`'s input for the fp32 (B, C, OI, OJ, OK)
    gradient ``grad_out`` of its output (`tio_interpolate_backward`), from the CSR tables of
    `tables.resize_adjoint_tables` / `tables.anisotropy_shared_adjoint_tables`.  Deterministic: a
    gather in a fixed order, no atomics."""
    grad_out = _batch(grad_out, "interpolate_backward", dtypes=(torch.float32,))
    b, c, oi, oj, ok = grad_out.shape
    i, j, k = (int(s) for s in in_shape)
    grad_in = torch.empty((b, c, i, j, k), dtype=torch.float32, device=grad_out.device)
    if grad_in.numel():
        if not grad_out.numel():
            return grad_in.zero_()
        ptr_d, ent_d, wt_d = upload(grad_out.device, ptr, ent, wt)
        _launch("tio_interpolate_backward", grad_out.device, _ptr(grad_out), _ptr(grad_in), b * c, i, j, k,
                oi, oj, ok, _ptr(ptr_d), _ptr(ent_d), _ptr(wt_d))
    return grad_in


def axis_resample_backward(grad_out: Tensor, axis: np.ndarray, w: np.ndarray, ptr: np.ndarray, ent: np.ndarray, *,
                           linear: bool) -> Tensor:
    """The fp32 gradient of `axis_resample`'s input for the fp32 gradient ``grad_out`` of its output
    (`tio_axis_resample_backward`): ``axis`` and ``w`` as in the forward call, (ptr, ent) from
    `tables.anisotropy_instance_adjoint_tables`.  Deterministic: a gather in a fixed order."""
    grad_out = _batch(grad_out, "axis_resample_backward", dtypes=(torch.float32,))
    b, c, i, j, k = grad_out.shape
    grad_in = torch.empty_like(grad_out)
    if grad_out.numel():
        if linear:
            axis_d, w_d, ptr_d, ent_d = upload(grad_out.device, axis, w, ptr, ent)
        else:
            (axis_d, ptr_d, ent_d), w_d = upload(grad_out.device, axis, ptr, ent), None
        _launch("tio_axis_resample_backward", grad_out.device, _ptr(grad_out), _ptr(grad_in), b, c, i, j, k,
                _ptr(axis_d), _ptr(ptr_d), _ptr(ent_d), _ptr(w_d), int(ptr.shape[1]) - 1, int(bool(linear)))
    return grad_in


# ---- Clamp, Mask, Swap (intensity/clamp.py, mask.py, swap.py) ----------------------------------


def _scalar_bytes(value: Tensor | None):
    """(keep-alive array, host address) of a one-element CPU tensor's bytes, or (None, None)."""
    if value is None:
        return None, None
    raw = value.reshape(1).contiguous().view(torch.uint8).numpy()
    return raw, raw.ctypes.data


def clamp(src: Tensor, lo: Tensor | None, hi: Tensor | None) -> Tensor:
    """``torch.clamp(src, lo, hi)`` in one pass (clamp.py:53-56) into a new tensor of the bounds' dtype:
    ``lo`` / ``hi`` are one-element CPU tensors holding the bounds as torch converts them to the
    result dtype (None: no bound), which is src's dtype or fp32 for an integer image."""
    src = _batch(src, "clamp", dtypes=IMAGE_DTYPE_CODES, ndim=None)
    bound = lo if lo is not None else hi
    if bound is None:
        raise ValueError("clamp: no bound")
    dst = torch.empty(src.shape, dtype=bound.dtype, device=src.device)
    (lo_keep, lo_ptr), (hi_keep, hi_ptr) = _scalar_bytes(lo), _scalar_bytes(hi)
    _launch("tio_clamp", src.device, _ptr(src), _ptr(dst), IMAGE_DTYPE_CODES[src.dtype], IMAGE_DTYPE_CODES[dst.dtype],
            src.numel(), lo_ptr, hi_ptr)
    del lo_keep, hi_keep
    return dst


def mask(data: Tensor, mask: Tensor, keys: np.ndarray | None, outside: Tensor) -> Tensor:
    """``torch.where(mask.expand_as(data), data, outside)`` (mask.py:61-71) for a (B, C, I, J, K) batch
    and the (1 or C, I, J, K) mask of one element (bool or a label dtype): inside = nonzero, or equal
    to one of ``keys`` (`tables.label_lut`'s keys).  ``outside`` is a one-element CPU tensor of the
    result dtype.  Same dtype: ``data`` is updated in place (only outside voxels are written) and
    returned; fp32 (an integer image): a new fp32 tensor."""
    data = _batch(data, "mask", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    mask = _batch(mask.view(torch.uint8) if mask.dtype == torch.bool else mask, "mask", dtypes=DTYPE_CODES, ndim=4)
    if mask.shape[0] not in (1, data.shape[1]) or mask.shape[1:] != data.shape[2:]:
        raise ValueError(f"mask: a {tuple(mask.shape)} mask for a {tuple(data.shape)} batch")
    b, c = data.shape[:2]
    promote = outside.dtype != data.dtype
    dst = torch.empty(data.shape, dtype=outside.dtype, device=data.device) if promote else data
    n = -1 if keys is None else int(keys.shape[0])
    (keys_d,) = upload(data.device, keys) if n > 0 else (None,)
    keep, outside_ptr = _scalar_bytes(outside)
    if data.numel():
        _launch("tio_mask", data.device, _ptr(mask), DTYPE_CODES[mask.dtype], mask.shape[0], _ptr(keys_d), n,
                _ptr(data), IMAGE_DTYPE_CODES[data.dtype], _ptr(dst), IMAGE_DTYPE_CODES[dst.dtype],
                b, c, data[0, 0].numel(), outside_ptr)
    del keep
    return dst


SWAP_EXCHANGE, SWAP_STAGED, SWAP_NOOP = 0, 1, 2


def swap_patches(data: Tensor, swaps: np.ndarray, patch_size) -> None:
    """In place: Swap's ordered patch exchanges (swap.py:195-364) on a contiguous (B, C, I, J, K)
    CUDA batch.  ``swaps``: int32 (1 or B, steps, 8) rows ``ai, aj, ak, bi, bj, bk, kind, 0`` (kind
    SWAP_EXCHANGE for a pair that does not overlap, SWAP_STAGED for one that may, SWAP_NOOP), one
    list for every element or one per element; checked against the volume before any launch."""
    data = _batch(data, "swap_patches", in_place=True)
    swaps = np.ascontiguousarray(swaps, dtype=np.int32)
    lists, steps = swaps.shape[:2]
    if steps == 0 or data.numel() == 0:
        return
    b, c, i, j, k = data.shape
    pi, pj, pk = (int(p) for p in patch_size)
    device_list = torch.empty(swaps.size, dtype=torch.int32, device=data.device)
    stage = None
    if bool((swaps[..., 6] == SWAP_STAGED).any()):
        stage = torch.empty(b * 2 * c * pi * pj * pk * data.element_size(), dtype=torch.uint8, device=data.device)
    _launch("tio_swap_patches", data.device, _ptr(data), data.element_size(), b, c, i, j, k, pi, pj, pk,
            swaps.ctypes.data, lists, steps, _ptr(device_list), _ptr(stage))


# ---- KeepLargestComponent (label/keep_largest.py) -----------------------------------------------

KEEP_KEYS, KEEP_VALUE, KEEP_SEARCH = 0, 1, 2  # tio_components' modes
KEEP_PRESENT, KEEP_NAN, KEEP_INF = 1, 2, 4     # its per-element flags


def _background_key(background_label, dtype: torch.dtype) -> tuple[int, int]:
    """(key, has_key) of ``int(v) != background_label`` for labels=None: has_key 0 when no value of a
    ``dtype`` map can equal the label (outside int64, or not exactly an fp32 value)."""
    if isinstance(background_label, float) and not background_label.is_integer():
        return 0, 0
    key = int(background_label)
    if not -2**63 <= key < 2**63:
        return 0, 0
    if dtype == torch.float32 and int(np.float32(key)) != key:
        return 0, 0
    return key, 1


def keep_largest(data: Tensor, labels, background_label, fully_connected: bool) -> tuple[Tensor, Tensor]:
    """In place on a (B, 1, I, J, K) CUDA label batch: within each element and each label, every
    connected component but the largest (ties: the one whose first voxel in C order comes first) is
    set to ``background_label`` (label/keep_largest.py:63-125).  ``labels``: the labels to filter
    (``data == label`` under torch's scalar rules, `tables.label_lut`), or None for every value with
    ``int(v) != background_label``; ``fully_connected``: 26 neighbours, else 6.

    Returns (data, roots): ``data`` is the input itself when it was contiguous; ``roots`` (B, I, J, K)
    int32, read as uint32, holds for each voxel that takes part the smallest C-order index of its
    component within its element, and -1 elsewhere.  Errors the reference raises (NaN / ±Inf with
    labels=None on fp32 maps, a background label the dtype cannot hold) are raised before anything
    is written, by the first element in batch order that would raise them."""
    if data.ndim != 5:
        raise ValueError(f"keep_largest expects (B, 1, I, J, K), got {tuple(data.shape)}")
    b, c, i, j, k = (int(s) for s in data.shape)
    if c != 1:
        raise ValueError(f"keep_largest expects single-channel label maps, got {c} channels")
    vox = i * j * k
    if vox >= 2**32:
        raise ValueError(f"keep_largest: {vox} voxels per element; component roots are 32-bit (at most 2**32 - 1)")
    if b > 65535:
        raise ValueError(f"keep_largest: {b} elements, at most 65535")
    data = _batch(data, "keep_largest", dtypes=DTYPE_CODES)
    dtype, dev = data.dtype, data.device
    fill, fill_error = None, None
    try:
        _, fill = tables.label_lut([(0, background_label)], dtype, dev)  # what t[mask] = label stores
    except (RuntimeError, ValueError, OverflowError, TypeError) as exc:
        fill_error = exc
    key, has_key = _background_key(background_label, dtype)
    if labels is not None:
        mode = KEEP_KEYS
        keys, _ = tables.label_lut([(label, 0) for label in labels], dtype, dev)
        n = int(keys.shape[0])
        (keys_d,) = upload(dev, keys) if n else (None,)
    else:
        mode = KEEP_VALUE if data.element_size() <= 2 else KEEP_SEARCH
        keys_d, n = None, 0
    roots = torch.empty((b, i, j, k), dtype=torch.int32, device=dev)
    count = torch.empty_like(roots)
    flags = torch.empty(b, dtype=torch.int32, device=dev)
    code = DTYPE_CODES[dtype]
    _launch("tio_components", dev, _ptr(data), code, b, i, j, k, mode, _ptr(keys_d), n, key, has_key,
            int(bool(fully_connected)), _ptr(roots), _ptr(count), _ptr(flags))
    if mode == KEEP_SEARCH and b * vox:
        values = torch.empty(b * vox, dtype=dtype, device=dev)
        n_values = torch.empty(1, dtype=torch.int32, device=dev)
        _launch("tio_component_roots", dev, _ptr(data), code, b, vox, _ptr(roots), _ptr(values), _ptr(n_values))
        found = values[:int(n_values.item())]  # the one read-back: the distinct labels present
        keys_d = torch.unique(found).to(torch.float32 if dtype == torch.float32 else torch.int64).contiguous()
        n = int(keys_d.numel())
        del values
    if (labels is None and dtype == torch.float32) or fill_error is not None:
        for bits in flags.tolist():
            if labels is None and bits & KEEP_INF:
                raise OverflowError("cannot convert float infinity to integer")
            if labels is None and bits & KEEP_NAN:
                raise ValueError("cannot convert float NaN to integer")
            if fill_error is not None and bits & KEEP_PRESENT:
                raise fill_error
    if fill_error is not None or not b * vox or (mode != KEEP_VALUE and n == 0):
        return data, roots  # nothing takes part
    slots = n if mode != KEEP_VALUE else (65536 if data.element_size() == 2 else 256)
    winner = torch.empty(b * slots, dtype=torch.int64, device=dev)
    keep, fill_ptr = _scalar_bytes(torch.from_numpy(np.ascontiguousarray(fill[:1])))
    _launch("tio_keep_largest", dev, _ptr(data), code, b, vox, mode, _ptr(keys_d), n, key, has_key, _ptr(roots),
            _ptr(count), _ptr(winner), fill_ptr)
    del keep
    return data, roots


# ---- Spike (intensity/spike.py) -----------------------------------------------------------------

SPIKE_MAX_AXIS = 4096              # tio_spectrum_peak's longest axis
SPECTRUM_WORKSPACE_BYTES = 512 << 20  # half-spectrum rows are transformed in chunks of about this size


def spike(data: Tensor, spikes: np.ndarray, intensity: np.ndarray) -> Tensor:
    """In place on a contiguous (B, C, I, J, K) CUDA batch of any image dtype: the reference's
    `_add_spikes` (spike.py:124-223) as x + A cos(...) per spike, with A = peak * intensity / (I J K)
    and peak = max |fftn(x.float())| of each (b, c), the sum when no voxel is negative.  ``spikes``:
    int32 (B, S, 4) rows ``u, v, w, 1`` (frequencies) padded with zeros, ``intensity``: fp32 (B,),
    0 for an element that stays untouched.  Stats, spectrum peak and spike pass stay on the device:
    no host sync."""
    data = _batch(data, "spike", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    b, c, i, j, k = (int(s) for s in data.shape)
    if max(i, j, k) > SPIKE_MAX_AXIS:
        raise NotImplementedError(
            f"Spike: spatial shape {(i, j, k)} has an axis longer than {SPIKE_MAX_AXIS} points, the"
            f" longest the spectrum peak supports")
    spikes = np.ascontiguousarray(spikes, dtype=np.int32)
    intensity = np.ascontiguousarray(intensity, dtype=np.float32)
    if spikes.ndim != 3 or spikes.shape[0] != b or spikes.shape[2] != 4 or intensity.shape != (b,):
        raise ValueError(f"spike: tables {spikes.shape} / {intensity.shape} for a batch of {b}")
    if data.numel() == 0 or spikes.shape[1] == 0:
        return data
    s = int(spikes.shape[1])
    spikes_d, intensity_d = upload(data.device, spikes, intensity)
    total, flags = spike_stats(data, intensity_d)
    peak = spectrum_peak(data, intensity_d, flags)
    tables_bytes = b * s * (i + j + k) * 8
    tables = torch.empty(tables_bytes, dtype=torch.uint8, device=data.device)
    _launch("tio_spike", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, i, j, k, _ptr(spikes_d), s,
            _ptr(intensity_d), _ptr(total), _ptr(flags), _ptr(peak), _ptr(tables), tables_bytes)
    return data


def spike_stats(data: Tensor, intensity: Tensor) -> tuple[Tensor, Tensor]:
    """(sum fp64 (B*C,), flags int32 (B*C,)) of `tio_spike_stats` for a contiguous (B, C, ...) CUDA
    batch; ``intensity``: fp32 (B,) on the device, 0 for an inactive element."""
    b, c = int(data.shape[0]), int(data.shape[1])
    total = torch.empty(b * c, dtype=torch.float64, device=data.device)
    flags = torch.empty(b * c, dtype=torch.int32, device=data.device)
    ws_bytes = _native.lib().tio_spike_stats_workspace_bytes(b * c)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=data.device)
    _launch("tio_spike_stats", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, data[0, 0].numel(),
            _ptr(intensity), _ptr(total), _ptr(flags), _ptr(ws), ws_bytes)
    return total, flags


def spectrum_peak(data: Tensor, intensity: Tensor, flags: Tensor, workspace_bytes: int | None = None) -> Tensor:
    """peak fp32 (B*C,) of `tio_spectrum_peak`: max |fftn(x.float())| of the active rows whose flags
    are 1 (signed and finite), 0 elsewhere; ``workspace_bytes`` bounds the half-spectrum chunk."""
    b, c, i, j, k = (int(s) for s in data.shape)
    row_bytes = i * j * (k // 2 + 1) * 8
    if workspace_bytes is None:
        workspace_bytes = min(b * c, max(1, SPECTRUM_WORKSPACE_BYTES // row_bytes)) * row_bytes
    peak = torch.empty(b * c, dtype=torch.float32, device=data.device)
    ws = torch.empty(workspace_bytes, dtype=torch.uint8, device=data.device)
    _launch("tio_spectrum_peak", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, i, j, k,
            _ptr(intensity), _ptr(flags), _ptr(peak), _ptr(ws), workspace_bytes)
    return peak


# ---- Ghosting (intensity/ghosting.py) -----------------------------------------------------------

GHOSTING_MAX_AXIS = 4096  # longest line tio_ghosting's shared-memory FFT holds


def ghosting(data: Tensor, table: np.ndarray, axis: np.ndarray, active: np.ndarray) -> Tensor:
    """In place on a contiguous (B, C, I, J, K) CUDA batch of any image dtype: the reference's
    `_add_ghosting` / `_add_ghosting_per_element` (ghosting.py:149-277) as one filter per line
    along each element's axis, ``ifft(Hs * fft(x))``.  ``table``: fp32 (B, n_max), element b's
    ``ifftshift(line_mask)`` in its first ``shape[axis[b]]`` entries; ``axis``: (B,) in 0..2;
    ``active``: (B,) bool, False for an element that stays untouched.  No host sync."""
    data = _batch(data, "ghosting", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    b, c, i, j, k = (int(s) for s in data.shape)
    table = np.ascontiguousarray(table, dtype=np.float32)
    axis = np.ascontiguousarray(axis, dtype=np.int32)
    active = np.ascontiguousarray(active, dtype=np.uint8)
    if table.ndim != 2 or table.shape[0] != b or axis.shape != (b,) or active.shape != (b,):
        raise ValueError(f"ghosting: tables {table.shape} / {axis.shape} / {active.shape} for a batch of {b}")
    ghosted = sorted({int(a) for a, on in zip(axis, active, strict=True) if on})
    if not ghosted or data.numel() == 0:
        return data
    if ghosted[0] < 0 or ghosted[-1] > 2:
        raise ValueError(f"ghosting: axis {ghosted[0] if ghosted[0] < 0 else ghosted[-1]} outside 0..2")
    longest = max(data.shape[2 + a] for a in ghosted)
    if longest > GHOSTING_MAX_AXIS:
        raise NotImplementedError(
            f"Ghosting: spatial shape {(i, j, k)} is ghosted along an axis longer than {GHOSTING_MAX_AXIS} points,"
            f" the longest the line FFT supports")
    if table.shape[1] < longest:
        raise ValueError(f"ghosting: table rows of {table.shape[1]} entries for an axis of {longest} points")
    table_d, axis_d, active_d = upload(data.device, table, axis, active)
    flags = torch.empty(b * c, dtype=torch.int32, device=data.device)
    _launch("tio_ghosting", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, i, j, k, _ptr(table_d),
            int(table.shape[1]), _ptr(axis_d), _ptr(active_d), sum(1 << a for a in ghosted), _ptr(flags))
    return data


# ---- Motion (intensity/motion.py) ---------------------------------------------------------------

MOTION_MAX_AXIS = 4096  # longest first axis tio_motion's shared-memory FFT holds


def motion(data: Tensor, theta: np.ndarray, active: np.ndarray) -> Tensor:
    """A new (B, C, I, J, K) CUDA tensor of ``data``'s dtype: the reference's `_apply_motion` /
    `_apply_motion_per_instance` (motion.py:140-561) as one k-space splice along the first axis,
    ``ifft_I(sum_s Hs_s * fft_I(x_s))``, with the rigidly resampled copies ``x_s`` gathered on the
    fly.  ``theta``: fp32 (B, N, 12), element b's `_affine_matrices` of segment s at ``[b, s - 1]``;
    ``active``: (B,) bool, False for an element that is copied unchanged.  Returns ``data`` itself
    when no element is active.  No host sync."""
    data = _batch(data, "motion", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    b, c, i, j, k = (int(s) for s in data.shape)
    theta = np.ascontiguousarray(theta, dtype=np.float32)
    active = np.ascontiguousarray(active, dtype=np.uint8)
    if theta.ndim != 3 or theta.shape[0] != b or theta.shape[1] < 1 or theta.shape[2] != 12 or active.shape != (b,):
        raise ValueError(f"motion: tables {theta.shape} / {active.shape} for a batch of {b}")
    if not active.any() or data.numel() == 0:
        return data
    segments = int(theta.shape[1]) + 1
    if i > MOTION_MAX_AXIS:
        raise NotImplementedError(
            f"Motion: spatial shape {(i, j, k)} has a first axis longer than {MOTION_MAX_AXIS} points, the longest"
            f" the line FFT supports")
    if i // segments == 0:
        raise ValueError(f"motion: {segments} segments for a first axis of {i} points")
    theta_d, active_d = upload(data.device, theta, active)
    out = torch.empty_like(data)
    flags = torch.empty(b * c, dtype=torch.int32, device=data.device)
    _launch("tio_motion", data.device, _ptr(data), _ptr(out), IMAGE_DTYPE_CODES[data.dtype], b, c, i, j, k,
            segments, _ptr(theta_d), _ptr(active_d), _ptr(flags))
    return out


# ---- PCA (intensity/pca.py) ---------------------------------------------------------------------

def pca_workspace(data: Tensor, q: int) -> Tensor:
    """Device scratch of `tio_pca_mean` and `tio_pca_gram_apply` for a (B, C, ...) batch and ``q``
    or one column; one workspace serves every pass of a call."""
    b, c = int(data.shape[0]), int(data.shape[1])
    vox = data[0, 0].numel()
    nbytes = max(_native.lib().tio_pca_workspace_bytes(b, c, cols, vox) for cols in (q, 1))
    return torch.empty(nbytes, dtype=torch.uint8, device=data.device)


def pca_mean(data: Tensor, workspace: Tensor) -> Tensor:
    """fp64 (B, C) channel means of float(x) for a contiguous (B, C, I, J, K) CUDA batch of any image
    dtype (pca.py:105), added in a fixed order."""
    data = _batch(data, "pca_mean", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    b, c = int(data.shape[0]), int(data.shape[1])
    mean = torch.empty(b, c, dtype=torch.float64, device=data.device)
    _launch("tio_pca_mean", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, data[0, 0].numel(),
            _ptr(mean), _ptr(workspace), workspace.numel())
    return mean


def pca_gram_apply(data: Tensor, mean: Tensor, w: np.ndarray, workspace: Tensor) -> Tensor:
    """fp64 (B, C, q) products G W of each element, G = A^T A for A = float(x) - mean (voxels x
    channels), from one read of the batch; ``w``: (B, C, q) float64 on the host, uploaded."""
    data = _batch(data, "pca_gram_apply", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    b, c = int(data.shape[0]), int(data.shape[1])
    w = np.ascontiguousarray(w, dtype=np.float64)
    if w.ndim != 3 or w.shape[:2] != (b, c) or w.shape[2] < 1:
        raise ValueError(f"pca_gram_apply: w {w.shape} for a batch of {b} x {c} channels")
    (w_d,) = upload(data.device, w)
    out = torch.empty(w.shape, dtype=torch.float64, device=data.device)
    _launch("tio_pca_gram_apply", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, data[0, 0].numel(),
            int(w.shape[2]), _ptr(mean), _ptr(w_d), _ptr(out), _ptr(workspace), workspace.numel())
    return out


def pca_project(data: Tensor, mean: Tensor, coef: np.ndarray, offset: float, clip: bool) -> Tensor:
    """fp32 (B, q, I, J, K): ``sum_c (float(x_c) - mean_c) coef[b, c, k] + offset`` in fp32, clamped
    to [0, 1] when ``clip`` (pca.py:111-130 with the scales folded into ``coef``: (B, C, q))."""
    data = _batch(data, "pca_project", dtypes=IMAGE_DTYPE_CODES, in_place=True)
    b, c = int(data.shape[0]), int(data.shape[1])
    coef = np.ascontiguousarray(coef, dtype=np.float32)
    if coef.ndim != 3 or coef.shape[:2] != (b, c) or coef.shape[2] < 1:
        raise ValueError(f"pca_project: coef {coef.shape} for a batch of {b} x {c} channels")
    q = int(coef.shape[2])
    (coef_d,) = upload(data.device, coef)
    out = torch.empty((b, q, *data.shape[2:]), dtype=torch.float32, device=data.device)
    _launch("tio_pca_project", data.device, _ptr(data), IMAGE_DTYPE_CODES[data.dtype], b, c, data[0, 0].numel(), q,
            _ptr(mean), _ptr(coef_d), float(offset), int(bool(clip)), _ptr(out))
    return out
