"""CPU oracle, part 2 (Python side): drive ``oracle/c/tio_oracle.c``.

TEST INFRASTRUCTURE — NOT PRODUCT CODE (see oracle/README.md).

Builds the parameter tables of include/tio_b200.h from the reference's
``params`` dictionaries with its own small numpy/torch code (independent of
``torchio_b200``'s host side, so a table-packing bug in the product cannot
hide behind an identical bug here) and calls the C restatement through ctypes.
"""

from __future__ import annotations

import ctypes
import math
import subprocess
from pathlib import Path

import numpy as np
import torch

from . import torch_port as tp

HERE = Path(__file__).resolve().parent
SRC = HERE / "c" / "tio_oracle.c"
LIB = HERE / "_build" / "libtio_oracle.so"

_DTYPES = {
    torch.float32: 0, torch.uint8: 1, torch.int8: 2,
    torch.int16: 3, torch.int32: 4, torch.int64: 5,
}


def build(force: bool = False) -> Path:
    """Compile the C oracle (gcc, strict fp32: no contraction)."""
    if LIB.exists() and not force and LIB.stat().st_mtime >= SRC.stat().st_mtime:
        return LIB
    LIB.parent.mkdir(exist_ok=True)
    cmd = [
        "gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared",
        "-o", str(LIB), str(SRC), "-lm",
    ]
    subprocess.run(cmd, check=True)
    return LIB


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(str(build()))
    return _lib


def _p(t):
    if t is None:
        return None
    return ctypes.c_void_p(t.data_ptr())


def _f32(x):
    return torch.as_tensor(np.asarray(x, dtype=np.float32)).contiguous()


# ---- spatial ---------------------------------------------------------------


def spatial_tables(params, batch, shape, affine0, a_out=None):
    """(mat[B,12], cp[B,ni,nj,nk,3]|None, flags[B], (ni,nj,nk)) or None if no-op.  ``a_out``: the
    target space's affine (spatial.py:1582-1601); with one, every element is resampled."""
    per_instance = "affine_matrix" in (params.get("_batched_keys") or [])
    if per_instance:
        mats, cps = params["affine_matrix"], params["control_points"]
    else:
        mats = [params["affine_matrix"]] * batch
        cps = [params["control_points"]] * batch
    if a_out is None and all(m is None for m in mats) and all(c is None for c in cps):
        return None
    mat = torch.zeros(batch, 12)
    flags = torch.zeros(batch, dtype=torch.uint8)
    grid_shape = None
    for c in cps:
        if c is not None:
            grid_shape = tuple(np.asarray(c).shape[:3])
    cp = None
    if grid_shape is not None:
        cp = torch.zeros(batch, *grid_shape, 3)
    for b in range(batch):
        m = tp.output_to_input_matrix(affine0, affine0 if a_out is None else a_out, mats[b])
        mat[b] = m[:3].reshape(12)
        if cps[b] is not None:
            cp[b] = torch.as_tensor(cps[b], dtype=torch.float32)
            flags[b] |= 2
        if a_out is None and per_instance and mats[b] is None and cps[b] is None:
            flags[b] |= 1
    return mat, cp, flags, grid_shape or (0, 0, 0)


def spatial(images, params):
    names = params.get("selected_images", [])
    if not names:
        return
    if (params.get("target") is not None or params.get("antialias", False)
            or params.get("label_interpolation") == "label"):
        # resampling onto another grid / the anti-alias pre-filter / partial-volume labels: the
        # torch restatement (F.grid_sample, F.pad + F.conv3d — the reference's own calls) is the oracle
        return tp.spatial(images, params)
    first = images[names[0]]
    shape = tuple(first["data"].shape[-3:])
    a0 = np.asarray(first["affines"][0], dtype=np.float64)
    batch = first["data"].shape[0]
    tables = spatial_tables(params, batch, shape, a0)
    if tables is None:
        return
    mat, cp, flags, (ni, nj, nk) = tables
    sp = _f32(tp.spacing_of(a0))
    for name in names:
        img = images[name]
        data = img["data"].contiguous()
        is_label = img["kind"] == "label"
        mode_name = params["label_interpolation"] if is_label else params["image_interpolation"]
        mode = {"nearest": 0, "linear": 1}[mode_name]
        fill = tp.fill_value_for(
            data, img["kind"], params["default_pad_value"], params["default_pad_label"]
        )
        c = data.shape[1]
        if isinstance(fill, torch.Tensor):
            fill_t = fill.float().contiguous()
        elif float(fill) != 0.0:
            fill_t = torch.full((c,), float(fill))
        else:
            fill_t = None
        out = torch.empty_like(data)
        rc = lib().orc_resample(
            _p(data), _p(out), _DTYPES[data.dtype],
            batch, c, *shape, *shape,
            _p(mat), _p(cp), _p(flags), ni, nj, nk,
            _p(sp), _p(sp), int(bool(params["affine_first"])), mode, _p(fill_t),
        )
        assert rc == 0
        img["data"] = out
        img["affines"] = [
            img["affines"][b] if flags[b] & 1 else a0.copy() for b in range(batch)
        ]


def _geometry_args(mat, cp, flags, spacing_in, spacing_out):
    mat = _f32(mat).reshape(-1, 12).contiguous()
    cp_t = None if cp is None else _f32(cp).contiguous()
    flags_t = None if flags is None else torch.as_tensor(np.asarray(flags, dtype=np.uint8)).contiguous()
    ni, nj, nk = (0, 0, 0) if cp is None else tuple(cp_t.shape[1:4])
    return mat, cp_t, flags_t, (ni, nj, nk), _f32(spacing_in), _f32(spacing_out)


def resample(src, out_shape, mat, cp, flags, spacing_in, spacing_out, *, affine_first, mode, fill):
    """orc_resample of fp32 ``src`` (B, C, I, J, K) onto ``out_shape``, with the packed tables of
    include/tio_b200.h as host arrays: mat (B, 12), cp (B, ni, nj, nk, 3) or None, flags (B,) or
    None; mode 0 nearest, 1 linear; fill (C,) or None (no mask step)."""
    src = src.float().contiguous()
    b, c = src.shape[:2]
    out = torch.empty((b, c, *out_shape), dtype=torch.float32)
    mat, cp_t, flags_t, grid, sp_in, sp_out = _geometry_args(mat, cp, flags, spacing_in, spacing_out)
    fill_t = None if fill is None else _f32(fill).reshape(-1).contiguous()
    rc = lib().orc_resample(_p(src), _p(out), 0, b, c, *src.shape[2:], *out_shape, _p(mat), _p(cp_t),
                            _p(flags_t), *grid, _p(sp_in), _p(sp_out), int(bool(affine_first)), int(mode),
                            _p(fill_t))
    assert rc == 0
    return out


def sampling_coords(out_shape, mat, cp, flags, spacing_in, spacing_out, *, affine_first):
    """orc_sampling_coords: the fp32 input-voxel coordinates (B, OI, OJ, OK, 3) at which `resample`
    (and the B-spline pull, through the same chain) samples every output voxel, with the geometry
    arguments of `resample`.  Pass-through elements get their own voxel indices."""
    mat, cp_t, flags_t, grid, sp_in, sp_out = _geometry_args(mat, cp, flags, spacing_in, spacing_out)
    b = mat.shape[0]
    q = torch.empty((b, *(int(v) for v in out_shape), 3), dtype=torch.float32)
    rc = lib().orc_sampling_coords(_p(q), b, *q.shape[1:4], _p(mat), _p(cp_t), _p(flags_t), *grid, _p(sp_in),
                                   _p(sp_out), int(bool(affine_first)))
    assert rc == 0
    return q


def resample_adjoint(grad_out, in_shape, mat, cp, flags, spacing_in, spacing_out, *, affine_first, mode,
                     fill):
    """orc_resample_adjoint: (grad64, abs64, count), each (B, C, *in_shape), for the fp32
    ``grad_out`` (B, C, OI, OJ, OK) of `resample` with the same geometry.  grad64 = sum of g * w
    in float64 over the output voxels reading an input voxel, abs64 = sum of |g * w|, count =
    the number of terms.  Only whether ``fill`` is None matters."""
    grad_out = torch.as_tensor(grad_out).float().contiguous()
    b, c = grad_out.shape[:2]
    shape = (b, c, *(int(v) for v in in_shape))
    grad64 = torch.empty(shape, dtype=torch.float64)
    abs64 = torch.empty(shape, dtype=torch.float64)
    count = torch.empty(shape, dtype=torch.int32)
    mat, cp_t, flags_t, grid, sp_in, sp_out = _geometry_args(mat, cp, flags, spacing_in, spacing_out)
    fill_t = None if fill is None else _f32(fill).reshape(-1).contiguous()
    rc = lib().orc_resample_adjoint(_p(grad_out), _p(grad64), _p(abs64), _p(count), b, c, *shape[2:],
                                    *grad_out.shape[2:], _p(mat), _p(cp_t), _p(flags_t), *grid, _p(sp_in),
                                    _p(sp_out), int(bool(affine_first)), int(mode), _p(fill_t))
    assert rc == 0, "orc_resample_adjoint: a pass-through element needs equal input and output shapes"
    return grad64, abs64, count


# ---- intensity ---------------------------------------------------------------


def bias_field(images, params, divide=False):
    std, seed, scale = params["std"], params["seed"], params["scale"]
    per_instance = "_batched_keys" in params
    if not per_instance and std == 0:
        return
    for img in images.values():
        if img["kind"] != "scalar":
            continue
        data = img["data"].contiguous()
        b, c = data.shape[:2]
        if per_instance and all(s == 0 for s in std):
            continue
        coarse = tp.coarse_bias_fields(data.shape, std, seed, scale).contiguous()
        ident = (
            torch.tensor([s == 0 for s in std], dtype=torch.uint8)
            if per_instance else None
        )
        out = torch.empty_like(data)
        rc = lib().orc_bias_field(
            _p(data), _p(out), b, c, *data.shape[2:], _p(coarse), *coarse.shape[2:],
            _p(ident), int(divide),
        )
        assert rc == 0
        img["data"] = out


def blur_tables(sigmas_vox, batch):
    """taps[3][B][2R+1], radius[3][B], R, identity[B] — or None when no-op."""
    sig = np.asarray(sigmas_vox, dtype=np.float64)
    if np.all(sig <= 0):
        return None
    if sig.ndim == 2 and np.all(sig == sig[0]):
        sig = sig[0]
    radius = torch.zeros(3, batch, dtype=torch.int32)
    rows = []
    if sig.ndim == 1:
        for axis in range(3):
            s = float(sig[axis])
            if s <= 0:
                rows.append(None)
                continue
            taps, r = tp.gaussian_taps_shared(s)
            radius[axis, :] = r
            rows.append(taps[None].expand(batch, -1))
        identity = torch.zeros(batch, dtype=torch.uint8)
    else:
        for axis in range(3):
            col = sig[:, axis]
            if np.all(col <= 0):
                rows.append(None)
                continue
            taps, _ = tp.gaussian_taps_stacked(col)
            pos = col > 0
            r = np.zeros(batch, dtype=np.int64)
            r[pos] = np.maximum(np.ceil(3 * col[pos]).astype(np.int64), 1)
            radius[axis] = torch.as_tensor(r, dtype=torch.int32)
            rows.append(taps)
        identity = torch.as_tensor(np.all(sig <= 0, axis=1)).to(torch.uint8)
    big_r = max((t.shape[1] - 1) // 2 for t in rows if t is not None)
    table = torch.zeros(3, batch, 2 * big_r + 1)
    for axis, t in enumerate(rows):
        if t is None:
            continue
        r = (t.shape[1] - 1) // 2
        table[axis, :, big_r - r: big_r + r + 1] = t
    return table.contiguous(), radius.contiguous(), big_r, identity


def blur(images, params):
    per_instance = "_batched_keys" in params
    for img in images.values():
        if img["kind"] != "scalar":
            continue
        data = img["data"].contiguous()
        b, c = data.shape[:2]
        if per_instance:
            mm = np.asarray(params["std"], dtype=np.float64)
            sp = np.asarray([tp.spacing_of(a) for a in img["affines"]], dtype=np.float64)
            vox = np.divide(mm, sp, out=np.zeros_like(mm), where=sp > 0)
        else:
            sp = np.asarray(tp.spacing_of(img["affines"][0]), dtype=np.float64)
            vox = [s / q if q > 0 else 0.0 for s, q in zip(params["std"], sp)]
        tables = blur_tables(vox, b)
        if tables is None:
            continue
        taps, radius, big_r, identity = tables
        out = torch.empty_like(data)
        rc = lib().orc_blur(
            _p(data), _p(out), None, b, c, *data.shape[2:], _p(taps), _p(radius),
            big_r, _p(identity),
        )
        assert rc == 0
        img["data"] = out


def randn_mt19937(seed: int, skip: int, n: int):
    """(z[n], words consumed): the C restatement of torch's CPU randn stream."""
    z = torch.empty(n)
    used = ctypes.c_uint64(0)
    rc = lib().orc_randn_mt19937(
        ctypes.c_uint64(seed), ctypes.c_uint64(skip), ctypes.c_uint64(n), _p(z),
        ctypes.byref(used),
    )
    assert rc == 0
    return z, used.value


def _vec(value, batch):
    if isinstance(value, list):
        return _f32(value)
    return torch.full((batch,), float(value))


def noise(images, params, use_c_rng=True):
    keep = params.get("_keep")
    skip = 0
    gen = torch.Generator(device="cpu")
    gen.manual_seed(params["seed"])
    for img in images.values():
        if img["kind"] != "scalar":
            continue
        data = img["data"].contiguous()
        b = data.shape[0]
        per = data[0].numel()
        n = data.numel()
        draws = []
        for _ in range(2 if params.get("rician", False) else 1):
            if use_c_rng and n >= 16:
                z, used = randn_mt19937(params["seed"], skip, n)
                skip += used
            else:
                z = torch.randn(data.shape, generator=gen).reshape(-1)
            draws.append(z.contiguous())
        keep_t = torch.tensor(keep, dtype=torch.uint8) if keep is not None else None
        mean, std = _vec(params["mean"], b), _vec(params["std"], b)
        out = torch.empty_like(data)
        rc = lib().orc_noise(
            _p(data), _p(out), b, ctypes.c_int64(per), _p(mean), _p(std), _p(keep_t),
            _p(draws[0]), _p(draws[1]) if len(draws) > 1 else None,
        )
        assert rc == 0
        img["data"] = out


def gamma(images, params, invert=False):
    lg = params["log_gamma"]
    if invert:
        lg = [-v for v in lg] if isinstance(lg, list) else -lg
    for img in images.values():
        if img["kind"] != "scalar":
            continue
        data = img["data"].contiguous()
        b = data.shape[0]
        if isinstance(lg, list):
            gam = torch.exp(torch.tensor(lg, dtype=torch.float32))
        else:
            gam = torch.full((b,), math.exp(lg))
        out = torch.empty_like(data)
        rc = lib().orc_gamma(
            _p(data), _p(out), b, ctypes.c_int64(data[0].numel()), _p(gam.contiguous())
        )
        assert rc == 0
        img["data"] = out


# ---- widened rows: Flip / Crop / Pad through orc_remap, patches through orc_crop_patches --

_PAD_MODES = {"constant": 0, "replicate": 1, "reflect": 2, "circular": 3}


def remap(data, out_shape, offsets, mode="constant", fill=0, flip_bits=None):
    data = data.contiguous()
    b, c, i, j, k = data.shape
    out = torch.empty((b, c, *out_shape), dtype=data.dtype)
    fill_t = torch.tensor([fill]).to(data.dtype)  # F.pad casts the value to the tensor's dtype
    flip_t = None if flip_bits is None else torch.as_tensor(np.asarray(flip_bits, dtype=np.uint8))
    rc = lib().orc_remap(_p(data), _p(out), data.element_size(), b, c, i, j, k, *[int(v) for v in out_shape],
                         int(offsets[0]), int(offsets[1]), int(offsets[2]), _PAD_MODES[mode], _p(fill_t),
                         _p(flip_t))
    assert rc == 0
    return out


def _shift_origin(img, voxels):
    shift = np.asarray(voxels, dtype=np.float64)
    for a in img["affines"]:
        a[:3, 3] += a[:3, :3] @ shift


def flip(images, params):
    axes = params["axes"]
    for img in images.values():
        b = img["data"].shape[0]
        per = axes if "_batched_keys" in params else [axes] * b
        bits = [sum(1 << int(a) for a in set(ax)) for ax in per]
        if any(bits):
            img["data"] = remap(img["data"], img["data"].shape[2:], (0, 0, 0), flip_bits=bits)


def crop(images, params):
    i0, i1, j0, j1, k0, k1 = params["cropping"]
    for img in images.values():
        si, sj, sk = img["data"].shape[-3:]
        img["data"] = remap(img["data"], (si - i0 - i1, sj - j0 - j1, sk - k0 - k1), (-i0, -j0, -k0))
        _shift_origin(img, (i0, j0, k0))


def pad(images, params):
    if params["padding_mode"] in ("mean", "median", "minimum"):
        return tp.pad(images, params)  # per-element statistic: the torch restatement is the oracle
    i0, i1, j0, j1, k0, k1 = params["padding"]
    for img in images.values():
        si, sj, sk = img["data"].shape[-3:]
        img["data"] = remap(img["data"], (si + i0 + i1, sj + j0 + j1, sk + k0 + k1), (i0, j0, k0),
                            mode=params["padding_mode"], fill=params["fill"])
        _shift_origin(img, (-i0, -j0, -k0))


def crop_patches(volume, corners, size):
    volume = volume.contiguous()
    c, i, j, k = volume.shape
    corners_t = torch.as_tensor(np.asarray(corners, dtype=np.int32).reshape(-1, 3)).contiguous()
    out = torch.empty((corners_t.shape[0], c, *size), dtype=volume.dtype)
    rc = lib().orc_crop_patches(_p(volume), _p(out), volume.element_size(), c, i, j, k, corners_t.shape[0],
                                _p(corners_t), *[int(v) for v in size])
    assert rc == 0
    return out


_APPLY = {
    "Spatial": spatial,
    "Resample": spatial, "Affine": spatial, "ElasticDeformation": spatial,
    "BiasField": bias_field, "Blur": blur, "Noise": noise, "Gamma": gamma,
    "Flip": flip, "Crop": crop, "Pad": pad,
    # elementwise fp32 maps with recorded constants: the torch restatement is the oracle
    "Standardize": tp.standardize, "Normalize": tp.normalize,
}


def replay(images, history):
    for step in history:
        _APPLY[step["name"]](images, step["params"])
    return images
