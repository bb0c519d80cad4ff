"""Anisotropy / Resize test infrastructure: the fixture cases, their seeded inputs, and the
reference's op sequences on plain torch ops (transforms/spatial/{anisotropy,resize}.py of TorchIO
2.0.0a2), runnable on CPU and on CUDA tensors.  ``tests/golden/generate_resolution.py`` runs the
reference's classes on these cases; nothing here is imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

GOLDEN = Path(__file__).resolve().parent / "golden"

I8, U8, I16, I32, I64, F32 = torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64, torch.float32

# transform: (class name, kwargs).  Inputs: a label map "seg" of `dtype` (blocks of labels 0..5,
# + 2**24 + 1 on a lattice when `large`) and a scalar image "t1" (fp32, NaN / +-Inf voxels when
# `nonfinite`), `batch` x `channels` x `shape`.
A, R = "Anisotropy", "Resize"
RESOLUTION_CASES = [
    dict(name="aniso_b1_axis0_i16", transform=(A, {"axes": (0,), "downsampling": (1.5, 5)}),
         batch=1, shape=(12, 10, 9), dtype=I16, seed=301),
    dict(name="aniso_b1_axis1_u8", transform=(A, {"axes": (1,), "downsampling": 3.0}),
         batch=1, shape=(9, 13, 8), dtype=U8, seed=302),
    dict(name="aniso_b1_axis2_i32", transform=(A, {"axes": (2,), "downsampling": (2, 4)}),
         batch=1, shape=(8, 9, 14), dtype=I32, seed=303),
    dict(name="aniso_b1_d_equals_l_i8", transform=(A, {"axes": (0,), "downsampling": 1.01}),
         batch=1, shape=(10, 6, 7), dtype=I8, nonfinite=True, seed=304),
    dict(name="aniso_b3_d_equals_l_i8", transform=(A, {"axes": (0,), "downsampling": 1.01}),
         batch=3, shape=(10, 6, 7), dtype=I8, nonfinite=True, seed=305),
    dict(name="aniso_b1_d1_f32", transform=(A, {"axes": (1,), "downsampling": 40.0}),
         batch=1, shape=(6, 9, 7), dtype=F32, seed=306),
    dict(name="aniso_b3_d1_u8", transform=(A, {"axes": (1,), "downsampling": 40.0}),
         batch=3, shape=(6, 9, 7), dtype=U8, seed=307),
    dict(name="aniso_b1_length1_i16", transform=(A, {"axes": (2,), "downsampling": 2.0}),
         batch=1, shape=(7, 8, 1), dtype=I16, seed=308),
    dict(name="aniso_b3_length1_i16", transform=(A, {"axes": (2,), "downsampling": 2.0}),
         batch=3, shape=(7, 8, 1), dtype=I16, seed=309),
    dict(name="aniso_b3_p05_i64", transform=(A, {"downsampling": (1.5, 5), "p": 0.5}),
         batch=3, shape=(11, 10, 12), dtype=I64, seed=310),
    dict(name="aniso_b3_shared_i32", transform=(A, {"downsampling": (2, 3), "per_instance": False}),
         batch=3, shape=(10, 11, 9), dtype=I32, seed=311),
    dict(name="aniso_b3_nearest_image_i16", transform=(A, {"downsampling": (1.5, 5), "image_interpolation": "nearest"}),
         batch=3, shape=(12, 11, 10), dtype=I16, seed=312),
    dict(name="aniso_b1_nearest_image_u8", transform=(A, {"downsampling": (1.5, 5), "image_interpolation": "nearest"}),
         batch=1, shape=(12, 11, 10), dtype=U8, seed=313),
    dict(name="aniso_b3_two_channels_f32", transform=(A, {"downsampling": (1.5, 5)}),
         batch=3, channels=2, shape=(9, 10, 11), dtype=F32, seed=314),
    dict(name="aniso_b1_two_channels_i8", transform=(A, {"downsampling": (1.5, 5)}),
         batch=1, channels=2, shape=(9, 10, 11), dtype=I8, seed=315),
    dict(name="aniso_b3_odd_shape_i16", transform=(A, {"downsampling": (1.5, 5)}),
         batch=3, shape=(37, 29, 23), dtype=I16, seed=316),
    dict(name="aniso_b1_odd_shape_i32", transform=(A, {"downsampling": (1.5, 5)}),
         batch=1, shape=(37, 29, 23), dtype=I32, seed=317),
    dict(name="aniso_b1_nonfinite_i16", transform=(A, {"axes": (1,), "downsampling": 2.5}),
         batch=1, shape=(9, 12, 10), dtype=I16, nonfinite=True, seed=318),
    dict(name="aniso_b3_nonfinite_i16", transform=(A, {"downsampling": (1.5, 5)}),
         batch=3, shape=(9, 12, 10), dtype=I16, nonfinite=True, seed=319),
    dict(name="aniso_b1_large_i64", transform=(A, {"axes": (2,), "downsampling": 3.0}),
         batch=1, shape=(8, 7, 12), dtype=I64, large=True, seed=320),
    dict(name="aniso_b3_large_i64", transform=(A, {"downsampling": (1.5, 5)}),
         batch=3, shape=(8, 7, 12), dtype=I64, large=True, seed=321),
    # L = 26, D = 22: ATen's fp32 nearest map and the per-instance int64 map pick different planes
    dict(name="aniso_b1_maps_differ_u8", transform=(A, {"axes": (0,), "downsampling": 26 / 22}),
         batch=1, shape=(26, 5, 6), dtype=U8, seed=322),
    dict(name="aniso_b3_maps_differ_u8", transform=(A, {"axes": (0,), "downsampling": 26 / 22}),
         batch=3, shape=(26, 5, 6), dtype=U8, seed=323),
    # round(L / f) at a .5 boundary: torch's int / Tensor is a reciprocal multiply (L = 33, f = 4.4:
    # D = 8; true division gives 7) and Python's round(L / f) of the shared path a true division
    dict(name="aniso_b3_round_boundary_f32", transform=(A, {"axes": (0,), "downsampling": 4.4}),
         batch=3, shape=(33, 22, 9), dtype=F32, seed=326),
    dict(name="aniso_b3_round_boundary_axis1_i16", transform=(A, {"axes": (1,), "downsampling": 1.76}),
         batch=3, shape=(33, 22, 9), dtype=I16, seed=327),
    dict(name="aniso_b1_round_boundary_u8", transform=(A, {"axes": (0,), "downsampling": 4.4}),
         batch=1, shape=(33, 22, 9), dtype=U8, seed=328),
    dict(name="aniso_b3_axis_error", transform=(A, {"axes": (3,), "downsampling": 2.0}),
         batch=3, shape=(6, 5, 4), dtype=I16, seed=324),
    dict(name="aniso_constructor_error", transform=(A, {"downsampling": (0.2, 0.5)}),
         batch=1, shape=(6, 5, 4), dtype=I16, seed=325),
    dict(name="resize_up_i16", transform=(R, {"target_shape": (9, 11, 13)}),
         batch=2, shape=(6, 5, 7), dtype=I16, nonfinite=True, seed=340),
    dict(name="resize_down_u8", transform=(R, {"target_shape": (5, 4, 3)}),
         batch=1, shape=(12, 10, 9), dtype=U8, seed=341),
    dict(name="resize_mixed_i32", transform=(R, {"target_shape": (15, 4, 9)}),
         batch=3, channels=2, shape=(10, 8, 9), dtype=I32, seed=342),
    dict(name="resize_same_shape_i64", transform=(R, {"target_shape": (7, 8, 9)}),
         batch=2, shape=(7, 8, 9), dtype=I64, large=True, nonfinite=True, seed=343),
    dict(name="resize_to_one_f32", transform=(R, {"target_shape": (8, 1, 10)}),
         batch=2, shape=(8, 9, 10), dtype=F32, seed=344),
    dict(name="resize_int_target_i8", transform=(R, {"target_shape": 6}),
         batch=1, shape=(9, 7, 8), dtype=I8, seed=345),
    dict(name="resize_label_linear_i16", transform=(R, {"target_shape": (13, 6, 11), "label_interpolation": "linear"}),
         batch=2, shape=(8, 9, 7), dtype=I16, seed=346),
]
RESOLUTION_CASES_BY_NAME = {c["name"]: c for c in RESOLUTION_CASES}


def label_map(case) -> torch.Tensor:
    """(B, C, I, J, K) labels of the case's dtype from its seed: 2-voxel blocks of 0..5."""
    g = torch.Generator().manual_seed(case["seed"] * 7919)
    b, c, shape = case["batch"], case.get("channels", 1), case["shape"]
    coarse = torch.randint(0, 6, (b, c, *(s // 2 + 1 for s in shape)), generator=g)
    data = coarse.repeat_interleave(2, 2).repeat_interleave(2, 3).repeat_interleave(2, 4)
    data = data[:, :, :shape[0], :shape[1], :shape[2]].clone()
    if case.get("large"):
        data[:, :, ::2, ::3] += 2**24 + 1  # not representable in fp32: rounds to 2**24
        data[:, :, 1::2, ::3] += 2**25 + 3
    return data.to(case["dtype"])


def scalar_image(case) -> torch.Tensor:
    g = torch.Generator().manual_seed(case["seed"] * 31)
    data = torch.rand((case["batch"], case.get("channels", 1), *case["shape"]), generator=g) * 100 - 50
    if case.get("nonfinite"):
        flat = data.view(-1)
        n = flat.numel()
        flat[n // 7] = float("nan")
        flat[n // 3] = float("inf")
        flat[n // 2 + 1] = float("-inf")
        flat[(2 * n) // 3] = -0.0
    return data


def affines(case) -> list[np.ndarray]:
    return [np.array([[0.0, -1.2, 0.0, 10.0], [1.0 + 0.25 * b, 0.0, 0.0, -5.0], [0.0, 0.0, 1.5, 2.0],
                      [0.0, 0.0, 0.0, 1.0]]) for b in range(case["batch"])]


def load_fixture(name) -> dict:
    """{"history", "out_seg", "out_t1", "aff_seg", "aff_t1" (B, 4, 4)} or {"history": [], "error":
    {"type", "message"}} (what the reference raised, at construction or when called)."""
    z = np.load(GOLDEN / f"{name}.npz")
    out = {"history": json.loads(bytes(z["history"]).decode())}
    if "error" in z:
        out["error"] = json.loads(bytes(z["error"]).decode())
    for key in ("out_seg", "out_t1"):
        if key in z:
            out[key] = torch.from_numpy(z[key])
    for key in ("aff_seg", "aff_t1"):
        if key in z:
            out[key] = z[key]
    return out


# ---- the reference's op sequences ---------------------------------------------------------------


def anisotropy_shared(data, axis, factor, mode):
    """_simulate_anisotropy (anisotropy.py:353-392): nearest F.interpolate down, then back up."""
    shape = list(data.shape[2:])
    down = list(shape)
    down[axis] = max(1, round(shape[axis] / factor))
    low = F.interpolate(data.float(), size=down, mode="nearest")
    if mode == "nearest":
        return F.interpolate(low, size=shape, mode="nearest").to(data.dtype)
    return F.interpolate(low, size=shape, mode="trilinear", align_corners=True).to(data.dtype)


def _instance_indices(length, down, mode, device):
    """(lower, upper, weight) along the axis for one element (anisotropy.py:219-331)."""
    def to_source(lowres):
        return torch.div(lowres * length, down, rounding_mode="floor").clamp(max=length - 1)

    m = torch.arange(length, device=device)
    if mode == "nearest":
        src = to_source(torch.div(m * down, length, rounding_mode="floor"))
        return src, src, None
    if length == 1:
        pos = torch.zeros(1, dtype=torch.float32, device=device)
    else:
        step = (torch.tensor(down, dtype=torch.float32, device=device) - 1.0) / (length - 1)
        pos = torch.arange(length, dtype=torch.float32, device=device) * step
    lower = pos.floor().long()
    upper = torch.minimum(lower + 1, torch.tensor(down - 1, device=device))
    return to_source(lower), to_source(upper), pos - lower.float()


def _along(rows, axis, like=None):
    """(B', L) rows -> shaped along spatial ``axis`` of a (B', C, I, J, K) tensor (expanded to
    ``like`` for a gather index)."""
    shape = [rows.shape[0], 1, 1, 1, 1]
    shape[axis + 2] = rows.shape[1]
    rows = rows.reshape(shape)
    return rows if like is None else rows.expand_as(like)


def anisotropy_per_instance(data, axes, factors, mode):
    """_simulate_anisotropy_per_instance (anisotropy.py:132-214): clone, then per axis a row mask,
    gathers of the float data, the four elementwise ops, the cast and a masked row assignment."""
    factors_t = torch.tensor(factors, dtype=torch.float64, device=data.device)
    axes_t = torch.tensor(axes, dtype=torch.long, device=data.device)
    active = factors_t > 1.0
    if not bool(active.any()):
        return data
    if bool(((axes_t[active] < 0) | (axes_t[active] > 2)).any()):
        raise ValueError(f"Anisotropy axis must be in {{0, 1, 2}}, got {sorted(set(axes))}")
    out = data.clone()
    for axis in range(3):
        mask = active & (axes_t == axis)
        if not bool(mask.any()):
            continue
        sub = data[mask]
        length = data.shape[axis + 2]
        downs = torch.round(length / factors_t[mask]).clamp_min(1).long().tolist()
        rows = [_instance_indices(length, d, mode, data.device) for d in downs]
        lower = torch.stack([r[0] for r in rows])
        x = sub.float()
        lo = torch.gather(x, axis + 2, _along(lower, axis, x))
        if mode == "nearest":
            out[mask] = lo.to(data.dtype)
            continue
        upper = torch.stack([r[1] for r in rows])
        weight = _along(torch.stack([r[2] for r in rows]), axis)
        hi = torch.gather(x, axis + 2, _along(upper, axis, x))
        out[mask] = (lo * (1.0 - weight) + hi * weight).to(data.dtype)
    return out


def resize(data, target, mode):
    """Resize.apply_transform for one image (resize.py:66-76)."""
    if mode == "nearest":
        return F.interpolate(data.float(), size=list(target), mode="nearest").to(data.dtype)
    return F.interpolate(data.float(), size=list(target), mode="trilinear", align_corners=True).to(data.dtype)


def resize_affine(affine, old_shape, target):
    out = np.array(affine, dtype=np.float64)
    for axis in range(3):
        out[:3, axis] *= old_shape[axis] / target[axis]
    return out


def reference_output(case, images, params):
    """{name: output} of the case's transform on ``images`` ({name: (data, is_label)}) with the
    recorded ``params``."""
    name, kwargs = case["transform"]
    out = {}
    for key, (data, is_label) in images.items():
        if name == "Resize":
            mode = kwargs.get("label_interpolation", "nearest") if is_label else kwargs.get(
                "image_interpolation", "linear")
            out[key] = resize(data, params["target_shape"], mode)
            continue
        mode = "nearest" if is_label else kwargs.get("image_interpolation", "linear")
        if "_batched_keys" in params:
            out[key] = anisotropy_per_instance(data, params["axis"], params["factor"], mode)
        elif params["factor"] > 1.0:
            out[key] = anisotropy_shared(data, params["axis"], params["factor"], mode)
        else:
            out[key] = data
    return out
