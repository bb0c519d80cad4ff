"""B-spline (orders 2-7) test infrastructure: a float64 restatement of the one ``torch-interpol`` call
the reference makes, the fixture cases and their seeded inputs.

``grid_pull`` restates ``interpol.grid_pull(data, grid, interpolation=order, bound="dct2",
extrapolate=False, prefilter=True)`` (transforms/spatial/spatial.py:1734-1761, 1860-1878 of
TorchIO 2.0.0a2) by its definition: per axis, the coefficients solve the collocation system of the
B-spline of that order with dct2 (half-sample-symmetric, period 2n) folding of the tap indices, and
the output is the spline at the grid, sum_t c[fold(t)] beta^n(x - t).  ``tests/golden/generate_bspline.py``
installs this module as ``interpol`` to run the unmodified reference.  Nothing here is imported by
the product.

Three facts about torch-interpol are assumptions, not read from its source:
  (a) a voxel is in bounds when -0.05 < x < n - 1 + 0.05 on every axis, both bounds strict;
  (b) out-of-bounds voxels are exactly 0, even when the coefficients are not finite;
  (c) the prefilter uses the dct2 bound on all three axes and runs in the input's fp32.
When torch-interpol is installed beside the reference, regenerating the fixtures with it settles them.
"""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"
ORDERS = (2, 3, 4, 5, 6, 7)
NAMES = {2: "quadratic", 3: "cubic", 4: "fourth", 5: "fifth", 6: "sixth", 7: "seventh"}
MARGIN = 0.05


# ---- the restatement ---------------------------------------------------------------------------

def weights(x: np.ndarray, order: int):
    """(P, order+1) float64 weights beta^order(x - t) and the taps t = t0 + j, t0 = floor(x - (order-1)/2),
    by the Cox-de Boor recursion on the fraction g in [0, 1)."""
    shift = 0.5 * (order - 1)
    f = np.floor(x - shift)
    g = x - shift - f
    w = [np.ones_like(g)]
    for k in range(1, order + 1):
        nw = [None] * (k + 1)
        nw[k] = g * w[k - 1] / k
        for j in range(k - 1, 0, -1):
            nw[j] = ((g + (k - j)) * w[j - 1] + ((j + 1) - g) * w[j]) / k
        nw[0] = (1 - g) * w[0] / k
        w = nw
    taps = f.astype(np.int64)[:, None] + np.arange(order + 1)[None, :]
    return np.stack(w, axis=1), taps


def fold(t: np.ndarray, n: int) -> np.ndarray:
    """dct2 reflection of tap indices: period 2n, -1 -> 0, n -> n - 1."""
    t = np.mod(t, 2 * n)
    return np.where(t < n, t, 2 * n - 1 - t)


def collocation(n: int, order: int) -> np.ndarray:
    """(n, n) matrix of the spline at the integer points: A[i, fold(t)] += beta^order(i - t)."""
    w, taps = weights(np.arange(n, dtype=np.float64), order)
    a = np.zeros((n, n))
    for j in range(order + 1):
        np.add.at(a, (np.arange(n), fold(taps[:, j], n)), w[:, j])
    return a


def coefficients(volume: np.ndarray, order: int) -> np.ndarray:
    """Interpolating coefficients of the trailing three axes, in float64 (direct solve per axis)."""
    c = np.asarray(volume, dtype=np.float64)
    for axis in (-3, -2, -1):
        n = c.shape[axis]
        if n > 1:
            c = np.moveaxis(np.linalg.solve(collocation(n, order), np.moveaxis(c, axis, 0).reshape(n, -1))
                            .reshape(np.moveaxis(c, axis, 0).shape), 0, axis)
    return c


def evaluate(coeff: np.ndarray, points: np.ndarray, order: int) -> np.ndarray:
    """Spline of (C, I, J, K) ``coeff`` at (P, 3) voxel ``points`` -> (C, P) float64, 0 outside the margin."""
    shape = coeff.shape[1:]
    points = np.asarray(points, dtype=np.float64)
    inside = np.ones(len(points), dtype=bool)
    for ax in range(3):
        inside &= (points[:, ax] > -MARGIN) & (points[:, ax] < shape[ax] - 1 + MARGIN)
    out = np.zeros((coeff.shape[0], len(points)))
    p = points[inside]
    if len(p) == 0:
        return out
    (wi, ti), (wj, tj), (wk, tk) = (weights(p[:, ax], order) for ax in range(3))
    ti, tj, tk = fold(ti, shape[0]), fold(tj, shape[1]), fold(tk, shape[2])
    acc = np.zeros((coeff.shape[0], len(p)))
    for x in range(order + 1):
        for y in range(order + 1):
            for z in range(order + 1):
                acc += coeff[:, ti[:, x], tj[:, y], tk[:, z]] * (wi[:, x] * wj[:, y] * wk[:, z])
    out[:, inside] = acc
    return out


def _pull64(data: torch.Tensor, grid: torch.Tensor, order: int) -> torch.Tensor:
    """The spline of every (b, c) volume of ``data`` at the voxel ``grid`` ((B|1, OI, OJ, OK, 3)), float64."""
    values = data.detach().cpu().numpy()
    g = grid.detach().cpu().numpy()
    if g.shape[0] != values.shape[0]:
        g = np.broadcast_to(g, (values.shape[0], *g.shape[1:]))
    out = np.empty((*values.shape[:2], *g.shape[1:4]))
    for b in range(values.shape[0]):
        out[b] = evaluate(coefficients(values[b], order), g[b].reshape(-1, 3), order).reshape(
            values.shape[1], *g.shape[1:4])
    return torch.from_numpy(out)


def grid_pull(input, grid, interpolation=1, bound="zero", extrapolate=False, prefilter=False, **kwargs):
    """The reference's call: (B, C, I, J, K) fp32 input, (B, OI, OJ, OK, 3) voxel grid -> fp32 output,
    computed in float64.  Any other argument than the reference passes is refused."""
    if kwargs or bound != "dct2" or extrapolate is not False or prefilter is not True:
        raise NotImplementedError("the restatement covers bound='dct2', extrapolate=False, prefilter=True only")
    order = int(interpolation)
    if order not in ORDERS:
        raise NotImplementedError(f"the restatement covers orders 2-7, got {interpolation}")
    return _pull64(input, grid, order).to(input.dtype)


def reference_pull(data: np.ndarray, points: np.ndarray, order: int) -> np.ndarray:
    """(C, I, J, K) data at (..., 3) points -> (C, ...) float64: the restatement without the fp32 casts."""
    return evaluate(coefficients(data, order), points.reshape(-1, 3), order).reshape(data.shape[0], *points.shape[:-1])


# ---- fixture cases -----------------------------------------------------------------------------

F32, F64, U8, I16, I32, I64 = (torch.float32, torch.float64, torch.uint8, torch.int16, torch.int32, torch.int64)
SHAPE = (14, 12, 10)
AFFINE = dict(scales=(0.9, 1.1), degrees=(-10, 10), translation=(-1, 1))
ELASTIC = dict(num_control_points=5, max_displacement=(2.0, 1.5, 1.0), locked_borders=1)
CASES_LIST = [
    *[dict(name=f"bspline_affine_o{o}", transform="Affine", kwargs=dict(AFFINE, image_interpolation=o))
      for o in ORDERS],
    dict(name="bspline_affine_shared_cubic", transform="Affine",
         kwargs=dict(AFFINE, image_interpolation="cubic", per_instance=False)),
    dict(name="bspline_elastic_fifth", transform="ElasticDeformation",
         kwargs=dict(ELASTIC, image_interpolation="fifth")),
    dict(name="bspline_spatial_affine_last_cubic", transform="Spatial",
         kwargs=dict(AFFINE, **ELASTIC, affine_first=False, image_interpolation="cubic")),
    dict(name="bspline_resample_antialias_quadratic", transform="Resample",
         kwargs=dict(target=(2.0, 1.5, 1.0), antialias=True, image_interpolation="quadratic")),
    dict(name="bspline_gated_seventh", transform="Affine", kwargs=dict(AFFINE, image_interpolation=7, p=0.5)),
    *[dict(name=f"bspline_cubic_{str(d).split('.')[-1]}", transform="Affine", dtype=d,
           kwargs=dict(AFFINE, image_interpolation="cubic")) for d in (U8, I16, I32, I64, F64)],
    dict(name="bspline_label_cubic", transform="Affine", seg=True,
         kwargs=dict(AFFINE, label_interpolation="cubic")),
    dict(name="bspline_label_mode_cubic", transform="Affine", seg=True,
         kwargs=dict(AFFINE, label_interpolation="label", one_hot_label_interpolation="cubic")),
    dict(name="bspline_label_mode_multichannel_cubic", transform="Affine", seg=True, seg_channels=3,
         kwargs=dict(AFFINE, label_interpolation="label", one_hot_label_interpolation="cubic")),
]
CASES = {c["name"]: c for c in CASES_LIST}
BATCH = 3


def seed(case) -> int:
    return 1000 + CASES_LIST.index(case)


def scalar_image(case) -> torch.Tensor:
    """(B, 1, *SHAPE) smooth values plus noise, in the case's dtype (u8 spans 0-255 so cubic overshoots)."""
    g = torch.Generator().manual_seed(seed(case))
    i, j, k = torch.meshgrid(*(torch.arange(n, dtype=torch.float64) for n in SHAPE), indexing="ij")
    smooth = torch.sin(i / 3) * torch.cos(j / 4) + 0.5 * torch.sin(k / 2)
    x = smooth[None, None].repeat(BATCH, 1, 1, 1, 1) + 0.3 * torch.randn(BATCH, 1, *SHAPE, generator=g,
                                                                         dtype=torch.float64)
    dtype = case.get("dtype", F32)
    if dtype == U8:
        blocks = (torch.rand(BATCH, 1, *SHAPE, generator=g) > 0.5).to(torch.float64)
        return (blocks * 255).to(U8)
    if not dtype.is_floating_point:
        return (x * 1000).round().to(dtype)
    return x.to(dtype)


def label_map(case) -> torch.Tensor | None:
    """(B, C, *SHAPE) int16 blobs of labels {0, 1, 3, 7}, or C one-hot-ish float channels."""
    if not case.get("seg"):
        return None
    g = torch.Generator().manual_seed(seed(case) + 1)
    coarse = torch.randint(0, 4, (BATCH, 1, 4, 4, 4), generator=g).double()
    up = torch.nn.functional.interpolate(coarse, size=SHAPE, mode="nearest")
    labels = torch.tensor([0, 1, 3, 7], dtype=torch.int16)[up.long()]
    channels = case.get("seg_channels", 1)
    if channels == 1:
        return labels
    return torch.cat([(labels == v).float() for v in (0, 1, 3)], dim=1)


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"{name}.npz") as z:
        return {k: z[k] for k in z.files}


def dtype_of(record, key: str) -> str:
    return json.loads(bytes(record[f"dtype_{key}"]).decode())


def params_of(record) -> list:
    return json.loads(bytes(record["history"]).decode())


# ---- the reference's op sequence for orders 2-7 ------------------------------------------------

_ORDER_OF = {**{v: k for k, v in NAMES.items()}, "nearest": 0, "linear": 1}


def spatial(images: dict, params: dict, exact: bool = False) -> None:
    """``Spatial.apply_transform`` (spatial.py:560-610, 1110-1272) with the images that use orders 2-7
    sampled through `grid_pull` (spatial.py:1734-1761, 1860-1878) and the others through
    ``oracle.torch_port.spatial``; the geometry is torch_port's (bit-exact with the reference).
    ``images`` as in torch_port, mutated in place.  ``exact``: scalar and label maps of orders 2-7
    keep the float64 spline values instead of the fp32 result cast to their dtype."""
    from oracle import torch_port as tp

    names = params.get("selected_images", [])

    def spline_order(img):
        mode = params["label_interpolation"] if img["kind"] == "label" else params["image_interpolation"]
        if mode == "label":
            mode = params.get("one_hot_label_interpolation", "linear")
        return _ORDER_OF[mode]

    splines = [n for n in names if spline_order(images[n]) >= 2]
    others = [n for n in names if n not in splines]
    if others:
        tp.spatial(images, {**params, "selected_images": others})
    if not splines:
        return
    per_instance = "affine_matrix" in (params.get("_batched_keys") or [])
    first = images[splines[0]]
    shape = tuple(first["data"].shape[-3:])
    a0 = np.asarray(first["affines"][0], dtype=np.float64)
    target = params["target"]
    out_shape = shape if target is None else tuple(int(v) for v in target["shape"])
    a_out = a0 if target is None else np.asarray(target["affine"], dtype=np.float64)
    if per_instance:
        mats, cps = params["affine_matrix"], params["control_points"]
        if target is None and all(m is None for m in mats) and all(c is None for c in cps):
            return
        grid = torch.stack([tp.sampling_grid(shape, a0, out_shape, a_out, mats[b], cps[b], params["affine_first"])
                            for b in range(len(mats))])
        passthrough = [] if target is not None else [
            b for b in range(len(mats)) if mats[b] is None and cps[b] is None]
    else:
        mat, cp = params["affine_matrix"], params["control_points"]
        if target is None and mat is None and cp is None:
            return
        grid = tp.sampling_grid(shape, a0, out_shape, a_out, mat, cp, params["affine_first"])[None]
        passthrough = []
    antialias_on = params.get("antialias", False)
    for name in splines:
        img = images[name]
        data, order = img["data"], spline_order(img)
        if img["kind"] == "label" and params["label_interpolation"] == "label":  # spatial.py:1342-1389
            if data.shape[1] > 1:
                smoothed = data.float()
                if antialias_on:
                    smoothed = tp.antialias(smoothed, a0, a_out)
                sampled = _pull64(smoothed, grid, order).float()
                out = sampled.to(data.dtype) if data.dtype.is_floating_point else sampled
            else:
                labels = torch.unique(data)
                one_hot = (data[:, 0][:, None] == labels.reshape(1, -1, 1, 1, 1)).float()
                if antialias_on:
                    one_hot = tp.antialias(one_hot, a0, a_out)
                sampled = _pull64(one_hot, grid, order).float()
                resampled = labels[sampled.argmax(dim=1)]
                in_bounds = sampled.sum(dim=1) > 0.5
                pad = torch.full_like(resampled, float(params["default_pad_label"]))
                out = torch.where(in_bounds, resampled, pad)[:, None].to(data.dtype)
        else:
            source = data
            if antialias_on and img["kind"] != "label":  # spatial.py:1256-1257
                source = tp.antialias(data, a0, a_out)
            values = _pull64(source.float(), grid, order)
            out = values if exact else values.float().to(source.dtype).to(data.dtype)
        if passthrough:  # spatial.py:1101-1106
            out = out.contiguous()
            for b in passthrough:
                out[b] = data[b]
        img["data"] = out
        img["affines"] = [img["affines"][b] if b in passthrough else a_out.copy()
                          for b in range(len(img["affines"]))]


def fixture_images(case) -> dict:
    """The case's inputs in torch_port's format: identity affines, as the generator's images have."""
    images = {"t1": {"kind": "scalar", "data": scalar_image(case), "affines": [np.eye(4)] * BATCH}}
    seg = label_map(case)
    if seg is not None:
        images["seg"] = {"kind": "label", "data": seg, "affines": [np.eye(4)] * BATCH}
    return images


def replay(case, exact: bool = False) -> dict:
    """The case's recorded history replayed on its inputs with `spatial`."""
    images = fixture_images(case)
    for step in params_of(load_fixture(case["name"])):
        spatial(images, step["params"], exact=exact)
    return images
