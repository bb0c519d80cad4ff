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
import math
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
    taps = f.astype(np.int64)[:, None] + np.arange(order + 1)[None, :]
    return cox_de_boor(x - shift - f, order), taps


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


# ---- float64 references and fp32 error bounds of the two kernels -------------------------------
#
# `prefilter64` runs the prefilter's documented algorithm (bspline.cu: filter_line) in float64 with
# the kernel's fp32 poles, its fp32 gain and its horizon rule, and carries two per-coefficient
# bounds through every pass by a running error analysis, following each recursion with |z|:
#   E  the kernel's fp32 rounding: |c_gpu - c64| <= E;
#   A  the algorithm's distance from the collocation solve: |c64 - coefficients(x)| <= A
#      (truncated initial sums, and the fp32 poles and gain standing in for the exact ones).
# `tap_sums` evaluates the spline at the kernel's own coordinates in float64 and gives the pull's
# bound gamma_m * sum |w_i w_j w_k| |c| (`pull_bound`).

U = 2.0**-24  # fp32 unit roundoff
_SQ = math.sqrt
EXACT_POLES = {
    2: [_SQ(8.0) - 3.0],
    3: [_SQ(3.0) - 2.0],
    4: [_SQ(664.0 - _SQ(438976.0)) + _SQ(304.0) - 19.0, _SQ(664.0 + _SQ(438976.0)) - _SQ(304.0) - 19.0],
    5: [_SQ(135.0 / 2.0 - _SQ(17745.0 / 4.0)) + _SQ(105.0 / 4.0) - 13.0 / 2.0,
        _SQ(135.0 / 2.0 + _SQ(17745.0 / 4.0)) - _SQ(105.0 / 4.0) - 13.0 / 2.0],
    6: [-0.48829458930304475513011803888378906211227916123938,
        -0.081679271076237512597937765737059080653379610398148,
        -0.0014141518083258177510872439765585925278641690553467],
    7: [-0.53528043079643816554240378168164607183392315234269,
        -0.12255461519232669051527226435935734360548654942730,
        -0.0091486948096082769285930216516478534156925639545994],
}


def gamma(m) -> float:
    """Bound on |prod of m factors (1 + d), |d| <= u| - 1|."""
    return m * U / (1 - m * U)


def kernel_poles(order):
    """The kernel's fp32 poles (as floats) and fp32 gain: prod (1 - z)(1 - 1/z) over the fp32 poles in
    double, rounded once (bspline.cu: poles_of)."""
    zs = [float(np.float32(z)) for z in EXACT_POLES[order]]
    g = 1.0
    for z in zs:
        g *= (1.0 - z) * (1.0 - 1.0 / z)
    return zs, float(np.float32(g))


def horizon_quotient(z) -> np.float32:
    """-24 ln 2 / ln|z| in fp32, as the kernel evaluates it before its ceil."""
    return np.float32(np.float32(-24.0) * np.float32(0.69314718)) / np.log(np.float32(abs(z)))


def horizon(z) -> int:
    """Decay horizon h of an fp32 pole: the kernel sums exactly over the dct2 period while n <= h and
    truncates the causal initial sum after h terms otherwise."""
    return int(np.ceil(horizon_quotient(z)))


def inverse_norm(order) -> float:
    """l1 norm of the exact inverse filter prod (1 - z)^2 / ((1 - zS)(1 - z/S)): prod ((1+|z|)/(1-|z|))^2,
    a bound on |A^-1| in the infinity norm for every n under the dct2 extension (2, 3, 4.8, 7.5, 11.8
    and 18.5 for orders 2-7)."""
    return float(np.prod([((1 + abs(z)) / (1 - abs(z))) ** 2 for z in EXACT_POLES[order]]))


def representation_norm(order) -> float:
    """l1 norm of the difference between the B-spline's samples (the filter the collocation solve
    inverts) and the filter the fp32 poles and gain invert exactly,
    (1/g32) prod (-1/z32)(1 - z32 S)(1 - z32/S)."""
    w, taps = weights(np.zeros(1), order)
    exact = dict(zip(taps[0].tolist(), w[0].tolist()))  # row 0 of the system: A[0, t] = beta(0 - t)
    zs, g32 = kernel_poles(order)
    poly = {0: 1.0}
    for z in zs:
        step = {-1: 1.0, 0: -(1.0 + z * z) / z, 1: 1.0}
        new = {}
        for a, va in poly.items():
            for b, vb in step.items():
                new[a + b] = new.get(a + b, 0.0) + va * vb
        poly = new
    keys = set(exact) | set(poly)
    return float(sum(abs(exact.get(k, 0.0) - poly.get(k, 0.0) / g32) for k in keys))


def _rnd(value, prop):
    """Error after one fp32 operation: the propagated error plus u times the computed result's size."""
    return prop + U * (np.abs(value) + prop)


def _pass(s, E, A, order, mirror="dct2"):
    """One prefilter pass over the lines of s (n, L) in float64 with the kernel's operation sequence;
    returns (s, E, A) after it.  The terms, per fp32 operation, each at most u * |result| on top of
    the errors its operands carry:
      gain multiply              s * g
      exact initial sum (n <= h) t = fma(z^n, s[n-1-e], s[e]); acc = fma(z^(e+1), t, acc);
                                 acc / (1 - z^n z^n)  (z^n from powf: 4 ulp = 8u; z^(e+1) after e
                                 products: gamma_e)
      truncated sum (n > h)      acc = fma(z^(e+1), s[e], acc), e < h
      c0 + acc, causal fma       prev = fma(z, prev, s[e])
      z / (z - 1)                two roundings: gamma_2
      anticausal                 prev = z * (prev - s[e]): the subtraction and the product
    A carries the truncated tail |z|^(h+1) / (1 - |z|) max|s| of each truncated initial sum and,
    after the pass, inverse_norm * representation_norm * max|c| per line; both through the same
    recursions.  ``mirror="dct1"`` starts the anticausal recursion as for a whole-sample mirror
    instead: a deliberately wrong spline for the mutation checks."""
    n = s.shape[0]
    zs, gain = kernel_poles(order)
    s = s * gain
    E = _rnd(s, abs(gain) * E)
    A = abs(gain) * A
    for z in zs:
        az, h = abs(z), horizon(z)
        if n <= h:
            zn = z**n
            ezn = 8 * U * abs(zn)
            acc = np.zeros(s.shape[1])
            e_acc, a_acc = np.zeros_like(acc), np.zeros_like(acc)
            zi, ezi = z, 0.0
            for e in range(n):
                lo, hi = s[e], s[n - 1 - e]
                t = zn * hi + lo
                e_t = _rnd(t, abs(zn) * E[n - 1 - e] + ezn * (np.abs(hi) + E[n - 1 - e]) + E[e])
                a_t = abs(zn) * A[n - 1 - e] + A[e]
                acc = zi * t + acc
                e_acc = _rnd(acc, abs(zi) * e_t + ezi * (np.abs(t) + e_t) + e_acc)
                a_acc = abs(zi) * a_t + a_acc
                zi, ezi = zi * z, gamma(e + 1) * abs(zi * z)
            zz = zn * zn
            e_zz = U * zz + 2 * abs(zn) * ezn + ezn**2
            d = 1.0 - zz
            e_d = U * abs(d) + e_zz
            acc = acc / d
            e_acc = _rnd(acc, (e_acc + np.abs(acc) * e_d) / (abs(d) - e_d))
            a_acc = a_acc / abs(d)
        else:
            acc = np.zeros(s.shape[1])
            e_acc, a_acc = np.zeros_like(acc), np.zeros_like(acc)
            zi, ezi = z, 0.0
            for e in range(h):
                acc = zi * s[e] + acc
                e_acc = _rnd(acc, abs(zi) * E[e] + ezi * (np.abs(s[e]) + E[e]) + e_acc)
                a_acc = abs(zi) * A[e] + a_acc
                zi, ezi = zi * z, gamma(e + 1) * abs(zi * z)
            a_acc = a_acc + az ** (h + 1) / (1 - az) * np.max(np.abs(s) + A, axis=0)
        s, E, A = s.copy(), E.copy(), A.copy()
        prev = s[0] + acc
        e_prev = _rnd(prev, E[0] + e_acc)
        a_prev = A[0] + a_acc
        s[0], E[0], A[0] = prev, e_prev, a_prev
        for e in range(1, n):
            prev = z * prev + s[e]
            e_prev = _rnd(prev, az * e_prev + E[e])
            a_prev = az * a_prev + A[e]
            s[e], E[e], A[e] = prev, e_prev, a_prev
        if mirror == "dct1":
            prev = z / (z * z - 1.0) * (prev + z * s[n - 2])
        q = 1.0 if mirror == "dct1" else z / (z - 1.0)
        e_prev = _rnd(prev * q, abs(q) * e_prev + gamma(2) * abs(q) * (np.abs(prev) + e_prev))
        prev, a_prev = prev * q, abs(q) * a_prev
        s[n - 1], E[n - 1], A[n - 1] = prev, e_prev, a_prev
        for e in range(n - 2, -1, -1):
            diff = prev - s[e]
            e_diff = _rnd(diff, e_prev + E[e])
            prev = z * diff
            e_prev = _rnd(prev, az * e_diff)
            a_prev = az * (a_prev + A[e])
            s[e], E[e], A[e] = prev, e_prev, a_prev
    A = A + inverse_norm(order) * representation_norm(order) * np.max(np.abs(s) + A, axis=0)
    return s, E, A


def prefilter64(x, order, E=None, mirror="dct2"):
    """Coefficients of the trailing three axes of ``x`` by the kernel's algorithm in float64, K pass
    first, axes of length 1 skipped: (c, E, A) as described above.  ``E`` seeds the rounding bound
    with an error the input already carries."""
    c = np.array(x, dtype=np.float64)
    E = np.zeros_like(c) if E is None else np.array(E, dtype=np.float64)
    A = np.zeros_like(c)
    for axis in (-1, -2, -3):
        n = c.shape[axis]
        if n < 2:
            continue
        moved = [np.moveaxis(t, axis, 0) for t in (c, E, A)]
        shape = moved[0].shape
        out = _pass(*(t.reshape(n, -1) for t in moved), order, mirror)
        c, E, A = (np.moveaxis(t.reshape(shape), 0, axis) for t in out)
    return c, E, A


def banded_coefficients(lines, order):
    """Coefficients of (n, L) lines by a banded float64 solve of the dct2 collocation system (the
    dense `collocation` solve, for axes too long to hold an n x n matrix)."""
    from scipy.linalg import solve_banded

    n = lines.shape[0]
    if n == 1:
        return np.array(lines, dtype=np.float64)
    w, taps = weights(np.arange(n, dtype=np.float64), order)
    rows = np.repeat(np.arange(n), order + 1)
    cols = fold(taps, n).reshape(-1)
    vals = w.reshape(-1)
    lower, upper = int(max(0, (rows - cols).max())), int(max(0, (cols - rows).max()))
    ab = np.zeros((lower + upper + 1, n))
    np.add.at(ab, (upper + rows - cols, cols), vals)
    return solve_banded((lower, upper), ab, np.asarray(lines, dtype=np.float64))


def coefficients_banded(volume, order):
    """`coefficients` with `banded_coefficients` per axis."""
    c = np.asarray(volume, dtype=np.float64)
    for axis in (-3, -2, -1):
        n = c.shape[axis]
        if n > 1:
            moved = np.moveaxis(c, axis, 0)
            c = np.moveaxis(banded_coefficients(moved.reshape(n, -1), order).reshape(moved.shape), 0, axis)
    return c


def kernel_mask(q, shape):
    """The pull's in-bounds test on fp32 coordinates (P, 3): -0.05f < q < (float)(n - 1) + 0.05f on
    every axis, in fp32; NaN fails it."""
    q = np.asarray(q, dtype=np.float32)
    inside = np.ones(len(q), dtype=bool)
    for ax in range(3):
        hi = np.float32(np.float32(shape[ax] - 1) + np.float32(MARGIN))
        inside &= (q[:, ax] > np.float32(-MARGIN)) & (q[:, ax] < hi)
    return inside


def kernel_fraction(q, order):
    """The pull's first step per axis: f = floor(q - (n-1)/2) and g = (q - (n-1)/2) - f, with
    q - (n-1)/2 rounded to fp32 as the kernel computes it (g is then exact).  The rounding moves the
    spline's argument only where q < (n-1)/2 + 1, by at most 2^-25 * 3.05 voxel."""
    shifted = np.asarray(q, dtype=np.float32) - np.float32(0.5 * (order - 1))
    f = np.floor(shifted)
    return f.astype(np.int64), (shifted - f).astype(np.float64)


def cox_de_boor(g, order):
    """(P, order+1) float64 weights beta^order(g + (order-1)/2 - j) of the fraction g in [0, 1)."""
    w = [np.ones_like(g)]
    for k in range(1, order + 1):
        nw = [None] * (k + 1)
        nw[k] = g * w[k - 1] / k
        for j in range(k - 1, 0, -1):
            nw[j] = ((g + (k - j)) * w[j - 1] + ((j + 1) - g) * w[j]) / k
        nw[0] = (1 - g) * w[0] / k
        w = nw
    return np.stack(w, axis=1)


def pull_terms(order) -> int:
    """Rounded operations m behind each tap of the pull's sum: the Cox-de Boor recursion gives each
    weight at most 5 per step (g + (k-j) or (j+1) - g, the product, the sum of two non-negative
    terms, the fp32 1/k, the product by it; g itself is exact), so 5n per weight and 15n for
    w_i w_j w_k; the three nested fma chains of n+1 terms add at most n+1 each."""
    return 15 * order + 3 * (order + 1)


def tap_sums(q, order, shape, coeff, extra=()):
    """The spline of ``coeff`` (C, I, J, K) at fp32 coordinates q (P, 3) with the kernel's taps and
    fractions, in float64: (value (C, P), sum |w c| (C, P), [sum |w| x for x in extra], inside (P,)).
    Voxels outside the mask are 0 in every sum."""
    q = np.asarray(q, dtype=np.float32).reshape(-1, 3)
    inside = kernel_mask(q, shape)
    C = coeff.shape[0]
    value, absum = np.zeros((C, len(q))), np.zeros((C, len(q)))
    sums = [np.zeros((x.shape[0], len(q))) for x in extra]
    p = q[inside]
    if len(p):
        taps, ws = [], []
        for ax in range(3):
            f, g = kernel_fraction(p[:, ax], order)
            ws.append(cox_de_boor(g, order))
            taps.append(fold(f[:, None] + np.arange(order + 1)[None, :], shape[ax]))
        acc, aacc = np.zeros((C, len(p))), np.zeros((C, len(p)))
        xacc = [np.zeros((x.shape[0], len(p))) for x in extra]
        with np.errstate(invalid="ignore", over="ignore"):
            for x in range(order + 1):
                for y in range(order + 1):
                    wxy = ws[0][:, x] * ws[1][:, y]
                    for z in range(order + 1):
                        w = wxy * ws[2][:, z]
                        idx = (taps[0][:, x], taps[1][:, y], taps[2][:, z])
                        c = coeff[(slice(None), *idx)]
                        acc += w * c
                        aacc += np.abs(w * c)
                        for xa, xs in zip(xacc, extra):
                            xa += np.abs(w) * xs[(slice(None), *idx)]
        value[:, inside], absum[:, inside] = acc, aacc
        for s_, xa in zip(sums, xacc):
            s_[:, inside] = xa
    return value, absum, sums, inside


def pull_bound(absum, order, cmax) -> np.ndarray:
    """|pull_gpu - value| <= gamma_m sum |w c| plus m 2^-149 (n+1)^3 max|c| for weights that underflow
    to subnormals (the kernel keeps them: no flush to zero)."""
    m = pull_terms(order)
    return gamma(m) * absum + m * 2.0**-149 * (order + 1) ** 3 * cmax


def end_to_end(x32, q, order, E_in=None):
    """The spline of `prefilter64`'s coefficients of fp32 ``x32`` (C, I, J, K) at fp32 coordinates
    q (P, 3), in float64, and the bound on the two kernels' fp32 result around it: sum |w| E over the
    taps (the prefilter's rounding carried through the weights) plus the pull's bound on the
    kernel's own coefficients.  The bound holds rounding only: prefilter64's distance from the
    collocation solve (its A, below 1e-7 of the coefficients) is checked on the CPU.  Returns
    (value (C, P), bound (C, P), inside (P,))."""
    shape = x32.shape[1:]
    c64, E, _ = prefilter64(x32, order, E_in)
    value, _, (carried, absum), inside = tap_sums(q, order, shape, c64, extra=(E, np.abs(c64) + E))
    cmax = float(np.max(np.abs(c64) + E, initial=0.0))
    return value, carried + pull_bound(absum, order, cmax), inside


def cast_check(got, value, bound, dtype):
    """The kernel's cast of its fp32 result: floating outputs within the bound (plus half an ulp of
    fp16 / bf16), integers the truncation of the float64 value wrapped to the dtype wherever that lies
    further than the bound from an integer, and within 1 (plus the bound, where it exceeds 1: integers
    above 2^24) elsewhere.  ``got``: floating results as
    float64.  Returns the largest |got - value| / bound (floating), or the share of voxels that lie
    within the bound of an integer (integers)."""
    got = np.asarray(got)
    if dtype in (torch.float16, torch.bfloat16):
        rel, tiny = (2.0**-11, 2.0**-25) if dtype == torch.float16 else (2.0**-8, 2.0**-134)
        bound = bound + rel * (np.abs(value) + bound) + tiny
    if not dtype.is_floating_point:
        bits = torch.iinfo(dtype).bits
        near = np.abs(value - np.round(value)) <= bound
        want = np.trunc(value).astype(np.int64)
        diff = got.astype(np.int64) - want
        if bits < 64:  # the cast wraps through int64 to the dtype
            diff = diff % (1 << bits)
            diff = np.where(diff > (1 << (bits - 1)), diff - (1 << bits), diff)
        assert np.all(diff[~near] == 0), (int((diff[~near] != 0).sum()), value[~near][diff[~near] != 0][:5])
        assert np.all(np.abs(diff[near]) <= np.floor(bound[near]) + 1)
        return float(np.mean(near))
    err = np.abs(got - value)
    assert np.all(err <= bound), (float(np.max(err / bound)), np.unravel_index(np.argmax(err / bound), err.shape))
    return float(np.max(err / bound, initial=0.0))


def step_coords(params, batch, shape):
    """A recorded spatial step's fp32 sampling coordinates (B, OI, OJ, OK, 3) from the C oracle, its
    output shape and its flags (images with identity affines, as the tests' batches have)."""
    from oracle import c_port, torch_port as tp

    a0 = np.eye(4)
    target = params["target"]
    out_shape = shape if target is None else tuple(int(v) for v in target["shape"])
    a_out = None if target is None else np.asarray(target["affine"], dtype=np.float64)
    mat, cp, flags, _ = c_port.spatial_tables(params, batch, shape, a0, a_out)
    q = c_port.sampling_coords(out_shape, mat.numpy(), None if cp is None else cp.numpy(), flags.numpy(),
                               tp.spacing_of(a0), tp.spacing_of(a0 if a_out is None else a_out),
                               affine_first=bool(params["affine_first"])).numpy()
    return q, out_shape, flags.numpy()


def check_end_to_end(data, out, params, order, source=None, source_error=None):
    """``out`` (B, C, ...) of one recorded spline step on ``data`` against `end_to_end` on
    data.float() (or on ``source``, whose values carry at most ``source_error``) with `cast_check`;
    0 outside the mask; passthrough elements bit-identical.  Returns the largest of `cast_check`'s
    results over the elements."""
    from concurrent.futures import ThreadPoolExecutor

    b = data.shape[0]
    q, _, flags = step_coords(params, b, tuple(data.shape[2:]))
    x32 = (data if source is None else source).float().double().numpy()

    def one(e):
        return end_to_end(x32[e], q[e].reshape(-1, 3), order, None if source_error is None else source_error[e])

    work = [e for e in range(b) if not flags[e] & 1]
    with ThreadPoolExecutor(8) as pool:  # numpy releases the GIL in the tap loops
        refs = dict(zip(work, pool.map(one, work)))
    worst = 0.0
    for e in range(b):
        if e not in refs:
            assert torch.equal(out[e].view(torch.uint8), data[e].view(torch.uint8))
            continue
        value, bound, inside = refs[e]
        assert inside.any()
        g = out[e].reshape(out.shape[1], -1)
        assert torch.all(g[:, torch.from_numpy(~inside)] == 0)
        got = g[:, torch.from_numpy(inside)]
        got = got.double().numpy() if out.dtype.is_floating_point else got.numpy()
        worst = max(worst, cast_check(got, value[:, inside], bound[:, inside], out.dtype))
    return worst
