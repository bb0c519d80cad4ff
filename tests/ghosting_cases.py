"""Ghosting test infrastructure: the fixture cases, their seeded inputs, the reference's op sequence
(transforms/intensity/ghosting.py:149-277 of TorchIO 2.0.0a2) restated on torch ops, runnable on CPU
and CUDA tensors, and a float64 numpy oracle of the one-axis filter the kernels compute.
``tests/golden/generate_ghosting.py`` runs the reference's class on these cases; nothing here is
imported by the product."""

from __future__ import annotations

import numpy as np
import torch

from spike_cases import (BF16, DTYPES, F16, F32, F64, GOLDEN, I8, I16, I32, I64, SHORT, U8,  # noqa: F401
                         as_float64, as_stored, load_fixture)

# Inputs: "t1" (ScalarImage, (B, C, *shape) of `dtype`, C = 2 unless the case says otherwise), kind
# "nonneg" (about 40 % zeros, the rest over [0, 400)), "signed" (over [-100, 400)) or "nonfinite"
# (signed, with one NaN in element 0, one +Inf in element 1 and one -Inf in element 2, channel 0
# only); integers rounded, within 0.8 of the dtype's range.  With `seg`, an int16 LabelMap "seg" of
# labels 0..3 that must stay untouched.  With `compose`, the reference's
# Compose([Spike(**spike), Ghosting(**kwargs), BiasField(**bias)]).
SMALL = (10, 12, 9)
CASES_LIST = [
    dict(name="ghosting_warn_default", batch=3, shape=SMALL, dtype=F32, kind="signed", kwargs=dict()),
    dict(name="ghosting_warn_zero_ghosts", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=0, intensity=0.8)),
    dict(name="ghosting_error_negative", batch=1, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=-1, intensity=0.8)),
    dict(name="ghosting_b1_f32", batch=1, channels=1, shape=(37, 29, 23), dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=5, intensity=0.5)),
    dict(name="ghosting_b3_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 10), intensity=(0.5, 1))),
    dict(name="ghosting_b3_many_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=40, intensity=(0.5, 1))),
    dict(name="ghosting_b3_strong_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 6), intensity=1.3)),
    dict(name="ghosting_b3_axis1_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(axes=(1,), intensity=(0.5, 1))),
    dict(name="ghosting_b3_axes02_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(axes=(0, 2), num_ghosts=(2, 8), intensity=(0.5, 1))),
    dict(name="ghosting_b3_restore01_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1), restore=0.1)),
    dict(name="ghosting_b3_restore05_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1), restore=0.5)),
    dict(name="ghosting_b3_restore15_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1), restore=1.5)),
    dict(name="ghosting_b3_shared_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1), per_instance=False)),
    dict(name="ghosting_b3_p05_f32", batch=3, shape=SMALL, dtype=F32, kind="signed",
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1), p=0.5)),
    dict(name="ghosting_b3_len1_f32", batch=3, shape=(1, 8, 13), dtype=F32, kind="signed",
         kwargs=dict(axes=(0, 1), num_ghosts=(2, 5), intensity=(0.5, 1), restore=0.25)),
    dict(name="ghosting_b3_seg_f32", batch=3, shape=SMALL, dtype=F32, kind="signed", seg=True,
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1))),
    dict(name="ghosting_b3_nonfinite_f32", batch=3, shape=SMALL, dtype=F32, kind="nonfinite",
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1))),
    dict(name="ghosting_compose_f32", batch=3, shape=SMALL, dtype=F32, kind="nonneg", compose=True,
         spike=dict(num_spikes=(1, 2), intensity=(1, 2)), bias=dict(std=0.3),
         kwargs=dict(num_ghosts=(2, 8), intensity=(0.5, 1))),
    *[dict(name=f"ghosting_b3_{SHORT[d]}", batch=3, shape=(9, 8, 7), dtype=d,
           kind="nonneg" if d == U8 else "signed", kwargs=dict(num_ghosts=(2, 6), intensity=(0.3, 0.8)))
      for d in DTYPES],
]
CASES = {c["name"]: c for c in CASES_LIST}


def seed(case) -> int:
    return 1300 + sorted(CASES).index(case["name"])


def random_values(rng: np.random.Generator, shape, dtype: torch.dtype, kind: str) -> torch.Tensor:
    n = int(np.prod(shape))
    lo, hi = (0.0 if kind == "nonneg" else -100.0), 400.0
    if not dtype.is_floating_point:
        lo, hi = max(lo, 0.8 * torch.iinfo(dtype).min), min(hi, 0.8 * torch.iinfo(dtype).max)
    x = rng.uniform(lo, hi, n)
    if kind == "nonneg":
        x[rng.random(n) < 0.4] = 0.0
    if not dtype.is_floating_point:
        info = torch.iinfo(dtype)
        x = np.clip(np.round(x), info.min, info.max)
    t = torch.as_tensor(x, dtype=torch.float64).reshape(shape)
    if kind == "nonfinite":
        for b, value in enumerate([float("nan"), float("inf"), float("-inf")][: shape[0]]):
            t[b, 0].view(-1)[b + 3] = value
    return t.to(dtype)


def scalar_image(case) -> torch.Tensor:
    rng = np.random.default_rng(seed(case))
    return random_values(rng, (case["batch"], case.get("channels", 2), *case["shape"]), case["dtype"], case["kind"])


def label_map(case) -> torch.Tensor | None:
    if not case.get("seg"):
        return None
    rng = np.random.default_rng(seed(case) + 1000)
    return torch.as_tensor(rng.integers(0, 4, (case["batch"], 1, *case["shape"])), dtype=torch.int16)


def per_element(params: dict, batch: int) -> tuple[list, list, list]:
    """(num_ghosts, axis, intensity) of every element from recorded params (shared or per instance)."""
    if "_batched_keys" in params:
        return params["num_ghosts"], params["axis"], params["intensity"]
    return [params["num_ghosts"]] * batch, [params["axis"]] * batch, [params["intensity"]] * batch


# ---- the reference's op sequence on torch tensors -----------------------------------------------

def line_mask(n: int, num_ghosts: int, intensity: float, restore: float, device=None) -> torch.Tensor:
    """ghosting.py:190-197: the fp32 mask in fftshift order."""
    mask = torch.ones(n, dtype=torch.float32, device=device)
    step = max(n // num_ghosts, 1)
    mask[::step] = 1 - intensity
    if restore > 0:
        mid = n // 2
        half = max(int(n * restore / 2), 1)
        mask[mid - half: mid + half] = 1
    return mask


def reference_ops(data: torch.Tensor, params: dict) -> torch.Tensor:
    """ghosting.py:149-277 on ``data`` (any device): the shared path returns ``data`` when not active,
    the per-element path keeps inactive elements through ``torch.where``."""
    dims = (-3, -2, -1)
    restore = params["restore"]
    if "_batched_keys" not in params:
        if not params["num_ghosts"] or params["intensity"] == 0:
            return data
        spectrum = torch.fft.fftshift(torch.fft.fftn(data.float(), dim=dims), dim=dims)
        axis = params["axis"]
        n = data.shape[2 + axis]
        mask = torch.ones(n, device=data.device)
        mask[:: max(n // params["num_ghosts"], 1)] = 1 - params["intensity"]
        shape = [1] * 5
        shape[2 + axis] = n
        corrupted = spectrum * mask.view(shape)
        if restore > 0:
            mid, half = n // 2, max(int(n * restore / 2), 1)
            index = [slice(None)] * 5
            index[2 + axis] = slice(mid - half, mid + half)
            corrupted[tuple(index)] = spectrum[tuple(index)]
        return torch.fft.ifftn(torch.fft.ifftshift(corrupted, dim=dims), dim=dims).real.to(data.dtype)
    spectrum = torch.fft.fftshift(torch.fft.fftn(data.float(), dim=dims), dim=dims)
    mask = torch.ones(data.shape[0], 1, *data.shape[2:], dtype=torch.float32, device=data.device)
    active = torch.zeros(data.shape[0], dtype=torch.bool, device=data.device)
    for b, (ghosts, axis, strength) in enumerate(zip(*per_element(params, data.shape[0]), strict=True)):
        if not ghosts or strength == 0:
            continue
        active[b] = True
        shape = [1] * 4
        shape[1 + axis] = data.shape[2 + axis]
        mask[b] = line_mask(data.shape[2 + axis], ghosts, strength, restore, data.device).view(shape)
    out = torch.fft.ifftn(torch.fft.ifftshift(spectrum * mask, dim=dims), dim=dims).real.to(data.dtype)
    return torch.where(active.view(-1, 1, 1, 1, 1), out, data)


# ---- float64 numpy oracle -----------------------------------------------------------------------

def one_axis(x: np.ndarray, params: dict) -> np.ndarray:
    """The identity the kernels compute, in float64, for float64 ``x`` (B, C, I, J, K): each line
    along the element's axis becomes Re(ifft(H fft(x))), H = ifftshift(line_mask) (fp32 values).
    Inactive elements keep x; a (b, c) with a non-finite voxel becomes NaN."""
    out = x.copy()
    for b, (ghosts, axis, strength) in enumerate(zip(*per_element(params, x.shape[0]), strict=True)):
        if not ghosts or strength == 0:
            continue
        n = x.shape[2 + axis]
        h = np.fft.ifftshift(line_mask(n, ghosts, strength, params["restore"]).double().numpy())
        shape = [1] * 4
        shape[1 + axis] = n
        with np.errstate(invalid="ignore"):  # the rows with a NaN or an Inf, overwritten below
            y = np.fft.ifft(h.reshape(shape) * np.fft.fft(x[b], axis=1 + axis), axis=1 + axis).real
        bad = ~np.isfinite(x[b]).all(axis=(1, 2, 3))
        y[bad] = np.nan
        out[b] = y
    return out


def check_against_oracle(got: np.ndarray, x: np.ndarray, params: dict, dtype: torch.dtype, rel: float = 1e-5) -> None:
    """Assert ``got`` (float64 values of an output of ``dtype``) is `one_axis` within the test
    tolerances: floats within rel * max|x| of the (b, c) row plus the output format's rounding;
    integers within 1 where the float64 value lies inside the dtype's range; NaN positions equal."""
    want = one_axis(x, params)
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
    inside = (w > info.min - 1) & (w < info.max + 1)  # the cast of an out-of-range value is not pinned
    assert np.all(np.abs(g[inside] - np.trunc(w[inside])) <= 1), f"max |diff| {np.abs(g - np.trunc(w)).max()}"
