"""Spike test infrastructure: the fixture cases, their seeded inputs, the reference's op sequence
(transforms/intensity/spike.py:124-223 of TorchIO 2.0.0a2) restated on torch ops, runnable on CPU
and CUDA tensors, and a float64 numpy oracle of the closed form the kernels use.
``tests/golden/generate_spike.py`` runs the reference's class on these cases; nothing here is
imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

F32, F16, BF16, F64 = torch.float32, torch.float16, torch.bfloat16, torch.float64
U8, I8, I16, I32, I64 = torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64
DTYPES = [F32, F16, BF16, F64, U8, I8, I16, I32, I64]
SHORT = {F32: "f32", F16: "f16", BF16: "bf16", F64: "f64", U8: "u8", I8: "i8", I16: "i16", I32: "i32", I64: "i64"}

# Inputs: "t1" (ScalarImage, (B, C, *shape) of `dtype`), kind "nonneg" (about 40 % zeros, the rest
# over [0, 400)), "signed" (over [-100, 400)) or "nonfinite" (signed, with one NaN in element 0, one
# +Inf in element 1 and one -Inf in element 2, channel 0 only); integers rounded, within 0.8 of the
# dtype's range so that small spikes stay inside it.  With `seg`, an int16 LabelMap "seg" of labels
# 0..3 that must stay untouched.
CASES_LIST = [
    dict(name="spike_b1_f32", batch=1, shape=(7, 6, 5), dtype=F32, kind="nonneg", kwargs=dict(intensity=1.5)),
    dict(name="spike_b3_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed", kwargs=dict(intensity=(1, 3))),
    dict(name="spike_b3_nonneg_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="nonneg",
         kwargs=dict(num_spikes=(1, 4), intensity=(1, 3))),
    dict(name="spike_b3_prime_f32", batch=3, shape=(13, 11, 7), dtype=F32, kind="signed",
         kwargs=dict(num_spikes=3, intensity=2.0)),
    dict(name="spike_b3_len1_f32", batch=3, shape=(1, 8, 13), dtype=F32, kind="signed",
         kwargs=dict(num_spikes=2, intensity=(0.5, 2))),
    dict(name="spike_b3_2d_f32", batch=3, shape=(12, 10, 1), dtype=F32, kind="nonneg",
         kwargs=dict(num_spikes=2, intensity=(1, 3))),
    dict(name="spike_b3_collide_f32", batch=3, shape=(4, 4, 4), dtype=F32, kind="signed",
         kwargs=dict(num_spikes=40, intensity=(1, 3))),
    dict(name="spike_b3_shared_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed",
         kwargs=dict(num_spikes=(1, 3), intensity=(1, 3), per_instance=False)),
    dict(name="spike_b3_p05_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed",
         kwargs=dict(intensity=(1, 3), p=0.5)),
    dict(name="spike_b3_p05_seed_f32", batch=3, shape=(9, 8, 7), dtype=F32, kind="nonneg",
         kwargs=dict(num_spikes=(1, 3), intensity=(1, 3), p=0.5)),
    dict(name="spike_b3_seg_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed", seg=True,
         kwargs=dict(intensity=(1, 3))),
    dict(name="spike_b3_include_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed", seg=True,
         kwargs=dict(intensity=(1, 3), include=["t1"])),
    dict(name="spike_b3_exclude_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed", seg=True,
         kwargs=dict(intensity=(1, 3), exclude=["t1"])),
    dict(name="spike_b3_nonfinite_f32", batch=3, shape=(7, 6, 5), dtype=F32, kind="nonfinite",
         kwargs=dict(intensity=(1, 3))),
    dict(name="spike_b3_u8", batch=3, shape=(9, 8, 7), dtype=U8, kind="nonneg", kwargs=dict(intensity=(0.05, 0.2))),
    dict(name="spike_b3_i16", batch=3, shape=(9, 8, 7), dtype=I16, kind="signed", kwargs=dict(intensity=(0.05, 0.2))),
    dict(name="spike_b3_f16", batch=3, shape=(9, 8, 7), dtype=F16, kind="signed", kwargs=dict(intensity=(1, 3))),
    dict(name="spike_b3_bf16", batch=3, shape=(9, 8, 7), dtype=BF16, kind="nonneg", kwargs=dict(intensity=(1, 3))),
    dict(name="spike_b3_f64", batch=3, shape=(9, 8, 7), dtype=F64, kind="signed", kwargs=dict(intensity=(1, 3))),
    dict(name="spike_warn_default", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed", kwargs=dict()),
    dict(name="spike_warn_zero_spikes", batch=3, shape=(7, 6, 5), dtype=F32, kind="signed",
         kwargs=dict(num_spikes=0, intensity=2.0)),
    dict(name="spike_error_negative", batch=1, shape=(7, 6, 5), dtype=F32, kind="signed",
         kwargs=dict(num_spikes=-1, intensity=2.0)),
]
CASES = {c["name"]: c for c in CASES_LIST}


def seed(case) -> int:
    return 900 + sorted(CASES).index(case["name"])


def random_values(rng: np.random.Generator, shape, dtype: torch.dtype, kind: str) -> torch.Tensor:
    n = int(np.prod(shape))
    lo, hi = (0.0 if kind == "nonneg" else -100.0), 400.0
    if not dtype.is_floating_point:  # room for the spikes inside the dtype's range
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


def per_element(params: dict, batch: int) -> tuple[list, list]:
    """(positions, intensity) of every element from recorded params (shared or per instance)."""
    if "_batched_keys" in params:
        return params["positions"], params["intensity"]
    return [params["positions"]] * batch, [params["intensity"]] * batch


# ---- the reference's op sequence on torch tensors -----------------------------------------------

def reference_ops(data: torch.Tensor, params: dict) -> torch.Tensor:
    """spike.py:124-223 on ``data`` (any device): fftn of data.float() over the spatial axes,
    fftshift, per-(b, c) peak of |spectrum|, ``+= peak * intensity`` at each spike's shifted index,
    ifftshift, ifftn, real part, cast back; elements that are not active keep their values."""
    positions, intensities = per_element(params, data.shape[0])
    active = [bool(p) and v != 0 for p, v in zip(positions, intensities, strict=True)]
    if not any(active):
        return data
    dims = (-3, -2, -1)
    shape = data.shape[2:]
    spectrum = torch.fft.fftshift(torch.fft.fftn(data.float(), dim=dims), dim=dims)
    peak = spectrum.abs().amax(dim=dims)
    for b, (pos_list, value) in enumerate(zip(positions, intensities, strict=True)):
        if not active[b]:
            continue
        for pos in pos_list:
            i, j, k = (int(p * s) % s for p, s in zip(pos, shape, strict=True))
            spectrum[b, :, i, j, k] += peak[b] * value
    out = torch.fft.ifftn(torch.fft.ifftshift(spectrum, dim=dims), dim=dims).real.to(data.dtype)
    keep = torch.as_tensor(active, device=data.device).view(-1, 1, 1, 1, 1)
    return torch.where(keep, out, data)


# ---- float64 numpy oracles ----------------------------------------------------------------------

def frequency(p: float, n: int) -> int:
    return (int(p * n) % n - n // 2) % n


def closed_form(x: np.ndarray, params: dict) -> tuple[np.ndarray, np.ndarray]:
    """(x + A cos(...) in float64, A (B, C)) for float64 ``x`` (B, C, I, J, K): the identity the
    kernels compute, with the peak taken as max |fftn(x)| in float64.  Inactive elements keep x;
    a (b, c) with a non-finite voxel becomes NaN."""
    b_count, c_count, ni, nj, nk = x.shape
    positions, intensities = per_element(params, b_count)
    out = x.copy()
    amp = np.zeros((b_count, c_count))
    ii, jj, kk = np.meshgrid(np.arange(ni), np.arange(nj), np.arange(nk), indexing="ij")
    for b in range(b_count):
        if not positions[b] or intensities[b] == 0:
            continue
        waves = np.zeros((ni, nj, nk))
        for pos in positions[b]:
            u, v, w = (frequency(p, n) for p, n in zip(pos, (ni, nj, nk), strict=True))
            phase = (u * ii % ni) / ni + (v * jj % nj) / nj + (w * kk % nk) / nk
            waves += np.cos(2 * np.pi * phase)
        for c in range(c_count):
            if not np.all(np.isfinite(x[b, c])):
                out[b, c] = np.nan
                continue
            peak = np.abs(np.fft.fftn(x[b, c])).max()
            amp[b, c] = peak * np.float32(intensities[b]) / (ni * nj * nk)
            out[b, c] = x[b, c] + amp[b, c] * waves
    return out, amp


def fft_steps(x: np.ndarray, params: dict) -> np.ndarray:
    """The reference's steps in float64 numpy (fftn, fftshift, peak, +=, ifftshift, ifftn, real)."""
    b_count = x.shape[0]
    positions, intensities = per_element(params, b_count)
    out = x.copy()
    shape = x.shape[2:]
    for b in range(b_count):
        if not positions[b] or intensities[b] == 0:
            continue
        spectrum = np.fft.fftshift(np.fft.fftn(x[b], axes=(-3, -2, -1)), axes=(-3, -2, -1))
        peak = np.abs(spectrum).max(axis=(-3, -2, -1))
        for pos in positions[b]:
            i, j, k = (int(p * s) % s for p, s in zip(pos, shape, strict=True))
            spectrum[:, i, j, k] += peak * np.float32(intensities[b])
        out[b] = np.fft.ifftn(np.fft.ifftshift(spectrum, axes=(-3, -2, -1)), axes=(-3, -2, -1)).real
    return out


def check_against_oracle(got: np.ndarray, x: np.ndarray, params: dict, dtype: torch.dtype, rel: float = 1e-5) -> None:
    """Assert ``got`` (float64 values of an output of ``dtype``) is the closed form within the test
    tolerances: floats within rel * (max|x| + sum|A|) plus the output format's rounding; integers
    within 1, and equal where the float64 value is farther than that tolerance from an integer;
    NaN positions equal."""
    want, amp = closed_form(x, params)
    finite_x = np.where(np.isfinite(x), np.abs(x), 0.0)
    n_spikes = max([len(p) for p in per_element(params, x.shape[0])[0]] + [1])
    scale = finite_x.max(axis=(2, 3, 4), keepdims=True) + n_spikes * np.abs(amp)[..., None, None, None]
    tol = rel * scale
    assert np.array_equal(np.isnan(got), np.isnan(want)), "NaN positions differ"
    ok = ~np.isnan(want)
    g, w, t = got[ok], want[ok], np.broadcast_to(tol, want.shape)[ok]
    if dtype.is_floating_point:
        ulp = {F16: 2.0**-10, BF16: 2.0**-7}.get(dtype, 0.0)
        bad = np.abs(g - w) > t + ulp * np.abs(w)
        assert not bad.any(), f"max |diff| {np.abs(g - w).max()}, tolerance {t.min()}"
        return
    info = torch.iinfo(dtype)
    in_range = (w > info.min - 1) & (w < info.max + 1)  # the cast of an out-of-range value is not pinned
    g, w, t = g[in_range], w[in_range], t[in_range]
    trunc = np.trunc(w)
    assert np.all(np.abs(g - trunc) <= 1), f"max |diff| {np.abs(g - trunc).max()}"
    far = np.abs(w - np.round(w)) > t
    assert np.array_equal(g[far], trunc[far]), f"{int((g[far] != trunc[far]).sum())} values differ"


def as_stored(t: torch.Tensor) -> np.ndarray:
    """A tensor as the fixtures store it (bf16 as its int16 bits)."""
    t = t.detach().cpu().contiguous()
    return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).numpy()


def as_float64(stored: np.ndarray, dtype: torch.dtype) -> np.ndarray:
    t = torch.from_numpy(np.ascontiguousarray(stored))
    return (t.view(torch.bfloat16) if dtype == BF16 else t).double().numpy()


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"{name}.npz") as z:
        out = {k: z[k] for k in z.files}
    for key in ("history", "error", "hydra", "repr", "init_warnings", "warnings", "dtype"):
        if key in out:
            out[key] = json.loads(out[key].tobytes().decode())
    return out
