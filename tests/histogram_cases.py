"""HistogramStandardization test infrastructure: the fixture cases, their seeded inputs, and the
reference's op sequence (transforms/intensity/histogram_standardization.py:216-303 of TorchIO
2.0.0a2) restated with np.percentile plus plain torch ops, runnable on CPU and on CUDA tensors.
``tests/golden/generate_histogram.py`` runs the reference's classes on these cases; nothing here is
imported by the product."""

from __future__ import annotations

import json
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

F32, F16, BF16, F64 = torch.float32, torch.float16, torch.bfloat16, torch.float64
U8, I8, I16, I32, I64 = torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64

DEFAULT_QUANTILES = (0.01, 0.10, 0.20, 0.25, 0.30, 0.40, 0.50, 0.60, 0.70, 0.75, 0.80, 0.90, 0.99)
EPS_F32 = float(np.float32(1e-5))

# input kinds ("t1", a ScalarImage, plus an untouched LabelMap "seg"):
#   background  60 % exact zeros, the rest spread over about [-100, 400] (integers for integer dtypes)
#   constant    every voxel 7
#   eps         22 % zeros, 22 % fp32(1e-5), the rest spread: two landmarks exactly fp32(1e-5) apart
#   nonfinite   background with a NaN voxel in element 0 and +-inf voxels in the others
# landmarks: "ramp" = linspace(0, 100, n); "negative" starts at -40 (uint8 wraps below the 1 % landmark)
HIST_CASES = [
    dict(name="histstd_b1_c1_f32", batch=1, channels=1, shape=(9, 8, 7), dtype=F32, kind="background", seed=401),
    dict(name="histstd_b3_c2_f32", batch=3, channels=2, shape=(9, 8, 7), dtype=F32, kind="background", seed=402),
    dict(name="histstd_b3_c1_f16", batch=3, channels=1, shape=(9, 8, 7), dtype=F16, kind="background", seed=403),
    dict(name="histstd_b1_c2_bf16", batch=1, channels=2, shape=(9, 8, 7), dtype=BF16, kind="background", seed=404),
    dict(name="histstd_b3_c1_f64", batch=3, channels=1, shape=(9, 8, 7), dtype=F64, kind="background", seed=405),
    dict(name="histstd_b3_c2_i16", batch=3, channels=2, shape=(9, 8, 7), dtype=I16, kind="background", seed=406),
    dict(name="histstd_b1_c1_u8_negative", batch=1, channels=1, shape=(9, 8, 7), dtype=U8, kind="background",
         landmarks="negative", seed=407),
    dict(name="histstd_b3_c1_u8_negative", batch=3, channels=1, shape=(9, 8, 7), dtype=U8, kind="background",
         landmarks="negative", seed=408),
    dict(name="histstd_b1_c1_f32_constant", batch=1, channels=1, shape=(6, 5, 4), dtype=F32, kind="constant", seed=409),
    dict(name="histstd_b3_c1_f32_eps", batch=3, channels=1, shape=(10, 9, 8), dtype=F32, kind="eps", seed=410),
    dict(name="histstd_b3_c1_f32_nonfinite", batch=3, channels=1, shape=(9, 8, 7), dtype=F32, kind="nonfinite",
         seed=411),
    dict(name="histstd_b1_c1_f32_n1", batch=1, channels=1, shape=(1, 1, 1), dtype=F32, kind="background", seed=412),
    dict(name="histstd_b3_c1_i16_odd", batch=3, channels=1, shape=(7, 5, 3), dtype=I16, kind="background", seed=413),
    dict(name="histstd_b3_c2_f32_odd", batch=3, channels=2, shape=(5, 3, 3), dtype=F32, kind="background", seed=414),
    dict(name="histstd_b3_c1_f32_cutoff", batch=3, channels=1, shape=(9, 8, 7), dtype=F32, kind="background",
         cutoff=(0.05, 0.95), seed=415),
    dict(name="histstd_b1_c1_f32_p0", batch=1, channels=1, shape=(6, 5, 4), dtype=F32, kind="background",
         kwargs={"p": 0.0}, seed=416),
    dict(name="histstd_b3_c1_f32_exclude", batch=3, channels=1, shape=(6, 5, 4), dtype=F32, kind="background",
         kwargs={"exclude": ["t1"]}, seed=417),
    dict(name="histstd_b3_c1_f32_include", batch=3, channels=1, shape=(6, 5, 4), dtype=F32, kind="background",
         kwargs={"include": ["t1"]}, seed=418),
    dict(name="histstd_b1_c1_f32_mismatch", batch=1, channels=1, shape=(6, 5, 4), dtype=F32, kind="background",
         landmark_count=15, seed=419),
]

# compute_histogram_landmarks: images of `dtype` from seeds, masking_method "positive" = x > 0
LANDMARK_CASES = [
    dict(name="histlm_unmasked_f32", dtype=F32, count=4, seed=431),
    dict(name="histlm_masked_f32", dtype=F32, count=4, masked=True, seed=432),
    dict(name="histlm_quantiles_f32", dtype=F32, count=3, quantiles=(0.01, 0.05, 0.5, 0.95, 0.99), seed=433),
    dict(name="histlm_unmasked_i16", dtype=I16, count=3, seed=434),
    dict(name="histlm_masked_u8", dtype=U8, count=3, masked=True, seed=435),
    dict(name="histlm_unmasked_f16", dtype=F16, count=3, seed=436),
    dict(name="histlm_cutoff_i8", dtype=I8, count=3, cutoff=(0.05, 0.95), seed=437),
    dict(name="histlm_error_few", dtype=F32, count=1, quantiles=(0.5,), cutoff=(0.5, 0.5), seed=438),
    dict(name="histlm_error_range", dtype=F32, count=1, quantiles=(0.01, 0.99, 1.5), seed=439),
    dict(name="histlm_error_cutoff", dtype=F32, count=1, quantiles=(0.1, 0.5, 0.9), seed=440),
]


def quantiles_for(cutoff) -> tuple[float, ...]:
    return tuple(sorted({*DEFAULT_QUANTILES, cutoff[0], cutoff[1]}))


def case_cutoff(case) -> tuple[float, float]:
    return tuple(case.get("cutoff", (0.01, 0.99)))


def landmarks(case) -> torch.Tensor:
    n = case.get("landmark_count", len(quantiles_for(case_cutoff(case))))
    start = -40.0 if case.get("landmarks") == "negative" else 0.0
    return torch.linspace(start, 100.0, n)


def _values(rng: np.random.Generator, n: int, kind: str, integer: bool) -> np.ndarray:
    if kind == "constant":
        return np.full(n, 7.0)
    x = rng.uniform(-100.0, 400.0, n)
    if integer:
        x = np.round(x)
    if kind == "eps":
        order = rng.permutation(n)
        x[order[: int(0.22 * n)]] = 0.0
        x[order[int(0.22 * n): int(0.44 * n)]] = EPS_F32
        return x
    x[rng.random(n) < 0.6] = 0.0
    return x


def scalar_image(case) -> torch.Tensor:
    """(B, C, I, J, K) of the case's dtype."""
    rng = np.random.default_rng(case["seed"])
    b, c, shape = case["batch"], case.get("channels", 1), case["shape"]
    dtype = case["dtype"]
    integer = not dtype.is_floating_point
    n = c * int(np.prod(shape))
    x = np.stack([_values(rng, n, case["kind"], integer) for _ in range(b)]).reshape(b, c, *shape)
    if dtype == U8:
        x = np.clip(x, 0, 255)
    elif dtype == I8:
        x = np.clip(x, -128, 127)
    t = torch.as_tensor(x, dtype=torch.float64)
    if case["kind"] == "nonfinite":
        flat = t.view(b, -1)
        flat[0, 3] = float("nan")
        for e in range(1, b):
            flat[e, 5], flat[e, 11] = float("inf"), float("-inf")
    return t.to(dtype)


def label_map(case) -> torch.Tensor:
    b, shape = case["batch"], case["shape"]
    return (torch.arange(b * int(np.prod(shape))).reshape(b, 1, *shape) % 3).to(torch.int16)


def training_images(case) -> list[torch.Tensor]:
    rng = np.random.default_rng(case["seed"])
    dtype = case["dtype"]
    out = []
    for i in range(case["count"]):
        shape = (1, 6 + i, 5, 4 + i)
        x = _values(rng, int(np.prod(shape)), "background", not dtype.is_floating_point) * (1 + 0.2 * i)
        if dtype == U8:
            x = np.clip(x, 0, 255)
        elif dtype == I8:
            x = np.clip(x, -128, 127)
        out.append(torch.as_tensor(x.reshape(shape)).to(dtype))
    return out


def positive_mask(tensor: torch.Tensor) -> torch.Tensor:
    return tensor > 0


# ---- the reference's op sequence --------------------------------------------------------------

def element_tables(element: torch.Tensor, lm: torch.Tensor, cutoff):
    """(input landmarks, slopes, intercepts, edges) of one (C, I, J, K) element, computed like
    _apply_histogram_standardization: np.percentile on the host, the rest as torch ops on
    element's device."""
    quantiles = quantiles_for(cutoff)
    percentiles = [100.0 * q for q in quantiles]
    flat = element.float().reshape(-1)
    pv = np.percentile(flat.cpu().numpy(), percentiles)
    dev = flat.device
    inp = torch.as_tensor(pv, dtype=torch.float32, device=dev)
    lm = lm.to(dev)
    d_in = torch.diff(inp)
    d_in = torch.where(d_in.abs() < 1e-5, torch.tensor(float("inf"), device=dev), d_in)
    slopes = torch.diff(lm) / d_in
    intercepts = lm[:-1] - slopes * inp[:-1]
    return inp, slopes, intercepts, inp[1:-1]


def reference_output(data: torch.Tensor, lm: torch.Tensor, cutoff) -> torch.Tensor:
    """The batch after the reference's per-element loop: each element mapped in fp32 and written
    back into a copy of ``data`` in its own dtype."""
    out = data.clone()
    for i in range(data.shape[0]):
        _, slopes, intercepts, edges = element_tables(data[i], lm, cutoff)
        flat = data[i].float().reshape(-1)
        bins = torch.bucketize(flat, edges, right=False)
        out[i] = (slopes[bins] * flat + intercepts[bins]).reshape(data[i].shape)
    return out


def reference_landmarks(images, *, quantiles=None, cutoff=(0.01, 0.99), masking_method=None) -> torch.Tensor:
    """compute_histogram_landmarks with np.percentile on each image's native dtype."""
    quantiles = quantiles_for(cutoff) if quantiles is None else tuple(sorted(set(quantiles)))
    rows = []
    for tensor in images:
        mask = torch.ones_like(tensor, dtype=torch.bool) if masking_method is None else masking_method(tensor)
        rows.append(np.percentile(tensor[mask].numpy(), [100.0 * q for q in quantiles]))
    db = np.vstack(rows)
    slopes = np.nan_to_num(100.0 / (db[:, -1] - db[:, 0]))
    return torch.as_tensor(slopes @ db / len(db) + float(np.mean(0.0 - slopes * db[:, 0])), dtype=torch.float32)


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"{name}.npz") as z:
        out = {k: z[k] for k in z.files}
    for key in ("history", "error", "hydra", "repr"):
        if key in out:
            out[key] = json.loads(out[key].tobytes().decode())
    return out
