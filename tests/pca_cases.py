"""PCA test infrastructure: the fixture cases, their seeded inputs, the reference's op sequence
(transforms/intensity/pca.py:83-140 of TorchIO 2.0.0a2, ``torch.pca_lowrank`` included) restated on
torch ops, runnable on CPU and CUDA tensors, and float64 numpy products G W for the host algebra.
``tests/golden/generate_pca.py`` runs the reference's class on these cases; nothing here is imported
by the product."""

from __future__ import annotations

import json
import math
from pathlib import Path

import numpy as np
import torch

GOLDEN = Path(__file__).resolve().parent / "golden"

F32, F16, BF16, F64 = torch.float32, torch.float16, torch.bfloat16, torch.float64
U8, I8, I16, I32, I64 = torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64
SHORT = {F32: "f32", F16: "f16", BF16: "bf16", F64: "f64", U8: "u8", I8: "i8", I16: "i16", I32: "i32", I64: "i64"}

# Inputs: image "t1" (and "t2" with `two`), a (B, C, *shape) ScalarImage of `dtype` built as
# offset + sum_k sigma_k z_k u_k over random orthonormal channel directions u_k and N(0, 1) voxel
# scores z_k, made orthonormal and centred when N > C so that the sample spectrum is sigma.  Spectra:
#   "gap"    the leading q components at sigma = 4^-k, the rest at 0.03 * 4^-(q-1): the sketch is
#            the reference's for any R to better than 1e-6 (ratio 0.03, raised to the 5th power)
#   "linear" sigma from 1 down to 0.25 over all C components (used with q = C: no tail)
#   "flat"   every sigma 1 and the raw scores: the sample spectrum has no gap, so the components
#            depend on R and only the same R reproduces them
# `offset` is the channel mean in units of the largest sigma.  Floats are scaled by 10; integers are
# scaled to a few percent of their range around its middle (0 when signed) and rounded.  `constant` makes that element 3.0 everywhere, `nan` puts a NaN voxel into that element.
CASES_LIST = [
    dict(name="pca_c3_q1", batch=1, channels=3, shape=(8, 8, 8), q=1, kwargs=dict(num_components=1)),
    dict(name="pca_c3_q3", batch=1, channels=3, shape=(8, 8, 8), q=3, spectrum="linear",
         kwargs=dict(num_components=3)),
    dict(name="pca_c4_q1", batch=1, channels=4, shape=(8, 8, 8), q=1, kwargs=dict(num_components=1)),
    dict(name="pca_c4_q3", batch=1, channels=4, shape=(8, 8, 8), q=3, kwargs=dict()),
    dict(name="pca_c4_q4", batch=1, channels=4, shape=(8, 8, 8), q=4, spectrum="linear",
         kwargs=dict(num_components=4)),
    dict(name="pca_c16_q1", batch=1, channels=16, shape=(8, 8, 8), q=1, kwargs=dict(num_components=1)),
    dict(name="pca_c16_q3", batch=3, channels=16, shape=(8, 8, 8), q=3, kwargs=dict()),
    dict(name="pca_c16_q16", batch=1, channels=16, shape=(8, 8, 8), q=16, spectrum="linear",
         kwargs=dict(num_components=16)),
    dict(name="pca_c64_q1", batch=1, channels=64, shape=(8, 8, 8), q=1, kwargs=dict(num_components=1)),
    dict(name="pca_c64_q3", batch=1, channels=64, shape=(8, 8, 8), q=3, kwargs=dict()),
    dict(name="pca_c64_q64", batch=1, channels=64, shape=(8, 8, 8), q=64, spectrum="linear",
         kwargs=dict(num_components=64, whiten=False)),
    dict(name="pca_b3_c4_q3", batch=3, channels=4, shape=(9, 7, 5), q=3, kwargs=dict()),
    dict(name="pca_nowhiten", batch=1, channels=16, shape=(8, 8, 8), q=3, kwargs=dict(whiten=False)),
    dict(name="pca_nonormalize", batch=1, channels=16, shape=(8, 8, 8), q=3, kwargs=dict(normalize=False)),
    dict(name="pca_noclip", batch=1, channels=16, shape=(8, 8, 8), q=3, kwargs=dict(clip=False)),
    dict(name="pca_plain", batch=1, channels=16, shape=(8, 8, 8), q=3,
         kwargs=dict(whiten=False, normalize=False, clip=False)),
    dict(name="pca_range_asym", batch=3, channels=4, shape=(8, 8, 8), q=3,
         kwargs=dict(values_range=(-1.0, 3.5), clip=False)),
    dict(name="pca_include", batch=3, channels=4, shape=(8, 8, 8), q=3, two=True, kwargs=dict(include=["t2"])),
    dict(name="pca_exclude", batch=3, channels=4, shape=(8, 8, 8), q=3, two=True, kwargs=dict(exclude=["t1"])),
    dict(name="pca_two_images", batch=3, channels=4, shape=(8, 8, 8), q=3, two=True, kwargs=dict()),
    *[dict(name=f"pca_dtype_{SHORT[d]}", batch=3, channels=4, shape=(8, 8, 8), q=3, dtype=d, kwargs=dict())
      for d in (F16, BF16, F64, U8, I8, I16, I32, I64)],
    dict(name="pca_constant", batch=3, channels=4, shape=(8, 8, 8), q=3, constant=1, kwargs=dict()),
    dict(name="pca_nan", batch=3, channels=4, shape=(8, 8, 8), q=3, nan=1, kwargs=dict()),
    dict(name="pca_n1", batch=2, channels=3, shape=(1, 1, 1), q=1, kwargs=dict(num_components=1)),
    dict(name="pca_n1_nonormalize", batch=2, channels=3, shape=(1, 1, 1), q=1,
         kwargs=dict(num_components=1, normalize=False)),
    dict(name="pca_n1_c1", batch=1, channels=1, shape=(1, 1, 1), q=1,
         kwargs=dict(num_components=1, normalize=False)),
    dict(name="pca_wide", batch=3, channels=16, shape=(2, 2, 2), q=3, kwargs=dict()),
    dict(name="pca_offset", batch=3, channels=4, shape=(8, 8, 8), q=3, offset=1e3, kwargs=dict(clip=False)),
    dict(name="pca_p05_gated", batch=3, channels=4, shape=(8, 8, 8), q=3, seed=1, kwargs=dict(p=0.5)),
    dict(name="pca_p05_applied", batch=3, channels=4, shape=(8, 8, 8), q=3, seed=3, kwargs=dict(p=0.5)),
    dict(name="pca_flat", batch=1, channels=16, shape=(8, 8, 8), q=3, spectrum="flat", kwargs=dict()),
    dict(name="pca_compose_normalize", batch=3, channels=4, shape=(8, 8, 8), q=3, compose=True, kwargs=dict()),
    dict(name="pca_error_components", batch=1, channels=4, shape=(8, 8, 8), q=0, kwargs=dict(num_components=0)),
    dict(name="pca_error_channels", batch=1, channels=2, shape=(8, 8, 8), q=3, kwargs=dict()),
    dict(name="pca_error_voxels", batch=1, channels=4, shape=(1, 1, 2), q=3, kwargs=dict()),
]
CASES = {c["name"]: c for c in CASES_LIST}


def seed(case) -> int:
    return case.get("seed", 1300 + sorted(CASES).index(case["name"]))


def sigmas(case) -> np.ndarray:
    c, q = case["channels"], max(case["q"], 1)
    kind = case.get("spectrum", "gap")
    if kind == "linear":
        return np.linspace(1.0, 0.25, c)
    if kind == "flat":
        return np.ones(c)
    lead = 4.0 ** -np.arange(min(q, c))
    return np.concatenate([lead, np.full(c - len(lead), 0.03 * lead[-1])])


def random_volume(rng: np.random.Generator, case, dtype: torch.dtype) -> torch.Tensor:
    b, c, shape = case["batch"], case["channels"], case["shape"]
    n = int(np.prod(shape))
    sig = sigmas(case)
    out = np.empty((b, c, n))
    for e in range(b):
        u = np.linalg.qr(rng.standard_normal((c, c)))[0]
        z = rng.standard_normal((c, n))
        if n > c and case.get("spectrum") != "flat":  # orthonormal centred scores: the sample spectrum is sigma
            z = np.linalg.qr((z - z.mean(axis=1, keepdims=True)).T)[0].T * math.sqrt(n - 1)
        out[e] = (u * sig) @ z + case.get("offset", 0.0) * rng.uniform(0.5, 1.0, (c, 1))
    if dtype.is_floating_point:
        out *= 10.0
    else:
        info = torch.iinfo(dtype)
        centre = 0.0 if info.min < 0 else 0.5 * info.max
        out = np.clip(np.round(centre + out * min(0.08 * info.max, 1e4)), info.min, info.max)
    if "constant" in case:
        out[case["constant"]] = 3.0
    t = torch.as_tensor(out).reshape(b, c, *shape)
    if "nan" in case:
        t[case["nan"], 1].view(-1)[5] = float("nan")
    return t.to(dtype)


def images(case) -> dict[str, torch.Tensor]:
    rng = np.random.default_rng(seed(case))
    dtype = case.get("dtype", F32)
    out = {"t1": random_volume(rng, case, dtype)}
    if case.get("two"):
        out["t2"] = random_volume(rng, case, dtype)
    return out


def options(case) -> dict:
    """PCA's constructor values of the case, defaults filled in."""
    kw = case["kwargs"]
    return dict(q=kw.get("num_components", 3), whiten=kw.get("whiten", True), normalize=kw.get("normalize", True),
                values_range=tuple(kw.get("values_range", (-2.3, 2.3))), clip=kw.get("clip", True))


def transformed_names(case) -> list[str]:
    names = ["t1", "t2"] if case.get("two") else ["t1"]
    kw = case["kwargs"]
    if "include" in kw:
        names = [n for n in names if n in kw["include"]]
    if "exclude" in kw:
        names = [n for n in names if n not in kw["exclude"]]
    return names


# ---- the reference's op sequence on torch tensors -----------------------------------------------

def reference_single(tensor: torch.Tensor, q: int, whiten: bool, normalize: bool, values_range, clip: bool):
    """pca.py:83-140 (`_pca_single`) on one (C, I, J, K) tensor on any device: the same torch calls,
    ``torch.pca_lowrank`` drawing its sketch from ``tensor``'s device generator."""
    c, si, sj, sk = tensor.shape
    if c < q:
        raise ValueError(f"Image has {c} channels but num_components={q}. Need at least as many channels as"
                         " components.")
    flat = tensor.float().reshape(c, -1).T
    centered = flat - flat.mean(dim=0, keepdim=True)
    _u, s, v = torch.pca_lowrank(centered, q=q)
    projected = centered @ v
    if whiten:
        n = flat.shape[0]
        denom = (n - 1) ** 0.5 if n > 1 else 1.0
        projected = projected / (s / denom).clamp(min=1e-8).unsqueeze(0)
    if normalize and projected.shape[1] > 0:
        projected = projected / projected[:, 0].std().clamp(min=1e-8)
    lo, hi = values_range
    projected = (projected - lo) / (hi - lo)
    if clip:
        projected = projected.clamp(0, 1)
    return projected.T.reshape(q, si, sj, sk)


def reference_ops(data: torch.Tensor, q: int, whiten: bool, normalize: bool, values_range, clip: bool):
    """The reference's `apply_transform` on one (B, C, I, J, K) image batch: element by element."""
    return torch.stack([reference_single(data[i], q, whiten, normalize, values_range, clip)
                        for i in range(data.shape[0])])


# ---- float64 products and comparisons -----------------------------------------------------------

def centred(data: torch.Tensor) -> np.ndarray:
    """(B, N, C) float64 of float(x) minus its float64 channel means."""
    a = data.float().double().reshape(data.shape[0], data.shape[1], -1).transpose(1, 2).cpu().numpy()
    return a - a.mean(axis=1, keepdims=True)


def gram_of(a: np.ndarray):
    """``gram(W) -> A^T (A W)`` over (B, N, C) float64 ``a``."""
    return lambda w: a.transpose(0, 2, 1) @ (a @ w)


def flipped(y: np.ndarray, values_range, clip: bool) -> np.ndarray:
    """The output ``y`` would be with the component's sign flipped: ``1 - y`` for a symmetric range
    (clipped or not), ``-y - 2 lo / (hi - lo)`` without clipping."""
    lo, hi = values_range
    if clip:
        assert lo == -hi, "a clipped output can be sign-flipped only for a symmetric range"
    return -y - 2 * lo / (hi - lo)


def sign_errors(got: np.ndarray, want: np.ndarray, values_range, clip: bool, *, shift: bool = False) -> np.ndarray:
    """(B, q) largest |got - want| of each component, with the better of the two signs; NaN must
    sit in the same places (a mismatch counts as inf).  With ``shift`` (unclipped outputs only), each
    component's median difference is removed first: a constant per component is what rounding the
    channel means differently adds."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    b, q = got.shape[:2]
    out = np.zeros((b, q))
    for e in range(b):
        for k in range(q):
            g, w = got[e, k].ravel(), want[e, k].ravel()
            best = math.inf
            for cand in (g, flipped(g, values_range, clip)):
                if not np.array_equal(np.isnan(cand), np.isnan(w)):
                    continue
                ok = ~np.isnan(w)
                diff = cand[ok] - w[ok]
                if shift and diff.size:
                    diff = diff - np.median(diff)
                best = min(best, float(np.abs(diff).max(initial=0.0)))
            out[e, k] = best
    return out


def spectral_gap(data: torch.Tensor, q: int) -> bool:
    """True when every element's float64 spectrum has sigma_{q+1} <= 0.1 sigma_q (or q = min(N, C)):
    the reference's result then does not depend on R to 1e-5."""
    a = centred(data)
    if q >= min(a.shape[1:]):
        return True
    if not np.isfinite(a).all():
        return False
    s = np.linalg.svd(a, compute_uv=False)
    return bool(np.all(s[:, q] <= 0.1 * s[:, q - 1]))


def as_stored(t: torch.Tensor) -> np.ndarray:
    """A tensor as the fixtures store it (bf16 as its int16 bits)."""
    t = t.detach().cpu().contiguous()
    return (t.view(torch.int16) if t.dtype == torch.bfloat16 else t).numpy()


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"{name}.npz") as z:
        out = {k: z[k] for k in z.files}
    for key in ("history", "error", "hydra", "repr", "dtype", "rng_after"):
        if key in out:
            out[key] = json.loads(out[key].tobytes().decode())
    return out
