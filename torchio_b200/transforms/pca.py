"""PCA (transforms/intensity/pca.py of TorchIO 2.0.0a2): reduce an image's channels to its leading
principal components.

Constructor, errors, ``repr``, ``to_hydra``, the batch-level ``p`` gate, history and the random draw
are the reference's.  The reference runs ``torch.pca_lowrank`` on A = (voxels x channels) minus the
channel means, then projects, whitens, normalises and maps ``values_range`` onto [0, 1].  Every step
of ``pca_lowrank`` depends on A only through products G W with G = A^T A and W a C x q matrix:

- an N x q basis ``Q = A Z`` has ``span(A^T Q) = span(G Z)``;
- ``orth(A W) = A W L^-T`` with ``L L^T = W^T G W`` (Cholesky), so the QR of a tall matrix is q x q work;
- ``Q^T A = Z^T G``, and the first component's std is ``sqrt(v0^T G v0 / (N - 1))`` times its scale.

So the volume is read by `ops.pca_mean`, three `ops.pca_gram_apply` passes (the sketch ``G R`` and the
two power iterations), one more for ``G v0`` when ``normalize``, and `ops.pca_project`; the C x q
algebra runs here in float64.  Each QR of the reference has a Q unique up to column signs, so the
subspace, S and V are the reference's for the same sketch R up to the sign of each component; the
sign is fixed here so that each loading vector's largest-magnitude entry is positive (the lowest
channel on a tie).

Each call reads a few C x q matrices back to the host (the sketch R and each G W), so the transform
synchronises with the device and cannot be captured in a CUDA graph.
"""

from __future__ import annotations

import math
from typing import Any

import numpy as np
import torch

from .. import ops
from ..data import SubjectsBatch
from .base import IntensityTransform, staged_source_device

_NONFINITE = "linalg.svd: The algorithm failed to converge because the input matrix contained non-finite values."


def _check_finite(*arrays: np.ndarray) -> None:
    """The reference's LAPACK SVD refuses a NaN or ±Inf input (a non-finite voxel spreads to every
    product of its element)."""
    if not all(np.isfinite(a).all() for a in arrays):
        raise torch.linalg.LinAlgError(_NONFINITE)


def _orthonormal_products(w: np.ndarray, gw: np.ndarray) -> np.ndarray:
    """G Z for the Z (C x q per element) with ``A Z`` an orthonormal basis of ``span(A w)``, from
    ``gw = G w``: ``Z = w L^-T`` with ``L L^T = w^T G w``.  A rank-deficient ``A w`` (a constant
    element) keeps only the directions with a nonzero norm; the others become zero columns."""
    out = np.empty_like(gw)
    for e in range(w.shape[0]):
        m = w[e].T @ gw[e]
        m = (m + m.T) / 2
        try:
            chol = np.linalg.cholesky(m)
            out[e] = np.linalg.solve(chol, gw[e].T).T
        except np.linalg.LinAlgError:
            lam, vec = np.linalg.eigh(m)
            keep = lam > lam.max(initial=0.0) * 1e-12
            inv = np.where(keep, 1.0 / np.sqrt(np.where(keep, lam, 1.0)), 0.0)
            out[e] = gw[e] @ (vec * inv)
    return out


def lowrank_tall(r: np.ndarray, gram, niter: int = 2) -> tuple[np.ndarray, np.ndarray]:
    """(S (B, q), V (B, C, q)) of ``torch.pca_lowrank(A, q)`` for N >= C, from the sketch ``r``
    (B, C, q) and ``gram(W) -> G W`` ((B, C, q) float64 in and out)."""
    gz = _orthonormal_products(r, gram(r))          # G Z0, A Z0 = qr(A R).Q
    for _ in range(niter):
        _check_finite(gz)
        basis = np.linalg.qr(gz)[0]                 # qr(A^T Q).Q
        gz = _orthonormal_products(basis, gram(basis))  # A Z = qr(A basis).Q
    _check_finite(gz)
    _, s, vh = np.linalg.svd(gz.transpose(0, 2, 1), full_matrices=False)  # B = Z^T G
    return s, vh.transpose(0, 2, 1)


def lowrank_wide(a: np.ndarray, r: np.ndarray, niter: int = 2) -> tuple[np.ndarray, np.ndarray]:
    """(S, V) of ``torch.pca_lowrank(A, q)`` for N < C, where torch sketches A^T: ``a`` (B, N, C)
    centred, ``r`` (B, N, q)."""
    _check_finite(a)
    t = a.transpose(0, 2, 1)                        # the tall C x N matrix torch works on
    basis = np.linalg.qr(t @ r)[0]
    for _ in range(niter):
        basis = np.linalg.qr(a @ basis)[0]
        basis = np.linalg.qr(t @ basis)[0]
    u, s, _ = np.linalg.svd(basis.transpose(0, 2, 1) @ t, full_matrices=False)
    return s, basis @ u


def fix_signs(v: np.ndarray) -> np.ndarray:
    """``v`` (B, C, q) with each column flipped so that its largest-|.| entry is positive."""
    idx = np.abs(v).argmax(axis=1)
    lead = np.take_along_axis(v, idx[:, None, :], axis=1)
    return v * np.where(lead < 0, -1.0, 1.0)


def projection(s: np.ndarray, v: np.ndarray, first_energy: np.ndarray | None, n: int, *, whiten: bool,
               normalize: bool, values_range) -> tuple[np.ndarray, float]:
    """(coef (B, C, q), offset) with output ``A coef + offset`` equal to pca.py:111-127:
    ``projected = A V``, divided by ``clamp(S / sqrt(N - 1), 1e-8)`` when whitening and by the
    first component's clamped std when normalising (``first_energy`` = v0^T G v0), then mapped by
    ``(x - lo) / (hi - lo)``.  A one-voxel element has no std: NaN, as torch.std gives."""
    scale = np.ones_like(s)
    if whiten:
        denom = math.sqrt(n - 1) if n > 1 else 1.0
        scale = 1.0 / np.maximum(s / denom, 1e-8)
    if normalize:
        with np.errstate(invalid="ignore", divide="ignore"):
            first = np.sqrt(first_energy / (n - 1)) * scale[:, 0] if n > 1 else np.full(len(s), np.nan)
        scale = scale / np.maximum(first, 1e-8)[:, None]
    lo, hi = values_range
    return v * (scale / (hi - lo))[:, None, :], -lo / (hi - lo)


def pca(data: torch.Tensor, q: int, *, whiten: bool, normalize: bool, values_range, clip: bool,
        generator_device: torch.device | None = None) -> torch.Tensor:
    """fp32 (B, q, I, J, K): `PCA._pca_single` of each element of a (B, C, I, J, K) CUDA batch.  One
    sketch ``torch.randn(C, q)`` per element is drawn on ``generator_device`` (default: the data's),
    element by element, as the reference draws it."""
    b, c = int(data.shape[0]), int(data.shape[1])
    n = math.prod(int(s) for s in data.shape[2:])
    if c < q:
        raise ValueError(f"Image has {c} channels but num_components={q}. Need at least as many channels"
                         " as components.")
    if q > min(n, c):
        raise ValueError(f"q(={q}) must be non-negative integer and not greater than min(m, n)={min(n, c)}")
    tall = n >= c
    device = data.device if generator_device is None else generator_device
    r = torch.stack([torch.randn(c if tall else n, q, dtype=torch.float32, device=device) for _ in range(b)])
    r = r.cpu().double().numpy()
    data = data.contiguous()
    workspace = ops.pca_workspace(data, q)
    mean = ops.pca_mean(data, workspace)

    def gram(w: np.ndarray) -> np.ndarray:
        return ops.pca_gram_apply(data, mean, w, workspace).cpu().numpy()

    if tall:
        s, v = lowrank_tall(r, gram)
        v = fix_signs(v)
        energy = np.einsum("bc,bc->b", v[:, :, 0], gram(v[:, :, :1])[:, :, 0]) if normalize else None
    else:
        eye = np.broadcast_to(np.eye(c, dtype=np.float32), (b, c, c))
        a = ops.pca_project(data, mean, eye, 0.0, False).reshape(b, c, n).cpu().double().numpy()
        a = a.transpose(0, 2, 1) - a.transpose(0, 2, 1).mean(axis=1, keepdims=True)
        s, v = lowrank_wide(a, r)
        v = fix_signs(v)
        energy = ((a @ v[:, :, :1]) ** 2).sum(axis=(1, 2))
    coef, offset = projection(s, v, energy, n, whiten=whiten, normalize=normalize, values_range=values_range)
    return ops.pca_project(data, mean, coef, offset, clip)


class PCA(IntensityTransform):
    """Reduce the channels of each scalar image to ``num_components`` principal components
    (intensity/pca.py:15-140), computed on the GPU; see the module docstring."""

    def __init__(self, num_components: int = 3, *, whiten: bool = True, normalize: bool = True,
                 values_range: tuple[float, float] = (-2.3, 2.3), clip: bool = True, **kwargs: Any) -> None:
        super().__init__(**kwargs)
        if num_components < 1:
            raise ValueError(f"num_components must be >= 1, got {num_components}")
        self.num_components = num_components
        self.whiten = whiten
        self.normalize = normalize
        self.values_range = values_range
        self.clip = clip

    def make_params(self, batch: SubjectsBatch) -> dict[str, Any]:
        return {}

    def apply_transform(self, batch: SubjectsBatch, params: dict[str, Any]) -> SubjectsBatch:
        for name, img_batch in self._get_images(batch).items():
            img_batch.data = pca(img_batch.data, self.num_components, whiten=self.whiten, normalize=self.normalize,
                                 values_range=self.values_range, clip=self.clip,
                                 generator_device=staged_source_device(name, img_batch.data))
        return batch
