"""Float64 adjoints of the Resize / Anisotropy passes, built as dense per-axis matrices: from the
forward tables (the matrix A of each axis) and from the CSR adjoint tables (Aᵀ), and applied to a
(B, C, I, J, K) gradient with torch on any device.  Shared by the table tests and the GPU tests."""

from __future__ import annotations

import numpy as np
import torch


def forward_matrix(idx: np.ndarray, lam: np.ndarray | None, n_in: int, n_out: int) -> np.ndarray:
    """(n_out, n_in) float64 A of one axis of a tio_interpolate table: the two taps (i0, i1) with
    weights (l0, l1) of each output (nearest: i0 with weight 1)."""
    a = np.zeros((n_out, n_in))
    o = np.arange(n_out)
    if lam is None:
        np.add.at(a, (o, idx[:n_out]), 1.0)
    else:
        np.add.at(a, (o, idx[:n_out]), lam[:n_out].astype(np.float64))
        np.add.at(a, (o, idx[n_out:]), lam[n_out:].astype(np.float64))
    return a


def forward_matrices(idx, lam, in_shape, out_shape) -> list[np.ndarray]:
    """A of each axis of packed (idx, lam) tables (`tables.resize_tables` layout)."""
    mats, base = [], 0
    for n_in, n_out in zip(in_shape, out_shape):
        mats.append(forward_matrix(idx[base:base + 2 * n_out], None if lam is None else lam[base:base + 2 * n_out],
                                   n_in, n_out))
        base += 2 * n_out
    return mats


def adjoint_matrices(ptr, ent, wt, in_shape, out_shape) -> list[np.ndarray]:
    """Aᵀ (n_in, n_out) of each axis of packed (ptr, ent, wt) adjoint tables."""
    mats, base = [], 0
    for n_in, n_out in zip(in_shape, out_shape):
        p = ptr[base:base + n_in + 1].astype(np.int64)
        m = np.zeros((n_in, n_out))
        for x in range(n_in):
            np.add.at(m, (x, ent[p[x]:p[x + 1]]), wt[p[x]:p[x + 1]].astype(np.float64))
        mats.append(m)
        base += n_in + 1
    return mats


def instance_forward_matrix(lo, hi, w, length: int, linear: bool) -> np.ndarray:
    """(L, L) float64 A of one element's axis of tio_axis_resample: (1 - w) rounded in fp32 on lo,
    w on hi (nearest: 1 on lo)."""
    a = np.zeros((length, length))
    o = np.arange(length)
    if not linear:
        np.add.at(a, (o, lo[:length]), 1.0)
        return a
    one_minus = (np.float32(1.0) - w[:length].astype(np.float32)).astype(np.float64)
    np.add.at(a, (o, lo[:length]), one_minus)
    np.add.at(a, (o, hi[:length]), w[:length].astype(np.float64))
    return a


def instance_adjoint_matrix(ptr_row, ent_row, w_row, length: int, linear: bool) -> np.ndarray:
    """Aᵀ (L, L) of one element's axis from its (ptr, ent) rows and the forward's weights."""
    m = np.zeros((length, length))
    for p in range(length):
        for code in ent_row[ptr_row[p]:ptr_row[p + 1]]:
            o, upper = int(code) >> 1, int(code) & 1
            if not linear:
                m[p, o] += 1.0
            elif upper:
                m[p, o] += float(w_row[o])
            else:
                m[p, o] += float(np.float32(1.0) - np.float32(w_row[o]))
    return m


def apply_separable(g: torch.Tensor, mats) -> torch.Tensor:
    """sum over (o, p, q) of M_i[x, o] M_j[y, p] M_k[z, q] g[..., o, p, q], in float64."""
    mi, mj, mk = (torch.as_tensor(m, dtype=torch.float64, device=g.device) for m in mats)
    g = g.double()
    g = torch.einsum("xo,bcopq->bcxpq", mi, g)
    g = torch.einsum("yp,bcxpq->bcxyq", mj, g)
    return torch.einsum("zq,bcxyq->bcxyz", mk, g)


def apply_along(g: torch.Tensor, mat, axis: int) -> torch.Tensor:
    """M applied to the spatial ``axis`` of a (C, I, J, K) gradient, in float64."""
    m = torch.as_tensor(mat, dtype=torch.float64, device=g.device)
    g = g.double().movedim(axis + 1, -1)
    return (g @ m.T).movedim(-1, axis + 1)


def gamma(m) -> np.ndarray:
    """γ_m = m u / (1 - m u) of fp32 (u = 2^-24)."""
    u = 2.0 ** -24
    m = np.asarray(m, dtype=np.float64)
    return m * u / (1 - m * u)
