"""The CSR adjoint tables of Resize and Anisotropy (`tables.*_adjoint_tables`) are the transposes of
the forward tables: for many (L, D) pairs, in both modes and on all three paths (Resize, Anisotropy's
shared pass, its per-instance rows), the dense matrix of the CSR tables equals Aᵀ of the dense
matrix of the forward tables, every tap the forward reads is an entry (zero weights included), and
a float64 adjoint from the CSR tables equals Aᵀ applied to a random gradient.  Host-only."""

import numpy as np
import pytest
import torch

from resolution_adjoint import (adjoint_matrices, apply_along, apply_separable, forward_matrices,
                                instance_adjoint_matrix, instance_forward_matrix)
from torchio_b200 import tables

# (in shape, out shape): up, down, mixed, same shape, unit axes on either side
RESIZE_CASES = [
    ((6, 5, 7), (9, 11, 13)),
    ((12, 10, 9), (5, 4, 3)),
    ((10, 8, 9), (15, 4, 9)),
    ((7, 8, 9), (7, 8, 9)),
    ((8, 9, 10), (8, 1, 10)),
    ((1, 6, 5), (4, 6, 1)),
    ((26, 5, 33), (22, 7, 8)),
]

# (L, factor): D = round(L / factor) down, D = L, D = 1, L = 1, and the (26, 22) and (33, 4.4) cases
# where ATen's nearest map and the per-instance map differ and where round(L / f) sits on .5
ANISO_CASES = [(12, 2.0), (13, 3.0), (9, 1.01), (9, 40.0), (1, 2.0), (26, 26 / 22), (33, 4.4), (37, 1.5),
               (64, 5.0), (2, 1.7)]


def _check_csr(ptr, ent_count, n_in):
    assert ptr[0] >= 0 and np.all(np.diff(ptr) >= 0) and len(ptr) == n_in + 1
    assert ptr[-1] - ptr[0] == ent_count


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("in_shape,out_shape", RESIZE_CASES)
def test_resize_adjoint_is_the_transpose(in_shape, out_shape, linear):
    idx, lam = tables.resize_tables(in_shape, out_shape, linear)
    ptr, ent, wt = tables.resize_adjoint_tables(in_shape, out_shape, linear)
    _compare(idx, lam, ptr, ent, wt, in_shape, out_shape)


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("length,factor", ANISO_CASES)
def test_anisotropy_shared_adjoint_is_the_transpose(length, factor, axis, linear):
    shape = [5, 4, 6]
    shape[axis] = length
    idx, lam = tables.anisotropy_shared_tables(shape, axis, factor, linear)
    ptr, ent, wt = tables.anisotropy_shared_adjoint_tables(shape, axis, factor, linear)
    _compare(idx, lam, ptr, ent, wt, shape, shape)


def _compare(idx, lam, ptr, ent, wt, in_shape, out_shape):
    assert ptr.dtype == np.int32 and ent.dtype == np.int32 and wt.dtype == np.float32
    taps = 2 if lam is not None else 1
    assert len(ent) == len(wt) == taps * sum(out_shape)  # every tap read, zero weights included
    base = 0
    for n_in, n_out in zip(in_shape, out_shape):
        p = ptr[base:base + n_in + 1]
        _check_csr(p, taps * n_out, n_in)
        for x in range(n_in):
            outs = ent[p[x]:p[x + 1]]
            assert np.all(np.diff(outs) >= 0), "entries of an input index in ascending output"
        base += n_in + 1
    a = forward_matrices(idx, lam, in_shape, out_shape)
    at = adjoint_matrices(ptr, ent, wt, in_shape, out_shape)
    for m, mt in zip(a, at):
        np.testing.assert_array_equal(mt, m.T)
    g = torch.randn((2, 1, *out_shape), generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    got = apply_separable(g, at)
    want = torch.einsum("oi,pj,qk,bcopq->bcijk", *(torch.as_tensor(m) for m in a), g)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_anisotropy_instance_adjoint_is_the_transpose(axis, linear):
    for length, factor in ANISO_CASES:
        shape = [5, 4, 6]
        shape[axis] = length
        # element 1 is gated out (factor 1): axis -1, empty rows
        axes, factors = [axis, axis, axis], [factor, 1.0, factor * 1.3]
        ax, lo, hi, w = tables.anisotropy_instance_tables(shape, axes, factors, linear)
        ptr, ent = tables.anisotropy_instance_adjoint_tables(shape, axes, factors, linear)
        width = max(shape)
        assert ptr.shape == (3, width + 1) and ent.shape == (3, 2 * width)
        assert ptr.dtype == np.int32 and ent.dtype == np.int32
        assert ax[1] == -1 and np.all(ptr[1] == 0)
        g = torch.randn((3, 2, *shape), generator=torch.Generator().manual_seed(4), dtype=torch.float64)
        for b in (0, 2):
            n = shape[axis]
            _check_csr(ptr[b, :n + 1], (2 if linear else 1) * n, n)
            assert np.all(ptr[b, n + 1:] == ptr[b, n])
            codes = ent[b, :ptr[b, n]]
            for p in range(n):
                row = ent[b, ptr[b, p]:ptr[b, p + 1]]
                assert np.all(np.diff(row) > 0), "entries of a plane in ascending output, lo before hi"
            assert sorted(codes.tolist()) == sorted(
                [2 * o for o in range(n)] + ([2 * o + 1 for o in range(n)] if linear else []))
            a = instance_forward_matrix(lo[b], hi[b], w[b], n, linear)
            at = instance_adjoint_matrix(ptr[b], ent[b], w[b], n, linear)
            np.testing.assert_array_equal(at, a.T)
            torch.testing.assert_close(apply_along(g[b], at, axis),
                                       apply_along(g[b], a.T, axis), rtol=1e-12, atol=1e-12)


def test_adjoint_tables_are_cached_per_axis():
    first = tables.resize_adjoint_tables((40, 30, 20), (17, 30, 50), True)
    tables._adjoint_axis.cache_clear()
    tables.resize_adjoint_tables((40, 30, 20), (17, 30, 50), True)
    misses = tables._adjoint_axis.cache_info().misses
    again = tables.resize_adjoint_tables((40, 30, 20), (17, 30, 50), True)
    assert tables._adjoint_axis.cache_info().misses == misses
    for x, y in zip(first, again):
        np.testing.assert_array_equal(x, y)


def test_invert_taps_assumes_no_monotonicity():
    src = np.array([3, 0, 3, 1, 0, 3])
    out = np.array([0, 1, 2, 3, 4, 0])
    ptr, order = tables.invert_taps(src, out, 5)
    assert ptr.tolist() == [0, 2, 3, 3, 6, 6]
    # input 3: outputs 0 (tap 0), 0 (tap 5, listed later), 2
    assert order.tolist() == [1, 4, 3, 0, 5, 2]
