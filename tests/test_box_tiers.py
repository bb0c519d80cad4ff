"""Host side of K1's per-element box: every output tile's pre-image fits its element's box.

`_affine_box_edges` bounds what `tile_bounds_kernel` (csrc/resample_tile.cuh) measures per tile.
Here that measurement is restated in numpy fp32 over every 16^3 tile of a 256^3 output, for the
bench's Affine draws and wider ones, and no tile may need more than its element's edge."""

import numpy as np
import pytest

from torchio_b200 import tables
from torchio_b200.data import AffineMatrix
from torchio_b200.transforms import spatial

S = 256


def _voxel_matrices(scales, degrees, translation):
    forwards = spatial.build_forward_affines(scales, degrees, translation, "image", (S, S, S), AffineMatrix())
    eye = np.eye(4)
    packed = tables.spatial_tables(list(forwards), [None] * len(forwards), len(forwards), eye, eye,
                                   per_instance=True, has_target=False)
    return packed


def _tile_needs(mat, out_shape):
    """(B, tiles, 3) planes of the box each tile needs per input axis, as tile_bounds_kernel
    counts them in fp32 (K with its origin rounded down to 4 elements)."""
    m = np.asarray(mat, dtype=np.float32).reshape(-1, 3, 4)
    starts = [np.arange(0, n, 16) for n in out_shape]
    lo = np.stack(np.meshgrid(*starts, indexing="ij"), axis=-1).reshape(-1, 3)
    hi = np.minimum(lo + 16, out_shape) - 1
    lo, hi = lo.astype(np.float32), hi.astype(np.float32)
    need = np.empty((len(m), len(lo), 3))
    for ax in range(3):
        qlo = np.broadcast_to(m[:, ax, 3][:, None], (len(m), len(lo))).astype(np.float32)
        qhi = qlo.copy()
        for bx in range(3):
            v0 = m[:, ax, bx][:, None] * lo[None, :, bx]
            v1 = m[:, ax, bx][:, None] * hi[None, :, bx]
            qlo = qlo + np.minimum(v0, v1)
            qhi = qhi + np.maximum(v0, v1)
        margin = np.float32(0.02) + np.float32(1e-5) * np.maximum(np.abs(qlo), np.abs(qhi))
        ilo = np.floor(qlo - margin).astype(np.int64)
        ihi = np.floor(qhi + margin).astype(np.int64) + 1
        if ax == 2:
            ilo &= ~3
        need[:, :, ax] = ihi - ilo + 1
    return need


@pytest.mark.parametrize("scales,degrees,translation", [
    ((0.9, 1.1), (-10, 10), (0, 0)),    # bench.py's Affine
    ((0.75, 1.25), (-20, 20), (-10, 10)),
    ((1.0, 1.0), (0, 0), (-300, 300)),  # pre-images partly or wholly outside the volume
], ids=["bench", "wide", "shifted"])
def test_no_tile_needs_more_than_its_elements_box(scales, degrees, translation):
    rng = np.random.default_rng(0)
    n = 48
    packed = _voxel_matrices(rng.uniform(*scales, (n, 3)), rng.uniform(*degrees, (n, 3)),
                             rng.uniform(*translation, (n, 3)))
    cap = 32  # no cap below the largest edge: every element gets the edge its tiles need
    edges = spatial._affine_box_edges(packed.mat, cap, (S, S, S))
    need = _tile_needs(packed.mat, (S, S, S))
    small = edges < cap
    assert small.any()
    bk = (edges + 7) // 4 * 4
    assert (need[small, :, 0] <= edges[small, None]).all()
    assert (need[small, :, 1] <= edges[small, None]).all()
    assert (need[small, :, 2] <= bk[small, None]).all()
    # the bound is tight: one step down would not hold some tile
    for b in np.nonzero(edges > min(spatial._BOX_EDGES))[0]:
        lower = spatial._BOX_EDGES[spatial._BOX_EDGES.index(int(edges[b])) - 1]
        fits = ((need[b, :, :2] <= lower).all(axis=1) & (need[b, :, 2] <= (lower + 7) // 4 * 4)).all()
        if edges[b] < cap:
            assert not fits, (b, edges[b])


def test_tiers_order_elements_by_edge_and_cover_the_batch():
    rng = np.random.default_rng(1)
    n = 32
    packed = _voxel_matrices(rng.uniform(0.9, 1.1, (n, 3)), rng.uniform(-10, 10, (n, 3)), np.zeros((n, 3)))
    cap = spatial._box_hint(packed, (1, 1, 1), (1, 1, 1), (S, S, S))
    assert cap == 24
    order, runs = spatial._box_tiers(packed, cap, (S, S, S))
    edges = spatial._affine_box_edges(packed.mat, cap, (S, S, S))
    assert order.dtype == np.int32 and sorted(order.tolist()) == list(range(n))
    assert [e for _, e in runs] == sorted({int(e) for e in edges})
    assert sum(c for c, _ in runs) == n
    assert (np.diff(edges[order]) >= 0).all()
    # identity matrices need the smallest box; one call of them is a single run at 20
    eye = _voxel_matrices(np.ones((4, 3)), np.zeros((4, 3)), np.zeros((4, 3)))
    assert spatial._box_tiers(eye, 24, (S, S, S))[1] == [(4, 20)]


def test_elastic_and_full_box_calls_keep_one_box():
    packed = _voxel_matrices(np.full((2, 3), 1.3), np.full((2, 3), 20.0), np.zeros((2, 3)))
    cap = spatial._box_hint(packed, (1, 1, 1), (1, 1, 1), (S, S, S))
    assert spatial._box_tiers(packed, cap, (S, S, S)) == (None, None)
    grid = tables.SpatialTables(packed.mat, np.zeros((2, 7, 7, 7, 3), np.float32), packed.flags, [])
    assert spatial._box_tiers(grid, 24, (S, S, S)) == (None, None)


def test_non_finite_matrices_take_the_launch_box():
    mat = np.zeros((2, 12), np.float32)
    mat[0, [0, 5, 10]] = 1
    mat[1] = np.nan
    assert spatial._affine_box_edges(mat, 24, (S, S, S)).tolist() == [20, 24]
