"""K1 with a box edge per batch element (`tio_resample_tiered`) against one box for the batch.

A tile takes the staged box or the fallback by the same test in both calls, so the output is
bit-identical, and so is every tile's record (box origin, fit code, in-bounds bit)."""

import ctypes

import numpy as np
import pytest
import torch

from torchio_b200 import _native, ops, tables
from torchio_b200.data import AffineMatrix
from torchio_b200.transforms import spatial

pytestmark = pytest.mark.gpu

SHAPE = (50, 44, 72)  # ragged: no axis a multiple of 16


def _batch():
    """Elements of every box edge (the 32 one's tiles fit no box: all fall back), a passthrough
    element and one mapped outside the volume."""
    scales = [(1, 1, 1), (0.8, 0.8, 0.8), (0.7, 0.75, 0.7), (1, 1, 1), (1, 1, 1), (0.95, 1.05, 0.9),
              (0.45, 0.5, 0.45)]
    degrees = [(10, 0, 0), (0, 0, 5), (8, -6, 4), (0, 0, 0), (0, 0, 0), (-9, 7, 3), (5, 5, 5)]
    shifts = [(0, 0, 0), (2, -3, 1), (0, 0, 0), (0, 0, 0), (500, 0, 0), (-6, 4, 8), (0, 0, 0)]
    forwards = list(spatial.build_forward_affines(np.array(scales, float), np.array(degrees, float),
                                                  np.array(shifts, float), "image", SHAPE, AffineMatrix()))
    forwards[3] = None
    eye = np.eye(4)
    packed = tables.spatial_tables(forwards, [None] * len(forwards), len(forwards), eye, eye,
                                   per_instance=True, has_target=False)
    packed.flags[3] = ops.FLAG_PASSTHROUGH
    return packed


def _call(x, packed, fill, box_hint, tiers):
    """dst and the per-tile records of one tio_resample[_tiered] call, records in element order."""
    b, c, i, j, k = x.shape
    dev = x.device
    mat = torch.tensor(packed.mat, device=dev)
    flags = torch.tensor(packed.flags, device=dev)
    dst = torch.empty_like(x)
    ws_bytes = _native.lib().tio_resample_workspace_bytes(b, i, j, k)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    sp = (ctypes.c_float * 3)(1, 1, 1)
    args = (x.data_ptr(), dst.data_ptr(), 0, b, c, i, j, k, i, j, k, mat.data_ptr(), None, flags.data_ptr(),
            0, 0, 0, ctypes.addressof(sp), ctypes.addressof(sp), 1, ops.LINEAR, fill.data_ptr(), box_hint)
    stream = torch.cuda.current_stream().cuda_stream
    if tiers is None:
        _native.call("tio_resample", *args, ws.data_ptr(), ws_bytes, stream)
        records = ws.view(torch.int32).view(b, -1, 4)
    else:
        order, runs = tiers
        elems = torch.tensor(order, device=dev)
        flat = np.asarray(runs, dtype=np.int32).reshape(-1)
        _native.call("tio_resample_tiered", *args, elems.data_ptr(), flat.ctypes.data, len(runs),
                     ws.data_ptr(), ws_bytes, stream)
        records = torch.empty_like(ws.view(torch.int32).view(b, -1, 4))
        records[elems.long()] = ws.view(torch.int32).view(b, -1, 4)
    torch.cuda.synchronize()
    return dst, records


@pytest.mark.parametrize("channels", [1, 2])
def test_tiered_call_is_the_single_box_call(channels):
    packed = _batch()
    cap = spatial._box_hint(packed, (1, 1, 1), (1, 1, 1), SHAPE)
    assert cap == 32
    order, runs = spatial._box_tiers(packed, cap, SHAPE)
    assert [e for _, e in runs] == [20, 22, 24, 28, 32]
    g = torch.Generator().manual_seed(5)
    x = torch.rand((len(packed.mat), channels, *SHAPE), generator=g).cuda()
    fill = torch.tensor([0.25, -1.0][:channels], device="cuda")
    one, rec_one = _call(x, packed, fill, cap, None)
    tiered, rec_tiered = _call(x, packed, fill, cap, (order, runs))
    assert torch.equal(tiered, one)
    assert torch.equal(rec_tiered, rec_one)
    codes = rec_one[..., 3] & 255
    assert set(codes.unique().tolist()) == {0, 1, 2, 3}  # fallback, fits, outside, passthrough
    assert torch.equal(one[3], x[3])


def test_transform_takes_the_tiered_path_and_matches_one_box():
    """`Affine` on an fp32 image passes tiers to ops.resample; the same call without them gives
    the same bits."""
    import torchio_b200 as tio

    calls = []
    raw = ops.resample

    def spy(*a, **kw):
        out = raw(*a, **kw)
        calls.append((a, kw, out))
        return out

    g = torch.Generator().manual_seed(11)
    x = torch.rand((8, 1, 64, 64, 64), generator=g).cuda()
    torch.manual_seed(3)
    ops.resample = spy
    try:
        batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(8)])})
        tio.Affine(scales=(0.8, 1.1), degrees=(-10, 10))(batch)
    finally:
        ops.resample = raw
    ((a, kw, out),) = calls
    assert kw["tiers"] is not None and len(kw["tiers"][1]) >= 2
    assert torch.equal(out, raw(*a, **{**kw, "tiers": None}))


def test_tiered_entry_point_refuses_bad_runs():
    x = torch.zeros((2, 1, 8, 8, 8), device="cuda")
    packed = tables.SpatialTables(np.tile(np.eye(4, dtype=np.float32)[:3].reshape(12), (2, 1)), None,
                                  np.zeros(2, np.uint8), [])
    fill = torch.zeros(1, device="cuda")
    with pytest.raises(RuntimeError, match="runs hold"):
        _call(x, packed, fill, 24, (np.arange(2, dtype=np.int32), [(1, 20)]))
    with pytest.raises(RuntimeError, match="ascending"):
        _call(x, packed, fill, 24, (np.arange(2, dtype=np.int32), [(1, 22), (1, 20)]))
