"""PatchAggregator against the reference on CPU: the restated op sequence regenerates every fixture of
tests/golden/generate_aggregator.py bit for bit, the host box resolution and the scaled locations
are the reference's, the constructor, attributes and errors equal it, and the C entry points check
their arguments before any launch."""

from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

import aggregator_cases as ac
import torchio_b200 as tio
from oracle.aggregator import OpSequence
from torchio_b200 import _native, ops
from torchio_b200.patches import PatchLocation

CASES = ac.CASES


@pytest.mark.parametrize("name", list(CASES))
def test_op_sequence_regenerates_the_fixture(name):
    case = CASES[name]
    got = ac.drive(case, OpSequence, PatchLocation, buffers=lambda aggregator, key: aggregator.buffers[key])
    ac.check_against_fixture(case, got)


BOXED = [n for n in CASES if "boxes" in ac.load_fixture(n)]


def test_most_cases_pin_their_boxes():
    assert len(BOXED) >= 25


@pytest.mark.parametrize("name", BOXED)
def test_host_boxes_are_the_references(name):
    case = CASES[name]
    fixture = ac.load_fixture(name)
    aggregator = tio.PatchAggregator(**ac.ctor(case))
    shape = ac.patch_shape(case)
    for (index, size), want in zip(ac.locations(case), ac.probe_rows(fixture["boxes"]), strict=True):
        dst_lo, dst_len, src_lo, src_len = aggregator._box(PatchLocation(index=index, size=size), shape)
        if want is None:  # the reference raised: the extents differ
            assert dst_len != src_len
        elif min(want[1]) == 0:  # nothing written
            assert min(dst_len) == 0
        else:
            assert (dst_lo, dst_len, src_lo) == want
            assert src_len == dst_len or case["deviation"]  # the broadcast case: refused, see below


@pytest.mark.parametrize("name", [n for n in CASES if CASES[n]["output_shape"] is not None])
def test_scaled_locations_are_the_references(name):
    case = CASES[name]
    scale = tuple(case["output_shape"][a] / case["shape"][a] for a in range(3))
    got = [[*loc.scaled(scale).index, *loc.scaled(scale).size]
           for loc in (PatchLocation(index=i, size=s) for i, s in ac.locations(case))]
    np.testing.assert_array_equal(np.asarray(got), ac.load_fixture(name)["scaled"])


def test_grid_locations_are_the_samplers():
    subject = tio.Subject(t1=tio.ScalarImage(torch.zeros(1, *ac.ODD)))
    for overlap in [(0, 0, 0), (2, 3, 4), (3, 5, 1)]:
        sampler = tio.GridSampler(subject, patch_size=ac.PATCH, patch_overlap=overlap)
        assert [(loc.index, loc.size) for loc in sampler.locations] == ac.grid_locations(ac.ODD, ac.PATCH, overlap)


# ---- errors the product raises before touching a device ---------------------------------------------

@pytest.mark.parametrize("name", [n for n in CASES if "error" in ac.load_fixture(n)])
def test_fixture_errors_are_raised_before_any_launch(name):
    case = CASES[name]
    before = ops.launches()
    got = ac.drive(case, tio.PatchAggregator, PatchLocation)
    assert ops.launches() == before
    ac.check_against_fixture(case, got)


def test_broadcast_box_is_refused():
    case = CASES["aggregator_broadcast_average"]
    assert "error" not in ac.load_fixture(case["name"])  # the reference broadcasts
    got = ac.drive(case, tio.PatchAggregator, PatchLocation)
    assert got["error"]["type"] == case["deviation"]


def test_constructor_and_attributes():
    a = tio.PatchAggregator(spatial_shape=(20, 18, 22), overlap_mode="hann", patch_overlap=3, output_shape=(10, 9, 11))
    assert a.input_spatial_shape == (20, 18, 22)
    assert a.spatial_shape == (10, 9, 11)
    assert a.overlap_mode == "hann"
    assert a.patch_overlap == (3, 3, 3)
    b = tio.PatchAggregator(spatial_shape=(10, 10, 10))
    assert b.overlap_mode == "crop" and b.patch_overlap == (0, 0, 0) and b.spatial_shape == (10, 10, 10)
    with pytest.raises(ValueError, match="overlap_mode"):
        tio.PatchAggregator(spatial_shape=(10, 10, 10), overlap_mode="invalid")


def test_missing_key_lists_the_available_ones():
    with pytest.raises(KeyError, match=r"No output for key None. Available: \[\]"):
        tio.PatchAggregator(spatial_shape=(4, 4, 4)).get_output()
    with pytest.raises(KeyError, match="'seg'"):
        tio.PatchAggregator(spatial_shape=(4, 4, 4)).get_output("seg")


def test_whole_batch_is_checked_first():
    """More locations than patches, or a dict whose second key fails, add nothing."""
    loc = PatchLocation(index=(0, 0, 0), size=(4, 4, 4))
    a = tio.PatchAggregator(spatial_shape=(4, 4, 4), overlap_mode="average")
    before = ops.launches()
    with pytest.raises(IndexError):
        a.add_batch(torch.zeros(1, 1, 4, 4, 4), [loc, loc])
    with pytest.raises(RuntimeError, match="Bool"):
        a.add_batch({"x": torch.zeros(1, 1, 4, 4, 4), "y": torch.zeros(1, 1, 4, 4, 4, dtype=torch.bool)}, [loc])
    with pytest.raises(RuntimeError, match="must match"):
        a.add_batch(torch.zeros(1, 3, 3, 4, 4), [loc])
    with pytest.raises(NotImplementedError, match="broadcasting"):
        a.add_batch(torch.zeros(1, 3, 4, 1, 4), [loc])
    assert ops.launches() == before
    assert a._outputs == {} and a._device is None


# ---- the C entry points ---------------------------------------------------------------------------

def test_entry_points_reject_bad_arguments_without_launching():
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    box = np.array([[0, 0, 0, 2, 2, 2, 0, 0, 0, 0]], dtype=np.int32)

    def call(patches=p, out=p + 4096, counts=p + 8192, dtype=0, mode=1, C=1, I=4, J=4, K=4, B=1, pi=2, pj=2, pk=2,
             n=1, boxes=box, boxes_device=p + 12288, window=p + 16384):
        _native.call("tio_aggregate_patches", patches, out, counts, dtype, mode, C, I, J, K, B, pi, pj, pk, n,
                     None if boxes is None else boxes.ctypes.data, boxes_device, window, None)

    def bad(row, **kw):
        b = box.copy()
        b[0] = row
        call(boxes=b, **kw)

    before = ops.launches()
    for missing in ("patches", "out", "boxes", "boxes_device"):
        with pytest.raises(RuntimeError, match="null pointer"):
            call(**{missing: None})
    with pytest.raises(RuntimeError, match="null counts"):
        call(counts=None)
    with pytest.raises(RuntimeError, match="null window"):
        call(mode=2, window=None)
    with pytest.raises(RuntimeError, match="mode 3 not in 0..2"):
        call(mode=3)
    with pytest.raises(RuntimeError, match="unknown dtype 9"):
        call(dtype=9)
    with pytest.raises(RuntimeError, match="hann needs a floating-point dtype"):
        call(mode=2, dtype=3)
    with pytest.raises(RuntimeError, match="bad shape"):
        call(n=2)  # more boxes than patches
    with pytest.raises(RuntimeError, match="bad shape"):
        call(K=0)
    with pytest.raises(RuntimeError, match="outside the buffer on axis 2"):
        bad([0, 0, 3, 2, 2, 5, 0, 0, 0, 0])
    with pytest.raises(RuntimeError, match="empty or outside the buffer on axis 0"):
        bad([1, 0, 0, 1, 2, 2, 0, 0, 0, 0])
    with pytest.raises(RuntimeError, match="outside its patch on axis 1"):
        bad([0, 0, 0, 2, 2, 2, 0, 1, 0, 0])
    with pytest.raises(RuntimeError, match="names patch 1 of 1"):
        bad([0, 0, 0, 2, 2, 2, 0, 0, 0, 1])
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_aggregate_finish", p, None, p, 0, 1, 64, None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_aggregate_finish", p, p, p, 0, 1, 0, None)
    with pytest.raises(RuntimeError, match="unknown dtype 11"):
        _native.call("tio_aggregate_finish", p, p, p, 11, 1, 64, None)
    assert ops.launches() == before
