"""PatchAggregator test infrastructure: the fixture cases, their seeded patches and locations, and one
driver that runs a case through any aggregator class (the reference's, `oracle.aggregator.OpSequence`
or `torchio_b200.PatchAggregator`) and records what it returns in the fixtures' format.
``tests/golden/generate_aggregator.py`` runs the reference on these cases; nothing here is imported
by the product."""

from __future__ import annotations

import json

import numpy as np
import torch

from spike_cases import BF16, F16, F32, F64, GOLDEN, I8, I16, I32, I64, U8, as_stored

BOOL = torch.bool
ALL_DTYPES = [F32, F16, BF16, F64, U8, I8, I16, I32, I64, BOOL]
FLOATS = [F32, F16, BF16, F64]
SHORT = {F32: "f32", F16: "f16", BF16: "bf16", F64: "f64", U8: "u8", I8: "i8", I16: "i16", I32: "i32", I64: "i64",
         BOOL: "bool"}
ERROR_DTYPES = {"hann": [d for d in ALL_DTYPES if d not in FLOATS], "average": [BOOL], "crop": []}

ODD = (23, 17, 29)
PATCH = (8, 6, 10)
ONE = {"__default__": (1, F32)}


def grid_locations(shape, patch, overlap) -> list[tuple[tuple[int, int, int], tuple[int, int, int]]]:
    """GridSampler's (index, size) pairs (data/sampler.py:70-162) of an unpadded volume."""
    per_axis = []
    for a in range(3):
        step = max(patch[a] - overlap[a], 1)
        starts = list(range(0, shape[a] - patch[a] + 1, step))
        if not starts or starts[-1] != shape[a] - patch[a]:
            starts.append(max(shape[a] - patch[a], 0))
        per_axis.append(starts)
    return [((i, j, k), tuple(patch)) for i in per_axis[0] for j in per_axis[1] for k in per_axis[2]]


def _case(name, mode, *, shape=ODD, patch=PATCH, overlap=(0, 0, 0), keys=ONE, splits=(None,), order="grid",
          output_shape=None, locations=None, patch_shape=None, deviation=None):
    """``splits``: patches per add_batch call, None = the rest; get_output of every key follows each
    call.  ``order``: "grid", "shuffle" (a seeded permutation) or "duplicate" (every location twice,
    the second pass reversed).  ``patch_shape``: the spatial shape of the patches when it is not
    ``patch`` scaled to ``output_shape``.  ``deviation``: the error the product raises where the
    reference does not."""
    return dict(name=name, mode=mode, shape=shape, patch=patch, overlap=overlap, keys=keys, splits=splits,
                order=order, output_shape=output_shape, locations=locations, patch_shape=patch_shape,
                deviation=deviation)


_OVERLAPS = {"o0": (0, 0, 0), "o234": (2, 3, 4), "odd": (3, 5, 1)}
CASES_LIST = [
    *[_case(f"aggregator_grid_{mode}_{tag}", mode, overlap=ov, splits=(1, 3, None))
      for mode in ("crop", "average", "hann") for tag, ov in _OVERLAPS.items()],
    # patch axes of 1 and 2 points: hann windows [1] and [0.75, 0.75]
    *[_case(f"aggregator_axes12_{mode}", mode, shape=(5, 6, 13), patch=(1, 2, 5), overlap=(0, 1, 2))
      for mode in ("crop", "average", "hann")],
    _case("aggregator_duplicate_crop", "crop", overlap=(2, 3, 4), order="duplicate"),
    _case("aggregator_duplicate_average", "average", overlap=(2, 3, 4), order="duplicate"),
    _case("aggregator_shuffle_hann", "hann", overlap=(3, 5, 1), order="shuffle", splits=(7, None)),
    *[_case(f"aggregator_dict_{mode}", mode, shape=(13, 11, 15), overlap=(2, 3, 4), keys={"seg": (2, F32), "emb": (5, F32)},
            splits=(1, 3, None)) for mode in ("crop", "average", "hann")],
    # output_shape halves (20, 18, 22): corners and sizes of 3 * odd land on .5 and round to even
    *[_case(f"aggregator_output_{mode}", mode, shape=(20, 18, 22), patch=(6, 6, 6), overlap=(3, 3, 3),
            output_shape=(10, 9, 11)) for mode in ("crop", "average", "hann")],
    *[_case(f"aggregator_dtypes_{mode}", mode, shape=(11, 9, 13), patch=(4, 5, 6), overlap=(1, 2, 3),
            keys={SHORT[d]: (2, d) for d in ALL_DTYPES if d not in ERROR_DTYPES[mode]}, splits=(3, None))
      for mode in ("crop", "average", "hann")],
    # 2100 patches on one voxel pair: uint8 counts wrap at 256, int8 at 128, bf16 stops at 256, fp16 at 2048
    _case("aggregator_counts_wrap", "average", shape=(3, 3, 4), patch=(1, 1, 2),
          keys={SHORT[d]: (1, d) for d in (U8, I8, F16, BF16)}, locations=[((1, 1, 1), (1, 1, 2))] * 2100),
    *[_case(f"aggregator_error_hann_{SHORT[d]}", "hann", shape=(9, 8, 7), patch=(4, 4, 4), overlap=(2, 2, 2),
            keys={"__default__": (1, d)}) for d in (I16, BOOL)],
    _case("aggregator_error_average_bool", "average", shape=(9, 8, 7), patch=(4, 4, 4), overlap=(2, 2, 2),
          keys={"__default__": (1, BOOL)}),
    # the third location runs past the end of the volume: its box is shorter than the patch
    *[_case(f"aggregator_error_mismatch_{mode}", mode, shape=(9, 8, 7), patch=(4, 4, 4),
            locations=[((0, 0, 0), (4, 4, 4)), ((2, 2, 2), (4, 4, 4)), ((6, 0, 0), (4, 4, 4))])
      for mode in ("crop", "average")],
    # a (1, 4, 4) patch broadcast over a (3, 4, 4) box: the reference accepts it, the product refuses
    _case("aggregator_broadcast_average", "average", shape=(6, 6, 6), patch=(3, 4, 4), patch_shape=(1, 4, 4),
          locations=[((0, 0, 0), (3, 4, 4))], deviation="NotImplementedError"),
    # negative corners and boxes that end past the volume, resolved by Python's slice rules
    *[_case(f"aggregator_slices_{mode}", mode, shape=(12, 10, 9), patch=(5, 4, 3), overlap=(2, 2, 2),
            locations=[((-8, 1, 0), (5, 4, 3)), ((7, 0, 6), (10, 4, 3)), ((3, -7, -4), (5, 4, 3)),
                       ((0, 0, 0), (5, 4, 3))])
      for mode in ("crop", "average")],
]
CASES = {c["name"]: c for c in CASES_LIST}


def locations(case) -> list[tuple[tuple[int, int, int], tuple[int, int, int]]]:
    locs = list(case["locations"]) if case["locations"] is not None else grid_locations(
        case["shape"], case["patch"], case["overlap"])
    if case["order"] == "shuffle":
        perm = torch.randperm(len(locs), generator=torch.Generator().manual_seed(seed(case)))
        locs = [locs[int(p)] for p in perm]
    elif case["order"] == "duplicate":
        locs = locs + locs[::-1]
    return locs


def patch_shape(case) -> tuple[int, int, int]:
    if case["patch_shape"] is not None:
        return tuple(case["patch_shape"])
    if case["output_shape"] is None:
        return tuple(case["patch"])
    return tuple(round(case["patch"][a] * case["output_shape"][a] / case["shape"][a]) for a in range(3))


def seed(case) -> int:
    return sum(ord(ch) * (i + 1) for i, ch in enumerate(case["name"])) % 100003


def random_patches(n: int, channels: int, shape, dtype: torch.dtype, seed_value: int,
                   device="cpu") -> torch.Tensor:
    """(n, C, *shape) of ``dtype``: floats over [-2, 3), integers over most of their range (so that
    sums wrap), bools half true."""
    g = torch.Generator().manual_seed(seed_value)
    u = torch.rand((n, channels, *shape), generator=g, dtype=torch.float64)
    if dtype == BOOL:
        t = u < 0.5
    elif dtype.is_floating_point:
        t = (u * 5 - 2).to(dtype)
    else:
        info = torch.iinfo(dtype)
        lo, hi = max(info.min, -(2 ** 40)), min(info.max, 2 ** 40)
        t = torch.floor(u * (hi - lo) + lo).to(torch.int64).to(dtype)
    return t.to(device)


def batch_ranges(case) -> list[tuple[int, int]]:
    total, out, start = len(locations(case)), [], 0
    for size in case["splits"]:
        stop = total if size is None else min(total, start + size)
        out.append((start, stop))
        start = stop
    return out


def batch_tensors(case, t: int, n: int, device="cpu") -> dict[str, torch.Tensor]:
    return {key: random_patches(n, channels, patch_shape(case), dtype, seed(case) * 31 + t * 7 + i, device)
            for i, (key, (channels, dtype)) in enumerate(case["keys"].items())}


def ctor(case) -> dict:
    kw = dict(spatial_shape=case["shape"], overlap_mode=case["mode"], patch_overlap=case["overlap"])
    if case["output_shape"] is not None:
        kw["output_shape"] = case["output_shape"]
    return kw


def drive(case, aggregator_cls, location_cls, device="cpu", buffers=None) -> dict:
    """Run ``case`` through ``aggregator_cls``: {"out_{t}_{key}": stored output, "dtype_...": str,
    "alias_...": bool} after each add_batch call t, or "error" {"type", "message", "batch"} where a
    call raised.  ``buffers(aggregator, key)``: the aggregator's own buffer of ``key``, for the alias
    check."""
    aggregator = aggregator_cls(**ctor(case))
    locs = [location_cls(index=i, size=s) for i, s in locations(case)]
    record: dict = {}
    for t, (start, stop) in enumerate(batch_ranges(case)):
        tensors = batch_tensors(case, t, stop - start, device)
        batch = tensors["__default__"] if list(tensors) == ["__default__"] else tensors
        try:
            aggregator.add_batch(batch, locs[start:stop])
        except Exception as exc:  # noqa: BLE001  (the fixture records what was raised)
            record["error"] = {"type": type(exc).__name__, "message": str(exc), "batch": t}
            return record
        for key in tensors:
            out = aggregator.get_output(None if key == "__default__" else key)
            record[f"out_{t}_{key}"] = as_stored(out).copy()  # crop returns the live buffer: snapshot it
            record[f"dtype_{t}_{key}"] = str(out.dtype)
            if buffers is not None:
                record[f"alias_{t}_{key}"] = out is buffers(aggregator, key)
    return record


def load_fixture(name: str) -> dict:
    with np.load(GOLDEN / f"{name}.npz") as z:
        out = {k: z[k] for k in z.files}
    for key in out:
        if key == "error" or key.startswith("dtype_"):
            out[key] = json.loads(out[key].tobytes().decode())
    return out


def check_against_fixture(case, got: dict) -> None:
    """``got`` (a `drive` record) equals the fixture of ``case`` bit for bit, aliasing included when
    ``got`` records it."""
    fixture = load_fixture(case["name"])
    if "error" in fixture:
        assert "error" in got, f"{case['name']}: expected {fixture['error']}"
        assert got["error"]["type"] == fixture["error"]["type"], got["error"]
        assert got["error"]["batch"] == fixture["error"]["batch"]
        return
    assert "error" not in got, got.get("error")
    outs = sorted(k for k in fixture if k.startswith("out_"))
    assert outs == sorted(k for k in got if k.startswith("out_"))
    for name in outs:
        want, have = fixture[name], got[name]
        assert want.dtype == have.dtype and want.shape == have.shape, (name, want.dtype, have.dtype)
        assert np.array_equal(want.view(np.uint8), np.ascontiguousarray(have).view(np.uint8)), name
        assert fixture["dtype_" + name[4:]] == got["dtype_" + name[4:]]
        if "alias_" + name[4:] in got:
            assert bool(fixture["alias_" + name[4:]]) == got["alias_" + name[4:]], name


def probe_rows(fixture_boxes: np.ndarray) -> list[tuple]:
    """The fixture's "boxes" rows as (dst lo, dst extent, src lo) or None where the reference raised."""
    rows = []
    for r in fixture_boxes:
        rows.append(None if r[0] == -2 else (tuple(int(v) for v in r[0:3]), tuple(int(v) for v in r[3:6]),
                                             tuple(int(v) for v in r[6:9])))
    return rows
