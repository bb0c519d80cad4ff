"""Generate the PatchAggregator golden vectors by running the UNMODIFIED reference on CPU.

TEST INFRASTRUCTURE, run like generate.py (the reference checkout plus the ``_shim/`` stubs):

    python tests/golden/generate_aggregator.py [case name ...]

For every case of ``tests/aggregator_cases.py`` it records what the reference's PatchAggregator
returns after each ``add_batch`` call (output, dtype and whether it is the internal buffer itself),
or the error it raised and in which call.  It also records, per location, the reference's
``PatchLocation.scaled`` result (``scaled``, (n, 6)) and where the reference writes a patch added
there (``boxes``, (n, 9): first destination voxel, extent, first source voxel), found by adding a
patch whose voxels hold their own index + 1 to a fresh aggregator; rows of -2 where that add raised.
"""

from __future__ import annotations

import json
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE / "_shim"))
sys.path.insert(1, "/root/reference/src")
sys.path.insert(2, str(HERE.parent))

import torchio as tio  # noqa: E402  (the reference)
from torchio.data.patch import PatchLocation  # noqa: E402

import aggregator_cases as ac  # noqa: E402


def _json(obj) -> np.ndarray:
    return np.frombuffer(json.dumps(obj).encode(), dtype=np.uint8)


def _probe(case, location) -> list[int]:
    """Where the reference writes a patch added at ``location``, read back from the output."""
    kw = ac.ctor(case)
    kw["overlap_mode"] = "crop" if case["mode"] == "crop" else "average"
    probe = tio.PatchAggregator(**kw)
    shape = ac.patch_shape(case)
    code = torch.arange(1, int(np.prod(shape)) + 1, dtype=torch.int64).reshape(1, 1, *shape)
    try:
        probe.add_batch(code, [location])
    except RuntimeError:
        return [-2] * 9
    written = probe.get_output()[0].to(torch.int64)
    where = written.nonzero()
    if where.numel() == 0:
        return [-1, -1, -1, 0, 0, 0, -1, -1, -1]
    lo, hi = where.min(0).values, where.max(0).values + 1
    first = int(written[tuple(lo.tolist())]) - 1
    src = np.unravel_index(first, shape)
    return [*lo.tolist(), *(hi - lo).tolist(), *(int(s) for s in src)]


def run_case(case) -> dict:
    record = ac.drive(case, tio.PatchAggregator, PatchLocation,
                      buffers=lambda aggregator, key: aggregator._outputs[key])
    if "error" in record:
        record["error"] = _json(record["error"])
    for key in [k for k in record if k.startswith("dtype_")]:
        record[key] = _json(record[key])
    locs = [PatchLocation(index=i, size=s) for i, s in ac.locations(case)]
    if len(locs) <= 256:
        record["boxes"] = np.asarray([_probe(case, loc) for loc in locs], dtype=np.int32)
        if case["output_shape"] is not None:
            scale = tuple(case["output_shape"][a] / case["shape"][a] for a in range(3))
            record["scaled"] = np.asarray([[*loc.scaled(scale).index, *loc.scaled(scale).size] for loc in locs],
                                          dtype=np.int64)
    return record


def main():
    torch.set_num_threads(1)
    names = set(sys.argv[1:])  # optional: regenerate only these cases
    for name, case in ac.CASES.items():
        if names and name not in names:
            continue
        path = HERE / f"{name}.npz"
        np.savez_compressed(path, **run_case(case))
        print(f"{name:45s} {path.stat().st_size / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()
