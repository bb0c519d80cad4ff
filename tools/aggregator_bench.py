"""Time PatchAggregator on the GPU against the reference's op sequence and the reference's own path.

    python tools/aggregator_bench.py [--iters 3] [--host-batches 2] [--out results.json]

Workloads, patches from a seed and resident in HBM before timing (one 256^3 volume, GridSampler's
grid, batches of 8 patches):
  (a) 96^3 patches, overlap 16, "hann", C = 4 fp32;
  (b) 64^3 patches, overlap 32, "average", C = 32 fp16;
  (c) 96^3 patches, overlap 16, "crop", C = 1 int64 labels;
  (d) (a) with output_shape = 128^3 (48^3 patches).
For each it reports, from CUDA events:
- ms per add_batch and per whole volume (every add_batch plus get_output), mean of ``--iters`` volumes
  after a warm-up volume;
- algorithmic bytes (each patch read once; each covered voxel's C channels and, for average and hann,
  its one count read and written once per add_batch; get_output reads the buffer and count and writes
  the result) and their share of 3.35 TB/s (H100 SXM HBM3, data sheet);
- the same for the reference's op sequence (oracle/aggregator.py) on the same CUDA tensors, one
  volume after a warm-up volume;
- the reference's own path (each batch moved to the host with .cpu(), accumulated there), ms per
  add_batch over the first ``--host-batches`` batches of one volume;
- whether the output is bit-identical to the op sequence's.
Prints the card, its power limit and maximum SM clock, and each workload as a JSON line; ``--out``
also writes all of it to one JSON file.
"""

from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))

from aggregator_cases import grid_locations  # noqa: E402
from oracle.aggregator import OpSequence  # noqa: E402
from spike_bench import _card  # noqa: E402
import torchio_b200 as tio  # noqa: E402
from torchio_b200.patches import PatchLocation  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet
SIZE, BATCH = 256, 8
WORKLOADS = {
    "a_hann_c4_f32": dict(patch=96, overlap=16, mode="hann", channels=4, dtype=torch.float32, output=None),
    "b_average_c32_f16": dict(patch=64, overlap=32, mode="average", channels=32, dtype=torch.float16, output=None),
    "c_crop_c1_i64": dict(patch=96, overlap=16, mode="crop", channels=1, dtype=torch.int64, output=None),
    "d_hann_c4_f32_half": dict(patch=96, overlap=16, mode="hann", channels=4, dtype=torch.float32, output=128),
}


def _inputs(w):
    """(batches of (patches, locations), output shape, patch shape) of a workload."""
    locs = [PatchLocation(index=i, size=s)
            for i, s in grid_locations((SIZE,) * 3, (w["patch"],) * 3, (w["overlap"],) * 3)]
    p = w["patch"] if w["output"] is None else round(w["patch"] * w["output"] / SIZE)
    g = torch.Generator(device="cuda").manual_seed(0)
    batches = []
    for start in range(0, len(locs), BATCH):
        chunk = locs[start:start + BATCH]
        shape = (len(chunk), w["channels"], p, p, p)
        if w["dtype"].is_floating_point:
            data = torch.rand(shape, generator=g, device="cuda").to(w["dtype"])
        else:
            data = torch.randint(0, 20, shape, generator=g, device="cuda", dtype=w["dtype"])
        batches.append((data, chunk))
    return batches, (SIZE if w["output"] is None else w["output"],) * 3, p


def _bytes(w, batches, out_shape, aggregator) -> tuple[list[int], int]:
    """Algorithmic bytes of each add_batch and of get_output."""
    elem = batches[0][0].element_size()
    counted = w["mode"] != "crop"
    per_batch = []
    for data, chunk in batches:
        covered = torch.zeros(out_shape, dtype=torch.bool)
        for row, loc in enumerate(chunk):
            lo, n, _, _ = aggregator._box(loc, tuple(data.shape[2:]))
            covered[lo[0]:lo[0] + n[0], lo[1]:lo[1] + n[1], lo[2]:lo[2] + n[2]] = True
        vox = int(covered.sum())
        rw = 1 if w["mode"] == "crop" else 2  # crop writes; average and hann read and write
        per_batch.append(data.numel() * elem + vox * (w["channels"] * rw + (2 if counted else 0)) * elem)
    total_vox = out_shape[0] * out_shape[1] * out_shape[2]
    out_elem = elem if w["dtype"].is_floating_point else 4
    finish = total_vox * (w["channels"] * elem + elem + w["channels"] * out_elem) if counted else 0
    return per_batch, finish


def _volume(make, batches):
    """CUDA-event times (ms) of each add_batch and of get_output for one volume."""
    aggregator = make()
    events = [torch.cuda.Event(enable_timing=True) for _ in range(len(batches) + 2)]
    events[0].record()
    for t, (data, chunk) in enumerate(batches):
        aggregator.add_batch(data, chunk)
        events[t + 1].record()
    out = aggregator.get_output()
    events[-1].record()
    torch.cuda.synchronize()
    steps = [events[t].elapsed_time(events[t + 1]) for t in range(len(batches) + 1)]
    return steps[:-1], steps[-1], out


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--iters", type=int, default=3)
    parser.add_argument("--host-batches", type=int, default=2)
    parser.add_argument("--out", default=None, help="also write the results as JSON to this file")
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("aggregator_bench: no CUDA device")
    result = {"card": _card(), "workloads": {}}
    print(json.dumps(result["card"]), flush=True)
    for name, w in WORKLOADS.items():
        batches, out_shape, p = _inputs(w)
        ctor = dict(spatial_shape=(SIZE,) * 3, overlap_mode=w["mode"], patch_overlap=w["overlap"],
                    output_shape=None if w["output"] is None else out_shape)
        per_batch_bytes, finish_bytes = _bytes(w, batches, out_shape, tio.PatchAggregator(**ctor))
        volume_bytes = sum(per_batch_bytes) + finish_bytes
        row = {"patch": p, "batches": len(batches), "bytes_per_volume": volume_bytes}
        for label, make in (("gpu", lambda: tio.PatchAggregator(**ctor)), ("op_sequence", lambda: OpSequence(**ctor))):
            _volume(make, batches)  # warm-up
            runs = [_volume(make, batches) for _ in range(args.iters if label == "gpu" else 1)]
            add_ms = sum(sum(r[0]) for r in runs) / len(runs)
            total_ms = add_ms + sum(r[1] for r in runs) / len(runs)
            row[label] = {
                "ms_per_add_batch": add_ms / len(batches),
                "ms_get_output": total_ms - add_ms,
                "ms_per_volume": total_ms,
                "add_batch_share_of_peak": sum(per_batch_bytes) / (add_ms * 1e-3) / PEAK_BYTES_PER_S,
                "volume_share_of_peak": volume_bytes / (total_ms * 1e-3) / PEAK_BYTES_PER_S,
            }
            row[f"_{label}_out"] = runs[-1][2]
        row["bit_identical"] = bool(torch.equal(_bits(row.pop("_gpu_out")), _bits(row.pop("_op_sequence_out"))))
        host = OpSequence(**ctor)
        torch.cuda.synchronize()
        start = time.perf_counter()
        for data, chunk in batches[:args.host_batches]:
            host.add_batch(data.cpu(), chunk)
        row["reference_host_path"] = {"ms_per_add_batch": (time.perf_counter() - start) * 1e3 / args.host_batches,
                                      "batches_timed": args.host_batches}
        result["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
        del batches, host
        torch.cuda.empty_cache()
    if args.out is not None:
        out = Path(args.out)
        out.parent.mkdir(parents=True, exist_ok=True)
        out.write_text(json.dumps(result, indent=1))


def _bits(t: torch.Tensor) -> torch.Tensor:
    view = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()]
    return t.contiguous().view(view)


if __name__ == "__main__":
    main()
