"""Time HistogramStandardization and compute_histogram_landmarks on the GPU.

    python tools/histogram_bench.py [--batch 32] [--size 256] [--volumes 64]

Inputs come from a seed: (B, 1, S^3) volumes with 60 % zero background.  For fp32 and int16 it
times, with CUDA events after warm-up, each pass of the transform separately (the batched select,
the table build, the in-place map), the whole transform, and one call of the reference's op sequence
from tests/histogram_cases.py on the same GPU, and checks that both outputs are bit-identical.  It then
times compute_histogram_landmarks over ``--volumes`` device-resident volumes of S^3.

Bytes per pass: the select reads every voxel once per radix level (3 levels: 3 x element size per
voxel), the map reads and writes it (2 x element size).  The algorithmic minimum is one read for
the statistics and one read + one write for the map (3 x element size; 12 B/voxel for fp32, of
which the map's 8 B are the DESIGN §3 figure).  Shares are against 3.35 TB/s (H100 SXM HBM3, data
sheet).  Prints the card, its power limit and maximum SM clock.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import histogram_cases as ref  # noqa: E402
import torchio_b200 as tio  # noqa: E402
from torchio_b200 import ops  # noqa: E402
from torchio_b200.transforms import compute_histogram_landmarks  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                              f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        power, clock = (v.strip() for v in out.stdout.strip().split(","))
        info.update(power_limit=power, max_sm_clock=clock)
    except (OSError, ValueError, subprocess.SubprocessError):
        info.update(power_limit="unknown", max_sm_clock="unknown")
    return info


def _time(fn, iters: int) -> float:
    """Mean milliseconds per call over ``iters`` calls, CUDA events."""
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def _volumes(b: int, s: int, dtype: torch.dtype, seed: int) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((b, 1, s, s, s), generator=g, device="cuda").mul_(300)
    x[torch.rand(x.shape, generator=g, device="cuda") < 0.6] = 0
    return x.to(dtype)


def _rate(ms: float, nbytes: float) -> dict:
    return {"ms": round(ms, 3), "TB/s": round(nbytes / ms / 1e9, 3),
            "share": round(nbytes / ms / 1e9 / (PEAK_BYTES_PER_S / 1e12), 3)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--volumes", type=int, default=64)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("histogram_bench needs a CUDA device")
    result = {"card": _card(), "batch": args.batch, "size": args.size}
    lm = torch.linspace(0, 100, 13)
    qs = np.asarray([100.0 * q for q in ref.DEFAULT_QUANTILES]) / 100.0
    for dtype in (torch.float32, torch.int16):
        data = _volumes(args.batch, args.size, dtype, 3)
        vox = data.numel()
        es = data.element_size()
        work = data.clone()
        values, weights, _, nan = ops.quantiles_batched(work, qs)
        tables = ops.histogram_tables(values, weights, nan, lm.cuda())
        t_select = _time(lambda: ops.quantiles_batched(work, qs), args.iters)
        t_tables = _time(lambda: ops.histogram_tables(values, weights, nan, lm.cuda()), args.iters)
        t_map = _time(lambda: ops.histogram_map(work, tables, 13), args.iters)  # input changes; the time does not

        transform = tio.HistogramStandardization(lm, copy=False)

        def run_transform():
            work.copy_(data)
            batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(work[b])) for b in range(len(work))])
            batch.images["t1"].data = work
            return transform(batch).images["t1"].data

        t_copy = _time(lambda: work.copy_(data), args.iters)
        t_total = _time(run_transform, args.iters) - t_copy
        got = run_transform().clone()
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        expected = ref.reference_output(data, lm, (0.01, 0.99))
        end.record()
        end.synchronize()
        t_ref = start.elapsed_time(end)  # one call: the host sorts dominate it
        result[str(dtype).split(".")[1]] = {
            "select": _rate(t_select, 3 * es * vox),
            "tables_ms": round(t_tables, 4),
            "map": _rate(t_map, 2 * es * vox),
            "transform": _rate(t_total, 5 * es * vox),
            "transform_vs_algorithmic": _rate(t_total, 3 * es * vox),
            "reference_ops_ms": round(t_ref, 2),
            "bit_identical": bool(torch.equal(got, expected)),
        }
        del data, work, got, expected
        torch.cuda.empty_cache()
    images = [tio.ScalarImage(_volumes(1, args.size, torch.float32, 5 + i)[0]) for i in range(args.volumes)]
    torch.cuda.synchronize()
    t_lm = _time(lambda: compute_histogram_landmarks(images), 1)
    result["landmarks_64_volumes_ms"] = round(t_lm, 1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
