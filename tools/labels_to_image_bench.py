"""Time LabelsToImage's one-pass kernel against the reference's op sequence on the same GPU.

    python tools/labels_to_image_bench.py [--batch 32] [--size 256] [--labels 32] [--iters 20]

A (B, 1, S, S, S) int16 label map with ``--labels`` labels is generated from a seed on the device,
per-element means and stds are drawn on the host.  ``ops.labels_to_image`` and the reference's
per-label torch ops (randn_like, * std, + mean, == label, cast, * mask, +=) are each timed with
CUDA events over ``--iters`` launches after warm-up, from the same CUDA generator state, and their
outputs are compared bit for bit.  Prints the card, its power limit and maximum SM clock, and the
kernel's rate over the 6 bytes per voxel it must move (int16 in, fp32 out) against 3.35 TB/s.
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

from labels_to_image_cases import reference_image  # noqa: E402
from torchio_b200 import ops, tables  # noqa: E402

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
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--labels", type=int, default=32)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reference-iters", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("labels_to_image_bench: needs a CUDA device")

    b, s, n = args.batch, args.size, args.labels
    labels = torch.empty((b, 1, s, s, s), dtype=torch.int16, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(1)
    labels.copy_(torch.randint(0, n, labels.shape, generator=g, device="cuda", dtype=torch.int16))
    rng = np.random.default_rng(2)
    mean = rng.uniform(0.1, 0.9, (b, n)).astype(np.float32)
    std = rng.uniform(0.01, 0.1, (b, n)).astype(np.float32)
    params = {"means": [{k: float(mean[e, k]) for k in range(n)} for e in range(b)],
              "stds": [{k: float(std[e, k]) for k in range(n)} for e in range(b)]}
    values, draw, mean_t, std_t = tables.label_synthesis_tables(params["means"], params["stds"], b)

    def ours():
        return ops.labels_to_image(labels, values, mean_t, std_t, draw)

    for _ in range(args.warmup):
        ours()
    kernel_ms = _time(ours, args.iters)
    reference_image(labels, params["means"], params["stds"])  # warm-up
    reference_ms = _time(lambda: reference_image(labels, params["means"], params["stds"]), args.reference_iters)

    torch.cuda.manual_seed(3)
    got = ours()
    torch.cuda.manual_seed(3)
    want = reference_image(labels, params["means"], params["stds"])
    identical = torch.equal(got.view(torch.int32), want.view(torch.int32))
    mismatches = int((got.view(torch.int32) != want.view(torch.int32)).sum())

    voxels = b * s**3
    rate = 6 * voxels / (kernel_ms * 1e-3)
    print(json.dumps({
        **_card(), "shape": [b, 1, s, s, s], "labels": n, "voxels": voxels,
        "kernel_ms": round(kernel_ms, 4), "reference_ms": round(reference_ms, 3),
        "speedup": round(reference_ms / kernel_ms, 1),
        "TB_per_s": round(rate / 1e12, 3), "fraction_of_3.35TBps": round(rate / PEAK_BYTES_PER_S, 3),
        "bit_identical": identical, "mismatches": mismatches,
    }))
    if not identical:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
