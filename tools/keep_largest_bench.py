"""Time KeepLargestComponent on the GPU; needs an H100 (or any CUDA device) and fails without one.

    python tools/keep_largest_bench.py [--batch 32] [--size 256] [--iters 20]

Inputs come from a seed: (B, 1, S^3) label maps with ~40 labels on a smooth map (8^3 blocks) plus
1 % salt noise, so every label has many small components.  Workloads: int16 and uint8 with
labels=None and labels=[1], each under 26- and 6-connectivity, and int32 with labels=None (the
distinct-values path, which reads back the roots' values once).  Each call runs on a fresh copy of
the map (the transform works in place); the copy is timed on its own and subtracted.  Times are CUDA
events, the mean of ``--iters`` calls after a warm-up.

Rate: the algorithmic bytes (the map read once plus the removed voxels written) over the time, as a
share of 3.35 TB/s (H100 SXM HBM3, data sheet).  The workspace traffic is reported beside it: the
parent array (4 B/voxel) is written by the tile pass, read and rewritten by the compress pass and
read by the winner and write passes, the count array (4 B/voxel) is zeroed, and the map is read
again by the merge, winner and write passes: about 24 B/voxel plus three more reads of the map.

Baseline (int16, 26 neighbours): the reference's op sequence (tests/keep_largest_cases.py) on the
same CUDA batch for ONE element, with the C oracle's labeller standing in for SimpleITK (whose speed cannot be measured
here); B times it is what the batch would take.  Prints the card, its power limit and SM clock.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import keep_largest_cases as ref  # noqa: E402
from torchio_b200 import ops  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader", f"--id={torch.cuda.current_device()}"],
                             capture_output=True, text=True, timeout=30)
        power, max_clock, clock = (v.strip() for v in out.stdout.strip().split(","))
        info.update(power_limit=power, max_sm_clock=max_clock, sm_clock=clock)
    except (OSError, ValueError, subprocess.SubprocessError):
        info.update(power_limit="unknown", max_sm_clock="unknown", sm_clock="unknown")
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


def label_batch(batch: int, size: int, dtype: torch.dtype) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(17)
    blocks = (size + 7) // 8 + 1
    coarse = torch.randint(0, 40, (batch, 1, blocks, blocks, blocks), generator=g, device="cuda")
    smooth = coarse.repeat_interleave(8, 2).repeat_interleave(8, 3).repeat_interleave(8, 4)
    labels = smooth[:, :, 3:3 + size, 5:5 + size, 1:1 + size].contiguous()
    salt = torch.rand(labels.shape, generator=g, device="cuda") < 0.01
    labels[salt] = torch.randint(0, 40, labels.shape, generator=g, device="cuda")[salt]
    return labels.to(dtype)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("keep_largest_bench needs a CUDA device")
    print(json.dumps(_card()))
    workloads = [(dtype, labels, fully) for dtype in (torch.int16, torch.uint8) for labels in (None, [1])
                 for fully in (True, False)]
    workloads += [(torch.int32, None, True), (torch.int32, None, False)]
    for dtype, labels, fully in workloads:
        data = label_batch(args.batch, args.size, dtype)
        work = torch.empty_like(data)
        copy_ms = _time(lambda: work.copy_(data), args.iters)
        total_ms = _time(lambda: ops.keep_largest(work.copy_(data), labels, 0, fully), args.iters)
        ms = total_ms - copy_ms
        out, _ = ops.keep_largest(data.clone(), labels, 0, fully)
        removed = int((out != data).sum())
        vox = data.numel()
        algorithmic = vox * data.element_size() + removed * data.element_size()
        reference_ms = same = None
        if dtype == torch.int16 and fully:  # ~40 host round trips per element: measured on two workloads
            torch.cuda.synchronize()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            want = ref.keep_largest_element(data[0, 0], labels, 0, fully, ref.c_labeller)
            end.record()
            end.synchronize()
            reference_ms = start.elapsed_time(end)
            same = torch.equal(want, out[0, 0])
        print(json.dumps({
            "dtype": str(dtype).replace("torch.", ""), "labels": labels, "fully_connected": fully,
            "shape": list(data.shape), "ms": round(ms, 3), "copy_ms": round(copy_ms, 3),
            "removed_voxels": removed, "algorithmic_bytes": algorithmic,
            "rate_TBps": round(algorithmic / (ms * 1e-3) / 1e12, 3),
            "share_of_3.35TBps": round(algorithmic / (ms * 1e-3) / PEAK_BYTES_PER_S, 3),
            "workspace_bytes_per_voxel": 24, "workspace_TBps": round(24 * vox / (ms * 1e-3) / 1e12, 3),
            "reference_one_element_ms_c_labeller": reference_ms and round(reference_ms, 1),
            "reference_batch_estimate_ms": reference_ms and round(reference_ms * args.batch, 1),
            "element0_bit_identical": same,
        }))
        del data, work, out


if __name__ == "__main__":
    main()
