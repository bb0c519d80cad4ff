"""Time the label-map kernels against the reference's op sequences on the same GPU.

    python tools/label_maps_bench.py [--batch 32] [--size 256] [--onehot-batch 4] [--classes 16]

Label maps are piecewise-constant blocks of random labels generated from a seed on the device.
Each kernel (through its `ops` function, tables built beforehand) and the reference's torch ops are
timed with CUDA events over ``--iters`` / ``--reference-iters`` calls after warm-up, and their
outputs are compared bit for bit:

    lut       RemapLabels, 100 entries, (B, 1, S^3) int16     4 B/voxel  (2 in, 2 out)
    lut_u8    the same on a uint8 map (256-entry shared LUT)   2 B/voxel
    contour   Contour, (B, 1, S^3) int16                       6 B/voxel  (2 in, 4 out)
    onehot    OneHot, (b, 1, S^3) int16, K classes             2 + 4K B/voxel
    argmax    OneHot's inverse, (b, K, S^3) fp32               4K + 4 B/voxel

Prints the card, its power limit and maximum SM clock, and each kernel's rate over the bytes it
must move against 3.35 TB/s (H100 SXM HBM3, data sheet).
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

import label_map_cases as ref  # noqa: E402
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


def _blocks(shape, high, seed, dtype):
    """Labels in [0, high) constant over 4^3 blocks."""
    b, c, s = shape[0], shape[1], shape[2]
    g = torch.Generator(device="cuda").manual_seed(seed)
    coarse = torch.randint(0, high, (b, c, s // 4, s // 4, s // 4), generator=g, device="cuda")
    return coarse.repeat_interleave(4, 2).repeat_interleave(4, 3).repeat_interleave(4, 4).to(dtype)


def _measure(name, ours, reference, voxels, bytes_per_voxel, args) -> dict:
    for _ in range(args.warmup):
        ours()
    kernel_ms = _time(ours, args.iters)
    reference()  # warm-up
    reference_ms = _time(reference, args.reference_iters)
    got, want = ours(), reference()
    identical = got.dtype == want.dtype and got.shape == want.shape and torch.equal(
        got.contiguous().view(torch.uint8), want.contiguous().view(torch.uint8))
    del got, want
    rate = bytes_per_voxel * voxels / (kernel_ms * 1e-3)
    return {"kernel": name, "voxels": voxels, "bytes_per_voxel": bytes_per_voxel,
            "kernel_ms": round(kernel_ms, 4), "reference_ms": round(reference_ms, 3),
            "speedup": round(reference_ms / kernel_ms, 1), "TB_per_s": round(rate / 1e12, 3),
            "fraction_of_3.35TBps": round(rate / PEAK_BYTES_PER_S, 3), "bit_identical": identical}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--onehot-batch", type=int, default=4)
    ap.add_argument("--classes", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reference-iters", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("label_maps_bench: needs a CUDA device")

    b, s, k = args.batch, args.size, args.classes
    results = []
    labels = _blocks((b, 1, s), 120, 1, torch.int16)
    voxels = labels.numel()
    remapping = {v: (v * 37 + 5) % 100 for v in range(100)}
    keys, values = tables.label_lut(list(remapping.items()), labels.dtype, labels.device)
    results.append(_measure("lut", lambda: ops.label_lut(labels, keys, values, identity=True),
                            lambda: ref.remap(labels, remapping), voxels, 4, args))
    labels_u8 = labels.to(torch.uint8)
    keys8, values8 = tables.label_lut(list(remapping.items()), labels_u8.dtype, labels.device)
    results.append(_measure("lut_u8", lambda: ops.label_lut(labels_u8, keys8, values8, identity=True),
                            lambda: ref.remap(labels_u8, remapping), voxels, 2, args))
    del labels_u8
    results.append(_measure("contour", lambda: ops.label_contour(labels), lambda: ref.contour(labels),
                            voxels, 6, args))
    del labels

    small = _blocks((args.onehot_batch, 1, s), k, 2, torch.int16)
    results.append(_measure("onehot", lambda: ops.onehot_classes(small, k), lambda: ref.one_hot(small, k),
                            small.numel(), 2 + 4 * k, args))
    scores = ref.one_hot(small, k) * torch.rand((args.onehot_batch, k, s, s, s), device="cuda")
    del small
    results.append(_measure("argmax", lambda: ops.channel_argmax(scores), lambda: ref.one_hot_inverse(scores),
                            scores[:, 0].numel(), 4 * k + 4, args))
    print(json.dumps({**_card(), "results": results}))
    if not all(r["bit_identical"] for r in results):
        raise SystemExit(1)


if __name__ == "__main__":
    main()
