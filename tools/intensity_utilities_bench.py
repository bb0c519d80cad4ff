"""Time Clamp, Mask and Swap on the GPU against the reference's op sequences.

    python tools/intensity_utilities_bench.py [--batch 32] [--size 256] [--iters 20]

Inputs come from a seed: (B, 1, S^3) volumes of fp32 and int16, and an int16 label map with 60 %
background in 8^3 blocks (labels 0..4).  For each case it times the kernel with CUDA events after warm-up (mean
over ``--iters`` calls), times one call of the reference's op sequence from
tests/intensity_utility_cases.py on the same GPU, and checks that both outputs are bit-identical:
- Swap at its defaults (patch 15, 100 iterations, per instance), and on one S^3 volume with patch 64
  and 100 iterations (one thread-block cluster does all the work);
- Mask in place (int16 images take an int outside value, so the dtype is kept), nonzero and labels;
- Clamp.
Clamp and Mask are reported as a share of 3.35 TB/s (H100 SXM HBM3, data sheet) against their
algorithmic bytes: Clamp one read and one write per voxel; Mask the mask read once plus the writes
of the outside voxels.  Prints the card, its power limit and maximum SM clock.
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

import intensity_utility_cases as ref  # noqa: E402
from torchio_b200 import ops  # noqa: E402
from torchio_b200.transforms.clamp_mask_swap import (clamp_bounds, sample_swap_locations, swap_table,  # noqa: E402
                                                     where_outside)

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


def _once(fn) -> tuple[float, torch.Tensor]:
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    out = fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end), out


def _report(name, dtype, ms, ref_ms, equal, algorithmic_bytes=None):
    line = {"case": name, "dtype": str(dtype).replace("torch.", ""), "kernel_ms": round(ms, 4),
            "reference_ms": round(ref_ms, 2), "bit_identical": bool(equal)}
    if algorithmic_bytes is not None:
        rate = algorithmic_bytes / (ms * 1e-3)
        line.update(algorithmic_gb=round(algorithmic_bytes / 1e9, 3), tb_per_s=round(rate / 1e12, 3),
                    share_of_peak=round(rate / PEAK_BYTES_PER_S, 3))
    print(json.dumps(line), flush=True)


def _swap(name, data, locations, patch, per_instance, iters):
    rows = locations if per_instance else [locations]
    table = swap_table(rows, patch)
    work = data.clone()
    ms = _time(lambda: ops.swap_patches(work, table, patch), iters)
    got = data.clone()
    ops.swap_patches(got, table, patch)
    ref_ms, expected = _once(lambda: ref.swap_reference(data, locations, patch, per_instance))
    _report(name, data.dtype, ms, ref_ms, torch.equal(got, expected))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps({"card": _card()}), flush=True)
    b, s = args.batch, args.size
    g = torch.Generator(device="cuda").manual_seed(1)
    # 60 % background in 8^3 blocks (a mask made of regions, not of scattered voxels), labels 1..4
    coarse = (torch.rand(1, 1, s // 8, s // 8, s // 8, generator=g, device="cuda") * 10).to(torch.int16) - 5
    labels = coarse.clamp_(min=0).repeat_interleave(8, 2).repeat_interleave(8, 3).repeat_interleave(8, 4).contiguous()
    background = float((labels == 0).double().mean())
    print(json.dumps({"mask_background_fraction": round(background, 4)}), flush=True)
    vox = s ** 3
    for dtype in (torch.float32, torch.int16):
        data = (torch.randn(b, 1, s, s, s, generator=g, device="cuda") * 300).to(dtype)
        esize = data.element_size()

        torch.manual_seed(0)
        locations = [sample_swap_locations((s, s, s), (15, 15, 15), 100) for _ in range(b)]
        _swap("swap_default_per_instance", data, locations, (15, 15, 15), True, args.iters)
        _swap("swap_b1_patch64", data[:1].contiguous(), sample_swap_locations((s, s, s), (64, 64, 64), 100),
              (64, 64, 64), False, args.iters)

        outside = where_outside(dtype, 0)
        for label_name, keys, ref_labels in (("nonzero", None, None),
                                             ("labels", ops_keys(labels, [1, 3]), [1, 3])):
            element = labels[0]
            work = data.clone()
            ms = _time(lambda: ops.mask(work, element, keys, outside), args.iters)
            got = ops.mask(data.clone(), element, keys, outside)
            ref_ms, expected = _once(lambda: ref.mask_reference(data, labels, "seg", ref_labels, 0))
            mask = element.bool() if keys is None else (element == 1) | (element == 3)
            outside_voxels = b * int((~mask).sum())
            _report(f"mask_{label_name}_in_place", dtype, ms, ref_ms, torch.equal(got, expected),
                    vox * labels.element_size() + outside_voxels * esize)

        lo, hi = clamp_bounds(dtype, -50, 200)
        ms = _time(lambda: ops.clamp(data, lo, hi), args.iters)
        got = ops.clamp(data, lo, hi)
        ref_ms, expected = _once(lambda: ref.clamp_reference(data, -50, 200))
        _report("clamp", dtype, ms, ref_ms, torch.equal(got, expected), 2 * b * vox * esize)
        del data, got, expected, work


def ops_keys(labels, values):
    from torchio_b200 import tables

    return tables.label_lut([(v, 1) for v in values], labels.dtype, labels.device)[0]


if __name__ == "__main__":
    main()
