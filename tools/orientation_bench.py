"""Time `tio_permute` (Reorient / Transpose) on the GPU against the reference's op sequence.

    python tools/orientation_bench.py [--batch 32] [--size 256] [--iters 20]

Inputs come from a seed: (B, 1, S^3) volumes of fp32, int16 and uint8.  Three permutations: PSR from
RAS (K moves, with a flip: the tile transpose), Transpose (K moves, no flip) and ARS (I <-> J, K stays
last: whole rows).  For each it times the kernel with CUDA events after warm-up (mean over ``--iters``
calls), times one call of the reference's op sequence (torch.flip per flipped axis, then
permute(...).contiguous(), reorient.py:63-91) on the same GPU, and checks that both outputs are
bit-identical.  Rates are against 2 x the tensor's bytes (one read, one write) and shares against
3.35 TB/s (H100 SXM HBM3, data sheet).  Prints the card, its power limit and maximum SM clock.
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

from torchio_b200 import ops  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet

# name -> (output axis -> input axis, flip bits by input axis)
PERMUTATIONS = {"PSR": ((1, 2, 0), 0b010), "Transpose": ((2, 1, 0), 0), "ARS": ((1, 0, 2), 0)}


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


def _reference(x: torch.Tensor, perm, bits: int) -> torch.Tensor:
    for ax in range(3):
        if bits >> ax & 1:
            x = torch.flip(x, [ax + 2])
    return x.permute(0, 1, *(p + 2 for p in perm)).contiguous()


def _events_ms(fn, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def main() -> None:
    parser = argparse.ArgumentParser()
    parser.add_argument("--batch", type=int, default=32)
    parser.add_argument("--size", type=int, default=256)
    parser.add_argument("--iters", type=int, default=20)
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("orientation_bench needs a CUDA device")
    print(json.dumps({"card": _card()}))
    shape = (args.batch, 1, args.size, args.size, args.size)
    g = torch.Generator(device="cuda").manual_seed(0)
    base = torch.randint(0, 1 << 30, shape, dtype=torch.int32, device="cuda", generator=g)
    for dtype in (torch.float32, torch.int16, torch.uint8):
        x = base.view(torch.float32).clone() if dtype == torch.float32 else (base % 20000).to(dtype)
        nbytes = 2 * x.numel() * x.element_size()
        for name, (perm, bits) in PERMUTATIONS.items():
            for _ in range(3):
                ops.permute(x, perm, bits)
            torch.cuda.synchronize()
            ms = _events_ms(lambda: ops.permute(x, perm, bits), args.iters)
            ref_ms = _events_ms(lambda: _reference(x, perm, bits), 1)
            equal = torch.equal(ops.permute(x, perm, bits).view(torch.uint8),
                                _reference(x, perm, bits).view(torch.uint8))
            rate = nbytes / (ms * 1e-3)
            print(json.dumps({"case": name, "dtype": str(dtype).replace("torch.", ""), "shape": list(shape),
                              "kernel_ms": round(ms, 4), "reference_ms": round(ref_ms, 3),
                              "tb_per_s": round(rate / 1e12, 3), "share_of_3.35": round(rate / PEAK_BYTES_PER_S, 3),
                              "bit_identical": bool(equal)}))
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
