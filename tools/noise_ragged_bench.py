"""Time exact `Noise` on the odd MNI 1 mm grid, where every draw is ragged.

    python tools/noise_ragged_bench.py [--batches 1 3 32] [--iters 5]

On (B, 1, 181, 217, 181) fp32 (7 109 137 voxels per element, an odd number, so a draw of the
whole batch is never a multiple of 16 normals) it times, with CUDA events, over ``--iters`` calls
after a warm-up call, the arms alternating within every iteration:

  noise     `Noise(std=(0, 0.25))` on a batch resident on the device: the normals replayed there
  compose   bench.py's six-transform Compose (Affine, ElasticDeformation, BiasField, Blur, Noise,
            Gamma) on the same batch
  replay    `ops.randn_mt19937` alone for the batch's draw, started at an unaligned stream word
  host      what such a draw cost when it stayed on the host: `torch.randn` of the batch's shape
            on a CPU generator into pinned memory, then the copy to the device

It prints the card, its power limit and the SM clock read while the kernels run, then
min / median / max per arm and batch.
"""

from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torchio_b200 as tio  # noqa: E402
from bench import pipeline_spec  # noqa: E402
from torchio_b200 import ops  # noqa: E402

SHAPE = (181, 217, 181)


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader", f"--id={torch.cuda.current_device()}"],
                             capture_output=True, text=True, timeout=30)
        power, max_clock, clock = (v.strip() for v in out.stdout.strip().split(","))
        info.update(power_limit=power, max_sm_clock=max_clock, sm_clock_now=clock)
    except (OSError, ValueError, subprocess.SubprocessError):
        info.update(power_limit="unknown", max_sm_clock="unknown", sm_clock_now="unknown")
    return info


def _timed(fn) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 3, 32])
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", torch.cuda.current_device())
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        noise = tio.Noise(std=(0, 0.25))
        compose = tio.Compose([getattr(tio, n)(**kw) for n, kw in pipeline_spec("full")], copy=False)
    card = None
    rows = []
    for b in args.batches:
        shape = (b, 1, *SHAPE)
        x = torch.rand(shape, generator=torch.Generator().manual_seed(b)).to(dev)
        affines = [tio.AffineMatrix() for _ in range(b)]
        batch = lambda: tio.SubjectsBatch({"t1": tio.ImagesBatch(x.clone(), list(affines))})  # noqa: E731
        n = x.numel()
        generator = torch.Generator().manual_seed(7)

        def host():
            z = torch.empty(shape, dtype=torch.float32, pin_memory=True)
            torch.randn(shape, generator=generator, out=z)
            return z.to(dev, non_blocking=True)

        arms = {"noise": lambda: noise(batch()), "compose": lambda: compose(batch()),
                "replay": lambda: ops.randn_mt19937(7, 12345, n, dev), "host": host}
        for fn in arms.values():  # warm-up of every arm
            fn()
        torch.cuda.synchronize()
        times = {name: [] for name in arms}
        for it in range(args.iters):
            for name, fn in arms.items():
                times[name].append(_timed(fn))
            if card is None and it == args.iters // 2:
                card = _card()  # read while the loop keeps the GPU busy
        for name, v in times.items():
            rows.append({"batch": b, "arm": name, "min_ms": round(min(v), 3),
                         "median_ms": round(statistics.median(v), 3), "max_ms": round(max(v), 3)})
        del x
        torch.cuda.empty_cache()
    print(json.dumps({"card": card or _card(), "shape": ["B", 1, *SHAPE], "iters": args.iters,
                      "torch": torch.__version__, "host_threads": torch.get_num_threads()}))
    for row in rows:
        print(json.dumps(row))


if __name__ == "__main__":
    main()
