"""Time the first intensity pass and the exact-noise normals as two launches and as one.

    python tools/pass1_normals_bench.py [--batch 32] [--size 256] [--iters 20]

On the bench shape (B x 1 x S^3 fp32, a 6^3 coarse bias grid, per-element blur sigmas in [0, 2]
voxels, one draw of B*S^3 normals; inputs from a seed) it times, with CUDA events around each call,
over ``--iters`` calls after a warm-up, the arms alternating within every iteration:

  a   `ops.randn_mt19937` then the first pass alone (`ops.intensity_fused` with bias and the I axis):
      what the chain ran before its J/K pass
  b   `ops.intensity_pass1_with_normals`: the same two outputs from one persistent kernel
  chain_a / chain_b   the whole chain bias -> blur -> noise -> gamma with the normals supplied / with
      the draw handed over as (seed, offset)

and checks that b's outputs equal a's.  It prints the card, its power limit and the SM clock read
while the kernels run, then min / median / max per arm.  The seed and jump launches of the replay
are inside both arms.
"""

from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from torchio_b200 import ops, tables  # noqa: E402


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
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    b, s, dev = args.batch, args.size, "cuda"
    rng = np.random.default_rng(0)
    x = torch.rand((b, 1, s, s, s), device=dev)
    t = tables.blur_tables(rng.uniform(0.0, 2.0, (b, 3)), b)
    first = dict(coarse=torch.as_tensor(rng.normal(0, 0.5, (b, 1, 6, 6, 6)).astype(np.float32)).to(dev),
                 taps=t.taps.to(dev), radius=t.radius.to(dev), big_r=t.big_r, axes_mask=t.axes_mask)
    rest = dict(mean=torch.zeros(b, device=dev), std=torch.as_tensor(rng.uniform(0, 0.25, b).astype(np.float32)).to(dev),
                noise_mode=1, gamma=torch.as_tensor(np.exp(rng.uniform(-0.3, 0.3, b)).astype(np.float32)).to(dev))
    seed, offset, n = 20240229, 0, x.numel()

    def arm_a():
        z = ops.randn_mt19937(seed, offset, n, dev)
        return ops.intensity_fused(x, **{**first, "axes_mask": first["axes_mask"] & 1}), z

    def arm_b():
        return ops.intensity_pass1_with_normals(x, seed, offset, **first)

    def chain_a():
        z = ops.randn_mt19937(seed, offset, n, dev).view(x.shape)
        return ops.intensity_fused(x, **first, **rest, z=z)

    def chain_b():
        return ops.intensity_fused(x, **first, **rest, z_replay=(seed, offset))

    arms = {"a_two_launches": arm_a, "b_one_kernel": arm_b, "chain_a": chain_a, "chain_b": chain_b}
    (want_first, want_z), (got_first, got_z) = arm_a(), arm_b()
    same = bool(torch.equal(got_first, want_first)) and bool(torch.equal(got_z.view(-1), want_z.view(-1)))
    del want_first, want_z, got_first, got_z
    same_chain = bool(torch.equal(chain_a(), chain_b()))
    for fn in arms.values():  # warm-up of every arm
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    card = None
    for it in range(args.iters):
        for name, fn in arms.items():
            times[name].append(_timed(fn))
        if it == args.iters // 2:
            card = _card()  # read while the loop keeps the GPU busy
    print(json.dumps({"card": card or _card(), "shape": list(x.shape), "iters": args.iters,
                      "pass1_and_normals_bit_identical": same, "chain_bit_identical": same_chain}))
    for name, v in times.items():
        print(json.dumps({"arm": name, "min_ms": round(min(v), 3), "median_ms": round(statistics.median(v), 3),
                          "max_ms": round(max(v), 3)}))


if __name__ == "__main__":
    main()
