"""Time Motion on the GPU against the reference's op sequence.

    python tools/motion_bench.py [--batch 32] [--size 256] [--iters 10]

Inputs come from a seed.  Cases: (B, 1, S^3) fp32 and int16 with N = 1, 2 and 4 rigid transforms
(degrees in U(-10, 10), translations in U(-5, 5) voxels per element), and one 181 x 217 x 181 fp32
volume (the 1 mm MNI grid) with N = 2.  For each it reports:
- the mean time of `ops.motion` over ``--iters`` calls after a warm-up call (CUDA events around
  each call);
- the rate over the algorithmic bytes (one read and one write of the batch: the gathers of the
  moved copies are served from the L2 and L1 caches), and its share of 3.35 TB/s (H100 SXM HBM3,
  data sheet);
- one call of the reference's op sequence (tests/motion_cases.py) on the same GPU, after one
  warm-up call;
- the peak memory each allocates beyond the input (``torch.cuda.max_memory_allocated``);
- the largest difference between the two outputs, over the output's range (units for int16).
Prints the card, its power limit and maximum SM clock.
"""

from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))

import motion_cases as ref  # noqa: E402
from spike_bench import _card, _peak_extra  # noqa: E402
from torchio_b200 import ops  # noqa: E402
from torchio_b200.transforms.motion import motion_theta  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet


def _params(b: int, n: int) -> dict:
    rng = np.random.default_rng(n)
    transforms = [[{"degrees": tuple(float(v) for v in rng.uniform(-10, 10, 3)),
                    "translation": tuple(float(v) for v in rng.uniform(-5, 5, 3))} for _ in range(n)]
                  for _ in range(b)]
    return {"transforms": transforms, "_batched_keys": ["transforms"]}


def _case(name, data, n, iters):
    b = data.shape[0]
    params = _params(b, n)
    theta, active = motion_theta(params["transforms"], data.shape[2:]), np.ones(b, dtype=bool)
    ops.motion(data, theta, active)  # warm-up
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(iters):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        out = ops.motion(data, theta, active)
        end.record()
        end.synchronize()
        total += start.elapsed_time(end)
        del out
    ms = total / iters
    ours_mem, got = _peak_extra(lambda: ops.motion(data, theta, active))
    ref.reference_ops(data, params)  # warm-up: cuFFT plans
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    expected = ref.reference_ops(data, params)
    end.record()
    end.synchronize()
    ref_ms = start.elapsed_time(end)
    del expected
    torch.cuda.empty_cache()
    ref_mem, expected = _peak_extra(lambda: ref.reference_ops(data, params))
    e = expected.double()
    span = (float(e.max() - e.min()) or 1.0) if data.dtype.is_floating_point else 1.0
    max_diff = float((got.double() - e).abs().max())
    del e
    algorithmic = 2 * data.numel() * data.element_size()
    rate = algorithmic / (ms * 1e-3)
    print(json.dumps({
        "case": name, "shape": list(data.shape), "dtype": str(data.dtype).replace("torch.", ""), "transforms": n,
        "kernel_ms": round(ms, 3), "algorithmic_gb": round(algorithmic / 1e9, 3), "tb_per_s": round(rate / 1e12, 3),
        "share_of_peak": round(rate / PEAK_BYTES_PER_S, 3), "reference_ms": round(ref_ms, 2),
        "speedup": round(ref_ms / ms, 2), "peak_mem_gb": round(ours_mem / 1e9, 3),
        "reference_peak_mem_gb": round(ref_mem / 1e9, 3), "max_diff": max_diff,
        "max_diff_over_range": max_diff / span}), flush=True)
    del got, expected
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    print(json.dumps({"card": _card()}), flush=True)
    b, s = args.batch, args.size
    g = torch.Generator(device="cuda").manual_seed(1)
    signed = torch.randn(b, 1, s, s, s, generator=g, device="cuda") * 100
    for n in (1, 2, 4):
        _case("fp32", signed, n, args.iters)
    int16 = (signed * 10).to(torch.int16)
    del signed
    torch.cuda.empty_cache()
    for n in (1, 2, 4):
        _case("int16", int16, n, args.iters)
    del int16
    torch.cuda.empty_cache()
    mni = torch.randn(1, 1, 181, 217, 181, generator=g, device="cuda") * 100
    _case("mni_fp32", mni, 2, args.iters)


if __name__ == "__main__":
    main()
