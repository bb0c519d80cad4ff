"""Time the B-spline (orders 2-7) prefilter passes and pull on the GPU.

    python tools/bspline_bench.py [--batch 32] [--size 256] [--iters 5] [--orders 2 3 5 7]

Workload: (B, 1, S^3) fp32 from a seed, per-instance geometry of
``Affine(scales=(0.9, 1.1), degrees=(-10, 10))`` followed by ``ElasticDeformation()`` folded into one
matrix and one control grid per element (what ``Spatial`` samples).  For each order it reports,
from CUDA events after a warm-up call:
- the whole prefilter and the pull, in ms, from CUDA events, with the rate over the bytes the
  algorithm needs (prefilter: 24 B/voxel, read the source plus three fp32 writes and two fp32
  reads; pull: read the coefficients once and write the output, 8 B/voxel) and its share of
  3.35 TB/s (H100 SXM HBM3, data sheet);
- each prefilter pass (K, J, I: the three `bspline_prefilter_kernel` launches of a call, in launch
  order) and the pull kernel, in ms, from a `torch.profiler` trace of separate calls (kernel
  durations; the trace slows the host, not the kernels), each pass at 8 B/voxel;
- the pull's voxels/s and taps/s ((n+1)^3 per voxel);
- the linear K1 call (`ops.resample`) on the same geometry in the same run, as the relative cost.
The reference's own GPU time is not measured: it needs torch-interpol.
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
sys.path.insert(0, str(ROOT / "tools"))

from spike_bench import _card  # noqa: E402
from torchio_b200 import ops, tables  # noqa: E402
from torchio_b200.data import AffineMatrix  # noqa: E402
from torchio_b200.transforms.spatial import Spatial  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet


def _events(fn, iters: int) -> float:
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def _kernel_times(fn, iters: int) -> dict:
    """Mean device time of each prefilter pass (K, J, I in launch order) and of the pull kernel over
    ``iters`` calls of ``fn``, from a profiler trace."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    kernels = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "bspline_" in e.name),
                     key=lambda e: e.time_range.start)
    prefilter = [e.time_range.elapsed_us() / 1e3 for e in kernels if "prefilter" in e.name]
    pull = [e.time_range.elapsed_us() / 1e3 for e in kernels if "pull" in e.name]
    if len(prefilter) != 3 * iters or len(pull) != iters:
        raise RuntimeError(f"expected {3 * iters} prefilter and {iters} pull kernels, traced "
                           f"{len(prefilter)} and {len(pull)}")
    out = {f"prefilter_{axis}": float(np.mean(prefilter[t::3])) for t, axis in enumerate("KJI")}
    out["pull_kernel"] = float(np.mean(pull))
    return out


def main():
    parser = argparse.ArgumentParser()
    parser.add_argument("--batch", type=int, default=32)
    parser.add_argument("--size", type=int, default=256)
    parser.add_argument("--iters", type=int, default=5)
    parser.add_argument("--orders", type=int, nargs="+", default=[2, 3, 5, 7])
    args = parser.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bspline_bench needs a GPU")
    b, s = args.batch, args.size
    shape = (s, s, s)
    torch.manual_seed(0)
    x = torch.randn(b, 1, *shape, device="cuda")
    spatial = Spatial(scales=(0.9, 1.1), degrees=(-10, 10), max_displacement=7.5)
    forwards, cps, _ = spatial._sample_batch_fast(b, None, shape, AffineMatrix(np.eye(4)))
    eye = np.eye(4)
    packed = tables.spatial_tables(forwards, cps, b, eye, eye, per_instance=True, has_target=False)
    mat, cp, flags = ops.upload(x.device, packed.mat, packed.cp, packed.flags)
    vox = b * s**3
    rows = {"card": _card(), "batch": b, "size": s, "orders": {}}

    def k1():
        return ops.resample(x, mat, cp, flags, (1, 1, 1), (1, 1, 1), affine_first=True, mode=ops.LINEAR,
                            fill=None)
    k1_ms = _events(k1, args.iters)
    rows["k1_linear_ms"] = k1_ms
    for order in args.orders:
        passes = {}
        total_ms = _events(lambda: ops.bspline_prefilter(x, order), args.iters)
        passes["prefilter_total_ms"] = total_ms
        passes["prefilter_total_GBps"] = 24 * vox / total_ms / 1e6
        passes["prefilter_total_share"] = 24 * vox / (total_ms * 1e-3) / PEAK_BYTES_PER_S
        c = ops.bspline_prefilter(x, order)

        def pull():
            return ops.bspline_resample(c, x, mat, cp, flags, (1, 1, 1), (1, 1, 1), affine_first=True,
                                        order=order)
        pull_ms = _events(pull, args.iters)
        for name, ms in _kernel_times(lambda: (ops.bspline_prefilter(x, order), pull()), args.iters).items():
            passes[f"{name}_ms"] = ms
            passes[f"{name}_share"] = 8 * vox / (ms * 1e-3) / PEAK_BYTES_PER_S
        passes["pull_ms"] = pull_ms
        passes["pull_share"] = 8 * vox / (pull_ms * 1e-3) / PEAK_BYTES_PER_S
        passes["pull_voxels_per_s"] = vox / (pull_ms * 1e-3)
        passes["pull_taps_per_s"] = vox * (order + 1) ** 3 / (pull_ms * 1e-3)
        passes["relative_to_k1"] = (total_ms + pull_ms) / k1_ms
        rows["orders"][order] = passes
        del c
    print(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
