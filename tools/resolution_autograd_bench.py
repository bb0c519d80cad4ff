"""Time the Resize / Anisotropy adjoint kernels against the reference's backward on the same GPU.

    python tools/resolution_autograd_bench.py [--batch 32] [--size 256] [--iters 20]

Inputs and cotangents are generated from a seed on the device.  Each adjoint (through its `ops`
function, tables built beforehand; the call includes its table upload) and the reference's
backward of its op sequence (`torch.autograd.grad` of F.interpolate / torch.gather and the four
elementwise ops, forward built once with ``retain_graph``) are timed with CUDA events over
``--iters`` calls after warm-up:

    resize_down / resize_up    Resize (B, 1, S^3) fp32 -> S/2 and 1.25 S, trilinear
    aniso_axis{0,1,2}          Anisotropy per-instance, (B, 1, S^3) fp32, factor 3 on one axis

Algorithmic bytes: grad_out read + grad_in written, 4 B each.  For the Resize cases also the bytes
the separable alternative (three 1-D gather passes, K then J then I, fp32 intermediates) must move
at least, and its time at 3.35 TB/s: a fused time below it means no separable schedule can be
faster.  Prints the card, its power limit and maximum SM clock, and each rate against 3.35 TB/s
(H100 SXM HBM3, data sheet).
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

import resolution_cases as ref  # noqa: E402
from torchio_b200 import ops, tables  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet


def _card() -> dict:
    info = {"name": torch.cuda.get_device_name()}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader",
                              f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        power, clock, current = (v.strip() for v in out.stdout.strip().split(","))
        info.update(power_limit=power, max_sm_clock=clock, sm_clock_at_start=current)
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


def _separable_bytes(batch: int, shape, target) -> int:
    """Least bytes of three 1-D adjoint passes, K then J then I: each reads its input and writes its
    output once (the cheapest order for both cases here)."""
    (i, j, k), (oi, oj, ok) = shape, target
    sizes = [oi * oj * ok, oi * oj * k, oi * j * k, i * j * k]
    return 4 * batch * sum(a + b for a, b in zip(sizes, sizes[1:]))


def _entry(ours_ms: float, ref_ms: float, nbytes: int) -> dict:
    return {"ms": round(ours_ms, 4), "reference_backward_ms": round(ref_ms, 4), "speedup": round(ref_ms / ours_ms, 2),
            "bytes": nbytes, "gb_per_s": round(nbytes / ours_ms / 1e6, 1),
            "hbm_share": round(nbytes / (ours_ms * 1e-3) / PEAK_BYTES_PER_S, 3)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    b, s = args.batch, args.size
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.rand((b, 1, s, s, s), device="cuda", generator=gen)
    result = {"card": _card(), "shape": [b, 1, s, s, s], "iters": args.iters, "cases": {}}

    for name, target in (("resize_down", (s // 2,) * 3), ("resize_up", (s * 5 // 4,) * 3)):
        adjoint = tables.resize_adjoint_tables((s,) * 3, target, True)
        g = torch.randn((b, 1, *target), device="cuda", generator=gen)
        ours = _time(lambda: ops.interpolate_backward(g, (s,) * 3, *adjoint), args.iters)
        leaf = x.detach().requires_grad_()
        y = ref.resize(leaf, target, "linear")
        theirs = _time(lambda: torch.autograd.grad(y, leaf, g, retain_graph=True), args.iters)
        entry = _entry(ours, theirs, 4 * (g.numel() + x.numel()))
        sep = _separable_bytes(b, (s,) * 3, target)
        entry.update(separable_min_bytes=sep, separable_floor_ms=round(sep / PEAK_BYTES_PER_S * 1e3, 4))
        result["cases"][name] = entry
        del g, y, leaf
        torch.cuda.empty_cache()

    g = torch.randn_like(x)
    for axis in range(3):
        axes, factors = [axis] * b, [3.0] * b
        ax, _, _, w = tables.anisotropy_instance_tables((s,) * 3, axes, factors, True)
        ptr, ent = tables.anisotropy_instance_adjoint_tables((s,) * 3, axes, factors, True)
        ours = _time(lambda: ops.axis_resample_backward(g, ax, w, ptr, ent, linear=True), args.iters)
        leaf = x.detach().requires_grad_()
        y = ref.anisotropy_per_instance(leaf, axes, factors, "linear")
        theirs = _time(lambda: torch.autograd.grad(y, leaf, g, retain_graph=True), args.iters)
        result["cases"][f"aniso_axis{axis}"] = _entry(ours, theirs, 8 * x.numel())
        del y, leaf
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
