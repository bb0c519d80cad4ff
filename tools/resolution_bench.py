"""Time the Anisotropy / Resize kernels against the reference's op sequences on the same GPU.

    python tools/resolution_bench.py [--batch 32] [--size 256]

Inputs are generated from a seed on the device.  Each kernel (through its `ops` function, tables
built beforehand) and the reference's torch ops are timed with CUDA events over ``--iters`` /
``--reference-iters`` calls after warm-up, and their outputs are compared bit for bit:

    aniso_axis{0,1,2}      Anisotropy per-instance, (B, 1, S^3) fp32, downsampling=(1.5, 5),
                           forced to one axis                                   8 B/voxel
    aniso_i16_axis{0,1,2}  the same on an int16 label map (nearest)             4 B/voxel
    aniso_shared           Anisotropy shared path (B = 1), (1, 1, S^3) fp32, axis 0, factor 3
    resize_down / _up      Resize (B, 1, S^3) fp32 -> S/2 and 1.25 S           4 (in + out) B

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

import resolution_cases as ref  # noqa: E402
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


def _measure(name, ours, reference, moved_bytes, args) -> dict:
    for _ in range(args.warmup):
        ours()
    kernel_ms = _time(ours, args.iters)
    reference()  # warm-up
    reference_ms = _time(reference, args.reference_iters)
    got, want = ours(), reference()
    identical = got.dtype == want.dtype and got.shape == want.shape and torch.equal(
        got.contiguous().view(torch.uint8), want.contiguous().view(torch.uint8))
    del got, want
    rate = moved_bytes / (kernel_ms * 1e-3)
    return {"kernel": name, "bytes": moved_bytes, "kernel_ms": round(kernel_ms, 4),
            "reference_ms": round(reference_ms, 3), "speedup": round(reference_ms / kernel_ms, 1),
            "TB_per_s": round(rate / 1e12, 3), "fraction_of_3.35TBps": round(rate / PEAK_BYTES_PER_S, 3),
            "bit_identical": identical}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reference-iters", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("resolution_bench: needs a CUDA device")

    b, s = args.batch, args.size
    shape = (s, s, s)
    g = torch.Generator(device="cuda").manual_seed(1)
    results = []
    gen = torch.Generator().manual_seed(2)
    factors = (torch.rand(b, generator=gen) * 3.5 + 1.5).tolist()  # downsampling=(1.5, 5)
    image = torch.rand((b, 1, *shape), generator=g, device="cuda")
    labels = torch.randint(0, 120, (b, 1, *shape), generator=g, device="cuda", dtype=torch.int16)
    for data, tag, linear in ((image, "", True), (labels, "_i16", False)):
        mode = "linear" if linear else "nearest"
        for axis in range(3):
            axes = [axis] * b
            tabs = tables.anisotropy_instance_tables(shape, axes, factors, linear)
            results.append(_measure(
                f"aniso{tag}_axis{axis}", lambda d=data, t=tabs, lin=linear: ops.axis_resample(d, *t, linear=lin),
                lambda d=data, a=axes, m=mode: ref.anisotropy_per_instance(d, a, factors, m),
                2 * data.numel() * data.element_size(), args))
    del labels
    single = image[:1].contiguous()
    del image
    idx, lam = tables.anisotropy_shared_tables(shape, 0, 3.0, True)
    results.append(_measure("aniso_shared", lambda: ops.interpolate(single, shape, idx, lam),
                            lambda: ref.anisotropy_shared(single, 0, 3.0, "linear"), 2 * single.numel() * 4, args))
    del single
    volumes = torch.rand((b, 1, *shape), generator=g, device="cuda")
    for name, n in (("resize_down", s // 2), ("resize_up", s * 5 // 4)):
        target = (n, n, n)
        idx, lam = tables.resize_tables(shape, target, True)
        results.append(_measure(name, lambda t=target, i=idx, w=lam: ops.interpolate(volumes, t, i, w),
                                lambda t=target: ref.resize(volumes, t, "linear"),
                                4 * (volumes.numel() + b * n ** 3), args))
    print(json.dumps({**_card(), "results": results}))
    if not all(r["bit_identical"] for r in results):
        raise SystemExit(1)


if __name__ == "__main__":
    main()
