"""Time Ghosting on the GPU against the reference's op sequence.

    python tools/ghosting_bench.py [--batch 32] [--size 256] [--iters 20]

Inputs come from a seed.  Cases: (B, 1, S^3) fp32 and int16 ghosted along each axis with 4 and with
10 ghosts, and one 181 x 217 x 181 fp32 volume (the 1 mm MNI grid) along each axis.  For each it
reports:
- the mean time of `ops.ghosting` over ``--iters`` calls after warm-up (CUDA events around each
  call; the input is restored between calls, outside the timed window, because the pass is in
  place);
- the rate over the algorithmic bytes (one read and one write of the batch), and its share of
  3.35 TB/s (H100 SXM HBM3, data sheet);
- one call of the reference's op sequence (tests/ghosting_cases.py) on the same GPU, after one
  warm-up call;
- the peak memory each allocates beyond the input (``torch.cuda.max_memory_allocated``);
- the largest difference between the two outputs, over the output's range (units for int16).
It also runs `Ghosting(num_ghosts=(4, 10), intensity=(0.5, 1))` on the fp32 batch with torch's sync
debug mode set to "warn" and reports how many synchronising calls it flagged.  Prints the card, its
power limit and maximum SM clock.
"""

from __future__ import annotations

import argparse
import json
import sys
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tools"))

import ghosting_cases as ref  # noqa: E402
import torchio_b200 as tio  # noqa: E402
from spike_bench import _card, _peak_extra, _time_in_place  # noqa: E402
from torchio_b200 import ops  # noqa: E402
from torchio_b200.transforms.ghosting import ghosting_table  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12  # H100 SXM HBM3, data sheet


def _case(name, data, axis, n_ghosts, iters):
    b = data.shape[0]
    ghosts, axes, strengths = [n_ghosts] * b, [axis] * b, [0.5 + 0.5 * e / max(b - 1, 1) for e in range(b)]
    table, ax, active = ghosting_table(ghosts, axes, strengths, 0.0, data.shape[2:])
    params = {"num_ghosts": ghosts, "axis": axes, "intensity": strengths, "restore": 0.0,
              "_batched_keys": ["num_ghosts", "axis", "intensity"]}
    work = torch.empty_like(data)
    ms = _time_in_place(lambda: ops.ghosting(work, table, ax, active), work, data, iters)
    work.copy_(data)
    ours_mem, got = _peak_extra(lambda: ops.ghosting(work, table, ax, active))
    ref.reference_ops(data, params)  # warm-up: cuFFT plans
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    expected = ref.reference_ops(data, params)
    end.record()
    end.synchronize()
    ref_ms = start.elapsed_time(end)
    del expected
    ref_mem, expected = _peak_extra(lambda: ref.reference_ops(data, params))
    e = expected.double()
    span = (float(e.max() - e.min()) or 1.0) if data.dtype.is_floating_point else 1.0
    max_diff = float((got.double() - e).abs().max())
    del e
    algorithmic = 2 * data.numel() * data.element_size()
    rate = algorithmic / (ms * 1e-3)
    print(json.dumps({
        "case": name, "shape": list(data.shape), "dtype": str(data.dtype).replace("torch.", ""), "axis": axis,
        "ghosts": n_ghosts, "kernel_ms": round(ms, 3), "algorithmic_gb": round(algorithmic / 1e9, 3),
        "tb_per_s": round(rate / 1e12, 3), "share_of_peak": round(rate / PEAK_BYTES_PER_S, 3),
        "reference_ms": round(ref_ms, 2), "peak_mem_gb": round(ours_mem / 1e9, 6),
        "reference_peak_mem_gb": round(ref_mem / 1e9, 3), "max_diff": max_diff,
        "max_diff_over_range": max_diff / span}), flush=True)
    del work, got, expected
    torch.cuda.empty_cache()


def _sync_check(data) -> None:
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(x)) for x in data])
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            tio.Ghosting(num_ghosts=(4, 10), intensity=(0.5, 1), copy=False)(batch)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    # the first warning only announces the (prototype) debug mode itself
    flagged = [str(w.message) for w in caught
               if "synchroniz" in str(w.message).lower() and "prototype feature" not in str(w.message)]
    print(json.dumps({"sync_debug_flagged": len(flagged), "messages": flagged[:3]}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    print(json.dumps({"card": _card()}), flush=True)
    b, s = args.batch, args.size
    g = torch.Generator(device="cuda").manual_seed(1)
    signed = torch.randn(b, 1, s, s, s, generator=g, device="cuda") * 100
    for axis in (0, 1, 2):
        for n_ghosts in (4, 10):
            _case("fp32", signed, axis, n_ghosts, args.iters)
    int16 = (signed * 10).to(torch.int16)
    for axis in (0, 1, 2):
        for n_ghosts in (4, 10):
            _case("int16", int16, axis, n_ghosts, args.iters)
    del int16
    _sync_check(signed.clone())
    del signed
    torch.cuda.empty_cache()
    mni = torch.randn(1, 1, 181, 217, 181, generator=g, device="cuda") * 100
    for axis in (0, 1, 2):
        _case("mni_fp32", mni, axis, 4, args.iters)


if __name__ == "__main__":
    main()
