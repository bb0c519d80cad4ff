"""Time Spike on the GPU against the reference's op sequence.

    python tools/spike_bench.py [--batch 32] [--size 256] [--iters 20]

Inputs come from a seed.  Cases: (B, 1, S^3) fp32 non-negative (the peak is the sum), fp32 signed
(the peak needs the forward FFT), int16 non-negative, and one 181 x 217 x 181 fp32 signed volume
(the 1 mm MNI grid), each with 1 and with 16 spikes.  For each it reports:
- the mean time of `ops.spike` over ``--iters`` calls after warm-up (CUDA events around each call; the
  input is restored between calls, outside the timed window, because the pass is in place);
- the rate over the algorithmic bytes, computed from the shapes, and its share of 3.35 TB/s (H100
  SXM HBM3, data sheet): the sum path reads the batch twice and writes it once; the FFT path adds
  the K pass (one read of the batch, one complex64 half-spectrum write), the J pass (half-spectrum
  read and write) and the I pass (half-spectrum read);
- one call of the reference's op sequence (tests/spike_cases.py) on the same GPU, after one
  warm-up call;
- the peak memory each allocates beyond the input (``torch.cuda.max_memory_allocated``);
- the largest difference between the two outputs, over the output's range.
It also runs `Spike(num_spikes=(1, 3), intensity=(1, 3))` on the fp32 batch with torch's sync debug
mode set to "warn" and reports how many synchronising calls it flagged.  Prints the card, its power
limit and maximum SM clock.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import warnings
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import spike_cases as ref  # noqa: E402
import torchio_b200 as tio  # noqa: E402
from torchio_b200 import ops  # noqa: E402
from torchio_b200.transforms.spike import spike_table  # noqa: E402

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


def _time_in_place(fn, work: torch.Tensor, source: torch.Tensor, iters: int) -> float:
    """Mean milliseconds of ``fn()`` over ``iters`` calls, ``work`` reset from ``source`` before each."""
    work.copy_(source)
    fn()
    total = 0.0
    for _ in range(iters):
        work.copy_(source)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn()
        end.record()
        end.synchronize()
        total += start.elapsed_time(end)
    return total / iters


def _peak_extra(fn) -> tuple[int, object]:
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def _algorithmic_bytes(shape, esize: int, fft: bool) -> int:
    b, c, i, j, k = shape
    n = b * c * i * j * k
    total = 3 * n * esize
    if fft:
        half = b * c * i * j * (k // 2 + 1) * 8
        total += n * esize + half + 2 * half + half
    return total


def _case(name, data, n_spikes, fft, iters):
    b = data.shape[0]
    gen = torch.Generator().manual_seed(n_spikes)
    rows = [torch.rand(n_spikes, 3, generator=gen).tolist() for _ in range(b)]
    intensities = [1.0 + 2.0 * float(torch.rand(1, generator=gen)) for _ in range(b)]
    table, ratio = spike_table(rows, intensities, data.shape[2:])
    params = {"positions": rows, "intensity": intensities, "_batched_keys": ["positions", "intensity"]}
    work = torch.empty_like(data)
    ms = _time_in_place(lambda: ops.spike(work, table, ratio), work, data, iters)
    work.copy_(data)
    ours_mem, got = _peak_extra(lambda: ops.spike(work, table, ratio))
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
    span = float(expected.double().max() - expected.double().min()) or 1.0
    max_diff = float((got.double() - expected.double()).abs().max())
    algorithmic = _algorithmic_bytes(tuple(data.shape), data.element_size(), fft)
    rate = algorithmic / (ms * 1e-3)
    print(json.dumps({
        "case": name, "shape": list(data.shape), "dtype": str(data.dtype).replace("torch.", ""), "spikes": n_spikes,
        "kernel_ms": round(ms, 3), "algorithmic_gb": round(algorithmic / 1e9, 3), "tb_per_s": round(rate / 1e12, 3),
        "share_of_peak": round(rate / PEAK_BYTES_PER_S, 3), "reference_ms": round(ref_ms, 2),
        "peak_mem_gb": round(ours_mem / 1e9, 3), "reference_peak_mem_gb": round(ref_mem / 1e9, 3),
        "max_diff": max_diff, "max_diff_over_range": max_diff / span}), flush=True)
    del work, got, expected


def _sync_check(data) -> None:
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(x)) for x in data])
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            tio.Spike(num_spikes=(1, 3), intensity=(1, 3), copy=False)(batch)
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
    for n_spikes in (1, 16):
        _case("fp32_nonneg_sum_path", signed.abs(), n_spikes, False, args.iters)
    for n_spikes in (1, 16):
        _case("fp32_signed_fft_path", signed, n_spikes, True, args.iters)
    for n_spikes in (1, 16):
        _case("int16_nonneg_sum_path", signed.abs().to(torch.int16), n_spikes, False, args.iters)
    _sync_check(signed.clone())
    del signed
    mni = torch.randn(1, 1, 181, 217, 181, generator=g, device="cuda") * 100
    for n_spikes in (1, 16):
        _case("mni_fp32_signed_fft_path", mni, n_spikes, True, args.iters)


if __name__ == "__main__":
    main()
