"""Time PCA on the GPU against the reference's op sequence.

    python tools/pca_bench.py [--iters 10] [--cases 1x4x256,4x16x128,1x64x128,1x256x96]

Cases are (B, C, S^3) fp32 batches with q = 3, made from a seed with a spectrum that has a gap at 3.
For each it reports:
- the mean time of one `PCA(num_components=3)` call on the CUDA batch (host clock around the call,
  which ends in a device-to-host read) over ``--iters`` calls after warm-up;
- the mean kernel time of `ops.pca_mean`, `ops.pca_gram_apply` (q = 3 and q = 1) and
  `ops.pca_project` (CUDA events around ``--iters`` launches), and each one's rate over the bytes it
  must move, computed from the shapes: B C N x 4 read (every pass), plus B q N x 4 written
  (projection); the share of 3.35 TB/s (H100 SXM HBM3, data sheet) and, for G W, its fp64 rate
  (2 C q FMAs per voxel, two flops each);
- the mean time of the reference's op sequence (tests/pca_cases.py `reference_ops`) on the same
  tensors over a few calls after one warm-up call;
- the largest difference between the two outputs up to each component's sign.
Prints the card, its power limit and maximum SM clock, and one JSON line per case.
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import torchio_b200 as tio  # noqa: E402
from torchio_b200 import ops  # noqa: E402

import pca_cases as pc  # noqa: E402

HBM = 3.35e12


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def make_batch(b: int, c: int, s: int) -> torch.Tensor:
    gen = torch.Generator(device="cuda").manual_seed(b * 1000 + c)
    sig = torch.cat([torch.tensor([8.0, 4.0, 2.0]), torch.full((c - 3,), 0.1)]).cuda()
    out = torch.empty(b, c, s ** 3, device="cuda")
    for e in range(b):
        u = torch.linalg.qr(torch.randn(c, c, device="cuda", generator=gen))[0]
        out[e] = (u * sig) @ torch.randn(c, s ** 3, device="cuda", generator=gen) + 50
    return out.reshape(b, c, s, s, s)


def kernel_ms(fn, iters: int) -> float:
    fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def run_case(b: int, c: int, s: int, iters: int) -> dict:
    q, n = 3, s ** 3
    x = make_batch(b, c, s)
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(x[e])) for e in range(b)])
    transform = tio.PCA(num_components=q, copy=False)

    def call():
        batch.images["t1"].data = x
        return transform(batch).images["t1"].data

    call()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        got = call()
    torch.cuda.synchronize()
    pca_ms = (time.perf_counter() - t0) * 1e3 / iters

    ws = ops.pca_workspace(x, q)
    mean = ops.pca_mean(x, ws)
    w3 = np.random.default_rng(0).standard_normal((b, c, q))
    coef = np.random.default_rng(1).standard_normal((b, c, q)).astype(np.float32) * 0.01
    read = b * c * n * 4
    kernels = {
        "mean": (kernel_ms(lambda: ops.pca_mean(x, ws), iters), read, 0),
        "gram_q3": (kernel_ms(lambda: ops.pca_gram_apply(x, mean, w3, ws), iters), read, 2 * c * q * b * n),
        "gram_q1": (kernel_ms(lambda: ops.pca_gram_apply(x, mean, w3[:, :, :1], ws), iters), read, 2 * c * b * n),
        "project": (kernel_ms(lambda: ops.pca_project(x, mean, coef, 0.5, True), iters), read + b * q * n * 4, 0),
    }
    kern = {}
    for name, (ms, nbytes, fma) in kernels.items():
        entry = {"ms": round(ms, 3), "GB/s": round(nbytes / ms / 1e6, 1), "hbm_share": round(nbytes / ms * 1e3 / HBM, 3)}
        if fma:
            entry["fp64_TFLOP/s"] = round(2 * fma / ms / 1e9, 2)
        kern[name] = entry

    torch.manual_seed(0)
    want = pc.reference_ops(x, q, True, True, (-2.3, 2.3), True)
    torch.cuda.synchronize()
    ref_iters = max(1, min(3, iters))
    t0 = time.perf_counter()
    for _ in range(ref_iters):
        torch.manual_seed(0)
        want = pc.reference_ops(x, q, True, True, (-2.3, 2.3), True)
    torch.cuda.synchronize()
    ref_ms = (time.perf_counter() - t0) * 1e3 / ref_iters
    torch.manual_seed(0)
    got = call()
    err = pc.sign_errors(got.cpu().numpy(), want.cpu().numpy(), (-2.3, 2.3), True)
    return {"case": f"B={b} C={c} {s}^3 q=3", "pca_ms": round(pca_ms, 3), "reference_ms": round(ref_ms, 3),
            "speedup": round(ref_ms / pca_ms, 2), "kernels": kern, "max_diff": float(err.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--cases", default="1x4x256,4x16x128,1x64x128,1x256x96")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pca_bench: no CUDA device")
    print(card())
    for spec in args.cases.split(","):
        b, c, s = (int(v) for v in spec.split("x"))
        print(json.dumps(run_case(b, c, s, args.iters)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
