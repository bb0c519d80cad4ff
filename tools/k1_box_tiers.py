"""K1's affine launch at the bench's own matrices: one box for the whole batch against a box per
element.

    python tools/k1_box_tiers.py [--reps 20] [--draws 2000]

Samples `Affine(scales=(0.9, 1.1), degrees=(-10, 10))` on a 32 x 1x256^3 fp32 batch as bench.py
does, captures the `ops.resample` call the transform makes, and times it with CUDA events (the
bounds pre-pass included):
  (a) the whole batch at the launch-wide box (today's single-box launch);
  (b) the elements whose per-element edge is 22, at box 22 (4 CTAs/SM) and at box 24 (3 CTAs/SM);
  (c) the same for the elements of edge 20;
  (d) the whole batch as one tiered call (a box per element).
Each pair of configurations is checked bit for bit.  The tier mix over `--draws` sampled
elements is computed on the host.  Prints the card, its power limit and SM clock."""

import argparse
import os
import subprocess
import sys
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import torchio_b200 as tio  # noqa: E402
from torchio_b200 import ops  # noqa: E402
from torchio_b200.transforms import spatial  # noqa: E402

B, S = 32, 256
AFFINE = {"scales": (0.9, 1.1), "degrees": (-10, 10)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        return "nvidia-smi unavailable"


def capture(transform, x):
    """The positional and keyword arguments of the one ops.resample call `transform` makes."""
    seen, raw = [], ops.resample

    def spy(*a, **kw):
        seen.append((a, kw))
        return raw(*a, **kw)

    ops.resample = spy
    try:
        batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(B)])})
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            transform(batch)
    finally:
        ops.resample = raw
    (call,) = seen
    return call


def timed(fn, reps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--draws", type=int, default=2000)
    args = ap.parse_args()
    print("card:", card())

    # tier mix over many of the bench's draws
    torch.manual_seed(0)
    transform = tio.Affine(**AFFINE)
    mats = []
    x_host = torch.zeros((B, 1, S, S, S), dtype=torch.float32, device="cuda")
    while len(mats) * B < args.draws:
        (a, kw) = capture(transform, x_host)
        mats.append(a[1].cpu().numpy())
    mats = np.concatenate(mats)
    cap = spatial._box_hint(spatial.tables.SpatialTables(mats, None, np.zeros(len(mats), np.uint8), []),
                            (1, 1, 1), (1, 1, 1), (S, S, S))
    edges = spatial._affine_box_edges(mats, cap, (S, S, S))
    for e in sorted(set(edges.tolist())):
        print(f"tier mix: edge {e}: {np.mean(edges == e) * 100:.1f} % of {len(edges)} elements")

    torch.manual_seed(1234)
    x = torch.rand((B, 1, S, S, S), device="cuda")
    (a, kw) = capture(transform, x)
    src, mat, cp, flags, sp_in, sp_out = a
    kw = {k: v for k, v in kw.items() if k not in ("box_hint", "tiers")}
    mat_h = mat.cpu().numpy()
    packed = spatial.tables.SpatialTables(mat_h, None, np.zeros(B, np.uint8), [])
    cap = spatial._box_hint(packed, sp_in, sp_out, (S, S, S))
    edges = spatial._affine_box_edges(mat_h, cap, (S, S, S))
    print("launch box", cap, "per-element edges", edges.tolist())

    def run(idx, hint, tiers=None):
        s, m = (x, mat) if idx is None else (x[idx], mat[idx])
        f = flags if flags is None or idx is None else flags[idx]
        extra = {} if tiers is None else {"tiers": tiers}
        return lambda: ops.resample(s, m, cp, f, sp_in, sp_out, box_hint=hint, **kw, **extra)

    rows = []
    ms_a, out_a = timed(run(None, cap), args.reps)
    rows.append(("(a) all %d elements, box %d" % (B, cap), ms_a))
    for tier, label in ((22, "(b)"), (20, "(c)")):
        idx = torch.tensor(np.nonzero(edges == tier)[0], device="cuda")
        if idx.numel() == 0:
            print(label, "no element of edge", tier)
            continue
        t_small, o_small = timed(run(idx, tier), args.reps)
        t_big, o_big = timed(run(idx, cap), args.reps)
        t_small2, _ = timed(run(idx, tier), args.reps)
        same = torch.equal(o_small, o_big)
        rows.append((f"{label} {idx.numel()} elements of edge {tier}: box {tier}", (t_small + t_small2) / 2))
        rows.append((f"{label} same elements: box {cap}", t_big))
        print(f"{label} box {tier} vs box {cap}: {(t_big / ((t_small + t_small2) / 2) - 1) * 100:+.1f} % faster,"
              f" bit-identical: {same}")
    order, runs = spatial._box_tiers(packed, cap, (S, S, S))
    tiers = (torch.tensor(order, device="cuda"), runs)
    print("runs (count, edge):", runs)
    ms_d, out_d = timed(run(None, cap, tiers), args.reps)
    ms_a2, _ = timed(run(None, cap), args.reps)
    rows.append(("(d) all %d elements, tiered" % B, ms_d))
    rows.append(("(a) again", ms_a2))
    print(f"(d) tiered vs single box: {((ms_a + ms_a2) / 2 / ms_d - 1) * 100:+.1f} % faster,"
          f" bit-identical: {torch.equal(out_d, out_a)}")
    for name, ms in rows:
        print(f"{name:48s} {ms:7.3f} ms")
    print("card:", card())


if __name__ == "__main__":
    main()
