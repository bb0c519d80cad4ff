"""Cost of the differentiable spatial path at 32 x 1 x 256^3 fp32; prints one JSON line.

- forward-with-grad and backward of the bench's spatial pair, Compose([Affine, ElasticDeformation]);
- the whole backward of an affine-only and an elastic-only batch (autograd included), and the K1ᵀ
  call alone (`ops.resample_backward` with the graph node's geometry: memset, bounds pre-pass, tile
  kernel) with its algorithmic bytes (8 B per voxel: read g, write grad_in) and share of 3.35 TB/s
  (H100 SXM HBM3);
- the reference's op sequence (F.grid_sample + ones-mask grid_sample + torch.where, forward and
  backward, on the same GPU, sampling grids built beforehand) per voxel, at --ref-batch elements.

    python tools/autograd_bench.py [--batch 32] [--ref-batch 4] [--reps 5]
"""

from __future__ import annotations

import argparse
import json
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

import torchio_b200 as tio  # noqa: E402
from torchio_b200 import ops  # noqa: E402

HBM = 3.35e12


def _gpu():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        out = torch.cuda.get_device_name()
    return out


def _events(fn, reps):
    """Median ms of ``fn`` over ``reps`` runs, CUDA events around each."""
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def _batch(x):
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(x.shape[0])])})


def _graph(transform, data):
    """(output, input leaf, transformed batch) of one differentiable call; the input is a fresh
    clone, which the no-grad timing below clones as well."""
    x = data.clone().requires_grad_()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = transform(_batch(x))
    return out.images["t1"].data, x, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ref-batch", type=int, default=4)
    ap.add_argument("--size", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    tio.set_differentiable(True)
    n = args.size
    voxels = args.batch * n**3
    torch.manual_seed(0)
    data = torch.rand((args.batch, 1, n, n, n), device="cuda")
    g = torch.randn_like(data)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        affine = tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10), copy=False)
        elastic = tio.ElasticDeformation(max_displacement=3.0, copy=False)
    pipeline = tio.Compose([affine, elastic], copy=False)

    result = {"gpu": _gpu(), "shape": [args.batch, 1, n, n, n]}
    # warm-up of every shape and path
    for t in (pipeline, affine, elastic):
        y, x, _ = _graph(t, data)
        y.backward(g)
    torch.cuda.synchronize()

    result["compose_forward_with_grad_ms"] = _events(lambda: _graph(pipeline, data), args.reps)
    result["compose_forward_no_grad_ms"] = _events(lambda: pipeline(_batch(data.clone())), args.reps)

    def backward_of(t):
        ys = []
        for _ in range(args.reps):
            y, _, _ = _graph(t, data)
            ys.append(y)
        torch.cuda.synchronize()
        it = iter(ys)
        return _events(lambda: next(it).backward(g), args.reps)

    result["compose_backward_ms"] = backward_of(pipeline)
    for name, t in (("affine", affine), ("elastic", elastic)):
        result[f"{name}_backward_ms"] = backward_of(t)
        # the kernel call alone, with the geometry the graph node holds (memset, bounds pre-pass, tile kernel)
        y, _, _ = _graph(t, data)
        node = y.grad_fn
        geometry = {k: node.geometry[k] for k in ("affine_first", "mode", "fill", "box_hint")}
        geo = node.geometry

        def k1t():
            ops.resample_backward(g, node.in_shape, geo["mat"], geo["cp"], geo["flags"], geo["spacing_in"],
                                  geo["spacing_out"], **geometry)

        k1t()
        ms = _events(k1t, 3 * args.reps)
        result[f"k1t_{name}_ms"] = ms
        result[f"k1t_{name}_bytes"] = 8 * voxels
        result[f"k1t_{name}_hbm_share"] = 8 * voxels / (ms * 1e-3) / HBM
        del y, node
    del g

    # the reference's op sequence, per element grids as spatial.py builds them (grid not timed)
    from oracle import torch_port

    rb = args.ref_batch
    _, _, out = _graph(pipeline, data[:rb])
    history = [{"name": h.name, "params": h.params} for h in out.applied_transforms]
    del out
    grids = []
    for step in history:
        p = step["params"]
        grid = torch.stack([torch_port.sampling_grid((n, n, n), np.eye(4), (n, n, n), np.eye(4), m, c, True)
                            for m, c in zip(p["affine_matrix"], p["control_points"])])
        grids.append(torch_port.normalise_grid(grid, (n, n, n)).cuda())
    x = data[:rb].clone()
    fill = x[0].min()

    def reference():
        v = x.detach().requires_grad_()
        y = v
        for grid in grids:
            t = y.permute(0, 1, 4, 3, 2)
            out = F.grid_sample(t, grid, mode="bilinear", padding_mode="zeros", align_corners=True)
            mask = F.grid_sample(torch.ones_like(t), grid, padding_mode="zeros", align_corners=True)
            y = torch.where(mask > 0.5, out, fill.detach()).permute(0, 1, 4, 3, 2)
        y.backward(torch.ones_like(y))

    reference()
    torch.cuda.synchronize()
    ms = _events(reference, max(3, args.reps // 3))
    result["reference_fwd_bwd_ms"] = ms
    result["reference_batch"] = rb
    result["reference_fwd_bwd_ns_per_voxel"] = ms * 1e6 / (rb * n**3)
    ours = result["compose_forward_with_grad_ms"] + result["compose_backward_ms"]
    result["ours_fwd_bwd_ns_per_voxel"] = ours * 1e6 / voxels
    print(json.dumps(result))


if __name__ == "__main__":
    main()
