"""The B-spline kernels (`tio_bspline_prefilter`, `tio_bspline_resample`) on every kernel path, voxel
by voxel against float64, with per-voxel bounds (tests/bspline_cases.py):

(a) prefilter: coefficients against `prefilter64` within its rounding bound E;
(b) pull: the output against sum w c_gpu in float64 at the C oracle's exact fp32 coordinates
    (`c_port.sampling_coords`), within gamma_m sum |w c_gpu|; no coordinate term;
(c) end to end through the public transforms: within sum |w| E plus the pull's bound, plus the
    cast's rounding, of the spline of prefilter64's coefficients of data.float().

Each case names the paths it reaches and prints its largest |gpu - ref| / bound; the coverage test
asserts that the cases together reach every path.
"""

from __future__ import annotations

import hashlib
import warnings
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

import bspline_cases as bc
from oracle import c_port
from torchio_b200 import ops

pytestmark = pytest.mark.gpu

INT_DTYPES = (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64)
KERNEL_DTYPES = (*INT_DTYPES, torch.float32)
LINES = 32  # kLines
SMEM_FLOATS = 200 * 1024 // 4  # kPrefilterSmem


def cta_lines(n):
    """bspline.cu: cta_lines_for(n | 1)."""
    return min(LINES, SMEM_FLOATS // (n | 1))


def _source(shape, dtype, seed, big=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    if dtype == torch.uint8:
        return (x.abs() * 90).clamp(0, 255).to(dtype)
    if dtype == torch.int8:
        return (x * 40).clamp(-128, 127).to(dtype)
    if dtype == torch.int16:
        return (x * 100).to(dtype)
    if dtype in (torch.int32, torch.int64):
        scale = 3e7 if big else 100.0  # above 2^24: the load rounds to fp32, as data.float() does
        return (x * scale).round().to(dtype)
    return x.to(dtype)


def _ratio(err, bound):
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.max(r, initial=0.0))


def check_prefilter(x, order, flags=None, in_place=False):
    """Coefficients of ``x`` (B, C, I, J, K) against prefilter64 within E (+ float64's own rounding);
    NaN and +-Inf where prefilter64 has them.  Returns (coefficients, largest ratio)."""
    xd = x.cuda()
    flags_d = None if flags is None else torch.as_tensor(flags, dtype=torch.uint8).cuda()
    got = ops.bspline_prefilter(xd, order, flags_d, in_place=in_place).cpu()
    ref_in = x.float().double().numpy()
    c64, E, _ = bc.prefilter64(ref_in, order)
    got64 = got.double().numpy()
    skip = np.zeros(x.shape[0], bool) if flags is None else (np.asarray(flags) & 1).astype(bool)
    work = ~skip
    g, c, e = got64[work], c64[work], E[work]
    finite = np.isfinite(c)
    assert np.array_equal(np.isnan(g), np.isnan(c)), "NaN classes differ"
    assert np.array_equal(np.isposinf(g), np.isposinf(c)) and np.array_equal(np.isneginf(g), np.isneginf(c))
    bound = e * (1 + 2.0**-28) + 2.0**-40 * np.abs(c)
    err = np.abs(g[finite] - c[finite])
    ratio = _ratio(err, bound[finite])
    assert ratio <= 1.0, ratio
    return got, ratio


# ---- prefilter ------------------------------------------------------------------------------------

PREFILTER_PATHS = {f"prefilter_{p}" for p in (
    "rows_dtype", "strided_dtype", "exact_and_truncated", "k_staging", "cta_lines_k", "cta_lines_j",
    "cta_lines_i", "ragged_volumes", "identity", "in_place", "passthrough", "nonfinite", "refusal")}


@pytest.mark.parametrize("dtype", KERNEL_DTYPES, ids=str)
def test_prefilter_rows_read_the_source_dtype(dtype):
    worst = 0.0
    for order in bc.ORDERS:
        x = _source((2, 1, 5, 6, 37), dtype, order, big=dtype == torch.int64)
        if dtype == torch.int64:
            assert x.abs().max() > 2**24
        worst = max(worst, check_prefilter(x, order)[1])
    print(f"[prefilter rows {dtype}] max |gpu - c64| / E = {worst:.3f}")


@pytest.mark.parametrize("dtype", (torch.uint8, torch.int8, torch.int16, torch.int64), ids=str)
@pytest.mark.parametrize("shape", [(9, 7, 1), (13, 1, 1)])
def test_prefilter_strided_first_pass_reads_the_source_dtype(shape, dtype):
    worst = 0.0
    for order in (3, 7):
        worst = max(worst, check_prefilter(_source((2, 2, *shape), dtype, 3, big=True), order)[1])
    print(f"[prefilter strided {shape} {dtype}] max ratio = {worst:.3f}")


@pytest.mark.parametrize("order", bc.ORDERS)
def test_prefilter_exact_and_truncated_initial_sums(order):
    """Every n in 2..64 on each axis: each pole's exact sum (n <= h) and truncated sum (n > h)."""
    ns = list(range(2, 65))
    for z in bc.kernel_poles(order)[0]:
        h = bc.horizon(z)
        assert h in ns and h + 1 in ns, (z, h)
    worst = 0.0
    for n in ns:
        for shape in ((2, 3, n), (3, n, 1), (n, 1, 2)):
            worst = max(worst, check_prefilter(_source((1, 1, *shape), torch.float32, n), order)[1])
    print(f"[prefilter n = 2..64 o{order}] horizons {[bc.horizon(z) for z in bc.kernel_poles(order)[0]]}, "
          f"max ratio = {worst:.3f}")


def test_prefilter_k_staging():
    """Row staging with (row, element) stepping and 8 loads in flight, K around the warp's 32."""
    worst = 0.0
    for k in (2, 3, 31, 32, 33, 255, 256, 257):
        worst = max(worst, check_prefilter(_source((1, 2, 3, 5, k), torch.int16, k), 5)[1])
    print(f"[prefilter K staging] max ratio = {worst:.3f}")


@pytest.mark.parametrize("shape,axis", [
    ((1, 40, 1599), 2), ((1, 40, 1600), 2), ((1, 30, 2100), 2), ((1, 2, 51199), 2), ((2, 1600, 20), 1),
    ((1700, 2, 20), 0),
], ids=str)
def test_prefilter_lines_per_cta(shape, axis):
    """Long lines: full CTAs of 32, 31, 24, 30 and 1 lines (up to 200 KiB of shared memory), several
    CTAs per volume, and a ragged last CTA."""
    n = shape[axis]
    per_cta = cta_lines(n)
    assert per_cta == {1599: 32, 1600: 31, 2100: 24, 51199: 1, 1700: 30}[n]
    lines = int(np.prod(shape)) // n  # lines per volume along the axis
    assert min(per_cta, lines) == per_cta and -(-lines // per_cta) >= 2
    assert per_cta == 1 or lines % per_cta != 0
    path = ("cta_lines_i", "cta_lines_j", "cta_lines_k")[axis]
    worst = 0.0
    for order in (2, 7):
        worst = max(worst, check_prefilter(_source((1, 1, *shape), torch.float32, n), order)[1])
    print(f"[prefilter {path} n={n}: {lines} lines per volume, {per_cta} per CTA, last CTA "
          f"{lines % per_cta or per_cta}] max ratio = {worst:.3f}")


def test_prefilter_ragged_last_cta_over_several_volumes():
    shape = (5, 7, 9)  # 35, 45 and 63 lines per volume along K, J, I: none a multiple of 32
    worst = check_prefilter(_source((3, 2, *shape), torch.float32, 8), 4)[1]
    print(f"[prefilter ragged B=3 C=2] max ratio = {worst:.3f}")


def test_prefilter_identity_pass():
    for dtype in KERNEL_DTYPES:
        x = _source((2, 3, 1, 1, 1), dtype, 1, big=True)
        before = ops.launches()
        got = ops.bspline_prefilter(x.cuda(), 3)
        torch.cuda.synchronize()
        assert ops.launches() - before == 1
        assert torch.equal(got.cpu(), x.float())
    x = torch.randn(2, 3, 1, 1, 1, device="cuda")
    keep = x.clone()
    before = ops.launches()
    ops.bspline_prefilter(x, 3, in_place=True)
    assert ops.launches() == before and torch.equal(x, keep)


def test_prefilter_in_place_equals_out_of_place():
    x = _source((2, 2, 11, 9, 40), torch.float32, 4)
    for order in bc.ORDERS:
        out = ops.bspline_prefilter(x.cuda(), order)
        inplace = x.cuda()
        ops.bspline_prefilter(inplace, order, in_place=True)
        assert torch.equal(out.view(torch.int32), inplace.view(torch.int32))
    check_prefilter(x, 6, in_place=True)


def test_prefilter_passthrough_keeps_its_bytes():
    x = _source((3, 3, 6, 5, 7), torch.float32, 5)
    flags = np.array([0, ops.FLAG_PASSTHROUGH, ops.FLAG_ELASTIC], np.uint8)
    xd = x.cuda()
    ops.bspline_prefilter(xd, 3, torch.as_tensor(flags).cuda(), in_place=True)
    assert torch.equal(xd[1].cpu().view(torch.int32), x[1].view(torch.int32))
    check_prefilter(x, 3, flags=flags)


def test_prefilter_nonfinite_classes():
    """NaN and +-Inf give prefilter64's classes (checked in check_prefilter): a non-finite value
    reaches every coefficient of its volume (an Inf as NaN, through Inf - Inf in the recursions) and
    no other volume."""
    x = _source((3, 1, 6, 5, 9), torch.float32, 6)
    x[0, 0, 2, 3, 4] = float("nan")
    x[1, 0, 4, 1, 2] = float("inf")
    x[1, 0, 0, 4, 7] = float("-inf")
    worst, counts = 0.0, []
    for order in (2, 5, 7):
        got, ratio = check_prefilter(x, order)
        assert torch.isnan(got[:2]).all() and torch.isfinite(got[2]).all()
        worst = max(worst, ratio)
        counts.append(f"o{order}: {int(torch.isnan(got).sum())} NaN")
    print(f"[prefilter nonfinite] {'; '.join(counts)}; max ratio over the finite volume = {worst:.3f}")


def test_prefilter_refuses_a_long_axis_before_any_launch():
    x = torch.zeros(1, 1, 1, 1, 51200, device="cuda")
    before = ops.launches()
    with pytest.raises(RuntimeError, match="does not fit"):
        ops.bspline_prefilter(x, 3)
    assert ops.launches() == before


# ---- pull -------------------------------------------------------------------------------------------

PULL_PATHS = {f"pull_{p}" for p in (
    "no_cp", "cp_mixed_flags", "cp_smem", "cp_smem_optin", "cp_global", "ragged_target", "single_voxel",
    "multi_period_fold", "mask", "casts", "channels", "batch_passthrough", "nonfinite", "refusal")}


def _mat(shape, out_shape=None, degrees=7.0, zoom=(1.0, 1.0, 1.0), shift=(0.3, -0.4, 0.2), seed=0):
    rng = np.random.default_rng(seed)
    out_shape = shape if out_shape is None else out_shape
    a = np.eye(3) + rng.uniform(-1, 1, (3, 3)) * np.radians(degrees)
    a = a @ np.diag(1.0 / np.asarray(zoom))
    c_in, c_out = (np.asarray(shape) - 1) / 2, (np.asarray(out_shape) - 1) / 2
    t = c_in - a @ c_out + np.asarray(shift)
    return np.concatenate([a, t[:, None]], axis=1).astype(np.float32).reshape(12)


def _shift(v):
    m = np.zeros((3, 4), np.float32)
    m[:, :3] = np.eye(3)
    m[:, 3] = v
    return m.reshape(12)


def _cp(grid, seed, amplitude=1.5):
    g = np.random.default_rng(seed).uniform(-amplitude, amplitude, (*grid, 3)).astype(np.float32)
    g[:1] = g[-1:] = 0
    return g


def run_pull(x, order, mats, *, cps=None, flags=None, out_shape=None, affine_first=True,
             spacing_in=(1.0, 1.0, 1.0), spacing_out=(1.0, 1.0, 1.0), coeff=None):
    """The pull of ``x``'s GPU coefficients (or ``coeff``) and the float64 reference at the oracle's
    coordinates: (got (B, C, ...) on the host, value, bound, inside, q)."""
    b = len(mats)
    shape = tuple(x.shape[2:])
    out_shape = shape if out_shape is None else tuple(out_shape)
    mat = np.stack(mats)
    fl = np.zeros(b, np.uint8) if flags is None else np.asarray(flags, np.uint8).copy()
    cp = None
    if cps is not None:
        grid = next(c for c in cps if c is not None).shape
        cp = np.zeros((b, *grid), np.float32)
        for e, c in enumerate(cps):
            if c is not None:
                cp[e] = c
                fl[e] |= ops.FLAG_ELASTIC
    xd = x.cuda()
    flags_d = torch.as_tensor(fl).cuda()
    if coeff is None:
        coeff = ops.bspline_prefilter(xd, order, flags_d)
    got = ops.bspline_resample(coeff, xd, torch.as_tensor(mat).cuda(), None if cp is None else torch.as_tensor(cp).cuda(),
                               flags_d, spacing_in, spacing_out, affine_first=affine_first, order=order,
                               out_shape=out_shape).cpu()
    q = c_port.sampling_coords(out_shape, mat, cp, fl, spacing_in, spacing_out, affine_first=affine_first).numpy()
    c_host = coeff.cpu().double().numpy()

    def one(e):
        if fl[e] & ops.FLAG_PASSTHROUGH:
            return None
        value, absum, _, inside = bc.tap_sums(q[e].reshape(-1, 3), order, shape, c_host[e])
        cmax = float(np.max(np.abs(c_host[e][np.isfinite(c_host[e])]), initial=0.0))
        return value, bc.pull_bound(absum, order, cmax), inside

    with ThreadPoolExecutor(8) as pool:
        refs = list(pool.map(one, range(b)))
    return got, refs, q, fl


def check_pull(got, refs, fl, x, out_shape=None):
    """Every voxel within the pull's bound (or the cast's rule), +0.0 bits outside the mask,
    NaN / Inf classes as in float64, passthrough elements as bit copies; every sampled element has
    voxels inside the mask.  Returns the largest ratio (integers: the largest share of voxels within
    the bound of an integer, from `cast_check`)."""
    worst = 0.0
    dtype = got.dtype
    for e, ref in enumerate(refs):
        if ref is None:
            assert torch.equal(got[e].view(torch.uint8), x[e].view(torch.uint8))
            continue
        value, bound, inside = ref
        assert inside.any(), f"element {e} has no voxel inside the mask"
        g = got[e].reshape(got.shape[1], -1)
        outside = g[:, torch.from_numpy(~inside)]
        assert torch.equal(outside.view(torch.uint8) if dtype.is_floating_point else outside,
                           torch.zeros_like(outside).view(torch.uint8) if dtype.is_floating_point
                           else torch.zeros_like(outside)), "outside the mask must be +0"
        g64 = g.double().numpy()[:, inside]
        v, bd = value[:, inside], bound[:, inside]
        if dtype.is_floating_point:
            assert np.array_equal(np.isnan(g64), np.isnan(v))
            assert np.array_equal(np.isposinf(g64), np.isposinf(v)) and np.array_equal(np.isneginf(g64), np.isneginf(v))
            fin = np.isfinite(v)
            worst = max(worst, bc.cast_check(g64[fin], v[fin], bd[fin], torch.float32))
        else:
            worst = max(worst, bc.cast_check(g.numpy()[:, inside], v, bd, dtype))
    return worst


def test_pull_no_control_grid():
    x = _source((3, 1, 12, 11, 10), torch.float32, 11)
    worst = 0.0
    for order in bc.ORDERS:
        got, refs, _, fl = run_pull(x, order, [_mat((12, 11, 10), seed=s) for s in range(3)])
        worst = max(worst, check_pull(got, refs, fl, x))
    print(f"[pull no_cp] max ratio = {worst:.3f}")


@pytest.mark.parametrize("affine_first", [True, False])
@pytest.mark.parametrize("grid,path", [((7, 6, 8), "cp_smem"), ((16, 16, 17), "cp_smem_optin"),
                                       ((21, 20, 20), "cp_global")])
def test_pull_control_grids(grid, path, affine_first):
    kib = np.prod(grid) * 12 / 1024
    assert {"cp_smem": kib <= 48, "cp_smem_optin": 48 < kib <= 96, "cp_global": kib > 96}[path]
    shape = (18, 16, 20)
    x = _source((3, 1, *shape), torch.float32, 12)
    mats = [_mat(shape, seed=1), _mat(shape, seed=2), _mat(shape, seed=3)]
    cps = [_cp(grid, 1), None, _cp(grid, 2)]  # an affine-only element in the same launch
    worst = 0.0
    for order in (3, 6):
        got, refs, _, fl = run_pull(x, order, mats, cps=cps, affine_first=affine_first,
                                    spacing_in=(1.0, 1.2, 0.9), spacing_out=(1.1, 0.9, 1.0))
        worst = max(worst, check_pull(got, refs, fl, x))
    print(f"[pull {path} {grid} ({kib:.0f} KiB) affine_first={affine_first}] max ratio = {worst:.3f}")


@pytest.mark.parametrize("out_shape", [(37, 7, 70), (1, 1, 1)], ids=str)
def test_pull_ragged_tiles_and_target_shapes(out_shape):
    assert out_shape == (1, 1, 1) or (out_shape[2] % 64 and out_shape[1] % 4 and out_shape[0] % 16)
    shape = (15, 13, 17)
    x = _source((2, 1, *shape), torch.float32, 13)
    mats = [_mat(shape, out_shape, zoom=np.asarray(out_shape) / np.asarray(shape), seed=s) for s in range(2)]
    worst = 0.0
    for order in (2, 5, 7):
        got, refs, _, fl = run_pull(x, order, mats, out_shape=out_shape)
        worst = max(worst, check_pull(got, refs, fl, x))
    print(f"[pull target {out_shape}] max ratio = {worst:.3f}")


def _plane_rotation(shape, flat, degrees, shift):
    """q = R (p - c) + c + shift with R a rotation in the plane of the two axes other than ``flat``,
    so that a 1-voxel axis stays inside the mask."""
    a, b = [ax for ax in range(3) if ax != flat]
    r = np.eye(3)
    t = np.radians(degrees)
    r[a, a], r[a, b], r[b, a], r[b, b] = np.cos(t), -np.sin(t), np.sin(t), np.cos(t)
    c = (np.asarray(shape, dtype=np.float64) - 1) / 2
    return np.concatenate([r, (c - r @ c + np.asarray(shift))[:, None]], axis=1).astype(np.float32).reshape(12)


def test_pull_taps_fold_over_more_than_one_period():
    worst = 0.0
    for shape in ((1, 2, 3), (3, 1, 2), (2, 3, 1)):
        x = _source((2, 2, *shape), torch.float32, 14)
        flat = shape.index(1)
        shift = [0.3, -0.2, 0.25]
        shift[flat] = 0.01
        mats = [_shift((0.02, -0.03, 0.04)), _plane_rotation(shape, flat, 20, shift)]
        got, refs, _, fl = run_pull(x, 7, mats)
        worst = max(worst, check_pull(got, refs, fl, x))
    print(f"[pull order 7 on axes of 1-3] max ratio = {worst:.3f}")


def test_pull_mask_edges():
    """q exactly at -0.05f and (n-1) + 0.05f (outside) and one fp32 step inside each, on every axis;
    outside voxels are +0.0 even where every coefficient is NaN."""
    shape = (6, 7, 5)
    x = _source((1, 1, *shape), torch.float32, 15)
    lo = np.float32(-0.05)
    worst = 0.0
    for ax in range(3):
        hi = np.float32(np.float32(shape[ax] - 1) + np.float32(0.05))
        for v, first in ((lo, True), (np.nextafter(lo, np.float32(1)), True),
                         (hi, False), (np.nextafter(hi, np.float32(0)), False)):
            t = np.zeros(3, np.float32)
            t[ax] = v if first else np.float32(v - np.float32(shape[ax] - 1))
            assert (np.float32(0) + t[ax] if first else np.float32(shape[ax] - 1) + t[ax]) == v
            got, refs, q, fl = run_pull(x, 3, [_shift(t)])
            plane = q[0][..., ax] == v
            assert plane.any()
            worst = max(worst, check_pull(got, refs, fl, x))
    nan_coeff = torch.full((1, 1, *shape), float("nan"), device="cuda")
    got, refs, _, fl = run_pull(x, 3, [_shift((-0.05, 0, 0))], coeff=nan_coeff)
    inside = refs[0][2]
    out = got[0, 0].reshape(-1)[torch.from_numpy(~inside)]
    assert (~inside).any() and torch.equal(out.view(torch.int32), torch.zeros_like(out).view(torch.int32))
    assert torch.isnan(got[0, 0].reshape(-1)[torch.from_numpy(inside)]).all()
    print(f"[pull mask edges] max ratio = {worst:.3f}")


@pytest.mark.parametrize("dtype", KERNEL_DTYPES, ids=str)
def test_pull_casts(dtype):
    """Integers: the truncation of the float64 value away from integers.  int64 holds values above
    2^24, where the fp32 result cannot resolve integers; the others must mostly fall under the
    exact-equality rule."""
    shape = (11, 9, 13)
    big = dtype == torch.int64
    x = _source((2, 1, *shape), dtype, 16, big=big)
    result = 0.0
    for order in (3, 7):
        got, refs, _, fl = run_pull(x, order, [_mat(shape, seed=7), _mat(shape, seed=8)])
        assert got.dtype == dtype
        result = max(result, check_pull(got, refs, fl, x))
    if dtype == torch.float32:
        print(f"[pull casts {dtype}] max ratio = {result:.3f}")
    else:
        assert big or result < 0.5, result
        print(f"[pull casts {dtype}] share within the bound of an integer = {result:.3f}")


def test_pull_channels_and_batch_with_passthrough():
    shape = (10, 9, 12)
    x = _source((2, 3, *shape), torch.float32, 17)
    got, refs, _, fl = run_pull(x, 4, [_mat(shape, seed=9), _mat(shape, seed=10)])
    r1 = check_pull(got, refs, fl, x)
    x = _source((32, 1, *shape), torch.float32, 18)
    flags = [ops.FLAG_PASSTHROUGH if e % 3 == 1 else 0 for e in range(32)]
    got, refs, _, fl = run_pull(x, 3, [_mat(shape, seed=e) for e in range(32)], flags=flags)
    r2 = check_pull(got, refs, fl, x)
    print(f"[pull C=3] max ratio = {r1:.3f}; [pull B=32 gated] max ratio = {r2:.3f}")


def test_pull_nonfinite_coefficients():
    """NaN and +-Inf coefficients give the classes float64 gives, 0 * Inf included: integer shifts
    put exact zero weights on taps."""
    shape = (9, 8, 10)
    x = _source((2, 1, *shape), torch.float32, 19)
    coeff = ops.bspline_prefilter(x.cuda(), 3)
    coeff[0, 0, 4, 4, 4] = float("nan")
    coeff[1, 0, 3, 3, 3] = float("inf")
    coeff[1, 0, 6, 5, 7] = float("-inf")
    got, refs, _, fl = run_pull(x, 3, [_mat(shape, seed=11), _shift((1.0, 0.0, -1.0))], coeff=coeff)
    ratio = check_pull(got, refs, fl, x)
    assert torch.isnan(got).any() and torch.isinf(got).any()
    print(f"[pull nonfinite] max ratio over the finite voxels = {ratio:.3f}")


def test_pull_refuses_a_grid_too_large_before_any_launch():
    b = 65536
    x = torch.zeros(b, 1, 1, 1, 1, device="cuda")
    mat = torch.as_tensor(np.tile(_shift((0, 0, 0)), (b, 1))).cuda()
    before = ops.launches()
    with pytest.raises(RuntimeError, match="grid too large"):
        ops.bspline_resample(x, x, mat, None, None, (1, 1, 1), (1, 1, 1), affine_first=True, order=3)
    assert ops.launches() == before


COVERAGE = {
    "test_prefilter_rows_read_the_source_dtype": {"prefilter_rows_dtype"},
    "test_prefilter_strided_first_pass_reads_the_source_dtype": {"prefilter_strided_dtype"},
    "test_prefilter_exact_and_truncated_initial_sums": {"prefilter_exact_and_truncated"},
    "test_prefilter_k_staging": {"prefilter_k_staging"},
    "test_prefilter_lines_per_cta": {"prefilter_cta_lines_k", "prefilter_cta_lines_j", "prefilter_cta_lines_i"},
    "test_prefilter_ragged_last_cta_over_several_volumes": {"prefilter_ragged_volumes"},
    "test_prefilter_identity_pass": {"prefilter_identity"},
    "test_prefilter_in_place_equals_out_of_place": {"prefilter_in_place"},
    "test_prefilter_passthrough_keeps_its_bytes": {"prefilter_passthrough"},
    "test_prefilter_nonfinite_classes": {"prefilter_nonfinite"},
    "test_prefilter_refuses_a_long_axis_before_any_launch": {"prefilter_refusal"},
    "test_pull_no_control_grid": {"pull_no_cp"},
    "test_pull_control_grids": {"pull_cp_smem", "pull_cp_smem_optin", "pull_cp_global", "pull_cp_mixed_flags"},
    "test_pull_ragged_tiles_and_target_shapes": {"pull_ragged_target", "pull_single_voxel"},
    "test_pull_taps_fold_over_more_than_one_period": {"pull_multi_period_fold"},
    "test_pull_mask_edges": {"pull_mask"},
    "test_pull_casts": {"pull_casts"},
    "test_pull_channels_and_batch_with_passthrough": {"pull_channels", "pull_batch_passthrough"},
    "test_pull_nonfinite_coefficients": {"pull_nonfinite"},
    "test_pull_refuses_a_grid_too_large_before_any_launch": {"pull_refusal"},
}


def test_cases_cover_every_path():
    """The cases together reach every path of both tables; each case asserts the shapes that put it
    on its path (lines per CTA, control-grid bytes, ragged remainders, horizons)."""
    assert all(callable(globals().get(name)) for name in COVERAGE)
    for name, paths in COVERAGE.items():  # a case claims paths of its own kernel only
        assert all(p.startswith(name.split("_")[1] + "_") for p in paths), name
    assert not PREFILTER_PATHS & PULL_PATHS
    reached = set().union(*COVERAGE.values())
    assert PREFILTER_PATHS | PULL_PATHS == reached, sorted((PREFILTER_PATHS | PULL_PATHS) ^ reached)


# ---- end to end through the public transforms ------------------------------------------------------

@pytest.mark.parametrize("transform", ["Affine", "ElasticDeformation", "Resample"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16, torch.float64], ids=str)
def test_public_transforms_end_to_end(transform, dtype):
    import torchio_b200 as tio

    shape = (14, 12, 16)
    worst, gated = {}, 0
    for order in bc.ORDERS:
        x = (torch.randn((4, 1, *shape), generator=torch.Generator().manual_seed(order)) * 2).to(dtype)
        kwargs = dict(image_interpolation=order, p=0.5)
        t = {"Affine": lambda: tio.Affine(scales=(0.9, 1.1), degrees=10, translation=1, **kwargs),
             "ElasticDeformation": lambda: tio.ElasticDeformation(max_displacement=2.0, **kwargs),
             "Resample": lambda: tio.Resample((1.5, 0.8, 1.2), **kwargs)}[transform]()
        for attempt in range(16):  # until the step applies: Resample gates the whole batch
            torch.manual_seed(20 + order + 100 * attempt)
            batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(x.cuda(), [tio.AffineMatrix() for _ in range(4)])})
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                out = t(batch)
            history = out.applied_transforms
            y = out.images["t1"].data.cpu()
            assert y.dtype == dtype
            if history:
                break
            gated += 1  # every element gated out
            assert torch.equal(y.view(torch.uint8), x.view(torch.uint8))
        (step,) = history
        worst[order] = bc.check_end_to_end(x, y, step.params, order)
    print(f"[end to end {transform} {dtype}] max ratio per order: "
          + ", ".join(f"o{o} {r:.3f}" for o, r in worst.items()) + f"; {gated} calls gated out")


def test_full_size_cubic():
    """2 x 1 x 256^3 order 3: every coefficient against the banded reference (within E + A) and the
    pull on a strided lattice plus one dense block."""
    shape = (256, 256, 256)
    x = torch.rand((2, 1, *shape), generator=torch.Generator().manual_seed(21))
    xd = x.cuda()
    coeff = ops.bspline_prefilter(xd, 3)
    c_gpu = coeff.cpu().double().numpy()
    worst_c = 0.0
    for e in range(2):
        c64, E, A = bc.prefilter64(x[e].double().numpy(), 3)
        exact = bc.coefficients_banded(x[e].double().numpy(), 3)
        bound = E * (1 + 2.0**-28) + A + 2.0**-40 * np.abs(exact)
        worst_c = max(worst_c, _ratio(np.abs(c_gpu[e] - exact), bound))
        del c64, E, A, exact, bound
    assert worst_c <= 1
    mats = [_mat(shape, seed=22), _mat(shape, degrees=12, seed=23)]
    got = ops.bspline_resample(coeff, xd, torch.as_tensor(np.stack(mats)).cuda(), None, None, (1, 1, 1), (1, 1, 1),
                               affine_first=True, order=3).cpu()
    digest = hashlib.sha256(got.numpy().tobytes()).hexdigest()
    q = c_port.sampling_coords(shape, np.stack(mats), None, None, (1, 1, 1), (1, 1, 1), affine_first=True).numpy()
    sel = np.zeros(shape, bool)
    sel[::7, ::5, ::3] = True
    sel[100:132, 64:96, 200:232] = True
    worst = 0.0
    for e in range(2):
        value, absum, _, inside = bc.tap_sums(q[e][sel], 3, shape, c_gpu[e])
        bound = bc.pull_bound(absum, 3, float(np.abs(c_gpu[e]).max()))
        g = got[e, 0].numpy()[sel].astype(np.float64)[None]
        assert np.all(g[:, ~inside] == 0)
        worst = max(worst, bc.cast_check(g[:, inside], value[:, inside], bound[:, inside], torch.float32))
    print(f"[256^3 cubic] coefficients max ratio {worst_c:.3f}; pull on {int(sel.sum())} voxels per element "
          f"max ratio {worst:.3f}; sha256 {digest}")
