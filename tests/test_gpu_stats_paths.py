"""The statistics kernels on every kernel path, against float64 and an exact sort:

(a) `tio_moments` (Standardize, Pad "mean"): the count exactly, the sum within n 2^-53 sum|x| of
    math.fsum, and the variance against a float64 two-pass variance within a bound derived below;
    constant selections give exactly 0;
(b) `tio_quantiles_batched` (Normalize, HistogramStandardization, Pad "median"): every order statistic
    bit for bit against a numpy sort on ATen's radix key (`bits ^ (sign ? 0xffffffff : 0x80000000)`,
    every NaN at 0xffffffff, above +Inf), the weights `index - lower` exactly, the count and the NaN
    flag exactly;
(c) `tio_min_sample0` (default_pad_value="minimum", Pad "minimum"): torch.amin's semantics, NaN when a
    value is NaN and otherwise the least value, whatever order the blocks finish in;
(d) end to end, the transforms against the reference's op sequence on the same CUDA tensors.

Each case names the kernel bodies it reaches and prints its largest error as a fraction of its bound;
the coverage test asserts that the cases together reach every body.
"""

from __future__ import annotations

import math
import warnings

import numpy as np
import pytest
import torch

from oracle import torch_port as tp
from torchio_b200 import ops

pytestmark = pytest.mark.gpu

U = 2.0**-53  # unit roundoff of float64
FLOAT_DTYPES = (torch.float16, torch.bfloat16, torch.float32, torch.float64)
IMAGE_DTYPES = (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, *FLOAT_DTYPES)
QUANT_PER_ROUND = 13  # kQuantPerRound: 26 targets per round of the select


def _on_device(x: torch.Tensor, offset: int = 0) -> torch.Tensor:
    """A CUDA copy of ``x`` whose first element lies ``offset`` elements into its storage (the
    caching allocator's blocks are 512-byte aligned, so offset 1 is a 4-byte misalignment for fp32)."""
    base = torch.empty(x.numel() + offset, dtype=x.dtype, device="cuda")
    view = base[offset:].view(x.shape)
    view.copy_(x)
    return view


NEG_NAN_BITS = {torch.float16: 0xFE00, torch.bfloat16: 0xFFC0, torch.float32: 0xFFC00000,
                torch.float64: 0xFFF8000000000000}
INT_OF_SIZE = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _nan(dtype=torch.float32, negative=True) -> torch.Tensor:
    """A quiet NaN of ``dtype`` made from its bits, as casts may change a NaN's sign.  The negative one
    is what x86 produces for inf - inf or 0 * inf on the host (0xffc00000 in fp32)."""
    inf = torch.tensor([math.inf])
    assert int((inf - inf).view(torch.int32)) & 0xFFFFFFFF == NEG_NAN_BITS[torch.float32]
    size = torch.finfo(dtype).bits // 8
    bits = NEG_NAN_BITS[dtype] - (1 << (8 * size))  # the same bits as a signed integer
    if not negative:
        bits += 1 << (8 * size - 1)  # clear the sign bit
    nan = torch.tensor([bits], dtype=INT_OF_SIZE[size]).view(dtype)
    assert torch.isnan(nan).all() and bool(torch.signbit(nan).all()) == negative
    return nan


def _neg_nan(dtype=torch.float32) -> torch.Tensor:
    return _nan(dtype, negative=True)


def _put_bits(x: torch.Tensor, index, values: torch.Tensor) -> None:
    """x[index] = values bit for bit (through an integer view: a float copy may canonicalise NaN)."""
    ints = INT_OF_SIZE[x.element_size()]
    x.view(ints)[index] = values.view(ints)


def _ratio(err: float, bound: float) -> float:
    return 0.0 if err == 0 else err / bound


# ---- (a) moments ------------------------------------------------------------------------------------

MOMENT_PATHS = {"moments_float4", "moments_float4_tail", "moments_unaligned", "moments_masked"}


def moment_bodies(x: torch.Tensor, mask) -> set:
    """Which bodies of both passes of moments_kernel a call on ``x`` runs."""
    if mask is not None:
        return {"moments_masked"}
    if x.data_ptr() % 16:
        return {"moments_unaligned"}
    return {"moments_float4"} | ({"moments_float4_tail"} if x.numel() % 4 else set())


def moments_reference(v: np.ndarray):
    """float64 references of a finite selection: (fsum, fsum |x|, two-pass sum of squared deviations)."""
    n = v.size
    s = math.fsum(v)
    abs_sum = math.fsum(np.abs(v))
    mean = s / n
    q = math.fsum((v - mean) ** 2)
    return s, abs_sum, q


def variance_bound(n: int, abs_sum: float, mean: float, q: float) -> float:
    """|var_gpu - var_ref| for var = Q / (n - 1), Q the sum of squared deviations.

    Device: its sum S^ is within n u sum|x| of the exact S in any order of the atomics, so its mean
    m = fl(S^ / n) is within d = u sum|x| (1 + u) + u |mu| of mu.  It sums fl(fl(x - m)^2): each term
    is (x - m)^2 (1 + 3u) at worst, and n - 1 additions of non-negative terms add (n - 1) u of their
    total; the total itself is Q + n (m - mu)^2, since sum (x - mu) = 0.  So
        |Q_gpu - Q| <= n d^2 + (n + 3) u (Q + n d^2).
    Reference: fsum's mean and the division are within 2u |mu|, each square within 3u, fsum's result
    within u:  |Q_ref - Q| <= n (2u mu)^2 + 4u (Q + n (2u mu)^2).
    Both quotients by n - 1 round once more (u var each).  Q is taken as Q_ref (1 + 1e-6)."""
    qq = q * (1 + 1e-6)
    d = U * abs_sum * (1 + U) + U * abs(mean)
    shift = n * d * d
    dev = shift + (n + 3) * U * (qq + shift)
    r = 2 * U * abs(mean)
    ref = n * r * r + 4 * U * (qq + n * r * r)
    return (dev + ref) / (n - 1) + 2 * U * qq / (n - 1)


def check_moments(x: torch.Tensor, mask: torch.Tensor | None = None, offset: int = 0, exact_zero=False):
    """ops.moments of the CUDA copy of the host fp32 ``x`` (at storage offset ``offset``) against
    float64.  Returns (bodies reached, largest error / bound of sum and variance)."""
    xd = _on_device(x, offset)
    md = None if mask is None else mask.cuda()
    bodies = moment_bodies(xd, md)
    s, dev, n = ops.moments(xd, md)
    v = (x if mask is None else x[mask.expand_as(x)]).reshape(-1).double().numpy()
    assert n == v.size
    ref_s, abs_sum, ref_q = moments_reference(v)
    sum_bound = v.size * U * abs_sum
    assert abs(s - ref_s) <= sum_bound, (s, ref_s, sum_bound)
    ratio = _ratio(abs(s - ref_s), sum_bound)
    if exact_zero:
        assert ref_q == 0 and dev == 0.0, dev
        return bodies, ratio
    var, ref_var = dev / (n - 1), ref_q / (n - 1)
    bound = variance_bound(v.size, abs_sum, ref_s / v.size, ref_q)
    assert abs(var - ref_var) <= bound, (var, ref_var, bound)
    return bodies, max(ratio, _ratio(abs(var - ref_var), bound))


def _moment_layouts(x: torch.Tensor, mask: torch.Tensor | None = None, seed: int = 0):
    """(values, mask, offset) reaching each body: aligned with n % 4 == 0, aligned with n % 4 != 0,
    at storage offset 1, and masked (``mask``, or a random one, over all of ``x``).  The unmasked
    layouts take the selected values of ``x`` when ``mask`` is given."""
    if mask is None:
        mask = torch.rand(x.shape, generator=torch.Generator().manual_seed(seed)) > 0.3
        v = x
    else:
        v = x[mask]
    n4 = v.numel() // 4 * 4
    return [(v[:n4], None, 0), (v[:n4 - 1], None, 0), (v[:n4 - 2], None, 1), (x, mask, 0)]


def test_moments_bodies_against_float64():
    worst, reached = 0.0, set()
    g = torch.Generator().manual_seed(1)
    for n in (6, 1000, 256 * 1056 * 4 + 8, 3_000_001):  # one block up to a grid-stride loop
        x = torch.randn(n, generator=g) * 3 - 1
        for xs, mask, off in _moment_layouts(x, seed=n):
            bodies, r = check_moments(xs, mask, off)
            reached |= bodies
            worst = max(worst, r)
    assert reached == MOMENT_PATHS
    print(f"[moments random] max error / bound = {worst:.3e}")


@pytest.mark.parametrize("value", [0.0, 1.0, -2.5, 123.456, 1000.1, -37000.7, 6.0e7, 3.0e30], ids=str)
def test_moments_constant_selection_has_zero_variance(value):
    """A constant selection: the variance is exactly 0 in every body (the raw-moment form
    (ss - s^2/n) leaves atomic-order noise here)."""
    reached, worst = set(), 0.0
    x = torch.full((1 << 20,), value, dtype=torch.float32)
    x[1::7] = -value - 1.0  # masked out below
    keep = x == np.float32(value)
    for xs, mask, off in _moment_layouts(x, keep):
        bodies, r = check_moments(xs, mask, off, exact_zero=True)
        reached |= bodies
        worst = max(worst, r)
    assert reached == MOMENT_PATHS
    print(f"[moments constant {value}] variance exactly 0, sum error / bound = {worst:.3e}")


def test_moments_constant_full_volume():
    """256^3 constants of the magnitudes where the raw-moment form is worst."""
    for value in (1000.1, 123.456):
        x = torch.full((256**3,), value, dtype=torch.float32)
        bodies, _ = check_moments(x, exact_zero=True)
        assert bodies == {"moments_float4"}


@pytest.mark.parametrize("center", [2.0**20, 1000.1, 123.456, -3.0e5], ids=str)
def test_moments_near_constant(center):
    """Values a few fp32 ulps around ``center``: mean / std up to ~2e6, where the raw moments cancel."""
    g = torch.Generator().manual_seed(7)
    c = np.float32(center)
    ulp = float(np.spacing(np.abs(c)))
    worst, reached, ratio = 0.0, set(), 0.0
    for n in (4096 * 37, 256**3 + 3) if center == 2.0**20 else (4096 * 37,):
        k = torch.randint(-8, 9, (n,), generator=g).to(torch.float64)
        x = (float(c) + k * ulp).to(torch.float32)
        assert torch.equal(x.double(), float(c) + k * ulp)  # every value representable
        ratio = max(ratio, abs(float(c)) / float(x.double().std()))
        for xs, mask, off in _moment_layouts(x, seed=n):
            bodies, r = check_moments(xs, mask, off)
            reached |= bodies
            worst = max(worst, r)
    assert reached == MOMENT_PATHS
    print(f"[moments near {center}] |mean| / std = {ratio:.2e}, max error / bound = {worst:.3e}")


def test_moments_nonfinite_follow_torch():
    """±Inf and NaN: the mean and variance are what torch's mean() and std() give (Inf or NaN)."""
    inf, reached = math.inf, set()
    g = torch.Generator().manual_seed(3)
    for specials in ([inf], [-inf], [inf, -inf], [math.nan], [inf, math.nan], [_neg_nan().item()]):
        x = torch.randn(4096 + 3, generator=g)
        pos = torch.randperm(x.numel() // 2, generator=g)[:len(specials)]  # kept by every layout
        x[pos] = torch.tensor(specials)
        mask = torch.rand(x.shape, generator=g) > 0.3
        mask[pos] = True
        for xs, mask, off in _moment_layouts(x, mask):
            xd = _on_device(xs, off)
            md = None if mask is None else mask.cuda()
            reached |= moment_bodies(xd, md)
            s, dev, n = ops.moments(xd, md)
            sel = xs if mask is None else xs[mask]
            assert n == sel.numel()
            want_mean, want_std = float(sel.double().mean()), float(sel.std())
            got_mean, got_var = s / n, dev / (n - 1)
            if math.isnan(want_mean):
                assert math.isnan(got_mean)
            else:
                assert got_mean == want_mean  # ±Inf
            assert math.isnan(want_std) and math.isnan(got_var)
    assert reached == MOMENT_PATHS


# ---- (b) radix select -------------------------------------------------------------------------------

SELECT_PATHS = {f"select_{p}" for p in (
    "uint4", "uint4_tail", "unaligned", "masked", "unmasked", "mask_single_voxel", "q_edges", "rounds",
    "shared_prefix", "range_walk", "runs", "specials", "nan_both_signs", "batch_1", "batch_3", "batch_40",
    "index_64bit")} | {f"select_dtype_{str(d)[6:]}" for d in IMAGE_DTYPES}


def order_keys(f: np.ndarray) -> np.ndarray:
    """ATen's radix key of fp32 values: bits ^ (sign ? 0xffffffff : 0x80000000), NaN -> 0xffffffff."""
    u = np.ascontiguousarray(f, dtype=np.float32).view(np.uint32)
    k = u ^ np.where(u >> 31 == 1, np.uint32(0xFFFFFFFF), np.uint32(0x80000000))
    k[np.isnan(f)] = 0xFFFFFFFF
    return k


def key_values(k: np.ndarray) -> np.ndarray:
    u = np.where(k >> 31 == 1, k ^ np.uint32(0x80000000), ~k).astype(np.uint32)
    return u.view(np.float32)


def select_bodies(x: torch.Tensor, mask) -> set:
    """Bodies of select_hist_kernel each element of ``x`` runs (element b starts at b * per_elem)."""
    size = x.element_size()
    per, v = x[0].numel(), 16 // size
    out = {"select_masked" if mask is not None else "select_unmasked", f"select_dtype_{str(x.dtype)[6:]}"}
    for b in range(x.shape[0]):
        if (x.data_ptr() + b * per * size) % 16:
            out.add("select_unaligned")
            continue
        if per >= v:
            out.add("select_uint4")
        if per % v:
            out.add("select_uint4_tail")
    return out


def round_structure(target_keys: np.ndarray, ranks: np.ndarray) -> set:
    """Per round of 13 quantiles: distinct ranks that share a level-1 histogram (the same top 11 key
    bits), and level-2 prefixes (top 22 bits) that share their top 11 bits, which walk `tab`'s range."""
    out = set()
    per = 2 * QUANT_PER_ROUND
    for r0 in range(0, target_keys.size, per):
        k, rk = target_keys[r0:r0 + per], ranks[r0:r0 + per]
        top = np.unique(k >> 21)
        if top.size < np.unique(rk).size:
            out.add("select_shared_prefix")
        if np.unique(k >> 10).size > top.size:
            out.add("select_range_walk")
    return out


def check_select(x: torch.Tensor, qs, mask: torch.Tensor | None = None) -> set:
    """ops.quantiles_batched of the CUDA tensor ``x`` (B, ...) against a numpy sort of each
    element's keys.  Returns the bodies and structures reached."""
    qs = np.asarray(qs, dtype=np.float64)
    vals, w, count, has_nan = (t.cpu().numpy() for t in ops.quantiles_batched(x, qs, mask))
    b_count = x.shape[0]
    flat = x.cpu().float().reshape(b_count, -1).numpy()
    sel = None if mask is None else mask.cpu().reshape(b_count, -1).numpy().astype(bool)
    reached = select_bodies(x, mask)
    if len(qs) > QUANT_PER_ROUND:
        reached.add("select_rounds")
    if 0.0 in qs and 1.0 in qs:
        reached.add("select_q_edges")
    for b in range(b_count):
        v = flat[b] if sel is None else flat[b][sel[b]]
        c = v.size
        if c == 1:
            reached.add("select_mask_single_voxel")
        nan = np.isnan(v)
        if nan.any() and (np.signbit(v[nan]).any() and (~np.signbit(v[nan])).any()):
            reached.add("select_nan_both_signs")
        keys = np.sort(order_keys(v))
        assert count[b] == c and bool(has_nan[b]) == bool(nan.any()), b
        index = qs * (c - 1)
        lower = np.floor(index)
        assert np.array_equal(w[b], index - lower), b
        ranks = np.stack([lower, np.minimum(lower + 1, c - 1)], 1).reshape(-1).astype(np.int64)
        want = key_values(keys[ranks])
        got = vals[b]
        want_nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), want_nan), (b, got, want)
        bad = got.view(np.uint32)[~want_nan] != want.view(np.uint32)[~want_nan]
        assert not bad.any(), (b, np.flatnonzero(bad)[:5], got[~want_nan][bad][:5], want[~want_nan][bad][:5])
        reached |= round_structure(keys[ranks], ranks)
    print(f"[select {str(x.dtype)[6:]} B={b_count} per_elem={x[0].numel()} m={len(qs)}"
          f"{' masked' if mask is not None else ''}] every order statistic, weight and count exact")
    return reached


def _values(shape, dtype, seed):
    """Random values of ``dtype`` with ties; int32 / int64 above 2^24, where .float() rounds."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g, dtype=torch.float64)
    if dtype == torch.uint8:
        return (x.abs() * 60).clamp(0, 255).to(dtype)
    if dtype == torch.int8:
        return (x * 40).clamp(-128, 127).to(dtype)
    if dtype == torch.int16:
        return (x * 3000).to(dtype)
    if dtype in (torch.int32, torch.int64):
        return (x * 3e8).round().to(dtype)
    return (x * 50).to(dtype)


def _specials(dtype) -> torch.Tensor:
    """±0, subnormals (of the dtype and, for fp64, of fp32 and below it), ±Inf, NaNs of both signs."""
    inf = math.inf
    vals = [0.0, -0.0, 0.0, -0.0, inf, -inf, inf]
    if dtype == torch.float16:
        vals += [6e-8, -6e-8, 3e-5]
    elif dtype == torch.bfloat16:
        vals += [1e-39, -1e-39]
    elif dtype == torch.float32:
        vals += [1e-45, -1e-45, 1e-40, -3e-39]
    else:  # fp64: fp32 subnormals, values that .float() rounds to ±0 and ±Inf
        vals += [1e-40, -1e-40, 1e-50, -1e-50, 1e39, -1e39, 3.4028235677973366e38]
    t = torch.tensor(vals, dtype=torch.float64).to(dtype)
    return torch.cat([t, _nan(dtype, negative=False), _neg_nan(dtype), _neg_nan(dtype)])


QS_MANY = np.concatenate([[0.0, 1.0], np.linspace(0.003, 0.997, 13), [0.5, 0.25]])  # 17: two rounds


@pytest.mark.parametrize("dtype", IMAGE_DTYPES, ids=str)
def test_select_every_dtype_and_body(dtype):
    """3 elements of 693 voxels: element 0 aligned (uint4 body and a tail), 1 and 2 unaligned; masked
    and unmasked; floats carry ±0, subnormals, ±Inf and NaNs of both signs."""
    shape = (3, 1, 7, 9, 11)
    x = _values(shape, dtype, 5)
    if dtype.is_floating_point:
        sp = _specials(dtype)
        flat = x.view(3, -1)
        for b in range(3):
            pos = torch.randperm(flat.shape[1], generator=torch.Generator().manual_seed(b))[:sp.numel()]
            _put_bits(flat, (b, pos), sp)
    xd = x.cuda()
    mask = torch.rand(shape, generator=torch.Generator().manual_seed(6)) > 0.4
    reached = check_select(xd, QS_MANY) | check_select(xd, QS_MANY, mask.cuda())
    want = {"select_uint4", "select_uint4_tail", "select_unaligned", "select_masked", "select_unmasked",
            "select_rounds", "select_q_edges", f"select_dtype_{str(dtype)[6:]}"}
    if dtype.is_floating_point:
        want.add("select_nan_both_signs")
    assert want <= reached, want - reached


def test_select_specials_order_like_aten():
    """A small fp32 volume of nothing but specials and a few finite values: every rank read, so each
    NaN, ±Inf, ±0 and subnormal is some order statistic."""
    sp = _specials(torch.float32)
    x = torch.cat([sp, torch.tensor([1.5, -2.0, 1e-30, -1e-30, 7.0]), _neg_nan(), sp]).repeat(3)
    n = x.numel()
    qs = np.arange(n) / (n - 1)  # every rank, several rounds
    reached = check_select(x.reshape(1, n).cuda(), qs)
    reached |= check_select(_on_device(x.reshape(1, n), 1), qs)  # unaligned
    assert {"select_nan_both_signs", "select_rounds", "select_q_edges", "select_uint4", "select_uint4_tail",
            "select_unaligned"} <= reached


@pytest.mark.parametrize("b", [1, 3, 40])
def test_select_masks_and_batches(b):
    """Per-element masks of different counts, one element of a single voxel, q = 0 and 1; aligned
    (per_elem % 4 == 0) and unaligned (odd per_elem) elements."""
    reached = set()
    for per in (4096, 1001):
        x = _values((b, per), torch.float32, b)
        g = torch.Generator().manual_seed(per + b)
        keep = torch.rand((b, 1), generator=g) * 0.9 + 0.05
        mask = torch.rand((b, per), generator=g) < keep
        mask[0] = False
        mask[0, per // 3] = True  # one voxel
        reached |= check_select(x.cuda(), [0.0, 0.31, 0.5, 1.0], mask.cuda())
        reached |= check_select(x.cuda(), [0.0, 0.31, 0.5, 1.0])
    assert {"select_mask_single_voxel", "select_q_edges", "select_masked", "select_unmasked"} <= reached
    assert ("select_unaligned" in reached) == (b > 1)


def test_select_shared_prefixes_and_range_walk():
    """Values packed into 4096 consecutive fp32 ulps above 1.0 (a range of 2^-11 relative): all ranks
    share their top 11 key bits (one level-1 histogram), their level-2 prefixes differ and share
    those 11 bits, so level 2 walks a range of `tab`.  13 quantiles: one full round."""
    g = torch.Generator().manual_seed(9)
    k = torch.randint(0, 4096, (2, 50_000), generator=g).to(torch.float64)
    x = (1.0 + k * 2.0**-23).to(torch.float32)
    qs = np.linspace(0.02, 0.98, 13)
    reached = check_select(x.cuda(), qs)
    reached |= check_select(x.cuda(), qs, (torch.rand(x.shape, generator=g) > 0.5).cuda())
    assert {"select_shared_prefix", "select_range_walk"} <= reached


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float32], ids=str)
def test_select_runs_of_ties(dtype):
    """A constant background with sparse islands: long runs of one bin in every thread's loads, which
    flush_run coalesces into one atomic."""
    g = torch.Generator().manual_seed(11)
    x = torch.zeros((3, 64, 64, 64), dtype=dtype)
    flat = x.view(3, -1)
    for b in range(3):
        idx = torch.randperm(flat.shape[1], generator=g)[:2000 * (b + 1)]
        flat[b, idx] = _values((idx.numel(),), dtype, b).abs().to(dtype) + 1
        flat[b, 1000:1000 + 100_000] = 7  # one long run of another value
    run = flat[0, 1000:1000 + 100_000]
    assert bool((run == run[0]).all()) and run.numel() >= 16 * 1024
    reached = check_select(x.cuda(), QS_MANY)
    assert {"select_uint4", "select_rounds"} <= reached


def test_select_more_than_2_to_the_31_voxels():
    """One uint8 element of 2^31 + 2^20 + 5 voxels (2.1 GB): 32 copies of a random 64 MiB block of
    values 1..254 and a tail past 2^31 that alone holds the 0s and the 255s, so the extreme order
    statistics come only from voxels at 64-bit indices.  Order statistics from np.bincount."""
    blk = 1 << 26
    block = np.random.default_rng(13).integers(1, 255, blk, dtype=np.uint8)
    tail = np.zeros((1 << 20) + 5, np.uint8)
    tail[::3] = 255
    tail[1::7] = np.random.default_rng(14).integers(1, 255, tail[1::7].size, dtype=np.uint8)
    n = 32 * blk + tail.size
    assert n > 2**31 and n % 16
    counts = 32 * np.bincount(block, minlength=256) + np.bincount(tail, minlength=256)
    assert counts.sum() == n
    x = torch.empty((1, n), dtype=torch.uint8, device="cuda")
    x[0, :32 * blk].view(32, blk).copy_(torch.from_numpy(block).cuda().expand(32, blk))
    x[0, 32 * blk:].copy_(torch.from_numpy(tail).cuda())
    qs = np.array([0.0, 1e-6, 0.25, 0.5, 0.75, 1 - 1e-6, 1.0])
    vals, w, count, has_nan = (t.cpu().numpy() for t in ops.quantiles_batched(x, qs))
    del x
    index = qs * (n - 1)
    lower = np.floor(index)
    ranks = np.stack([lower, np.minimum(lower + 1, n - 1)], 1).reshape(-1).astype(np.int64)
    want = np.searchsorted(np.cumsum(counts), ranks, side="right").astype(np.float32)
    assert count[0] == n and has_nan[0] == 0
    assert np.array_equal(w[0], index - lower)
    assert np.array_equal(vals[0], want), (vals[0], want)
    assert want[0] == 0 and want[-1] == 255


# ---- (c) minimum of sample 0 ------------------------------------------------------------------------

MIN_PATHS = {"min_vector", "min_scalar", "min_c1", "min_c3", "min_signed_zero_blocks", "min_nan"}


def check_min(x: torch.Tensor) -> set:
    """ops.min_sample0 of the CUDA (B, C, ...) ``x`` against torch.amin's semantics per channel of
    element 0: NaN if any NaN, else the least value (compared by value, so -0.0 == 0.0)."""
    got = ops.min_sample0(x).cpu().numpy()
    c = x.shape[1]
    v = x[0].reshape(c, -1).cpu().numpy()
    for ch in range(c):
        nan = np.isnan(v[ch])
        want = math.nan if nan.any() else float(v[ch].min())
        if math.isnan(want):
            assert math.isnan(got[ch]), (ch, got[ch])
        else:
            assert got[ch] == want, (ch, got[ch], want)
    n = v.shape[1]
    print(f"[min C={c} n={n}] {got} equals amin's")
    vec = x.data_ptr() % 16 == 0 and n % 4 == 0
    return {"min_vector" if vec else "min_scalar", f"min_c{c}"} | ({"min_nan"} if np.isnan(v).any() else set())


@pytest.mark.parametrize("c", [1, 3])
def test_min_bodies(c):
    reached = set()
    g = torch.Generator().manual_seed(c)
    for shape in ((16, 16, 16), (5, 7, 3), (64, 64, 65)):
        x = torch.randn((2, c, *shape), generator=g) * 10 + 3
        reached |= check_min(x.cuda())
    assert {"min_vector", "min_scalar", f"min_c{c}"} <= reached


@pytest.mark.parametrize("where", ["last", "first"])
def test_min_negative_zero_and_a_negative_in_other_blocks(where):
    """Channels of -0.0 and positives with one small negative region: the blocks that see only -0.0
    and positives end with -0.0, and their atomics race the negative block's.  One wave of blocks
    (n = 2^20: 1024 blocks of 256 float4), so the finishing order is the scheduler's."""
    reached = set()
    for c in (1, 3):
        n = 1 << 20
        g = torch.Generator().manual_seed(17 + c)
        x = torch.rand((2, c, n), generator=g) + 0.5
        x[:, :, ::5] = -0.0
        neg = slice(n - 300, n - 200) if where == "last" else slice(100, 200)
        x[0, :, neg] = -torch.rand((c, 100), generator=g) - 1.0
        for layout in (x, x[:, :, :-1].contiguous()):  # vector and scalar bodies
            for _ in range(3):
                reached |= check_min(layout.reshape(2, c, -1, 1, 1).cuda())
    assert {"min_vector", "min_scalar", "min_c1", "min_c3"} <= reached


def test_min_nan_wins():
    """NaN of either sign anywhere in a channel gives NaN, as amin does; other channels keep their min."""
    reached = set()
    for n in (1 << 16, (1 << 16) + 1):
        x = torch.randn((1, 3, n), generator=torch.Generator().manual_seed(n))
        x[0, 0, n // 2] = math.nan
        x[0, 1, 7] = _neg_nan()
        x[0, 1, n - 3] = -1e30
        reached |= check_min(x.reshape(1, 3, -1, 1, 1).cuda())
        assert np.isfinite(ops.min_sample0(x.reshape(1, 3, -1, 1, 1).cuda()).cpu().numpy()[2])
    assert {"min_nan", "min_vector", "min_scalar"} <= reached


COVERAGE = {
    "test_moments_bodies_against_float64": MOMENT_PATHS,
    "test_moments_constant_selection_has_zero_variance": MOMENT_PATHS,
    "test_moments_near_constant": MOMENT_PATHS,
    "test_moments_nonfinite_follow_torch": MOMENT_PATHS,
    "test_select_every_dtype_and_body": {"select_uint4", "select_uint4_tail", "select_unaligned", "select_masked",
                                         "select_unmasked", "select_rounds", "select_q_edges",
                                         "select_nan_both_signs"}
                                        | {f"select_dtype_{str(d)[6:]}" for d in IMAGE_DTYPES},
    "test_select_specials_order_like_aten": {"select_specials", "select_nan_both_signs"},
    "test_select_masks_and_batches": {"select_mask_single_voxel", "select_batch_1", "select_batch_3",
                                      "select_batch_40", "select_masked"},
    "test_select_shared_prefixes_and_range_walk": {"select_shared_prefix", "select_range_walk"},
    "test_select_runs_of_ties": {"select_runs"},
    "test_select_more_than_2_to_the_31_voxels": {"select_index_64bit"},
    "test_min_bodies": {"min_vector", "min_scalar", "min_c1", "min_c3"},
    "test_min_negative_zero_and_a_negative_in_other_blocks": {"min_signed_zero_blocks"},
    "test_min_nan_wins": {"min_nan"},
}


def test_cases_cover_every_path():
    """The cases together reach every body of the three kernels; each case asserts the layouts and
    data that put it on its bodies."""
    assert all(callable(globals().get(name)) for name in COVERAGE)
    for name, paths in COVERAGE.items():  # a case claims bodies of its own kernel only
        kernel = {"moments": "moments_", "select": "select_", "min": "min_"}[name.split("_")[1]]
        assert all(p.startswith(kernel) for p in paths), name
    reached = set().union(*COVERAGE.values())
    everything = MOMENT_PATHS | SELECT_PATHS | MIN_PATHS
    assert everything == reached, sorted(everything ^ reached)


# ---- (d) end to end against the reference's op sequence --------------------------------------------

def _batch(x: torch.Tensor):
    import torchio_b200 as tio

    return tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(x.shape[0])])})


def _same(got: float, want: float) -> bool:
    return (math.isnan(got) and math.isnan(want)) or got == want


@pytest.mark.parametrize("value", [1000.1, 123.456, -7.25, 0.0], ids=str)
@pytest.mark.parametrize("masked", [False, True])
def test_standardize_constant_image_raises(value, masked):
    """The reference's Welford std() of a constant is exactly 0, and Standardize raises."""
    import torchio_b200 as tio

    x = torch.full((2, 1, 256, 256, 256), value, device="cuda")
    method = None
    if masked:
        x[0, 0, :, :, :100] = value + 5.0
        method = lambda t: t == np.float32(value)  # noqa: E731
        sel = x[0][method(x[0])]
    else:
        sel = x[0].reshape(-1)
    assert float(sel.float().std()) == 0.0  # the reference's statistic
    with pytest.raises(RuntimeError, match="Standard deviation is zero"):
        tio.Standardize(masking_method=method)(_batch(x))


def test_standardize_near_constant_and_single_voxel():
    """std of values a few ulps around 1000.1 and 2^20, within fp32 rounding of float64's; a mask of one
    voxel gives NaN, as the reference's std() of one value does."""
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(21)
    for center in (1000.1, 2.0**20):
        c = np.float32(center)
        k = torch.randint(-4, 5, (1, 1, 128, 128, 128), generator=g).double()
        x = (float(c) + k * float(np.spacing(c))).float()
        out = tio.Standardize()(_batch(x.repeat(2, 1, 1, 1, 1).cuda()))
        mean, std = out.applied_transforms[0].params["stats"]["t1"]
        v = x.double().reshape(-1)
        want_mean, want_std = float(v.mean()), float(v.std())
        assert abs(std - want_std) <= 2.0**-23 * want_std * 1.01, (std, want_std)
        assert abs(mean - want_mean) <= float(np.spacing(np.float32(want_mean))), (mean, want_mean)
        print(f"[Standardize near {center}] std {std:.6e} vs float64 {want_std:.6e}")
    x = torch.randn((2, 1, 8, 8, 8), generator=g).cuda()
    single = lambda t: t == t[0, 3, 4, 5]  # noqa: E731
    assert int(single(x[0]).sum()) == 1 and x[0][single(x[0])].float().std().isnan()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = tio.Standardize(masking_method=single)(_batch(x))
    mean, std = out.applied_transforms[0].params["stats"]["t1"]
    assert mean == float(x[0, 0, 3, 4, 5]) and math.isnan(std)


def _signed_data(shape, seed, dtype=torch.float32):
    """randn with -0.0 runs and host-made negative NaNs (0xffc00000 in fp32)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(shape, generator=g) * 4
    flat = x.view(shape[0], -1)
    flat[:, 5:40] = -0.0
    pos = torch.randperm(flat.shape[1], generator=g)[:9]
    _put_bits(flat, (slice(None), pos), _neg_nan().expand(shape[0], 9))
    return x.to(dtype)


def test_normalize_percentiles_with_negative_nans():
    """in_ranges against compute_quantile (kthvalue + lerp) on the same CUDA tensor, which sorts every
    NaN above +Inf."""
    import torchio_b200 as tio

    x = _signed_data((2, 1, 1, 73, 137), 23).cuda()  # 10001 voxels: these percentiles need no lerp
    for low, high in ((0.0, 95.0), (1.0, 99.0), (2.5, 100.0)):
        assert all(q / 100 * 10000 == int(q * 100) for q in (low, high))
        out = tio.Normalize(percentile_low=low, percentile_high=high)(_batch(x))
        got = out.applied_transforms[0].params["in_ranges"]["t1"]
        values = x[0].reshape(-1).float()
        want = (float(tp._quantile(values, low / 100)), float(tp._quantile(values, high / 100)))
        assert all(_same(a, b) for a, b in zip(got, want)), (low, high, got, want)


def _reference_pad_statistic(data: torch.Tensor, mode: str) -> torch.Tensor:
    """_compute_padding_statistic (_padding.py:43-69) on the CUDA tensor."""
    flat = data.flatten(start_dim=1)
    if mode == "minimum":
        return flat.amin(dim=1)
    float_flat = flat if data.dtype in (torch.float32, torch.float64) else flat.float()
    if mode == "mean":
        statistic = float_flat.mean(dim=1)
    else:
        statistic = torch.stack([tp._quantile(values, 0.5) for values in float_flat])
    return statistic.to(data.dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64, torch.float16, torch.int16], ids=str)
@pytest.mark.parametrize("mode", ["minimum", "mean", "median"])
def test_pad_statistics_match_the_reference(mode, dtype):
    """Pad's statistic modes on data with -0.0 and negative NaNs (element 1 has no NaN), fp64 kept in
    fp64; the padded voxels against the reference's statistic."""
    import torchio_b200 as tio

    x = _signed_data((3, 1, 21, 15, 13), 29)  # 4095 voxels: the median needs no lerp
    x[1].nan_to_num_(0.5)
    x[2, 0, 3, 4, 5] = -1e3  # element 2's minimum
    if dtype == torch.int16:
        x = x.nan_to_num(0.0).mul(100)
    x = x.to(dtype).cuda()
    if dtype == torch.float64:  # values fp32 cannot hold
        x = x + 1e-9 * torch.arange(x.numel(), device="cuda", dtype=torch.float64).view(x.shape)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = tio.Pad(padding=(2, 1, 0, 3, 1, 1), padding_mode=mode)(_batch(x)).images["t1"].data
        want = _reference_pad_statistic(x, mode)
    assert out.dtype == dtype
    assert torch.equal(out[:, :, 2:-1, 0:-3, 1:-1].contiguous().view(torch.uint8), x.view(torch.uint8))
    for b in range(3):
        pad = out[b, :, :2].reshape(-1).double().cpu()
        w = float(want[b])
        if math.isnan(w):
            assert bool(pad.isnan().all()), (mode, b, pad[0])
        elif mode == "mean" and dtype != torch.float64:
            # fp64 sums rounded once to fp32 (then cast): within rounding of the float64 mean.  The
            # reference's fp32 cascade sum is within its own, larger, rounding error of it.
            exact = float(x[b].double().mean())
            tol = 1.0 if dtype == torch.int16 else float(np.spacing(np.float32(abs(exact))))
            if dtype == torch.float16:
                tol += float(np.spacing(np.float16(abs(exact))))
            assert bool(((pad - exact).abs() <= tol).all()), (b, pad[0], exact, w)
        else:
            assert bool((pad == w).all()), (mode, b, pad[0], w)


def test_default_pad_value_minimum_with_signed_zero_and_nan():
    """default_pad_value="minimum" of a transform that moves every voxel out of the volume: every output
    voxel is element 0's channel minimum (amin: NaN when the channel holds a NaN)."""
    import torchio_b200 as tio

    n = 64
    x = torch.rand((2, 2, n, n, n), generator=torch.Generator().manual_seed(31)) + 0.5
    x[0, :, ::3] = -0.0
    x[0, 0, -2:, -3:] = -torch.rand((2, 3, n)) - 2.0  # a negative region in the last blocks
    x[0, 1, 40, 40, 40] = _neg_nan()
    xd = x.cuda()
    want = tp.fill_value_for(xd, "scalar", "minimum", 0)
    assert float(want[0]) < -2.0 and math.isnan(float(want[1]))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = tio.Affine(translation=(500.0, 500.0), default_pad_value="minimum")(_batch(xd))
    y = out.images["t1"].data.cpu()
    assert bool((y[:, 0] == float(want[0])).all())
    assert bool(y[:, 1].isnan().all())
