"""Every kernel path of the intensity chain (bias -> blur -> noise -> gamma, `tio_intensity_fused`)
against a plain float64 reference, and against each other.

Depending on the table radius R, K % 4, 16-byte alignment and the blurred axes, the chain runs
one of seven kernel bodies:
    pass 1 (bias + I axis)   march6_kernel (R <= 6, aligned, K % 4 == 0), march_kernel<4>,
                             march_kernel<1>
    pass 2 (K then J axis)   jk6_kernel (TMA: R <= 6, aligned, K % 4 == 0), jk_kernel<6>,
                             jk_kernel<16>
    R > 16                   axis_kernel, one launch per blurred axis
The tests below force each one through its dispatch condition: a table zero-padded to a larger
R (the element radii stay the same), K % 4 != 0, or a source view at storage offset 1.

`ref64` is written from the reference's semantics (TorchIO's bias_field.py, blur.py, noise.py,
gamma.py), not from the kernels: align-corners trilinear upsampling, exp, multiply or divide;
per-axis convolution with the element's own taps and clamped indices, for any radius; additive
or Rician noise; sign(x) |x|^gamma with sign(+-0) = 0.  Everything is float64 numpy.

Error bound.  With u = 2^-24, a chain of fp32 operations whose exact inputs are x and whose
partial results are bounded in magnitude by S differs from the exact result by at most
n u S (first order), where n counts the roundings on the chain.  `ref64` returns S, the same
linear chain applied to |x| and |taps|, and n per voxel:
  bias      the three lerp levels (fma + product) round six times, at most M each, M = max
            |coarse| of the element; each axis's fp32 weight is within 4 u (s - 1) of the exact
            one (s = coarse size, source coordinates <= s - 1) and multiplies a difference of at
            most 2 M: the exponent is within (6 + 8 sum(s - 1)) u M.  expf is within 2 ulp (4 u)
            and the multiply or divide adds one rounding: n += (6 + 8 sum(s - 1)) M + 8 with
            S = |x f|.
  blur      one fma per tap: n += 2r + 1 per blurred axis (2 (2r + 1) for a chain of separately
            rounded products and sums, as the C oracle computes); S is convolved with |taps|.
  noise     n1 = mean + std z (two roundings), v + n1 (one): n += 3, S += |mean| + |std z|.
            Rician sqrt((v + n1)^2 + n2^2): with s = v + n1 the derivative of the result is
            at most 1 in s and in n2, and the squares, sum and sqrt add four roundings of at
            most the result: n += 8, S += |n1| + |n2|.
  gamma     |x|^g = ex2(g lg2|x|) on the SFU.  The PTX ISA states lg2.approx.f32 to within
            2^-22 absolute on [0.5, 2] and 2 ulp elsewhere, ex2.approx.f32 to within 2 ulp
            (2^-22 relative); so with E = ln2 (g 2^-22 max(1, |log2 x|) + u |g log2 x|)
            + 2^-22 + u the SFU result is within E relative (plus 2^-149 absolute below the
            normal range).  The input error e = n u S is carried through the monotone
            |x|^g exactly: the output may be anywhere in [(|v| - e)^g, (|v| + e)^g], and where
            e >= |v| the sign may flip.
Each case prints the largest observed |got - ref64| / bound, so a later change sees its margin.
"""

from __future__ import annotations

import ctypes
import math

import numpy as np
import pytest
import torch

from torchio_b200 import tables

U = 2.0 ** -24
E_SFU = 2.0 ** -22


# ---------------------------------------------------------------------------------------------
# the float64 reference
# ---------------------------------------------------------------------------------------------


def _lerp64(n_in: int, n_out: int):
    """align_corners=True source indices and weights of one axis."""
    o = np.arange(n_out)
    if n_in == n_out:
        return o, o, np.ones(n_out), np.zeros(n_out)
    scale = (n_in - 1) / (n_out - 1) if n_out > 1 else 0.0
    real = scale * o
    i0 = np.minimum(np.floor(real).astype(np.int64), n_in - 1)
    i1 = np.minimum(i0 + 1, n_in - 1)
    l1 = np.clip(real - i0, 0.0, 1.0)
    return i0, i1, 1.0 - l1, l1


def upsample64(g: np.ndarray, shape) -> np.ndarray:
    """Trilinear align-corners upsampling of (..., si, sj, sk) to (..., I, J, K)."""
    out = np.asarray(g, dtype=np.float64)
    for axis, n_out in enumerate(shape):
        ax = out.ndim - 3 + axis
        i0, i1, l0, l1 = _lerp64(out.shape[ax], n_out)
        bshape = [1] * out.ndim
        bshape[ax] = n_out
        out = np.take(out, i0, ax) * l0.reshape(bshape) + np.take(out, i1, ax) * l1.reshape(bshape)
    return out


def blur_axis64(x: np.ndarray, taps: np.ndarray, axis: int) -> np.ndarray:
    """Convolution of x (..., I, J, K) along spatial `axis` with 2r+1 centred taps, replicate
    (clamped) indices, any r, including r larger than the axis."""
    r = (len(taps) - 1) // 2
    ax = x.ndim - 3 + axis
    n = x.shape[ax]
    out = np.zeros_like(x)
    for t in range(-r, r + 1):
        idx = np.clip(np.arange(n) + t, 0, n - 1)
        out = out + float(taps[t + r]) * np.take(x, idx, ax)
    return out


class Ref:
    def __init__(self, y, pre, n, s, gamma):
        self.y, self.pre, self.n, self.s, self.gamma = y, pre, n, s, gamma

    def bound(self) -> np.ndarray:
        e = self.n * U * self.s
        if self.gamma is None:
            return e
        g = self.gamma.reshape(-1, *([1] * (self.pre.ndim - 1)))
        with np.errstate(all="ignore"):
            a = np.abs(self.pre)
            hi = a + e
            lo = np.maximum(a - e, 0.0)
            p, phi, plo = a ** g, hi ** g, lo ** g
            lg = np.maximum(np.abs(np.log2(np.maximum(hi, 1e-300))), np.abs(np.log2(np.maximum(lo, 1e-300))))
            sfu = math.log(2) * (g * E_SFU * np.maximum(1.0, lg) + U * g * lg) + E_SFU + U
            swing = np.maximum(phi - p, p - plo)
            swing = np.where(e >= a, p + phi, swing)  # the sign may flip
            out = swing + phi * sfu + 2.0 ** -148
        return np.where(g == 1.0, e, out)


def ref64(x, *, coarse=None, bias_identity=None, divide=False, taps=None, radius=None, axes_mask=0,
          mean=None, std=None, keep=None, z=None, z2=None, rician=False, gamma=None,
          roundings_per_tap=1) -> Ref:
    """float64 chain on (B, C, I, J, K) numpy data; every table as the kernels receive it."""
    x = np.asarray(x, dtype=np.float64)
    b_n = x.shape[0]
    shape = x.shape[2:]
    y = x.copy()
    s = np.abs(x)
    n = np.zeros(x.shape)
    with np.errstate(all="ignore"):
        for b in range(b_n):
            if coarse is not None and not (bias_identity is not None and bias_identity[b]):
                f = np.exp(upsample64(coarse[b], shape))
                y[b] = y[b] / f if divide else y[b] * f
                s[b] = np.abs(y[b])
                n[b] += (6 + 8 * (sum(coarse.shape[2:]) - 3)) * float(np.abs(coarse[b]).max()) + 8
            if taps is not None:
                big_r = (taps.shape[2] - 1) // 2
                for axis in range(3):
                    r = int(radius[axis, b])
                    if not (axes_mask >> axis) & 1 or r == 0:
                        continue
                    row = np.asarray(taps[axis, b, big_r - r: big_r + r + 1], dtype=np.float64)
                    y[b] = blur_axis64(y[b], row, axis)
                    s[b] = blur_axis64(s[b], np.abs(row), axis)
                    n[b] += roundings_per_tap * (2 * r + 1)
            if z is not None and (keep is None or keep[b]):
                n1 = float(mean[b]) + float(std[b]) * z[b].astype(np.float64)
                if rician:
                    n2 = float(mean[b]) + float(std[b]) * z2[b].astype(np.float64)
                    y[b] = np.sqrt((y[b] + n1) ** 2 + n2 ** 2)
                    s[b] = s[b] + np.abs(n1) + np.abs(n2)
                    n[b] += 8
                else:
                    y[b] = y[b] + n1
                    s[b] = s[b] + abs(float(mean[b])) + np.abs(float(std[b]) * z[b])
                    n[b] += 3
        pre = y.copy()
        g = None
        if gamma is not None:
            g = np.asarray(gamma, dtype=np.float64)
            gb = g.reshape(-1, 1, 1, 1, 1)
            y = np.where(gb == 1.0, y, np.sign(y) * np.abs(y) ** gb)
    return Ref(y, pre, n, s, g)


def classes(a) -> np.ndarray:
    """0 finite, 1 NaN, 2 +Inf, 3 -Inf."""
    a = np.asarray(a)
    c = np.zeros(a.shape, dtype=np.int8)
    c[np.isnan(a)] = 1
    c[np.isposinf(a)] = 2
    c[np.isneginf(a)] = 3
    return c


def check_bound(got, ref: Ref, label: str) -> float:
    """Classes equal; finite voxels within the bound.  Returns the largest fraction used."""
    got = np.asarray(got, dtype=np.float64)
    cg, cr = classes(got), classes(ref.y)
    bad = np.argwhere(cg != cr)
    assert bad.size == 0, (f"{label}: {len(bad)} voxels of another class than ref64, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, ref64 {ref.y[tuple(bad[0])]!r}")
    fin = cr == 0
    bound = ref.bound()
    err = np.abs(got - ref.y)
    over = fin & (err > bound)
    if over.any():
        first = tuple(np.argwhere(over)[0])
        raise AssertionError(f"{label}: {int(over.sum())} voxels beyond the bound, first at {first}: got "
                             f"{got[first]!r}, ref64 {ref.y[first]!r}, bound {bound[first]:.3e}")
    with np.errstate(all="ignore"):
        frac = np.where(fin & (bound > 0), err / np.where(bound > 0, bound, 1.0), 0.0)
    worst = float(frac.max()) if frac.size else 0.0
    print(f"{label}: max |got - ref64| / bound = {worst:.3f}")
    return worst


def sigma_for_radius(r: int) -> float:
    """A sigma whose taps have radius max(ceil(3 sigma), 1) == r (0 = no blur)."""
    return 0.0 if r == 0 else (r - 0.5) / 3.0


def pad_table(taps: torch.Tensor, new_r: int) -> torch.Tensor:
    """The same taps centred in a table of half-width new_r (zero beyond)."""
    big_r = (taps.shape[2] - 1) // 2
    out = torch.zeros((3, taps.shape[1], 2 * new_r + 1), dtype=taps.dtype)
    out[:, :, new_r - big_r: new_r + big_r + 1] = taps
    return out


# ---------------------------------------------------------------------------------------------
# CPU: ref64 against the C oracle and the torch restatement
# ---------------------------------------------------------------------------------------------


def _c():
    from oracle import c_port

    return c_port


def _random_tables(rng, b, per_element, radii_choice=(0, 1, 2, 3, 5, 8)):
    if per_element:
        sig = np.array([[sigma_for_radius(int(rng.choice(radii_choice))) for _ in range(3)] for _ in range(b)])
        sig[0] = 0.0  # an identity row
        if np.all(sig <= 0):
            sig[-1, 1] = 1.0
    else:
        sig = np.array([sigma_for_radius(int(rng.choice(radii_choice[1:]))) for _ in range(3)])
    return sig, tables.blur_tables(sig, b)


@pytest.mark.parametrize("seed", range(4))
def test_ref64_matches_c_oracle(seed):
    c_port = _c()
    lib, p = c_port.lib(), c_port._p
    rng = np.random.default_rng(seed)
    b, c, shape = 3, 2, (int(rng.integers(1, 9)), int(rng.integers(1, 9)), int(rng.integers(1, 12)))
    x = torch.as_tensor(rng.normal(0, 50, (b, c, *shape)).astype(np.float32))
    # bias
    coarse = torch.as_tensor(rng.normal(0, 0.4, (b, c, 2, 1, 3)).astype(np.float32))
    ident = torch.tensor([0, 1, 0], dtype=torch.uint8)
    for divide in (0, 1):
        out = torch.empty_like(x)
        assert lib.orc_bias_field(p(x), p(out), b, c, *shape, p(coarse), 2, 1, 3, p(ident), divide) == 0
        ref = ref64(x.numpy(), coarse=coarse.numpy(), bias_identity=ident.numpy(), divide=bool(divide))
        check_bound(out.numpy(), ref, f"orc_bias_field divide={divide}")
    # blur, shared and per-element
    for per_element in (False, True):
        _, t = _random_tables(rng, b, per_element)
        out = torch.empty_like(x)
        assert lib.orc_blur(p(x), p(out), None, b, c, *shape, p(t.taps), p(t.radius), t.big_r, p(t.identity)) == 0
        ref = ref64(x.numpy(), taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask,
                    roundings_per_tap=2)
        check_bound(out.numpy(), ref, f"orc_blur per_element={per_element}")
    # noise, Gaussian and Rician, one gated row
    mean = torch.tensor([0.5, -1.0, 2.0])
    std = torch.tensor([3.0, 0.5, 1.0])
    keep = torch.tensor([1, 0, 1], dtype=torch.uint8)
    z = torch.as_tensor(rng.normal(size=x.shape).astype(np.float32))
    z2 = torch.as_tensor(rng.normal(size=x.shape).astype(np.float32))
    for rician in (False, True):
        out = torch.empty_like(x)
        per = x[0].numel()
        assert lib.orc_noise(p(x), p(out), b, ctypes.c_int64(per), p(mean), p(std), p(keep), p(z),
                             p(z2) if rician else None) == 0
        ref = ref64(x.numpy(), mean=mean.numpy(), std=std.numpy(), keep=keep.numpy(), z=z.numpy(),
                    z2=z2.numpy(), rician=rician)
        check_bound(out.numpy(), ref, f"orc_noise rician={rician}")
    # gamma
    gam = torch.tensor([0.7, 1.0, 1.6])
    out = torch.empty_like(x)
    assert lib.orc_gamma(p(x), p(out), b, ctypes.c_int64(x[0].numel()), p(gam)) == 0
    check_bound(out.numpy(), ref64(x.numpy(), gamma=gam.numpy()), "orc_gamma")


def _nonfinite_input(rng, shape, frac=0.02):
    x = rng.normal(0, 10, shape).astype(np.float32)
    flat = x.reshape(-1)
    idx = rng.choice(flat.size, min(flat.size, max(3, int(frac * flat.size))), replace=False)
    flat[idx[0::3]] = np.nan
    flat[idx[1::3]] = np.inf
    flat[idx[2::3]] = -np.inf
    if x.shape[2] > 2 and x.shape[3] > 2:  # a NaN background block
        x[..., : x.shape[2] // 3, : x.shape[3] // 2, :] = np.nan
    return x


@pytest.mark.parametrize("per_element", [False, True])
def test_ref64_nonfinite_masks_match_c_oracle(per_element):
    c_port = _c()
    lib, p = c_port.lib(), c_port._p
    rng = np.random.default_rng(11 + per_element)
    b, c, shape = 3, 1, (9, 7, 10)
    x = torch.as_tensor(_nonfinite_input(rng, (b, c, *shape)))
    _, t = _random_tables(rng, b, per_element, radii_choice=(0, 1, 2, 4, 12))
    out = torch.empty_like(x)
    assert lib.orc_blur(p(x), p(out), None, b, c, *shape, p(t.taps), p(t.radius), t.big_r, p(t.identity)) == 0
    ref = ref64(x.numpy(), taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask)
    np.testing.assert_array_equal(classes(out.numpy()), classes(ref.y))


def test_ref64_nonfinite_masks_match_torch_port_shared():
    """Shared sigma: each element's radius is the table's, so the reference's own op sequence
    (F.pad replicate + F.conv3d per axis, CPU) spreads non-finite values exactly as ref64."""
    from oracle import torch_port

    rng = np.random.default_rng(5)
    x = _nonfinite_input(rng, (2, 2, 10, 9, 11))
    sig = [sigma_for_radius(2), 0.0, sigma_for_radius(4)]
    t = tables.blur_tables(sig, 2)
    want = torch_port.gaussian_smooth(torch.as_tensor(x), sig).numpy()
    ref = ref64(x, taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask)
    np.testing.assert_array_equal(classes(ref.y), classes(want))
    fin = classes(want) == 0
    assert np.all(np.abs(ref.y - want)[fin] <= 1e-5 * np.abs(want[fin]).max())


def test_sigma_for_radius():
    for r in range(0, 41):
        t = tables.blur_tables([sigma_for_radius(r), 0.0, 0.0] if r else [0.0, 1.0, 0.0], 1)
        assert int(t.radius[0, 0]) == r


# ---------------------------------------------------------------------------------------------
# GPU: the path matrix
# ---------------------------------------------------------------------------------------------

DEV = "cuda"
MAGNITUDES = {"milli": 1e-3, "unit": 1.0, "u12": 4095.0, "ct": None, "1e5": 1e5}


def _make_cases():
    """A seeded covering list: every listed size, radius, mask, stage and magnitude appears."""
    rng = np.random.default_rng(2024)
    sizes_i, sizes_j = [1, 5, 16, 17, 40], [1, 3, 7, 32, 33]
    sizes_k = [1, 3, 4, 8, 12, 64, 68, 132]
    wide = [7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 24, 40]
    cases = []
    n = 60
    for idx in range(n):
        i, j, k = sizes_i[idx % 5], sizes_j[(idx // 5) % 5], sizes_k[idx % 8]
        per_element = idx % 2 == 1
        mask = idx % 8
        b = 1 + idx % 3
        c = 1 + 2 * ((idx // 3) % 2)
        while b * c * i * j * k > 120_000 and (b > 1 or c > 1):
            b, c = max(1, b - 1), 1
        if idx < 21:  # radius 0..6 on each axis in turn, the others random
            radius_axis = (idx // 7) % 3
            fixed = idx % 7
            mask |= 1 << radius_axis
        else:
            radius_axis, fixed = None, None
        if idx >= 40:  # 7..16, 17, 24, 40 on one axis
            mask |= 1 << (idx % 3)
        def draw(axis):
            if not (mask >> axis) & 1:
                return 0
            if radius_axis == axis:
                return fixed
            if idx >= 40 and axis == (idx % 3):
                return wide[idx % len(wide)]
            return int(rng.integers(0, 7))
        if per_element:
            radii = np.array([[draw(a) for a in range(3)] for _ in range(b)])
            if b > 1:
                radii[0] = 0  # identity row
        else:
            radii = np.array([draw(a) for a in range(3)])
        if idx in (12, 20):  # TMA halo outside both K edges, and J < rj
            k, j = (4 if idx == 12 else 8), 3
            radii = np.array([0, 6, 6]) if not per_element else np.array([[0, 6, 6]] * b)
            mask = 6
        cases.append(dict(
            idx=idx, shape=(b, c, i, j, k), radii=radii, mask=mask,
            bias=[None, "mul", "div"][idx % 3], coarse=[(2, 3, 2), (1, 2, 3), (3, 1, 1)][(idx // 3) % 3],
            noise=[None, "gauss", "rician", "gauss"][(idx // 2) % 4], gated=idx % 5 == 0,
            gamma=[None, 0.7, 1.4, 1.0][(idx // 4) % 4], mag=list(MAGNITUDES)[idx % 5]))
    return cases


CASES = _make_cases()


def _inputs(case, nonfinite=False):
    rng = np.random.default_rng(1000 + case["idx"])
    b, c, i, j, k = case["shape"]
    shape = (b, c, i, j, k)
    scale = MAGNITUDES[case["mag"]]
    if nonfinite:
        x = _nonfinite_input(rng, shape)
    elif scale is None:
        x = rng.uniform(-1024, 3071, shape).astype(np.float32)
    else:
        x = (rng.uniform(0.2, 1.0, shape) * scale).astype(np.float32)
    scale = scale or 1000.0
    radii = case["radii"]
    if radii.ndim == 1:
        sig = [sigma_for_radius(int(r)) for r in radii]
    else:
        sig = [[sigma_for_radius(int(r)) for r in row] for row in radii]
    t = tables.blur_tables(sig, b)
    kw = {}
    ref_kw = {}
    if case["bias"]:
        coarse = rng.normal(0, 0.3, (b, c, *case["coarse"])).astype(np.float32)
        ident = np.zeros(b, np.uint8)
        if case["gated"]:
            ident[0] = 1
        kw.update(coarse=torch.as_tensor(coarse).to(DEV), bias_identity=torch.as_tensor(ident).to(DEV),
                  bias_divide=case["bias"] == "div")
        ref_kw.update(coarse=coarse, bias_identity=ident, divide=case["bias"] == "div")
    if t is not None:
        kw.update(taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask)
        ref_kw.update(taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask)
    if case["noise"]:
        mean = np.full(b, 0.05 * scale, np.float32)
        std = np.full(b, 0.1 * scale, np.float32)
        keep = np.ones(b, np.uint8)
        if case["gated"]:
            keep[0] = 0
        z = rng.normal(size=shape).astype(np.float32)
        z2 = rng.normal(size=shape).astype(np.float32)
        rician = case["noise"] == "rician"
        kw.update(mean=torch.as_tensor(mean).to(DEV), std=torch.as_tensor(std).to(DEV),
                  keep=torch.as_tensor(keep).to(DEV), z=torch.as_tensor(z).to(DEV),
                  z2=torch.as_tensor(z2).to(DEV) if rician else None, noise_mode=1, rician=rician)
        ref_kw.update(mean=mean, std=std, keep=keep, z=z, z2=z2 if rician else None, rician=rician)
    if case["gamma"] is not None:
        gam = np.full(b, case["gamma"], np.float32)
        if case["gated"]:
            gam[0] = 1.0
        kw["gamma"] = torch.as_tensor(gam).to(DEV)
        ref_kw["gamma"] = gam
    return x, kw, ref_kw


def _misaligned(x: torch.Tensor) -> torch.Tensor:
    """The same values in a contiguous view at storage offset 1 (4 bytes past 16-byte alignment)."""
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    v = buf[1:].view(x.shape)
    v.copy_(x)
    assert v.data_ptr() % 16 == 4 and v.is_contiguous()
    return v


def variants(case):
    """(name, table half-width or None for the case's own, misaligned source)."""
    out = [("natural", None, False), ("misaligned", None, True)]
    big_r = int(np.max(case["radii"]))
    if case["mask"] and big_r <= 16:
        out.append(("R16", 16, False))
        out.append(("R16-misaligned", 16, True))
    if case["mask"] and big_r <= 6:
        out.append(("R9", 9, False))
    if case["mask"]:
        out.append(("R20" if big_r <= 20 else "R+4", max(20, big_r + 4), False))
    return out


def run_variant(x_np, kw, new_r=None, misaligned=False):
    from torchio_b200 import ops

    x = torch.as_tensor(x_np).to(DEV)
    if misaligned:
        x = _misaligned(x)
    kw = dict(kw)
    if "taps" in kw:
        taps = kw["taps"] if new_r is None else pad_table(kw["taps"], new_r)
        kw["taps"] = taps.to(DEV)
        if new_r is not None:
            kw["big_r"] = new_r
    out = ops.intensity_fused(x, **kw)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _bits(a: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.int32)


def _first_diff(a, b):
    d = np.argwhere(_bits(a) != _bits(b))
    return len(d), (tuple(d[0]) if len(d) else None)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"case{c['idx']}")
def test_path_matrix(case):
    """Every variant within the ref64 bound; all variants bit-identical (int32, so the sign of
    zero counts); gated rows bit copies."""
    x, kw, ref_kw = _inputs(case)
    ref = ref64(x, **ref_kw)
    results = {}
    for name, new_r, mis in variants(case):
        got = run_variant(x, kw, new_r, mis)
        check_bound(got, ref, f"case{case['idx']} {case['shape']} {name}")
        results[name] = got
    base = results["natural"]
    for name, got in results.items():
        n, first = _first_diff(base, got)
        assert n == 0, f"{name} differs from natural in {n} voxels, first at {first}"
    if case["gated"] and case["shape"][0] > 1 and (case["bias"] or case["noise"] or case["gamma"] is not None):
        # element 0: bias identity, no noise, gamma 1; its radii are 0 when per-element
        if case["radii"].ndim == 2 or not case["mask"]:
            assert np.array_equal(_bits(base[0]), _bits(x[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in CASES if c["mask"]][::2], ids=lambda c: f"case{c['idx']}")
def test_path_matrix_nonfinite(case):
    """Scattered NaN, +Inf, -Inf and a NaN block: each voxel's class equals ref64's on every path
    (a voxel is NaN / Inf only within its own element's radius of a non-finite input)."""
    x, kw, ref_kw = _inputs(case, nonfinite=True)
    ref = ref64(x, **ref_kw)
    want = classes(ref.y)
    for name, new_r, mis in variants(case):
        got = classes(run_variant(x, kw, new_r, mis))
        bad = np.argwhere(got != want)
        assert bad.size == 0, (f"case{case['idx']} {name}: {len(bad)} voxels of another class than ref64, "
                               f"first at {tuple(bad[0])} (got {got[tuple(bad[0])]}, ref64 {want[tuple(bad[0])]})")


@pytest.mark.gpu
def test_gated_rows_are_bit_copies_with_nan_payloads():
    b, shape = 3, (1, 6, 9, 16)
    rng = np.random.default_rng(3)
    x = rng.normal(size=(b, *shape)).astype(np.float32)
    payloads = np.array([0x7FC00123, 0xFFC45670, 0x7F800001, 0x80000000], dtype=np.uint32)
    x.reshape(b, -1)[0, :4] = payloads.view(np.float32)
    sig = [[0.0, 0.0, 0.0], [sigma_for_radius(2), sigma_for_radius(3), sigma_for_radius(1)],
           [sigma_for_radius(1), 0.0, sigma_for_radius(5)]]
    t = tables.blur_tables(sig, b)
    kw = dict(coarse=torch.zeros((b, 1, 2, 2, 2), device=DEV), bias_identity=torch.tensor([1, 0, 0], dtype=torch.uint8, device=DEV),
              taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask,
              mean=torch.zeros(b, device=DEV), std=torch.ones(b, device=DEV),
              keep=torch.tensor([0, 1, 1], dtype=torch.uint8, device=DEV),
              z=torch.ones((b, *shape), device=DEV), noise_mode=1,
              gamma=torch.tensor([1.0, 0.8, 1.2], device=DEV))
    for name, new_r, mis in [("natural", None, False), ("misaligned", None, True), ("R16", 16, False),
                             ("R20", 20, False)]:
        got = run_variant(x, kw, new_r, mis)
        assert np.array_equal(_bits(got[0]), _bits(x[0])), name


# ---------------------------------------------------------------------------------------------
# which kernel runs
# ---------------------------------------------------------------------------------------------


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


FORCED = [
    # name, expected kernel substring, shape, per-axis radii, table half-width, misaligned
    ("march6", "march6_kernel", (2, 1, 9, 8, 16), (3, 0, 0), None, False),
    ("march<4>", "march_kernel<4", (2, 1, 9, 8, 16), (3, 0, 0), 10, False),
    ("march<1> K%4", "march_kernel<1", (2, 1, 9, 8, 13), (3, 0, 0), None, False),
    ("march<1> offset", "march_kernel<1", (2, 1, 9, 8, 16), (3, 0, 0), None, True),
    ("jk6", "jk6_kernel", (2, 1, 9, 8, 16), (0, 2, 3), None, False),
    ("jk<6>", "jk_kernel<6", (2, 1, 9, 8, 16), (0, 2, 3), None, True),
    ("jk<16>", "jk_kernel<16", (2, 1, 9, 8, 16), (0, 2, 3), 10, False),
    ("axis R>16", "axis_kernel", (2, 1, 9, 8, 16), (1, 2, 3), 20, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("forced", FORCED, ids=[f[0] for f in FORCED])
def test_forced_path_launches_its_kernel(forced):
    name, kernel, shape, radii, new_r, mis = forced
    t = tables.blur_tables([sigma_for_radius(r) for r in radii], shape[0])
    x = np.random.default_rng(0).normal(size=shape).astype(np.float32)
    kw = dict(taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask,
              gamma=torch.full((shape[0],), 0.9, device=DEV))
    run_variant(x, kw, new_r, mis)  # warm-up: module load outside the trace
    names = _kernel_names(lambda: run_variant(x, kw, new_r, mis))
    assert any(kernel in n for n in names), f"{name}: {kernel} did not launch; launched {names}"


# ---------------------------------------------------------------------------------------------
# gamma: signed zeros and subnormals
# ---------------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("g", [0.8, 1.3, 2.5])
def test_gamma_signed_zero_and_subnormal_match_torch(g):
    """sign(x) |x|^g on +-0 and subnormal inputs, on every path, against torch's
    x.sign() * x.abs().pow(g) on the same CUDA tensor: zero signs exactly, values within the SFU
    bound (torch's pow is correctly rounded to within an ulp)."""
    special = np.array([0.0, -0.0, 1e-40, -1e-40, 1e-45, -1e-45, 1.1754942e-38, -3e-39, 1e-30, -1e-30,
                        1e-20, 0.5, -2.0], dtype=np.float32)
    b, shape = 2, (1, 3, 4, 16)
    x = np.resize(special, (b, *shape)).astype(np.float32)
    xt = torch.as_tensor(x).to(DEV)
    want = (xt.sign() * xt.abs().pow(g)).cpu().numpy()
    # element 0 has all radii 0 (a copy through every blur pass), element 1 blurs along J: the
    # J/K pass and its epilogue run, and element 0 still sees the pure gamma map
    sig = [[0.0, 0.0, 0.0], [0.0, sigma_for_radius(1), 0.0]]
    t = tables.blur_tables(sig, b)
    gam = torch.full((b,), g, device=DEV)
    configs = {
        "march6": dict(gamma=gam),
        "march<1>": dict(gamma=gam, _mis=True),
        "jk6": dict(gamma=gam, taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask),
        "jk<6>": dict(gamma=gam, taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask, _mis=True),
        "axis": dict(gamma=gam, taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask, _r=20),
    }
    for name, kw in configs.items():
        mis, new_r = kw.pop("_mis", False), kw.pop("_r", None)
        got = run_variant(x, kw, new_r, mis)[0]
        w = want[0]
        zero = w == 0
        sb = np.signbit(got[zero]) != np.signbit(w[zero])
        assert not sb.any() and np.all(got[zero] == 0), (
            f"{name} g={g}: {int(sb.sum()) + int((got[zero] != 0).sum())} zero results differ from torch, "
            f"inputs {x[0][zero][sb | (got[zero] != 0)][:4]}, got {got[zero][sb | (got[zero] != 0)][:4]}")
        nz = ~zero
        lg = np.abs(np.log2(np.abs(w[nz]).astype(np.float64)))
        tol = np.abs(w[nz]) * (math.log(2) * (g * E_SFU * np.maximum(1, lg) + U * g * lg) + E_SFU + 2 * U) + 2.0 ** -148
        err = np.abs(got[nz].astype(np.float64) - w[nz])
        assert np.all(err <= tol), (f"{name} g={g}: {int((err > tol).sum())} values differ from torch beyond the "
                                    f"SFU bound; inputs {x[0][nz][err > tol][:4]}, got {got[nz][err > tol][:4]}, "
                                    f"torch {w[nz][err > tol][:4]}")


# ---------------------------------------------------------------------------------------------
# transforms and edges
# ---------------------------------------------------------------------------------------------


def _vox_sigmas(params, affines):
    from oracle import torch_port as tp

    if "_batched_keys" in params:
        mm = np.asarray(params["std"], dtype=np.float64)
        sp = np.asarray([tp.spacing_of(a) for a in affines], dtype=np.float64)
        return np.divide(mm, sp, out=np.zeros_like(mm), where=sp > 0)
    sp = np.asarray(tp.spacing_of(affines[0]), dtype=np.float64)
    return [s / q if q > 0 else 0.0 for s, q in zip(params["std"], sp)]


@pytest.mark.gpu
@pytest.mark.parametrize("per_instance", [False, True])
def test_blur_fine_spacing_large_sigma(per_instance):
    """Blur(std up to 2 mm) on 0.35 mm in-plane spacing: radius 17..18 voxels."""
    import warnings

    import torchio_b200 as tio
    from oracle import torch_port

    torch.manual_seed(3)
    affine = np.diag([1.0, 0.35, 0.35, 1.0])
    subjects = [tio.Subject(t1=tio.ScalarImage(torch.rand((1, 6, 40, 44), generator=torch.Generator().manual_seed(s)) * 100,
                                               affine=affine.copy())) for s in range(3)]
    batch = tio.SubjectsBatch.from_subjects(subjects).to(DEV)
    data_in = batch.images["t1"].data.clone()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = tio.Blur(std=(1.9, 2.0), per_instance=per_instance)(batch)
    got = out.images["t1"].data.cpu().numpy()
    params = out.applied_transforms[-1].params
    affines = [np.asarray(a, dtype=np.float64) for a in batch.images["t1"].affines]
    vox = _vox_sigmas(params, affines)
    t = tables.blur_tables(vox, 3)
    assert t.big_r > 16
    ref = ref64(data_in.cpu().numpy(), taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask)
    check_bound(got, ref, f"Blur 0.35 mm per_instance={per_instance} R={t.big_r}")
    want = torch_port.gaussian_smooth(data_in.cpu(), vox).numpy()  # its taps live on the CPU
    rng = float(want.max() - want.min())
    assert float(np.abs(got - want).max()) <= 1e-4 * rng


@pytest.mark.gpu
def test_resample_antialias_factor_14():
    """Anti-aliased downsampling by 14 along K: the pre-filter radius is 18."""
    from torchio_b200.transforms import spatial

    import torchio_b200 as tio

    a_in = tio.AffineMatrix(np.eye(4))
    a_out = tio.AffineMatrix(np.diag([1.0, 1.0, 14.0, 1.0]))
    x = torch.as_tensor(np.random.default_rng(4).normal(size=(2, 1, 5, 6, 70)).astype(np.float32)).to(DEV)
    got = spatial._antialias(x, a_in, a_out).cpu().numpy()
    sig = spatial._antialias_sigmas(np.array([1.0, 1.0, 14.0]), np.ones(3))
    t = tables.blur_tables([float(v) for v in sig], 2)
    assert t.big_r > 16
    check_bound(got, ref64(x.cpu().numpy(), taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask),
                "antialias x14")
    import warnings

    subject = tio.Subject(t1=tio.ScalarImage(x[0].clone(), affine=np.eye(4)))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        down = tio.Resample((1.0, 1.0, 14.0), antialias=True)(subject)
    assert down.t1.spatial_shape[2] < 10 and torch.isfinite(down.t1.data).all()


@pytest.mark.gpu
def test_compose_nan_background_fused_and_unfused():
    import copy
    import warnings

    import torchio_b200 as tio

    g = torch.Generator().manual_seed(9)
    vols = []
    for _ in range(2):
        v = torch.rand((1, 64, 64, 64), generator=g)
        v[:, :12] = float("nan")
        v[:, :, :, 50:] = float("nan")
        vols.append(v)
    def make():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return tio.Compose([tio.BiasField(), tio.Blur(std=(0.5, 2.0)), tio.Noise(std=(0, 0.1)),
                                tio.Gamma(log_gamma=(-0.3, 0.3))])
    outs = []
    for fuse in (True, False):
        batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(v.clone())) for v in vols]).to(DEV)
        pipe = make()
        pipe.fuse = fuse
        torch.manual_seed(21)
        out = pipe(batch)
        history = [(t.name, copy.deepcopy(t.params)) for t in out.applied_transforms]
        outs.append((out.images["t1"].data.cpu().numpy(), history))
    (fused, h_fused), (unfused, h_unfused) = outs
    assert repr(h_fused) == repr(h_unfused)
    blur_params = next(p for name, p in h_fused if name == "Blur")
    vox = _vox_sigmas(blur_params, [np.eye(4)] * 2)
    t = tables.blur_tables(vox, 2)
    x = np.stack([v.numpy() for v in vols])
    # bias, noise and gamma map finite values to finite values: the classes are the blur's
    want = classes(ref64(x, taps=t.taps.numpy(), radius=t.radius.numpy(), axes_mask=t.axes_mask).y)
    np.testing.assert_array_equal(classes(fused), want)
    np.testing.assert_array_equal(classes(unfused), want)


@pytest.mark.gpu
def test_pass2_grid_limit():
    """B * C * ceil(I / 16) = 65535 tiles of pass 2 run and match ref64 on every element; one
    tile more is refused before any kernel launches."""
    from torchio_b200 import ops

    b, shape = 65535, (1, 16, 4, 4)
    rng = np.random.default_rng(8)
    x = rng.normal(size=(b, *shape)).astype(np.float32)
    sig = [0.0, sigma_for_radius(2), sigma_for_radius(1)]
    t = tables.blur_tables(sig, b)
    kw = dict(taps=t.taps.to(DEV), radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask)
    got = ops.intensity_fused(torch.as_tensor(x).to(DEV), **kw).cpu().numpy()
    # shared taps: ref64's chain on the whole batch at once
    y, s, n = x.astype(np.float64), np.abs(x.astype(np.float64)), 0
    for axis in (1, 2):
        r = int(t.radius[axis, 0])
        row = t.taps[axis, 0, t.big_r - r: t.big_r + r + 1].numpy().astype(np.float64)
        y, s, n = blur_axis64(y, row, axis), blur_axis64(s, np.abs(row), axis), n + 2 * r + 1
    check_bound(got, Ref(y, y, np.full(y.shape, float(n)), s, None), "65535 tiles")
    b2, shape2 = 16384, (1, 64, 4, 4)
    t2 = tables.blur_tables([sigma_for_radius(1)] * 3, b2)
    kw2 = dict(taps=t2.taps.to(DEV), radius=t2.radius.to(DEV), big_r=t2.big_r, axes_mask=t2.axes_mask,
               coarse=torch.zeros((b2, 1, 2, 2, 2), device=DEV))
    x2 = torch.zeros((b2, *shape2), device=DEV)
    torch.cuda.synchronize()

    def refused():
        with pytest.raises(RuntimeError, match="too large for the blur grid"):
            ops.intensity_fused(x2, **kw2)

    names = _kernel_names(refused)
    assert not any("march" in n or "jk" in n for n in names), names


@pytest.mark.gpu
def test_full_size_forced_paths_bit_identical():
    """2 x 1 x 256^3 with sprinkled NaN / Inf: march6 against march<1> (misaligned view) and jk6
    against jk<6>, bit for bit (NaNs compared as a class: their payload is the hardware's)."""
    rng = np.random.default_rng(17)
    shape = (2, 1, 256, 256, 256)
    x = rng.normal(0, 100, shape).astype(np.float32)
    flat = x.reshape(-1)
    idx = rng.choice(flat.size, 3000, replace=False)
    flat[idx[:1000]] = np.nan
    flat[idx[1000:2000]] = np.inf
    flat[idx[2000:]] = -np.inf
    sig_i = [[sigma_for_radius(3), 0.0, 0.0], [sigma_for_radius(6), 0.0, 0.0]]
    sig_jk = [[0.0, sigma_for_radius(2), sigma_for_radius(5)], [0.0, sigma_for_radius(6), sigma_for_radius(1)]]
    gam = torch.tensor([0.8, 1.25], device=DEV)
    for label, sig in (("march6 vs march<1>", sig_i), ("jk6 vs jk<6>", sig_jk)):
        t = tables.blur_tables(sig, 2)
        kw = dict(taps=t.taps, radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask, gamma=gam)
        a = run_variant(x, kw, None, False)
        bb = run_variant(x, kw, None, True)
        ca, cb = classes(a), classes(bb)
        assert np.array_equal(ca, cb), f"{label}: {int((ca != cb).sum())} voxels of another class"
        a[ca == 1] = 0.0
        bb[cb == 1] = 0.0
        n, first = _first_diff(a, bb)
        assert n == 0, f"{label}: {n} voxels differ, first at {first}"
        print(f"{label}: bit-identical, {int((ca == 1).sum())} NaN, {int((ca >= 2).sum())} Inf voxels")
