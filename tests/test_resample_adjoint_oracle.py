"""The float64 adjoint of the resample in the C oracle (`orc_resample_adjoint`), on the CPU.

- Against the reference's own backward: torch autograd through `oracle.torch_port.replay`
  (F.grid_sample + torch.where).  The reference adds the same fp32 products g * w as the oracle,
  in fp32, so every voxel lies within gamma_m * abs64 of grad64 (`adjoint_bound`), and its NaN and
  Inf voxels are the oracle's.
- Against the oracle's own forward: <orc_resample(x), g> == <x, grad64> up to the forward's fp32
  rounding, a bound stated in `test_adjoint_of_the_oracle_forward`.

`adjoint_bound` is also the per-voxel bound of the GPU kernel (tests/test_gpu_resample_adjoint.py).
"""

import copy

import numpy as np
import pytest
import torch

from oracle import c_port
from oracle import torch_port as tp

U32 = 2.0**-24  # unit roundoff of fp32
U64 = 2.0**-53


def gamma(m, u=U32):
    """gamma_m = m u / (1 - m u) (Higham, Accuracy and Stability, §3.1)."""
    m = np.asarray(m, dtype=np.float64)
    return m * u / (1.0 - m * u)


def adjoint_bound(abs64, count):
    """Largest |fp32 adjoint - grad64| of a voxel with m = ``count`` terms whose |g * w| sum to
    ``abs64``, for any order of fp32 additions.

    fp32 rounds each product g * w once and each of at most m - 1 additions once, so any summation
    tree of the m products (a sequential loop, shared-memory partial sums flushed into a zeroed
    buffer, atomics in any order) ends within gamma_m * abs64 of the exact sum; a product that
    underflows adds at most 2^-150 more.  grad64 itself is within gamma_m(2^-53) * abs64 of the
    exact sum.  No term covers a weight that differs from the oracle's."""
    abs64 = np.asarray(abs64, dtype=np.float64)
    return (gamma(count) + gamma(count, U64)) * abs64 + count * 2.0**-150


def check_adjoint(got, grad64, abs64, count, *, round_to=None):
    """Assert ``got`` (fp32, or fp16 / bf16 when ``round_to`` gives its unit roundoff and the
    smallest subnormal's half) against the oracle voxel by voxel.  Returns the largest
    |got - grad64| / bound over the finite voxels with a nonzero bound."""
    got = torch.as_tensor(got).cpu().double().numpy()
    grad64, abs64, count = (torch.as_tensor(t).numpy() for t in (grad64, abs64, count))
    assert got.shape == grad64.shape
    finite = np.isfinite(grad64)
    # NaN and Inf voxels: the same values (NaN * 0 reaches zero-weight taps in both)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(grad64))
    np.testing.assert_array_equal(got[~finite & ~np.isnan(grad64)], grad64[~finite & ~np.isnan(grad64)])
    bound = adjoint_bound(np.where(finite, abs64, 0.0), count)
    if round_to is not None:  # one more rounding at the cast: |rn(v) - v| <= u |v| + eta
        u, eta = round_to
        bound = bound + u * (np.abs(np.where(finite, grad64, 0.0)) + bound) + eta
    with np.errstate(invalid="ignore"):  # inf - inf off the finite voxels
        err = np.abs(np.where(finite, got - grad64, 0.0))
    worst = np.unravel_index(np.argmax(err - bound), err.shape)
    assert (err <= bound).all(), (
        f"voxel {worst}: got {got[worst]!r} grad64 {grad64[worst]!r} m={count[worst]} "
        f"abs64={abs64[worst]!r} bound={bound[worst]!r}")
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1.0), 0.0)
    return float(ratio.max()) if ratio.size else 0.0


# ---- against the reference's backward -----------------------------------------------------------

SHAPE = (21, 18, 23)
FILLS = [0.0, 1.5, "minimum", "mean", "otsu"]
A0 = np.diag([1.0, 1.2, 0.9, 1.0])  # anisotropic: the displacement divides by the spacing


def _world(rng, shape, deg=20.0, two_d=False):
    """A forward world transform about the volume's centre (degrees, scales, shift)."""
    from scipy.spatial.transform import Rotation

    angles = rng.uniform(-deg, deg, 3)
    if two_d:
        angles[:2] = 0
    r = Rotation.from_euler("xyz", angles, degrees=True).as_matrix() @ np.diag(rng.uniform(0.8, 1.2, 3))
    c = A0[:3, :3] @ ((np.asarray(shape, dtype=np.float64) - 1) / 2)
    t = np.eye(4)
    t[:3, :3] = r
    t[:3, 3] = c - r @ c + rng.uniform(-3, 3, 3) * (np.array([1, 1, 0]) if two_d else 1)
    return t


def _history(kind, b, fill, seed):
    """(params, input shape) of one Spatial step of the reference."""
    rng = np.random.default_rng(seed)
    shape = (34, 29, 1) if kind == "2d" else SHAPE
    mats = [_world(rng, shape, two_d=kind == "2d") for _ in range(b)]
    cps = [None] * b
    if kind.startswith("elastic"):
        cps = [rng.uniform(-4, 4, (6, 5, 7, 3)).astype(np.float32) for _ in range(b)]
        if b > 1:
            mats[1] = None  # elastic-only element
    if kind == "passthrough":
        mats[b // 2] = None
    target = None
    if kind == "target":
        a_out = np.diag([1.3, 1.3, 1.3, 1.0])
        target = {"shape": tuple(int(s * a / 1.3) for s, a in zip(shape, np.diag(A0))), "affine": a_out}
    params = {
        "selected_images": ["t1"], "_batched_keys": ["affine_matrix", "control_points"],
        "affine_matrix": mats, "control_points": cps, "target": target,
        "affine_first": kind != "elastic_last",
        "image_interpolation": "nearest" if kind == "nearest" else "linear",
        "label_interpolation": "nearest", "default_pad_value": fill, "default_pad_label": 0,
    }
    return params, shape


def _oracle_tables(params, b, shape):
    """(mat, cp, flags, spacing_in, spacing_out, out_shape) of a Spatial step, packed here from
    the params (independent of the product's packing)."""
    target = params["target"]
    a_out = A0 if target is None else np.asarray(target["affine"])
    out_shape = shape if target is None else tuple(target["shape"])
    mat = np.zeros((b, 12), np.float32)
    flags = np.zeros(b, np.uint8)
    cp = None
    grids = [c for c in params["control_points"] if c is not None]
    if grids:
        cp = np.zeros((b, *grids[0].shape), np.float32)
    for e in range(b):
        m, c = params["affine_matrix"][e], params["control_points"][e]
        mat[e] = tp.output_to_input_matrix(A0, a_out, m)[:3].reshape(12).numpy()
        if c is not None:
            cp[e] = c
            flags[e] |= 2
        if m is None and c is None and target is None:
            flags[e] |= 1
    return mat, cp, flags, tp.spacing_of(A0), tp.spacing_of(a_out), out_shape


def _fill_of(data, pad_value):
    """The oracle's fill argument: None when the reference skips the mask step (a fill of 0)."""
    fill = tp.fill_value_for(data, "scalar", pad_value, 0)
    if isinstance(fill, torch.Tensor):
        return fill.numpy()
    return None if float(fill) == 0.0 else np.full(data.shape[1], float(fill), np.float32)


def _cotangent(shape, seed, nonfinite):
    g = torch.randn(shape, generator=torch.Generator().manual_seed(seed))
    if nonfinite:  # NaN and +-Inf, some on voxels whose taps carry zero weight
        flat = g.view(-1)
        n = flat.numel()
        flat[[n // 7, n // 3]] = float("nan")
        flat[n // 2] = float("inf")
        flat[(2 * n) // 3] = float("-inf")
    return g


KINDS = ["affine", "elastic", "elastic_last", "nearest", "target", "2d", "passthrough"]


@pytest.mark.parametrize("c", [1, 3])
@pytest.mark.parametrize("b", [1, 3])
@pytest.mark.parametrize("fill", FILLS)
@pytest.mark.parametrize("kind", KINDS)
def test_oracle_adjoint_matches_reference_autograd(kind, fill, b, c):
    if kind == "passthrough" and b == 1:
        pytest.skip("a pass-through element needs a batch")
    params, shape = _history(kind, b, fill, seed=b * 10 + c)
    x = torch.rand((b, c, *shape), generator=torch.Generator().manual_seed(3)) * 3 - 1
    xr = x.clone().requires_grad_()
    images = {"t1": {"kind": "scalar", "data": xr, "affines": [A0.copy() for _ in range(b)]}}
    y = tp.replay(images, copy.deepcopy([{"name": "Spatial", "params": params}]))["t1"]["data"]
    g = _cotangent(y.shape, seed=11, nonfinite=c == 3)
    y.backward(g)
    mat, cp, flags, sp_in, sp_out, out_shape = _oracle_tables(params, b, shape)
    assert tuple(y.shape[2:]) == out_shape
    mode = 0 if kind == "nearest" else 1
    grad64, abs64, count = c_port.resample_adjoint(
        g, shape, mat, cp, flags, sp_in, sp_out, affine_first=params["affine_first"], mode=mode,
        fill=_fill_of(x, fill))
    ratio = check_adjoint(xr.grad, grad64, abs64, count)
    assert count.sum() > 0
    print(f"[oracle adjoint {kind} fill={fill} B={b} C={c}] max |ref - grad64| / bound = {ratio:.3f}")


# ---- adjoint of the oracle's forward -----------------------------------------------------------

@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("fill", [None, 0.7])
@pytest.mark.parametrize("kind", ["affine", "elastic", "elastic_last", "target", "2d", "passthrough"])
def test_adjoint_of_the_oracle_forward(kind, fill, mode):
    """<y, g> - <x, grad64> with y = orc_resample(x) and its filled voxels taken out.

    A linear output voxel is the fp32 dot product of at most 8 taps with their weights, so it
    lies within gamma_8 * sum_t |x_t w_t| of the exact one (one rounding per product and per
    addition, the output's own rounding included); nearest and pass-through voxels copy x exactly.
    Summed against g: |<y, g> - <x, grad64>| <= gamma_8 * sum_o |g_o| sum_t |x_t w_t|
    = gamma_8 * <|x|, abs64>, plus the float64 sums' own gamma_n(2^-53) terms."""
    b, c = 3, 2
    params, shape = _history(kind, b, 0.0, seed=5)
    mat, cp, flags, sp_in, sp_out, out_shape = _oracle_tables(params, b, shape)
    gen = torch.Generator().manual_seed(4)
    x = torch.rand((b, c, *shape), generator=gen) * 2 - 0.5
    g = torch.randn((b, c, *out_shape), generator=gen)
    fill_a = None if fill is None else np.full(c, fill, np.float32)
    geometry = dict(affine_first=params["affine_first"], mode=mode, fill=fill_a)
    y = c_port.resample(x, out_shape, mat, cp, flags, sp_in, sp_out, **geometry)
    if fill is not None:  # filled voxels do not depend on x
        y = y - c_port.resample(torch.zeros_like(x), out_shape, mat, cp, flags, sp_in, sp_out, **geometry)
    grad64, abs64, count = c_port.resample_adjoint(g, shape, mat, cp, flags, sp_in, sp_out, **geometry)
    lhs = float((y.double() * g.double()).sum())
    rhs = float((x.double() * grad64).sum())
    n = max(y.numel(), x.numel())
    bound = (float(gamma(8)) * float((x.double().abs() * abs64).sum())
             + float(gamma(n, U64)) * (float((y.double() * g.double()).abs().sum())
                                       + float((x.double() * grad64).abs().sum())))
    if mode == 0:
        bound -= float(gamma(8)) * float((x.double().abs() * abs64).sum())  # copies: no fp32 rounding
    print(f"[oracle forward/adjoint {kind} fill={fill} mode={mode}] |lhs - rhs| = {abs(lhs - rhs):.3e}"
          f" bound {bound:.3e}")
    assert abs(lhs - rhs) <= bound, (lhs, rhs, bound)


def test_adjoint_counts_and_filled_voxels():
    """Hand-checkable geometry: a shift of -0.5 voxel along I on a 33-plane axis (33 - 1 = 2^5,
    so the normalise round trip gives u = -0.5 exactly).  Plane 0 of the output then has a linear
    mask of exactly 0.5 and counts as filled (!(msum > 0.5)); every other plane sends g / 2 to
    planes oi - 1 and oi, each with a zero-weight tap on j + 1 and k + 1."""
    shape = (33, 4, 5)
    mat = np.array([[1, 0, 0, -0.5, 0, 1, 0, 0, 0, 0, 1, 0]], np.float32)
    g = torch.randn((1, 1, *shape), generator=torch.Generator().manual_seed(0))
    geo = dict(affine_first=True, mode=1)
    filled64, _, filled_count = c_port.resample_adjoint(g, shape, mat, None, None, (1, 1, 1), (1, 1, 1),
                                                         fill=np.ones(1, np.float32), **geo)
    plain64, _, plain_count = c_port.resample_adjoint(g, shape, mat, None, None, (1, 1, 1), (1, 1, 1),
                                                       fill=None, **geo)
    g64 = g.double()[0, 0]
    want = torch.zeros_like(g64)
    want[:-1] += 0.5 * g64[1:]
    want[1:] += 0.5 * g64[1:]
    assert torch.equal(filled64[0, 0], want)
    want[0] += 0.5 * g64[0]  # without a fill, plane 0 also sends g / 2 to input plane 0
    assert torch.equal(plain64[0, 0], want)
    # taps (i, i + 1) x (j, j + 1) x (k, k + 1), the + 1 ones inside the volume but of weight 0
    assert int(filled_count[0, 0, 0, 0, 0]) == 1 and int(plain_count[0, 0, 0, 0, 0]) == 2
    assert int(filled_count[0, 0, 5, 2, 3]) == 8  # two planes, two rows, two columns
