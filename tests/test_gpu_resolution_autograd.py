"""Gradients through Resize and Anisotropy (`set_differentiable`, `autograd.interpolate`,
`autograd.axis_resample`, the kernels `tio_interpolate_backward` / `tio_axis_resample_backward`).

- Against the reference: torch autograd through the reference's op sequences (`F.interpolate`,
  `torch.gather` and the four elementwise ops, `resolution_cases`) on the same CUDA input and cotangent.
- Float64 bound: every voxel within γ_m·Σ|w·g| of a float64 adjoint, m from the summation shape.
- Adjoint identity <A x, g> == <x, Aᵀ g> in fp64 sums; determinism, also under
  torch.use_deterministic_algorithms; the forward with grad is the forward without it.
- Non-finite cotangents spread to the same voxels as in the reference; label maps are refused.
"""

import json
import subprocess
import sys
import warnings
from pathlib import Path

import numpy as np
import pytest
import torch

import resolution_cases as rc
import torchio_b200 as tio
from resolution_adjoint import adjoint_matrices, apply_along, apply_separable, gamma, instance_adjoint_matrix
from torchio_b200 import ops, tables
from torchio_b200.data import AffineMatrix
from torchio_b200.transforms import resolution

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
DEV = "cuda"


@pytest.fixture(autouse=True)
def differentiable():
    previous = tio.set_differentiable(True)
    try:
        yield
    finally:
        tio.set_differentiable(previous)


def _data(shape, dtype=torch.float32, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) * 4 - 2).to(dtype)


def _cotangent(shape, dtype, seed):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(dtype).to(DEV)


def _batch(x, label=False):
    kwargs = dict(image_class=tio.LabelMap) if label else {}
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [AffineMatrix() for _ in range(x.shape[0])], **kwargs)})


def _run(transform, data, seed):
    """(output, params, cotangent, grad of the input) of ``transform`` on CUDA ``data``."""
    x = data.to(DEV).requires_grad_()
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = transform(_batch(x))
    y = out.images["t1"].data
    params = out.applied_transforms[-1].params if out.applied_transforms else None
    cot = _cotangent(y.shape, y.dtype, seed + 1)
    y.backward(cot)
    return y.detach(), params, cot, x.grad


def _reference_grad(fn, data, cot):
    x = data.to(DEV).requires_grad_()
    y = fn(x)
    y.backward(cot)
    return y.detach(), x.grad


def _compare(got, ref, dtype):
    """Same non-finite voxels; finite ones within 1e-5 of the gradient's largest magnitude, or one
    rounding of fp16 / bf16 there (the fp32 sums differ in their last bits: the reference adds with
    atomics)."""
    assert got.dtype == ref.dtype == dtype and got.shape == ref.shape
    assert torch.equal(torch.isfinite(got), torch.isfinite(ref))
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    finite = torch.isfinite(ref)
    if not finite.any():
        return 0.0
    diff = (got.double() - ref.double())[finite].abs().max().item()
    scale = ref.double()[finite].abs().max().item() or 1.0
    eps = {torch.float16: 2.0**-10, torch.bfloat16: 2.0**-7}.get(dtype, 1e-5)
    assert diff <= eps * scale, (diff, scale)
    return diff


def _resize_ref(target, mode):
    return lambda x: rc.resize(x, target, mode)


def _aniso_ref(params, mode):
    case = {"transform": ("Anisotropy", {"image_interpolation": mode})}
    return lambda x: rc.reference_output(case, {"t1": (x, False)}, params)["t1"]


# ---- against the reference's op sequence ----------------------------------------------------------

RESIZE = {
    "up": ((6, 5, 7), (9, 11, 13)),
    "down": ((12, 10, 9), (5, 4, 3)),
    "mixed": ((10, 8, 9), (15, 4, 9)),
    "same": ((7, 8, 9), (7, 8, 9)),
    "unit_out": ((8, 9, 10), (8, 1, 10)),
    "unit_in": ((1, 6, 5), (4, 6, 1)),
    "large_k": ((9, 7, 150), (5, 11, 301)),  # several 128-wide chunks per row
}
DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.float64]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("case", list(RESIZE))
def test_resize_gradient_matches_reference(case, mode, dtype):
    shape, target = RESIZE[case]
    data = _data((2, 2, *shape), dtype, seed=1)
    out, _, cot, grad = _run(tio.Resize(target, image_interpolation=mode, copy=False), data, 3)
    _, ref_grad = _reference_grad(_resize_ref(target, mode), data, cot)
    err = _compare(grad, ref_grad, dtype)
    print(f"[resize {case} {mode} {dtype}] max |grad - ref| = {err:.3e}")


ANISO_SHAPE = (13, 10, 11)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("downsampling", [2.5, 1.01, 40.0])  # D < L, D == L, D == 1
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("b", [1, 3])
def test_anisotropy_shared_gradient_matches_reference(b, axis, downsampling, mode, dtype):
    """B = 1, or per_instance=False: one tio_interpolate pass and its adjoint."""
    data = _data((b, 2, *ANISO_SHAPE), dtype, seed=2)
    transform = tio.Anisotropy(axes=(axis,), downsampling=downsampling, image_interpolation=mode,
                               per_instance=b == 1, copy=False)
    out, params, cot, grad = _run(transform, data, 5)
    assert "_batched_keys" not in params
    ref_out, ref_grad = _reference_grad(_aniso_ref(params, mode), data, cot)
    err = _compare(grad, ref_grad, dtype)
    print(f"[anisotropy shared B={b} axis={axis} f={downsampling} {mode} {dtype}] max |grad - ref| = {err:.3e}")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("axes", [(0,), (1,), (2,), (0, 1, 2)])
@pytest.mark.parametrize("b", [3, 8])
def test_anisotropy_per_instance_gradient_matches_reference(b, axes, mode, dtype):
    """Per-element axes and factors, with rows gated out by p = 0.6 (copied, axis -1)."""
    data = _data((b, 2, *ANISO_SHAPE), dtype, seed=3)
    transform = tio.Anisotropy(axes=axes, downsampling=(1.0, 5.0), image_interpolation=mode, p=0.6, copy=False)
    out, params, cot, grad = _run(transform, data, 7)
    assert "_batched_keys" in params
    ref_out, ref_grad = _reference_grad(_aniso_ref(params, mode), data, cot)
    err = _compare(grad, ref_grad, dtype)
    print(f"[anisotropy per-instance B={b} axes={axes} {mode} {dtype}] factors={params['factor']}"
          f" max |grad - ref| = {err:.3e}")


@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("factors", [[2.5], [1.01], [1.0, 3.0, 1.01, 26 / 22, 4.4, 1.0, 40.0, 1.7]])
def test_per_instance_rows_match_reference(factors, axis, mode):
    """The per-instance path itself at B = 1 and B = 8, D == L and gated rows included."""
    b = len(factors)
    data = _data((b, 2, *ANISO_SHAPE), seed=4)
    axes = [axis] * b
    x = data.to(DEV).requires_grad_()
    y = resolution._degrade_per_instance(x, axes, factors, mode == "linear", graph=True)
    cot = _cotangent(y.shape, y.dtype, 11)
    y.backward(cot)
    ref_out, ref_grad = _reference_grad(lambda t: rc.anisotropy_per_instance(t, axes, factors, mode), data, cot)
    assert torch.equal(y.detach(), ref_out)
    err = _compare(x.grad, ref_grad, torch.float32)
    print(f"[per-instance rows axis={axis} {mode} factors={factors}] max |grad - ref| = {err:.3e}")


def test_compose_with_affine_matches_reference():
    from oracle import torch_port

    data = _data((2, 2, 14, 12, 13), seed=6)
    pipeline = tio.Compose([tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)),
                            tio.Anisotropy(downsampling=(2, 4)), tio.Resize((9, 15, 10))], copy=False)
    x = data.to(DEV).requires_grad_()
    torch.manual_seed(9)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = pipeline(_batch(x))
    history = [{"name": t.name, "params": t.params} for t in out.applied_transforms]
    assert [h["name"] for h in history] == ["Affine", "Anisotropy", "Resize"]
    y = out.images["t1"].data
    cot = _cotangent(y.shape, y.dtype, 10)
    y.backward(cot)

    # the oracle's Affine replay runs on the host; its output moves to the GPU inside the graph
    leaf = data.clone().requires_grad_()
    images = {"t1": {"kind": "scalar", "data": leaf, "affines": [np.eye(4) for _ in range(data.shape[0])]}}
    t = torch_port.replay(images, history[:1])["t1"]["data"].to(DEV)
    t = _aniso_ref(history[1]["params"], "linear")(t)
    rc.resize(t, (9, 15, 10), "linear").backward(cot)
    err = _compare(x.grad.cpu(), leaf.grad, torch.float32)
    print(f"[compose affine + anisotropy + resize] max |grad - ref| = {err:.3e}")


# ---- float64 bound, adjoint identity, determinism -----------------------------------------------

def _interpolate_case(case, mode):
    """(in shape, out shape, forward tables, adjoint tables) of a Resize or shared Anisotropy case."""
    linear = mode == "linear"
    if case in RESIZE:
        shape, target = RESIZE[case]
        return shape, target, tables.resize_tables(shape, target, linear), tables.resize_adjoint_tables(
            shape, target, linear)
    axis, factor = {"aniso_i": (0, 2.5), "aniso_j": (1, 26 / 22), "aniso_k": (2, 4.4)}[case]
    shape = (26, 22, 33)
    return shape, shape, tables.anisotropy_shared_tables(shape, axis, factor, linear), \
        tables.anisotropy_shared_adjoint_tables(shape, axis, factor, linear)


INTERP_CASES = [*RESIZE, "aniso_i", "aniso_j", "aniso_k"]


@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("case", INTERP_CASES)
def test_interpolate_backward_within_float64_bound(case, mode):
    """Each voxel sums n = n_i*n_j*n_k terms ((w_i*w_j)*w_k)*g: 3 roundings per term and n - 1 adds,
    so |got - exact| <= γ_{n+2} Σ|w g|."""
    shape, target, _, (ptr, ent, wt) = _interpolate_case(case, mode)
    g = _cotangent((3, 2, *target), torch.float32, 12)
    got = ops.interpolate_backward(g, shape, ptr, ent, wt).double()
    mats = adjoint_matrices(ptr, ent, wt, shape, target)
    exact = apply_separable(g, mats)
    mags = apply_separable(g.abs(), [np.abs(m) for m in mats])
    counts = [np.diff(ptr[s:s + n + 1]) for s, n in zip((0, shape[0] + 1, shape[0] + shape[1] + 2), shape)]
    n = np.einsum("i,j,k->ijk", *counts)
    bound = torch.as_tensor(gamma(n + 2), device=DEV) * mags
    err = (got - exact).abs()
    assert torch.all(err <= bound)
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    print(f"[interpolate_backward {case} {mode}] max |err| / γ_m Σ|w g| = {ratio:.3f} (m <= {int(n.max()) + 2})")


def _instance_case(mode, b=8):
    axes = [0, 1, 2, 0, 1, 2, 0, 2][:b]
    factors = [2.5, 1.0, 4.4, 26 / 22, 1.01, 40.0, 1.0, 1.7][:b]
    shape = (26, 22, 33)
    linear = mode == "linear"
    ax, lo, hi, w = tables.anisotropy_instance_tables(shape, axes, factors, linear)
    ptr, ent = tables.anisotropy_instance_adjoint_tables(shape, axes, factors, linear)
    return shape, (ax, lo, hi, w), (ptr, ent), linear


@pytest.mark.parametrize("mode", ["linear", "nearest"])
def test_axis_resample_backward_within_float64_bound(mode):
    """A plane sums n terms g*c (c = 1 - w rounded as in the forward, or w): |got - exact| <=
    γ_n Σ|c g|; elements with axis -1 copy g exactly."""
    shape, (ax, lo, hi, w), (ptr, ent), linear = _instance_case(mode)
    g = _cotangent((len(ax), 2, *shape), torch.float32, 13)
    got = ops.axis_resample_backward(g, ax, w, ptr, ent, linear=linear).double()
    worst = 0.0
    for b, a in enumerate(ax.tolist()):
        if a < 0:
            assert torch.equal(got[b], g[b].double())
            continue
        n = shape[a]
        m = instance_adjoint_matrix(ptr[b], ent[b], w[b], n, linear)
        exact = apply_along(g[b], m, a)
        mags = apply_along(g[b].abs(), np.abs(m), a)
        count = np.diff(ptr[b, :n + 1]).astype(np.float64)
        view = [1, 1, 1, 1]
        view[a + 1] = n
        bound = torch.as_tensor(gamma(count), device=DEV).reshape(view) * mags
        err = (got[b] - exact).abs()
        assert torch.all(err <= bound)
        worst = max(worst, (err / bound.clamp_min(1e-300)).max().item())
    print(f"[axis_resample_backward {mode}] max |err| / γ_n Σ|c g| = {worst:.3f}")


@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("case", INTERP_CASES)
def test_interpolate_adjoint_identity(case, mode):
    shape, target, (idx, lam), (ptr, ent, wt) = _interpolate_case(case, mode)
    x = _data((2, 2, *shape), seed=14).to(DEV)
    g = _cotangent((2, 2, *target), torch.float32, 15)
    y = ops.interpolate(x, target, idx, lam)
    gin = ops.interpolate_backward(g, shape, ptr, ent, wt)
    lhs, rhs = (y.double() * g.double()).sum().item(), (x.double() * gin.double()).sum().item()
    scale = (y.double() * g.double()).abs().sum().item()
    assert abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


@pytest.mark.parametrize("mode", ["linear", "nearest"])
def test_axis_resample_adjoint_identity(mode):
    shape, (ax, lo, hi, w), (ptr, ent), linear = _instance_case(mode)
    x = _data((len(ax), 2, *shape), seed=16).to(DEV)
    g = _cotangent(x.shape, torch.float32, 17)
    y = ops.axis_resample(x, ax, lo, hi, w, linear=linear)
    gin = ops.axis_resample_backward(g, ax, w, ptr, ent, linear=linear)
    lhs, rhs = (y.double() * g.double()).sum().item(), (x.double() * gin.double()).sum().item()
    scale = (y.double() * g.double()).abs().sum().item()
    assert abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


def _grads_twice(transform_factory, data):
    grads = []
    for _ in range(2):
        _, _, _, grad = _run(transform_factory(), data, 19)
        grads.append(grad)
    return grads


FACTORIES = {
    "resize": lambda: tio.Resize((9, 17, 8), copy=False),
    "aniso_shared": lambda: tio.Anisotropy(downsampling=(2, 4), per_instance=False, copy=False),
    "aniso_per_instance": lambda: tio.Anisotropy(downsampling=(1.5, 4), p=0.7, copy=False),
}


@pytest.mark.parametrize("kind", list(FACTORIES))
def test_backward_is_deterministic(kind):
    data = _data((4, 2, *ANISO_SHAPE), seed=18)
    a, b = _grads_twice(FACTORIES[kind], data)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    previous = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        with warnings.catch_warnings():
            warnings.simplefilter("error")  # no warning and no error: the backward is deterministic
            c, d = _grads_twice(FACTORIES[kind], data)
    finally:
        torch.use_deterministic_algorithms(previous)
    assert torch.equal(a.view(torch.int32), c.view(torch.int32))
    assert torch.equal(c.view(torch.int32), d.view(torch.int32))


# ---- the forward with grad is the forward without it ---------------------------------------------

def _forward(factory, data, grad):
    x = data.clone().requires_grad_(grad)
    torch.manual_seed(21)
    torch.cuda.synchronize()
    before = ops.launches()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = factory()(_batch(x)).images["t1"].data
    torch.cuda.synchronize()
    return out, ops.launches() - before


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", list(FACTORIES))
def test_forward_with_grad_is_the_forward_without_it(kind, dtype):
    data = _data((4, 2, *ANISO_SHAPE), dtype, seed=20).to(DEV)
    data[0, 0, 1, 2, 3] = float("nan")
    _forward(FACTORIES[kind], data, False)
    with_grad, n_grad = _forward(FACTORIES[kind], data, True)
    without, n_plain = _forward(FACTORIES[kind], data, False)
    tio.set_differentiable(False)
    switched_off, n_off = _forward(FACTORIES[kind], data, False)
    assert with_grad.requires_grad and not without.requires_grad
    bits = {torch.float64: torch.int64, torch.float32: torch.int32}.get(dtype, torch.int16)
    assert torch.equal(with_grad.detach().view(bits), without.view(bits))
    assert torch.equal(without.view(bits), switched_off.view(bits))
    assert n_grad == n_plain == n_off


def test_no_grad_mode_runs_the_usual_path():
    data = _data((3, 1, *ANISO_SHAPE), seed=22).to(DEV)
    plain, n_plain = _forward(FACTORIES["aniso_per_instance"], data, False)
    with torch.no_grad():
        out, n = _forward(FACTORIES["aniso_per_instance"], data, True)
    assert not out.requires_grad and torch.equal(out, plain) and n == n_plain


# ---- non-finite cotangents, refusals, full size -----------------------------------------------------

def _nonfinite(cot):
    flat = cot.view(-1)
    n = flat.numel()
    flat[n // 7] = float("nan")
    flat[n // 3] = float("inf")
    flat[n // 2 + 1] = float("-inf")
    flat[(5 * n) // 6] = float("inf")
    return cot


@pytest.mark.parametrize("mode", ["linear", "nearest"])
@pytest.mark.parametrize("kind", ["resize_up", "resize_down", "aniso_shared", "aniso_per_instance"])
def test_nonfinite_cotangents_spread_as_in_the_reference(kind, mode):
    data = _data((3, 1, *ANISO_SHAPE), seed=23)
    if kind.startswith("resize"):
        target = (19, 15, 16) if kind == "resize_up" else (6, 5, 7)
        transform = tio.Resize(target, image_interpolation=mode, copy=False)
    else:
        transform = tio.Anisotropy(downsampling=(2, 4), per_instance=kind == "aniso_per_instance",
                                   image_interpolation=mode, copy=False)
    x = data.to(DEV).requires_grad_()
    torch.manual_seed(24)
    out = transform(_batch(x))
    y = out.images["t1"].data
    params = out.applied_transforms[-1].params
    cot = _nonfinite(_cotangent(y.shape, y.dtype, 25))
    y.backward(cot)
    ref = _resize_ref(params["target_shape"], mode) if kind.startswith("resize") else _aniso_ref(params, mode)
    _, ref_grad = _reference_grad(ref, data, cot)
    assert (~torch.isfinite(ref_grad)).any()
    assert torch.equal(torch.isfinite(x.grad), torch.isfinite(ref_grad))
    assert torch.equal(torch.isnan(x.grad), torch.isnan(ref_grad))
    print(f"[non-finite {kind} {mode}] {(~torch.isfinite(x.grad)).sum().item()} non-finite voxels, as the reference")


@pytest.mark.parametrize("make", [
    lambda: tio.Resize((5, 6, 7), copy=False),
    lambda: tio.Anisotropy(downsampling=3.0, per_instance=False, copy=False),
    lambda: tio.Anisotropy(downsampling=3.0, copy=False),
])
def test_label_maps_that_require_grad_are_refused(make):
    x = torch.rand((2, 1, 12, 12, 12), device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError, match=r"(Resize|Anisotropy) \(label map \"t1\"\).*no GPU gradient"):
        make()(_batch(x, label=True))


def test_switch_off_keeps_refusing():
    tio.set_differentiable(False)
    x = torch.rand((1, 1, 12, 12, 12), device=DEV, requires_grad=True)
    with pytest.raises(NotImplementedError, match="forward-only"):
        tio.Resize((5, 6, 7), copy=False)(_batch(x))


@pytest.mark.parametrize("kind", ["resize", "aniso_per_instance"])
def test_gradients_at_256_match_reference(kind):
    data = _data((2, 1, 256, 256, 256), seed=26)
    if kind == "resize":
        transform, target = tio.Resize((200, 320, 128), copy=False), (200, 320, 128)
    else:
        transform = tio.Anisotropy(downsampling=(2, 5), copy=False)
    out, params, cot, grad = _run(transform, data, 27)
    ref = _resize_ref(target, "linear") if kind == "resize" else _aniso_ref(params, "linear")
    _, ref_grad = _reference_grad(ref, data, cot)
    err = _compare(grad, ref_grad, torch.float32)
    print(f"[256^3 B=2 {kind}] max |grad - ref| = {err:.3e}")


# ---- launches: the library's count against the tio:: kernels of a trace ----------------------------

def _launch_cases():
    g_i = _cotangent((2, 2, 9, 11, 13), torch.float32, 30)
    shape, (ax, _, _, w), (ptr, ent), _ = _instance_case("linear", b=3)
    _, _, (ptr_n, ent_n), _ = _instance_case("nearest", b=3)
    g_a = _cotangent((3, 2, *shape), torch.float32, 31)
    adj = tables.resize_adjoint_tables((6, 5, 7), (9, 11, 13), True)
    return {
        "interpolate_backward": lambda: ops.interpolate_backward(g_i, (6, 5, 7), *adj),
        "axis_resample_backward_linear": lambda: ops.axis_resample_backward(g_a, ax, w, ptr, ent, linear=True),
        "axis_resample_backward_nearest": lambda: ops.axis_resample_backward(g_a, ax, None, ptr_n, ent_n,
                                                                             linear=False),
    }


def count_case(name: str, out_path: str) -> None:
    """[ops.launches() delta, tio:: kernels in a CUDA trace] of one call of case ``name``, as JSON
    (test_launch_count's method).  The call runs once before the traced one: what is traced is a
    call of a process whose tables, staging ring and kernels are already set up."""
    out = Path(out_path)
    trace = out.with_suffix(".trace.json")
    call = _launch_cases()[name]
    call()
    torch.cuda.synchronize()
    before = ops.launches()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    counted = ops.launches() - before
    prof.export_chrome_trace(str(trace))
    events = json.loads(trace.read_text())["traceEvents"]
    kernels = [e["name"] for e in events if e.get("cat") == "kernel" and "tio::" in e.get("name", "")]
    out.write_text(json.dumps([counted, len(kernels), kernels]))


LAUNCH_CASES = ["interpolate_backward", "axis_resample_backward_linear", "axis_resample_backward_nearest"]


@pytest.fixture(scope="module")
def counts(tmp_path_factory):
    """Each case is traced in a process of its own, in that process's only profiler session: a
    later session of one process can miss kernel records or report an earlier session's."""
    results = {}
    for name in LAUNCH_CASES:
        out = tmp_path_factory.mktemp("resolution_launch_count") / f"{name}.json"
        code = (f"import sys; sys.path[:0] = {[str(ROOT), str(ROOT / 'tests')]!r}; "
                f"import test_gpu_resolution_autograd as t; t.count_case({name!r}, {str(out)!r})")
        subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], check=True)
        results[name] = json.loads(out.read_text())
    return results


@pytest.mark.parametrize("name", LAUNCH_CASES)
def test_backward_launch_count_equals_the_kernels_in_a_trace(name, counts):
    counted, traced, kernels = counts[name]
    assert traced >= 2, kernels  # the table upload and the adjoint kernel
    assert counted == traced, (counted, kernels)
