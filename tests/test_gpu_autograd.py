"""Gradients through the spatial transforms (`set_differentiable`, `torchio_b200.autograd`).

- Against the reference: torch autograd through `oracle.torch_port.replay` of the same history
  (F.grid_sample + torch.where, the reference's op sequence) on the same input and cotangent.
- Adjoint identity of the kernel pair: <K1 x, g> == <x, K1ᵀ g> in fp64 sums.
- The forward with grad is the forward without it: same bits, same launches.
- Refusals: everything outside the differentiable set, deterministic mode, host batches, submit.
"""

import copy
import math
import warnings

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import ops, tables
from torchio_b200.data import AffineMatrix
from torchio_b200.transforms import spatial

pytestmark = pytest.mark.gpu

SHAPE = (21, 18, 23)  # odd: ragged tiles on every axis


@pytest.fixture(autouse=True)
def differentiable():
    previous = tio.set_differentiable(True)
    try:
        yield
    finally:
        tio.set_differentiable(previous)


def _transform(kind, fill, p):
    kwargs = dict(copy=False, p=p, default_pad_value=fill)
    if kind == "affine":
        return tio.Affine(scales=(0.8, 1.2), degrees=(-20, 20), translation=(-3, 3), **kwargs)
    if kind == "elastic":
        return tio.ElasticDeformation(max_displacement=(4, 3, 5), num_control_points=6, **kwargs)
    if kind == "spatial":
        return tio.Spatial(scales=(0.9, 1.1), degrees=(-10, 10), max_displacement=2.0, affine_first=False,
                           **kwargs)
    if kind == "nearest":
        return tio.Affine(degrees=(-15, 15), translation=(-2, 2), image_interpolation="nearest", **kwargs)
    if kind == "target":
        return tio.Resample(1.3, **kwargs)
    raise ValueError(kind)


def _inputs(b, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    data = (torch.rand((b, 1, *SHAPE), generator=g) * 3 - 1).to(dtype)
    return data


def _run(transform, data, seed):
    """(output, history, grad of the input) for a seeded cotangent."""
    x = data.cuda().requires_grad_()
    batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [AffineMatrix() for _ in range(data.shape[0])])})
    torch.manual_seed(seed)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = transform(batch)
    y = out.images["t1"].data
    history = [{"name": t.name, "params": t.params} for t in out.applied_transforms]
    cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(seed + 1)).to(y.dtype)
    if y.requires_grad:
        y.backward(cot.cuda())
    return y.detach().cpu(), history, cot, x.grad


def _reference(data, history, cot):
    from oracle import torch_port

    x = data.clone().requires_grad_()
    images = {"t1": {"kind": "scalar", "data": x, "affines": [np.eye(4) for _ in range(data.shape[0])]}}
    y = torch_port.replay(images, copy.deepcopy(history))["t1"]["data"]
    if y.requires_grad:
        y.backward(cot)
    return y.detach(), x.grad


def _bar(dtype, ref):
    """1e-4 of the reference gradient's range, or one rounding of the dtype at that range: the
    fp32 gradients differ in their last bits (atomics), which can round to the neighbouring
    fp16 / bf16 value."""
    rng = float(ref.double().nan_to_num(0, 0, 0).max() - ref.double().nan_to_num(0, 0, 0).min()) or 1.0
    eps = {torch.float16: 2.0**-10, torch.bfloat16: 2.0**-7}.get(dtype, 0.0)
    return max(1e-4, eps) * rng


def _compare(got, ref, dtype):
    got, ref = got.cpu(), ref.cpu()
    assert got.dtype == ref.dtype and got.shape == ref.shape
    assert torch.equal(torch.isnan(got), torch.isnan(ref))
    finite = ~torch.isnan(ref)
    err = float((got.double() - ref.double())[finite].abs().max()) if finite.any() else 0.0
    bar = _bar(dtype, ref)
    assert err <= bar, (err, bar)
    return err


FILLS = [0.0, 1.5, "minimum", "mean", "otsu"]


@pytest.mark.parametrize("kind", ["affine", "elastic", "spatial", "nearest", "target"])
@pytest.mark.parametrize("fill", FILLS)
@pytest.mark.parametrize("b", [1, 3])
def test_gradient_matches_reference_autograd(kind, fill, b, coords):
    if kind == "target" and b == 3:
        pytest.skip("a target space applies to the whole batch: B = 1 covers it")
    dtype = torch.float32
    data = _inputs(b, dtype, 7)
    transform = _transform(kind, fill, p=0.5 if b == 3 and kind != "target" else 1.0)
    out, history, cot, grad = _run(transform, data, 5)
    assert history, "the gate drew nothing: pick another seed"
    ref_out, ref_grad = _reference(data, history, cot)
    assert ref_grad is not None and grad is not None
    err = _compare(grad, ref_grad, dtype)
    print(f"[autograd {kind} fill={fill} B={b} {coords}] max |grad - ref| = {err:.3e}")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float64])
@pytest.mark.parametrize("kind", ["affine", "elastic"])
def test_gradient_of_other_float_dtypes_matches_reference(kind, dtype):
    data = _inputs(3, dtype, 9)
    out, history, cot, grad = _run(_transform(kind, "minimum", 0.5), data, 6)
    ref_out, ref_grad = _reference(data, history, cot)
    assert grad.dtype == dtype
    _compare(grad, ref_grad, dtype)


def test_compose_of_spatial_transforms_matches_reference():
    data = _inputs(2, torch.float32, 3)
    pipeline = tio.Compose([tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)),
                            tio.ElasticDeformation(max_displacement=3.0)], copy=False)
    out, history, cot, grad = _run(pipeline, data, 8)
    assert [h["name"] for h in history] == ["Affine", "ElasticDeformation"]
    ref_out, ref_grad = _reference(data, history, cot)
    _compare(grad, ref_grad, torch.float32)


def test_inverse_is_differentiable():
    data = _inputs(2, torch.float32, 4).cuda()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        forward = tio.Affine(degrees=(-10, 10), copy=False)(
            tio.SubjectsBatch({"t1": tio.ImagesBatch(data.clone(), [AffineMatrix(), AffineMatrix()])}))
        x = forward.images["t1"].data.detach().requires_grad_()
        forward.images["t1"].data = x
        back = tio.apply_inverse_transform(forward, warn=False)
    y = back.images["t1"].data
    assert y.requires_grad
    y.sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()


# ---- the kernel pair: adjoint identity ---------------------------------------------------------

def _geometry(case, b):
    """(packed tables, in shape, out shape, a_out) of one adjoint case."""
    shape = (34, 29, 1) if case == "2d" else (37, 30, 41)
    a_in = np.eye(4)
    a_out = np.eye(4)
    out_shape = shape
    rng = np.random.default_rng(1)
    deg = {"rotated": 45.0, "2d": 20.0}.get(case, 12.0)
    degrees = rng.uniform(-deg, deg, (b, 3))
    if case == "2d":
        degrees[:, :2] = 0
    scales = rng.uniform(0.85, 1.15, (b, 3))
    shifts = rng.uniform(-3, 3, (b, 3))
    if case == "outside":
        shifts[0] = (400, 0, 0)
    forwards = list(spatial.build_forward_affines(scales, degrees, shifts, "image", shape, AffineMatrix()))
    cps = [None] * b
    if case == "elastic":
        cps = [rng.uniform(-4, 4, (7, 7, 7, 3)).astype(np.float32) for _ in range(b)]
        for cp in cps:
            cp[:2] = cp[-2:] = 0
    if case == "passthrough":
        forwards[1] = None
    if case == "target":
        a_out = np.diag([1.3, 1.3, 1.3, 1.0])
        out_shape = tuple(int(math.floor(s / 1.3)) for s in shape)
    packed = tables.spatial_tables(forwards, cps, b, a_in, a_out, per_instance=True,
                                   has_target=case == "target")
    return packed, shape, out_shape, a_out


@pytest.mark.parametrize("mode", [ops.LINEAR, ops.NEAREST])
@pytest.mark.parametrize("fill", [None, 0.7])
@pytest.mark.parametrize("case", ["plain", "rotated", "outside", "elastic", "2d", "target", "passthrough"])
def test_adjoint_identity(case, fill, mode, coords):
    b = 3
    packed, shape, out_shape, a_out = _geometry(case, b)
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(2)
    x = torch.rand((b, 2, *shape), generator=gen).to(dev)
    g = torch.randn((b, 2, *out_shape), generator=gen).to(dev)
    mat, cp, flags = ops.upload(dev, packed.mat, packed.cp, packed.flags)
    fill_d = None if fill is None else torch.full((2,), fill, device=dev)
    sp_out = AffineMatrix(a_out).spacing
    box = spatial._box_hint(packed, (1.0, 1.0, 1.0), sp_out, out_shape)
    geometry = dict(affine_first=True, mode=mode, fill=fill_d, box_hint=box)
    y = ops.resample(x, mat, cp, flags, (1.0, 1.0, 1.0), sp_out, out_shape=out_shape, **geometry)
    before = ops.launches()
    gin = ops.resample_backward(g, shape, mat, cp, flags, (1.0, 1.0, 1.0), sp_out, **geometry)
    assert ops.launches() - before == 2  # bounds pre-pass + tile kernel (the memset is no kernel)
    if fill is not None:  # filled voxels do not depend on x: take them out of <K1 x, g>
        y = y - ops.resample(torch.zeros_like(x), mat, cp, flags, (1.0, 1.0, 1.0), sp_out, out_shape=out_shape,
                             **geometry)
    lhs = float((y.double() * g.double()).sum())
    rhs = float((x.double() * gin.double()).sum())
    scale = float((y.double() * g.double()).abs().sum()) or 1.0
    print(f"[adjoint {case} fill={fill} mode={mode} {coords}] |lhs - rhs| / sum|y g| = {abs(lhs - rhs) / scale:.2e}")
    assert abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)


# ---- forward unchanged ---------------------------------------------------------------------------

def _pipeline():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return tio.Compose([tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)),
                            tio.ElasticDeformation(max_displacement=3.0)], copy=False)


def _forward(data, grad):
    x = data.clone().requires_grad_(grad)
    batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [AffineMatrix() for _ in range(data.shape[0])])})
    torch.manual_seed(21)
    before = ops.launches()
    out = _pipeline()(batch).images["t1"].data
    torch.cuda.synchronize()
    return out, ops.launches() - before


def test_forward_with_grad_is_the_forward_without_it(coords):
    data = torch.rand((3, 1, 48, 40, 36), generator=torch.Generator().manual_seed(0)).cuda()
    _forward(data, False)  # first calls of a process also launch the library's one-time probes
    with_grad, n_grad = _forward(data, True)
    without, n_plain = _forward(data, False)
    tio.set_differentiable(False)
    switched_off, n_off = _forward(data, False)
    assert with_grad.requires_grad and not without.requires_grad
    assert torch.equal(with_grad.detach(), without) and torch.equal(without, switched_off)
    assert n_grad == n_plain == n_off


def test_no_grad_mode_runs_the_usual_path():
    data = torch.rand((2, 1, *SHAPE), generator=torch.Generator().manual_seed(1)).cuda()
    _forward(data, False)
    with torch.no_grad():
        out, n = _forward(data, True)
    plain, n_plain = _forward(data, False)
    assert not out.requires_grad and torch.equal(out, plain) and n == n_plain


@pytest.mark.parametrize("b", [2])
def test_gradients_at_256_match_reference(b):
    """The bench's spatial pair at 256^3, B = 2, against the reference's op sequence."""
    data = torch.rand((b, 1, 256, 256, 256), generator=torch.Generator().manual_seed(5))
    out, history, cot, grad = _run(_pipeline(), data, 30)
    ref_out, ref_grad = _reference(data, history, cot)
    err = _compare(grad, ref_grad, torch.float32)
    print(f"[autograd 256^3 B={b}] max |grad - ref| = {err:.3e}")


# ---- refusals ----------------------------------------------------------------------------------

def _batch(device="cuda"):
    x = torch.rand((1, 1, 12, 12, 12), device=device, requires_grad=True)
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [AffineMatrix()])})


@pytest.mark.parametrize("make", [
    lambda: tio.Gamma(log_gamma=(-0.3, 0.3), copy=False),
    lambda: tio.Noise(std=0.1, copy=False),
    lambda: tio.Flip(axes=(0,), copy=False),
    lambda: tio.Compose([tio.BiasField(), tio.Gamma()], copy=False),
])
def test_transforms_outside_the_set_raise_naming_themselves(make):
    transform = make()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        with pytest.raises(NotImplementedError, match=r"(Gamma|Noise|Flip|BiasField).*no GPU gradient"):
            transform(_batch())


@pytest.mark.parametrize("kwargs,why", [
    (dict(image_interpolation="cubic"), "cubic"),
    (dict(antialias=True, target=2.0), "antialias"),
])
def test_out_of_set_spatial_configurations_raise(kwargs, why):
    with pytest.raises(NotImplementedError, match=why):
        tio.Spatial(degrees=10, copy=False, **kwargs)(_batch())


def test_label_maps_never_carry_grad():
    with pytest.raises(NotImplementedError, match="label map"):
        x = torch.rand((1, 1, 12, 12, 12), device="cuda", requires_grad=True)
        tio.Affine(degrees=10, copy=False)(
            tio.SubjectsBatch({"seg": tio.ImagesBatch(x, [AffineMatrix()], image_class=tio.LabelMap)}))


def test_switch_off_keeps_refusing():
    tio.set_differentiable(False)
    with pytest.raises(NotImplementedError, match="forward-only"):
        tio.Affine(degrees=10, copy=False)(_batch())


def test_host_batches_and_submit_refuse():
    with pytest.raises(NotImplementedError, match="CUDA tensors only"):
        tio.Affine(degrees=10, copy=False)(_batch(device="cpu"))
    with pytest.raises(NotImplementedError, match="submit"):
        _pipeline().submit(_batch())


def test_deterministic_mode_raises_like_the_reference():
    from oracle import torch_port  # noqa: F401  (the reference op sequence below is its grid_sample)

    x = torch.rand((1, 1, 12, 12, 12), device="cuda", requires_grad=True)
    y = tio.Affine(degrees=(10, 10), copy=False)(
        tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [AffineMatrix()])})).images["t1"].data
    grid = torch.rand((1, 12, 12, 12, 3), device="cuda") * 2 - 1
    ref = torch.nn.functional.grid_sample(x, grid, align_corners=True)
    previous = torch.are_deterministic_algorithms_enabled()
    try:
        torch.use_deterministic_algorithms(True)
        with pytest.raises(RuntimeError, match="deterministic"):
            y.sum().backward(retain_graph=True)
        with pytest.raises(RuntimeError, match="deterministic"):
            ref.sum().backward(retain_graph=True)
        torch.use_deterministic_algorithms(True, warn_only=True)
        with pytest.warns(UserWarning, match="deterministic"):
            y.sum().backward()
    finally:
        torch.use_deterministic_algorithms(previous)
