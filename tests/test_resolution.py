"""Anisotropy and Resize: params, history, index tables and errors against the reference's
fixtures and torch's own choices (CPU), and the kernels against the reference's op sequences on the
same CUDA tensors and against the CPU fixtures (GPU)."""

from __future__ import annotations

import hashlib
import json
import re
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resolution_cases as ref
from resolution_cases import RESOLUTION_CASES, affines, label_map, load_fixture, scalar_image

CASES = {c["name"]: c for c in RESOLUTION_CASES}
CASE_NAMES = list(CASES)
DTYPES = [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float32]
ALL_DTYPES = DTYPES + [torch.float16, torch.bfloat16, torch.float64]  # images computed in fp32


def _batch(case, device=None, seg=None, t1=None):
    import torchio_b200 as tio

    seg = label_map(case) if seg is None else seg
    t1 = scalar_image(case) if t1 is None else t1
    if device is not None:
        seg, t1 = seg.to(device), t1.to(device)
    aff = [tio.AffineMatrix(a) for a in affines(case)]
    return tio.SubjectsBatch({"seg": tio.ImagesBatch(seg, aff, image_class=tio.LabelMap),
                              "t1": tio.ImagesBatch(t1, [a.clone() for a in aff], image_class=tio.ScalarImage)})


def _transform(case):
    import torchio_b200 as tio

    name, kwargs = case["transform"]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return getattr(tio, name)(**kwargs)


def _history(batch):
    return json.dumps([{"name": t.name, "params": t.params} for t in batch.applied_transforms])


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Equal dtype, shape and bits (NaN payloads and the sign of zero included)."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _images(case, device=None):
    seg, t1 = label_map(case), scalar_image(case)
    if device is not None:
        seg, t1 = seg.to(device), t1.to(device)
    return {"seg": (seg, True), "t1": (t1, False)}


# ---- CPU ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", CASE_NAMES)
def test_op_sequence_regenerates_the_fixture(name):
    """The restated op sequences are the reference: outputs and errors, from the recorded params."""
    case = CASES[name]
    fixture = load_fixture(name)
    if "error" in fixture:
        kwargs = case["transform"][1]
        if "axes" in kwargs and kwargs["axes"] == (3,):
            with pytest.raises(ValueError, match=f"^{re.escape(fixture['error']['message'])}$"):
                ref.anisotropy_per_instance(label_map(case), [3] * case["batch"], [2.0] * case["batch"], "nearest")
        return
    (entry,) = fixture["history"]
    out = ref.reference_output(case, _images(case), entry["params"])
    assert _same(out["seg"], fixture["out_seg"])
    assert _same(out["t1"], fixture["out_t1"])
    if case["transform"][0] == "Resize":
        target = entry["params"]["target_shape"]
        for b, a in enumerate(affines(case)):
            np.testing.assert_array_equal(ref.resize_affine(a, case["shape"], target), fixture["aff_seg"][b])
    else:
        np.testing.assert_array_equal(np.stack(affines(case)), fixture["aff_seg"])


@pytest.mark.parametrize("name", CASE_NAMES)
def test_params_and_errors_match_the_reference(name):
    """Gating, make_params and history on a host batch (kernels stubbed out), and the reference's
    errors at construction or from apply_transform."""
    case = CASES[name]
    fixture = load_fixture(name)
    if fixture.get("error", {}).get("message", "").startswith("downsampling range"):
        with pytest.raises(ValueError, match=f"^{re.escape(fixture['error']['message'])}$"):
            _transform(case)
        return
    transform = _transform(case)
    batch = _batch(case)
    torch.manual_seed(case["seed"])
    gated = transform._forward_batch.__func__
    apply = type(transform).apply_transform
    type(transform).apply_transform = lambda self, b, p: b
    try:
        out = gated(transform, batch)
    finally:
        type(transform).apply_transform = apply
    if "error" in fixture:
        params = json.loads(_history(out))[0]["params"]
        with pytest.raises(ValueError, match=f"^{re.escape(fixture['error']['message'])}$"):
            transform.apply_transform(_batch(case), params)
        return
    assert _history(out) == json.dumps(fixture["history"])


LENGTHS = list(range(1, 301))


def test_aten_tables_equal_torch_interpolate_on_probe_volumes():
    """The fp32 index / weight builders against F.interpolate on CPU, read back from index-coded
    probes: nearest picks the coded plane; linear on a probe of 0 / 1 at one source plane gives
    that plane's weight per output (nearest: every L <= 300 against a spread of output sizes)."""
    from torchio_b200 import tables

    for n_in in LENGTHS:
        probe = torch.arange(n_in, dtype=torch.float32).reshape(1, 1, n_in, 1, 1)  # fp32, as data.float()
        for n_out in sorted({1, 2, 3, max(1, n_in // 3), max(1, n_in - 1), n_in, n_in + 1, 2 * n_in, 301}):
            got = F.interpolate(probe, size=(n_out, 1, 1), mode="nearest").flatten().long().numpy()
            np.testing.assert_array_equal(tables.aten_nearest_axis(n_in, n_out), got, err_msg=f"{n_in}->{n_out}")
    for n_in in (1, 2, 3, 7, 26, 97, 255, 256, 300):
        for n_out in (1, 2, 5, 22, 128, 257, 300, 320):
            i0, i1, l0, l1 = tables.aten_linear_axis(n_in, n_out)
            for plane in sorted({0, n_in // 2, n_in - 1}):
                probe = torch.zeros(1, 1, n_in, 1, 1, dtype=torch.float32)
                probe[0, 0, plane] = 1.0
                got = F.interpolate(probe, size=(n_out, 1, 1), mode="trilinear",
                                    align_corners=True).flatten().double().numpy()
                want = np.where(i0 == plane, l0.astype(np.float64), 0.0)
                want = want + np.where(i1 == plane, l1.astype(np.float64), 0.0)
                if n_in == n_out:
                    want = (np.arange(n_out) == plane).astype(np.float64)
                np.testing.assert_allclose(got, want, rtol=0, atol=2e-7, err_msg=f"{n_in}->{n_out} plane {plane}")


def _instance_rows_cuda_rule(length, down, linear):
    """The reference's index helpers with its scale division as ATen runs it on a CUDA tensor
    (a multiply by the fp32 reciprocal of the Python-scalar divisor), on CPU torch ops."""
    lower, upper, weight = ref._instance_indices(length, down, "linear" if linear else "nearest", "cpu")
    if not linear or length == 1:
        return lower, upper, weight
    step = (torch.tensor(down, dtype=torch.float32) - 1.0) * (torch.tensor(1.0) / torch.tensor(float(length - 1)))
    pos = torch.arange(length, dtype=torch.float32) * step
    lo = pos.floor().long()
    hi = torch.minimum(lo + 1, torch.tensor(down - 1))

    def src(x):
        return torch.div(x * length, down, rounding_mode="floor").clamp(max=length - 1)

    return src(lo), src(hi), pos - lo.float()


def test_instance_tables_equal_the_reference_helpers():
    """The per-instance (lo, hi, w) rows equal the reference's index helpers for every L <= 300 and
    a spread of factors (the fp32 scale as a CUDA batch computes it), and differ from ATen's
    composed map where the two paths disagree (L = 26, D = 22, low-res plane 11: 13 vs 12)."""
    from torchio_b200 import tables

    for length in range(1, 513):  # the down size against _downsample_sizes, two-decimal factors
        factors = torch.arange(101, 1001, dtype=torch.float64) / 100
        want = torch.round(length / factors).clamp_min(1).long().tolist()
        assert [tables.anisotropy_down_size(length, f) for f in factors.tolist()] == want, length
    assert tables.anisotropy_down_size(33, 4.4) == 8 and tables.anisotropy_down_size(22, 1.76) == 13
    for length in LENGTHS:
        for factor in (1.01, 1.5, 1.76, 2.0, 2.48, 2.5, 3.3, 4.4, 5.0, 5.2, 9.2, 1000.0):
            down = tables.anisotropy_down_size(length, factor)
            assert down == int(torch.round(length / torch.tensor([factor], dtype=torch.float64)).clamp_min(1))
            for linear in (False, True):
                axis, lo, hi, w = tables.anisotropy_instance_tables((length, 1, 1), [0], [factor], linear)
                lower, upper, weight = _instance_rows_cuda_rule(length, down, linear)
                assert axis.tolist() == [0]
                np.testing.assert_array_equal(lo[0, :length], lower.numpy())
                if linear:
                    np.testing.assert_array_equal(hi[0, :length], upper.numpy())
                    assert np.array_equal(w[0, :length].view(np.uint32), weight.numpy().view(np.uint32))
    _, lo, _, _ = tables.anisotropy_instance_tables((26, 1, 1), [0], [26 / 22], False)
    assert tables.aten_nearest_axis(26, 22)[11] == 12 and min(11 * 26 // 22, 25) == 13
    shared, _ = tables.anisotropy_shared_tables((26, 1, 1), 0, 26 / 22, False)
    assert not np.array_equal(lo[0, :26], shared[:26])


@pytest.mark.gpu
def test_instance_tables_equal_the_reference_helpers_on_cuda():
    """The same rows against the reference's helpers run on CUDA tensors, every L <= 300."""
    from torchio_b200 import tables

    for length in LENGTHS:
        for factor in (1.01, 1.5, 1.76, 2.0, 2.48, 2.5, 3.3, 4.4, 5.0, 5.2, 9.2, 1000.0):
            down = tables.anisotropy_down_size(length, factor)
            _, lo, hi, w = tables.anisotropy_instance_tables((length, 1, 1), [0], [factor], True)
            lower, upper, weight = ref._instance_indices(length, down, "linear", "cuda")
            np.testing.assert_array_equal(lo[0, :length], lower.cpu().numpy())
            np.testing.assert_array_equal(hi[0, :length], upper.cpu().numpy())
            assert np.array_equal(w[0, :length].view(np.uint32), weight.cpu().numpy().view(np.uint32)), length


def test_shared_tables_compose_the_down_map():
    """One tio_interpolate table set equals the two F.interpolate of the shared path on an index-coded
    probe (CPU, fp32 as the reference's data.float(); every index below 2**24 is exact)."""
    from torchio_b200 import tables

    for shape, axis, factor in [((26, 5, 6), 0, 26 / 22), ((9, 13, 8), 1, 3.0), ((8, 9, 14), 2, 2.7),
                                ((10, 6, 7), 0, 1.01), ((6, 9, 7), 1, 40.0), ((7, 8, 1), 2, 2.0)]:
        probe = torch.arange(int(np.prod(shape)), dtype=torch.float32).reshape(1, 1, *shape)
        want = ref.anisotropy_shared(probe, axis, factor, "nearest").flatten().long().numpy()
        idx, lam = tables.anisotropy_shared_tables(shape, axis, factor, False)
        assert lam is None
        i, j, k = shape
        ii, jj, kk = idx[:i], idx[2 * i:2 * i + j], idx[2 * (i + j):2 * (i + j) + k]
        got = ((ii[:, None, None] * j + jj[None, :, None]) * k + kk[None, None, :]).flatten()
        np.testing.assert_array_equal(got, want)


def test_constructors_warning_repr_and_hydra():
    import torchio_b200 as tio
    from torchio_b200.transforms.base import _TRANSFORM_REGISTRY

    with pytest.warns(UserWarning, match="Anisotropy is a no-op"):
        tio.Anisotropy()
    with pytest.raises(ValueError, match="upper bound must be >= 1, got 0.9"):
        tio.Anisotropy(downsampling=0.9)
    with pytest.raises(ValueError, match="non-negative"):
        tio.Anisotropy(downsampling=(-1, 2))
    with pytest.raises(TypeError):
        tio.Anisotropy((2,))  # keyword-only, as in the reference
    assert repr(tio.Anisotropy(axes=(2,), downsampling=(1.5, 5))) == "Anisotropy(axes=(2,), downsampling=(1.5, 5))"
    assert tio.Anisotropy(downsampling=4).to_hydra() == {"_target_": "torchio.Anisotropy", "downsampling": 4}
    assert repr(tio.Resize(4)) == "Resize(target_shape=(4, 4, 4))"
    assert tio.Resize((4, 5, 6), label_interpolation="linear").to_hydra() == {
        "_target_": "torchio.Resize", "target_shape": [4, 5, 6], "label_interpolation": "linear"}
    assert "Anisotropy" in _TRANSFORM_REGISTRY and "Resize" in _TRANSFORM_REGISTRY
    assert not tio.Anisotropy(downsampling=2).invertible and not tio.Resize(3).invertible
    batch = _batch(CASES["aniso_b3_p05_i64"])
    assert tio.Anisotropy(downsampling=2).supports_chunks(batch)
    assert not tio.Resize(3).supports_chunks(batch)


def test_ops_refuse_host_tensors():
    from torchio_b200 import ops, tables

    data = torch.zeros((1, 1, 4, 5, 6), dtype=torch.int16)
    idx, lam = tables.resize_tables((4, 5, 6), (2, 2, 2), True)
    with pytest.raises(RuntimeError, match="expected a CUDA tensor"):
        ops.interpolate(data, (2, 2, 2), idx, lam)
    axis, lo, hi, w = tables.anisotropy_instance_tables((4, 5, 6), [1], [2.0], True)
    with pytest.raises(RuntimeError, match="expected a CUDA tensor"):
        ops.axis_resample(data, axis, lo, hi, w, linear=True)


# ---- GPU ----------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_fixture_on_the_device(name):
    """History and affines equal the CPU reference's; every output equals the reference's op
    sequence on the same CUDA tensors bit for bit, and the CPU reference bit for bit except where
    the reference's own CUDA and CPU results differ (printed, finite differences bounded)."""
    case = CASES[name]
    fixture = load_fixture(name)
    if fixture.get("error", {}).get("message", "").startswith("downsampling range"):
        return
    transform = _transform(case)
    batch = _batch(case, device="cuda")
    torch.manual_seed(case["seed"])
    if "error" in fixture:
        with pytest.raises(ValueError, match=f"^{re.escape(fixture['error']['message'])}$"):
            transform(batch)
        return
    out = transform(batch)
    assert _history(out) == json.dumps(fixture["history"])
    params = fixture["history"][0]["params"]
    on_cuda = ref.reference_output(case, _images(case, device="cuda"), params)
    for key in ("seg", "t1"):
        got = out.images[key].data
        assert got.is_cuda
        np.testing.assert_array_equal(np.stack([a.numpy() for a in out.images[key].affines]), fixture[f"aff_{key}"])
        assert _same(got, on_cuda[key]), key  # the reference's op sequence on the same CUDA tensors
        want = fixture[f"out_{key}"]
        if _same(got, want):
            continue
        # The reference itself differs between CPU and CUDA here: ATen's CUDA trilinear copies
        # equal shapes and reads zero-weight taps of unchanged axes, and a CUDA tensor divides by a
        # Python scalar through its reciprocal (per-instance weights).  Label maps never differ.
        assert key == "t1" and got.dtype == torch.float32, key
        g, w = got.cpu(), want
        x = scalar_image(case)
        both_nan = torch.isnan(g) & torch.isnan(w)  # a NaN made by 0 * Inf: x86's default NaN is negative
        differ = (g.view(torch.int32) != w.view(torch.int32)) & ~both_nan
        both_finite = torch.isfinite(g) & torch.isfinite(w)
        err = (g[both_finite].double() - w[both_finite].double()).abs()
        bound = _cpu_cuda_bound(x)
        one_sided = differ & ~both_finite
        nan_bits = int((both_nan & (g.view(torch.int32) != w.view(torch.int32))).sum())
        print(f"{name} {key}: {int(differ.sum())} of {g.numel()} voxels differ from the CPU reference "
              f"({int(one_sided.sum())} non-finite on one side; {nan_bits} NaN on both with other bits), "
              f"max finite difference "
              f"{float(err.max()) if err.numel() else 0.0:.3g} <= bound {bound:.3g}")
        assert (float(err.max()) if err.numel() else 0.0) <= bound
        # a non-finite value on one side only comes from a non-finite input among the voxel's taps,
        # which lie within ceil(factor) + 1 voxels (Anisotropy) or 1 voxel (Resize to the same shape)
        if one_sided.any():
            assert g.shape == x.shape, "non-finite differences from a Resize that changes the shape"
            factor = params.get("factor", 1.0)
            reach = int(np.ceil(max(factor) if isinstance(factor, list) else factor)) + 1
            bad = (~torch.isfinite(x)).float().flatten(0, 1).unsqueeze(1)
            near = F.max_pool3d(bad, 2 * reach + 1, stride=1, padding=reach).reshape(x.shape) > 0
            assert bool(near[one_sided].all())


def _cpu_cuda_bound(x: torch.Tensor) -> float:
    """Largest |CUDA - CPU| of a finite fp32 output voxel, from the two causes that reach finite
    values.  Per-instance weights: the scale (D - 1) / (L - 1) is a true division on CPU and a
    multiply by the rounded reciprocal on CUDA, so it differs by <= 2 ulp, pos = i * scale by
    <= 3 ulp(L) (one more rounding), and w = pos - floor(pos) (exact) by the same; the output
    lo * (1 - w) + hi * w then moves by <= |hi - lo| * dw <= range(x) * 3 ulp(L), also when floor(pos)
    steps to the neighbouring plane (w goes from ~0 to ~1 and the value from x[lo] to ~x[lo]).
    Trilinear: both devices evaluate the same nested fma(a, x, rn(b * y)) from the same fp32
    weights (§3), so at most a rounding per combine level, 4 ulp of the largest |x|."""
    finite = x[torch.isfinite(x)].double()
    top = float(finite.abs().max())
    longest = max(x.shape[2:])
    return (float(finite.max() - finite.min()) * 3 * float(np.spacing(np.float32(longest)))
            + 4 * float(np.spacing(np.float32(top))))


def _inputs(dtype, batch_size, shape, seed, channels=1):
    g = torch.Generator().manual_seed(seed)
    if dtype.is_floating_point:
        data = torch.randn((batch_size, channels, *shape), generator=g) * 10
        flat = data.view(-1)
        flat[::97] = float("nan")
        flat[5::89] = float("inf")
        flat[7::83] = float("-inf")
        flat[11::79] = -0.0
        data = data.to(dtype) if dtype != torch.float64 else data.double() + 1e-9  # not fp32-exact
    else:
        lo = 0 if dtype == torch.uint8 else -50
        data = torch.randint(lo, 100, (batch_size, channels, *shape), generator=g).to(dtype)
        if dtype == torch.int64:
            data[:, :, ::3] += 2**40 + 2**25 + 1
    return data.cuda()


def _run(transform, data, is_label):
    import torchio_b200 as tio

    b = data.shape[0]
    cls = tio.LabelMap if is_label else tio.ScalarImage
    batch = tio.SubjectsBatch({"x": tio.ImagesBatch(data.clone(), [tio.AffineMatrix(np.eye(4)) for _ in range(b)],
                                                    image_class=cls)})
    out = transform(batch)
    return out.images["x"].data, out.applied_transforms[0].params if out.applied_transforms else None


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [1, 3])
@pytest.mark.parametrize("dtype", ALL_DTYPES)
def test_every_dtype_and_axis_equals_the_op_sequence_on_cuda(dtype, batch_size):
    """Both Anisotropy paths (B = 1: shared; B = 3: per-instance and per_instance=False) on each axis,
    nearest and linear, D = L, D = 1 and .5-boundary down sizes included, and Resize up / down /
    same shape, against the reference's op sequences on the same CUDA tensors, bit for bit; every
    label dtype, and fp16 / bf16 / fp64 images computed in fp32 and cast back."""
    import torchio_b200 as tio

    data = _inputs(dtype, batch_size, (10, 19, 13), seed=batch_size * 10 + ALL_DTYPES.index(dtype))
    boundary = _inputs(dtype, batch_size, (33, 22, 9), seed=batch_size * 10 + ALL_DTYPES.index(dtype) + 100)
    runs = [(data, axis, downsampling) for axis in range(3) for downsampling in ((1.5, 5), 1.01, 40.0)]
    runs += [(boundary, 0, 4.4), (boundary, 1, 1.76)]  # round(L / f) at a .5 boundary: 33 / 4.4, 22 / 1.76
    checked = 0
    for x, axis, downsampling in runs:
        for per_instance in (True, False):
            for is_label, interp in ((True, "linear"), (False, "linear"), (False, "nearest")):
                transform = tio.Anisotropy(axes=(axis,), downsampling=downsampling, image_interpolation=interp,
                                           per_instance=per_instance)
                torch.manual_seed(axis)
                got, params = _run(transform, x, is_label)
                mode = "nearest" if is_label else interp
                if "_batched_keys" in params:
                    want = ref.anisotropy_per_instance(x, params["axis"], params["factor"], mode)
                elif params["factor"] > 1.0:
                    want = ref.anisotropy_shared(x, params["axis"], params["factor"], mode)
                else:
                    want = x
                assert _same(got, want), (x.shape, axis, downsampling, per_instance, is_label, interp)
                checked += 1
    for target in ((5, 23, 13), (10, 19, 13), (20, 7, 1), (1, 1, 1)):
        for label_interp in ("nearest", "linear"):
            for is_label in (True, False):
                got, _ = _run(tio.Resize(target, label_interpolation=label_interp), data, is_label)
                mode = label_interp if is_label else "linear"
                assert _same(got, ref.resize(data, target, mode)), (target, label_interp, is_label)
                checked += 1
    print(f"{dtype} B={batch_size}: {checked} transforms bit-identical to the op sequences on CUDA")


@pytest.mark.gpu
def test_misaligned_and_ragged_rows_take_the_scalar_path():
    from torchio_b200 import ops, tables

    flat = _inputs(torch.float32, 1, (5 * 7 * 9 + 1, 1, 1), seed=4).flatten()
    view = flat[1:].reshape(1, 1, 5, 7, 9)  # 4 bytes past the allocation, K = 9
    for linear in (False, True):
        idx, lam = tables.resize_tables((5, 7, 9), (6, 3, 11), linear)
        assert _same(ops.interpolate(view, (6, 3, 11), idx, lam),
                     ref.resize(view, (6, 3, 11), "linear" if linear else "nearest"))
        axes, factors = [2], [2.5]
        axis, lo, hi, w = tables.anisotropy_instance_tables((5, 7, 9), axes, factors, linear)
        assert _same(ops.axis_resample(view, axis, lo, hi, w, linear=linear),
                     ref.anisotropy_per_instance(view, axes, factors, "linear" if linear else "nearest"))


def _force_axis(axis):
    import torchio_b200 as tio

    return tio.Anisotropy(axes=(axis,), downsampling=(1.5, 5), copy=False)


@pytest.mark.gpu
def test_full_size_anisotropy_every_voxel():
    """32 x 1 x 256^3 fp32 and int16 through the per-instance path, forced to each axis."""
    g = torch.Generator(device="cuda").manual_seed(17)
    for dtype in (torch.float32, torch.int16):
        if dtype == torch.float32:
            data = torch.rand((32, 1, 256, 256, 256), generator=g, device="cuda")
        else:
            data = torch.randint(0, 120, (32, 1, 256, 256, 256), generator=g, device="cuda", dtype=torch.int16)
        for axis in range(3):
            torch.manual_seed(axis)
            ours, params = _run(_force_axis(axis), data, dtype != torch.float32)
            mode = "nearest" if dtype != torch.float32 else "linear"
            expected = ref.anisotropy_per_instance(data, params["axis"], params["factor"], mode)
            equal = _same(ours, expected)
            digest = hashlib.sha256(ours.cpu().numpy().tobytes()).hexdigest()
            print(f"Anisotropy axis {axis} 32x256^3 {dtype}: sha256 {digest}, bit-identical={equal}")
            assert equal
            del ours, expected


@pytest.mark.gpu
def test_full_size_resize():
    import torchio_b200 as tio

    g = torch.Generator(device="cuda").manual_seed(18)
    data = torch.rand((2, 1, 256, 256, 256), generator=g, device="cuda")
    ours, _ = _run(tio.Resize((160, 192, 224)), data, False)
    equal = _same(ours, ref.resize(data, (160, 192, 224), "linear"))
    digest = hashlib.sha256(ours.cpu().numpy().tobytes()).hexdigest()
    print(f"Resize 2x256^3 -> (160, 192, 224) fp32: sha256 {digest}, bit-identical={equal}")
    assert equal


def _chain_batch(device="cuda"):
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(21)
    labels = torch.randint(0, 6, (3, 1, 32, 28, 24), generator=g).to(torch.int16)
    t1 = torch.rand((3, 1, 32, 28, 24), generator=g)
    if device is not None:
        labels, t1 = labels.to(device), t1.to(device)
    affine = [tio.AffineMatrix(np.diag([1.0, 1.0, 1.2, 1.0])) for _ in range(3)]
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(t1, affine, image_class=tio.ScalarImage),
                              "seg": tio.ImagesBatch(labels, [a.clone() for a in affine], image_class=tio.LabelMap)})


@pytest.mark.gpu
def test_compose_synthseg_chain_equals_one_by_one():
    import torchio_b200 as tio

    def chain():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return [tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.LabelsToImage("seg"),
                    tio.Anisotropy(downsampling=(1.5, 5)), tio.BiasField(std=0.3), tio.Blur(std=(0, 1)),
                    tio.Noise(std=(0, 0.1)), tio.Gamma(log_gamma=(-0.3, 0.3))]

    torch.manual_seed(31)
    torch.cuda.manual_seed(32)
    batch = _chain_batch()
    for transform in chain():
        batch = transform(batch)
    torch.manual_seed(31)
    torch.cuda.manual_seed(32)
    composed = tio.Compose(chain())(_chain_batch())
    for name in ("t1", "seg", "image_from_labels"):
        assert _same(composed.images[name].data, batch.images[name].data), name
    assert _history(composed) == _history(batch)


@pytest.mark.gpu
def test_host_batch_comes_back_on_the_host_and_streams_like_the_plain_call():
    import torchio_b200 as tio

    def chain():
        return [tio.Anisotropy(downsampling=(1.5, 5)), tio.Anisotropy(axes=(1,), downsampling=3.0, p=0.5)]

    torch.manual_seed(5)
    on_device = tio.Compose(chain())(_chain_batch())
    one_shot = tio.Compose(chain())
    one_shot.chunk_size = 0
    torch.manual_seed(5)
    plain = one_shot(_chain_batch(device=None))
    streamed_pipe = tio.Compose(chain())
    streamed_pipe.chunk_size = 1
    assert streamed_pipe._chunk_size(_chain_batch(device=None)) == 1
    torch.manual_seed(5)
    streamed = list(streamed_pipe.stream([_chain_batch(device=None)]))
    for out in (plain, *streamed):
        for name in ("t1", "seg"):
            assert out.images[name].data.device.type == "cpu"
            assert _same(out.images[name].data, on_device.images[name].data), name
        assert _history(out) == _history(on_device)
    resized = tio.Resize((20, 30, 10))(_chain_batch(device=None))
    assert resized.images["seg"].data.device.type == "cpu"
    assert _same(resized.images["seg"].data, ref.resize(_chain_batch(device=None).images["seg"].data, (20, 30, 10),
                                                        "nearest"))
