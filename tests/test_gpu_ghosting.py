"""Ghosting on the GPU: the fixtures of tests/golden/generate_ghosting.py, every image dtype on every
axis against a float64 one-axis filter and against the reference's op sequence on the same CUDA
tensors, inactive and non-finite rows, 32 x 1 x 256^3 batches, pipelines, host batches streamed
through a Compose, and the reference's own Ghosting tests."""

from __future__ import annotations

import math
import warnings
import zlib

import numpy as np
import pytest
import torch

import ghosting_cases as gc
import torchio_b200 as tio
from test_gpu_vectorization import _batch as _vectorization_batch
from test_gpu_vectorization import assert_vectorized
from torchio_b200 import ops
from torchio_b200.transforms.ghosting import ghosting_table

pytestmark = pytest.mark.gpu

CASES = gc.CASES


def _batch(data: torch.Tensor, seg: torch.Tensor | None = None) -> tio.SubjectsBatch:
    subjects = []
    for b in range(data.shape[0]):
        images = {"t1": tio.ScalarImage(data[b])}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b])
        subjects.append(tio.Subject(**images))
    return tio.SubjectsBatch.from_subjects(subjects)


def _run(transform, data, seg=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return transform(_batch(data, seg))


def _check_close(got: torch.Tensor, ref: torch.Tensor, exact: torch.Tensor | None = None, rel: float = 1e-4) -> float:
    """Within rel of the reference's range (floats; plus one unit in the last place of fp16 / bf16),
    within 1 (integers where the float value, ``exact`` when given, lies inside the dtype's range:
    the cast of a value outside it is not pinned); NaN positions equal.  Returns the largest
    difference (over the range for floats)."""
    assert got.dtype == ref.dtype and got.shape == ref.shape
    g, r = got.double(), ref.double()
    assert torch.equal(torch.isnan(g), torch.isnan(r)), "NaN positions differ"
    ok = ~torch.isnan(r)
    if not bool(ok.any()):
        return 0.0
    if got.dtype.is_floating_point:
        span = float(r[ok].max() - r[ok].min()) or 1.0
        ulp = {torch.float16: 2.0**-10, torch.bfloat16: 2.0**-7}.get(got.dtype, 0.0)
        diff = (g[ok] - r[ok]).abs()
        assert bool((diff <= rel * span + ulp * r[ok].abs()).all()), f"max |diff| {float(diff.max())}, span {span}"
        return float(diff.max()) / span
    info = torch.iinfo(got.dtype)
    if exact is None:
        inside = ok & (r > info.min) & (r < info.max)
    else:
        inside = ok & (exact.to(r.device) > info.min + 1) & (exact.to(r.device) < info.max - 1)
    diff = float((g[inside] - r[inside]).abs().max()) if bool(inside.any()) else 0.0
    assert diff <= 1
    return diff


def _one_axis_device(x: torch.Tensor, params: dict) -> tuple[torch.Tensor, torch.Tensor]:
    """(float64 one-axis filter of float(x), per-voxel error bound) on the device.  The bound per line
    is 16 ceil(log2 n) 2^-24 max|H| ||x_line||_2: an fp32 FFT has a relative L2 error of at most
    about log2(n) eta, eta ~ u + 4u sqrt(2) ~ 7u with rounded twiddles (Higham, Accuracy and Stability
    of Numerical Algorithms, Theorem 24.2), and the filter is two FFTs and a multiply."""
    xf = x.float().double()
    out = xf.clone()
    bound = torch.zeros_like(xf)
    ghosts, axes, strengths = gc.per_element(params, x.shape[0])
    for b, (g, axis, s) in enumerate(zip(ghosts, axes, strengths, strict=True)):
        if not g or s == 0:
            continue
        n = x.shape[2 + axis]
        h = torch.fft.ifftshift(gc.line_mask(n, g, s, params["restore"], x.device).double())
        shape = [1] * 4
        shape[1 + axis] = n
        dim = 1 + axis
        out[b] = torch.fft.ifft(h.view(shape) * torch.fft.fft(xf[b], dim=dim), dim=dim).real
        norm = torch.linalg.vector_norm(xf[b], dim=dim, keepdim=True)
        bound[b] = 16 * max(1, math.ceil(math.log2(n))) * 2.0**-24 * float(h.abs().max()) * norm
        out[b][~torch.isfinite(xf[b]).flatten(1).all(dim=1)] = float("nan")  # a non-finite voxel: all NaN
    return out, bound


def _check_one_axis(got: torch.Tensor, x: torch.Tensor, params: dict) -> float:
    want, bound = _one_axis_device(x, params)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), "NaN positions differ"
    ok = ~torch.isnan(want)
    g, want, bound = got.double()[ok], want[ok], bound[ok]
    if got.dtype.is_floating_point:
        ulp = {torch.float16: 2.0**-10, torch.bfloat16: 2.0**-7}.get(got.dtype, 0.0)  # the output's rounding
        excess = (g - want).abs() - bound - ulp * want.abs()
        assert float(excess.max()) <= 0, f"over the bound by {float(excess.max())}"
        return float(((g - want).abs() / (bound + 1e-30)).max())
    info = torch.iinfo(got.dtype)
    inside = (want > info.min) & (want < info.max)
    diff = float((g - torch.trunc(want)).abs()[inside].max()) if bool(inside.any()) else 0.0
    assert diff <= 1
    return diff


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_are_reproduced_on_the_device(name):
    case = CASES[name]
    fx = gc.load_fixture(name)
    data, seg = gc.scalar_image(case), gc.label_map(case)
    if "error" in fx:
        with pytest.raises(ValueError, match=fx["error"]["message"]):
            tio.Ghosting(**case["kwargs"])
        return
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = tio.Ghosting(**case["kwargs"])
        if case.get("compose"):
            transform = tio.Compose([tio.Spike(**case["spike"]), transform, tio.BiasField(**case["bias"])])
    torch.manual_seed(gc.seed(case))
    out = _run(transform, data.cuda(), None if seg is None else seg.cuda())
    assert [{"name": t.name, "params": t.params} for t in out.applied_transforms] == fx["history"]
    got = out.images["t1"].data
    assert str(got.dtype) == fx["dtype"] and got.is_cuda
    if seg is not None:
        assert torch.equal(out.images["seg"].data.cpu(), seg)
    want = torch.from_numpy(gc.as_float64(fx["out_t1"], case["dtype"])).to(case["dtype"])
    if not fx["history"]:
        assert np.array_equal(gc.as_stored(got), fx["out_t1"], equal_nan=True)
        return
    if case.get("compose"):
        _check_close(got.cpu(), want)
        return
    params = fx["history"][0]["params"]
    _check_close(got.cpu(), want, torch.from_numpy(gc.one_axis(data.double().numpy(), params)))
    _check_one_axis(got, data.cuda(), params)


SHAPES = [(37, 29, 23), (64, 64, 64), (181, 217, 181), (4096, 3, 2), (12, 1, 10)]


def _values(shape, dtype, key) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))
    if dtype.is_floating_point:
        return (torch.randn(shape, generator=g, device="cuda") * 100 + 50).to(dtype)
    info = torch.iinfo(dtype)
    lo, hi = max(-1000.0, 0.4 * info.min), min(1000.0, 0.4 * info.max)
    if dtype == torch.uint8:
        lo, hi = 60.0, 200.0
    return (torch.rand(shape, generator=g, device="cuda") * (hi - lo) + lo).round().to(dtype)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("mode", ["shared_0", "shared_1", "shared_2", "each_0", "each_1", "each_2", "each_mixed"])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("dtype", gc.DTYPES, ids=gc.SHORT.get)
def test_every_dtype_axis_and_shape(dtype, batch, mode, shape):
    data = _values((batch, 1, *shape), dtype, (gc.SHORT[dtype], batch, mode, shape))
    kind, axis = mode.split("_")
    ghosts, strengths = [3, 7, 5][:batch], [0.6, 1.0, 1.3][:batch]
    if kind == "shared":
        params = {"num_ghosts": 4, "axis": int(axis), "intensity": 0.8, "restore": 0.1}
    else:
        axes = [b % 3 for b in range(batch)] if axis == "mixed" else [int(axis)] * batch
        params = {"num_ghosts": ghosts, "axis": axes, "intensity": strengths, "restore": 0.2,
                  "_batched_keys": ["num_ghosts", "axis", "intensity"]}
    source = data.clone()
    ghost_axes = gc.per_element(params, batch)
    table, ax, active = ghosting_table(*ghost_axes, params["restore"], shape)
    got = ops.ghosting(data, table, ax, active)
    assert got.data_ptr() == data.data_ptr()
    _check_close(got, gc.reference_ops(source, params), _one_axis_device(source, params)[0])
    _check_one_axis(got, source, params)


def test_inactive_rows_keep_their_bits():
    shape = (4, 2, 20, 18, 16)
    data = torch.randint(-2**31, 2**31 - 1, shape, device="cuda", dtype=torch.int32).view(torch.float32)
    source = data.clone()
    # elements 1 (intensity 0) and 3 (no ghosts) are not active; 0 and 2 ghost different axes
    table, axis, active = ghosting_table([4, 4, 3, 0], [0, 2, 1, 1], [0.5, 0.0, 1.0, 0.7], 0.0, shape[2:])
    ops.ghosting(data, table, axis, active)
    for b in (1, 3):
        assert torch.equal(data[b].view(torch.int32), source[b].view(torch.int32))
    for b in (0, 2):
        assert not torch.equal(data[b].view(torch.int32), source[b].view(torch.int32))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.float64], ids=str)
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_non_finite_rows_become_nan_and_leave_their_neighbours(dtype, axis):
    data = (torch.randn(2, 3, 24, 20, 16, device="cuda") * 10).to(dtype)
    data[0, 1, 5, 6, 7] = float("nan")
    data[1, 2, 0, 0, 0] = float("inf")
    data[1, 0, 23, 19, 15] = float("-inf")
    params = {"num_ghosts": [4, 6], "axis": [axis, axis], "intensity": [0.8, 0.5], "restore": 0.0,
              "_batched_keys": ["num_ghosts", "axis", "intensity"]}
    source = data.clone()
    ref = gc.reference_ops(source, params)
    got = ops.ghosting(data, *ghosting_table(*gc.per_element(params, 2), 0.0, data.shape[2:]))
    for b, c in [(0, 1), (1, 2), (1, 0)]:
        assert bool(torch.isnan(got[b, c]).all())
        print(f"reference on CUDA, row ({b}, {c}): all NaN {bool(torch.isnan(ref[b, c]).all())}, "
              f"NaN share {float(torch.isnan(ref[b, c]).double().mean()):.3f}")
    for b, c in [(0, 0), (0, 2), (1, 1)]:
        assert not bool(torch.isnan(got[b, c]).any())
        _check_close(got[b, c], ref[b, c])


def test_a_storage_offset_view():
    base = torch.randn(1 + 3 * 2 * 30 * 20 * 10, device="cuda")
    data = base[1:].view(3, 2, 30, 20, 10)
    assert data.storage_offset() == 1 and data.is_contiguous()
    source, before = data.clone(), base[0].clone()
    torch.manual_seed(3)
    out = tio.Ghosting(num_ghosts=(2, 6), intensity=(0.5, 1), copy=False)(_batch(data))
    params = out.applied_transforms[-1].params
    got = out.images["t1"].data
    _check_close(got, gc.reference_ops(source, params))
    assert torch.equal(base[0], before)


def test_shared_intensity_zero_returns_the_same_tensor():
    data = torch.rand(3, 1, 8, 8, 8, device="cuda")
    batch = _batch(data)
    before = batch.images["t1"].data
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tio.Ghosting(intensity=0.0, per_instance=False, copy=False)(batch)
    assert batch.images["t1"].data is before


def test_no_host_sync_on_a_large_cuda_batch():
    data = torch.randn(32, 1, 256, 256, 256, device="cuda")
    batch = _batch(data)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            tio.Ghosting(num_ghosts=(4, 10), intensity=(0.5, 1), copy=False)(batch)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    flagged = [str(w.message) for w in caught
               if "synchroniz" in str(w.message).lower() and "prototype feature" not in str(w.message)]
    assert flagged == []
    del data, batch
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", [torch.float32, torch.int16], ids=str)
@pytest.mark.parametrize("axis", [0, 1, 2])
def test_a_32_x_256_cubed_batch_on_every_voxel(dtype, axis):
    g = torch.Generator(device="cuda").manual_seed(axis)
    data = (torch.randn(32, 1, 256, 256, 256, generator=g, device="cuda") * 300).to(dtype)
    ghosts = [4 + b % 7 for b in range(32)]
    strengths = [0.5 + 0.5 * (b % 5) / 4 for b in range(32)]
    params = {"num_ghosts": ghosts, "axis": [axis] * 32, "intensity": strengths, "restore": 0.0,
              "_batched_keys": ["num_ghosts", "axis", "intensity"]}
    source = data.clone()
    ops.ghosting(data, *ghosting_table(ghosts, [axis] * 32, strengths, 0.0, data.shape[2:]))
    worst_ref, worst_bound = 0.0, 0.0
    for b0 in range(0, 32, 4):
        chunk = {**params, **{k: params[k][b0:b0 + 4] for k in params["_batched_keys"]}}
        exact = _one_axis_device(source[b0:b0 + 4], chunk)[0]
        worst_ref = max(worst_ref, _check_close(data[b0:b0 + 4], gc.reference_ops(source[b0:b0 + 4], chunk), exact))
        del exact
        worst_bound = max(worst_bound, _check_one_axis(data[b0:b0 + 4], source[b0:b0 + 4], chunk))
    print(f"{dtype} axis {axis}: largest difference from the reference's op sequence {worst_ref:.3e}"
          f" ({'of range' if dtype.is_floating_point else 'units'}), from float64"
          f" {worst_bound:.3e} ({'of the bound' if dtype.is_floating_point else 'units'})")
    del data, source
    torch.cuda.empty_cache()


def _pipeline():
    return [tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.Ghosting(num_ghosts=(2, 8), intensity=(0.5, 1)),
            tio.BiasField(), tio.Blur(std=(0, 2)), tio.Noise(std=(0, 0.25)), tio.Gamma(log_gamma=(-0.3, 0.3))]


def test_compose_equals_the_transforms_one_by_one():
    data = torch.rand(4, 1, 40, 36, 32, device="cuda") + 0.5
    torch.manual_seed(11)
    composed = tio.Compose(_pipeline())(_batch(data))
    torch.manual_seed(11)
    step = _batch(data)
    for t in _pipeline():
        step = t(step)
    assert [t.name for t in composed.applied_transforms] == [t.name for t in step.applied_transforms]
    assert [t.params for t in composed.applied_transforms] == [t.params for t in step.applied_transforms]
    got, want = composed.images["t1"].data, step.images["t1"].data
    span = float(want.max() - want.min())
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5 * span)


def test_compose_stream_on_a_host_batch_equals_the_plain_call():
    g = torch.Generator().manual_seed(21)
    batches = [(torch.randn(6, 1, 24, 22, 20, generator=g) * 100 + 50) for _ in range(3)]

    def pipeline():
        return [tio.ZNormalization(), tio.Ghosting(num_ghosts=(2, 8), intensity=(0.5, 1))]

    streamed_pipeline = tio.Compose(pipeline())
    streamed_pipeline.chunk_size = 2
    torch.manual_seed(17)
    streamed = list(streamed_pipeline.stream(_batch(b) for b in batches))
    torch.manual_seed(17)
    for data, out in zip(batches, streamed, strict=True):
        plain = tio.Compose(pipeline())(_batch(data))
        assert out.images["t1"].data.device.type == "cpu"
        assert [t.params for t in out.applied_transforms] == [t.params for t in plain.applied_transforms]
        torch.testing.assert_close(out.images["t1"].data, plain.images["t1"].data.cpu(), rtol=1e-5, atol=1e-5)


def test_an_axis_longer_than_4096_is_refused_only_when_ghosted():
    data = torch.rand(1, 1, 4097, 2, 3, device="cuda")
    with pytest.raises(NotImplementedError, match="longer than 4096"):
        tio.Ghosting(axes=(0,), intensity=0.5)(_batch(data))
    out = tio.Ghosting(axes=(2,), intensity=0.5)(_batch(data))  # the other axes are not bounded
    _check_close(out.images["t1"].data, gc.reference_ops(data, out.applied_transforms[-1].params))


# ---- the reference's tests/test_ghosting.py ------------------------------------------------------

def _subject(with_label: bool = True) -> tio.Subject:
    data = torch.rand(1, 10, 10, 10) * 100
    kwargs: dict = {"t1": tio.ScalarImage(data)}
    if with_label:
        seg = torch.zeros(1, 10, 10, 10, dtype=torch.float32)
        seg[0, 2:5, 2:5, 2:5] = 1
        seg[0, 6:9, 6:9, 6:9] = 2
        kwargs["seg"] = tio.LabelMap(seg)
    return tio.Subject(**kwargs)


def test_changes_data():
    subject = _subject(with_label=False)
    original = subject.t1.data.clone()
    result = tio.Ghosting(num_ghosts=5, intensity=0.8)(subject)
    assert not torch.allclose(result.t1.data.cpu(), original)


def test_zero_intensity_is_identity():
    subject = _subject(with_label=False)
    original = subject.t1.data.clone()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        result = tio.Ghosting(intensity=0.0)(subject)
    torch.testing.assert_close(result.t1.data.cpu(), original)


def test_leaves_labels_unchanged():
    subject = _subject()
    original_seg = subject.seg.data.clone()
    result = tio.Ghosting(num_ghosts=5, intensity=0.8)(subject)
    torch.testing.assert_close(result.seg.data.cpu(), original_seg)


def test_specific_axis():
    subject = _subject(with_label=False)
    original = subject.t1.data.clone()
    result = tio.Ghosting(axes=(1,), intensity=0.8)(subject)
    assert not torch.allclose(result.t1.data.cpu(), original)


def test_restore_fraction():
    subject = _subject(with_label=False)
    result = tio.Ghosting(restore=0.2, intensity=0.8)(subject)
    assert result.t1.data.shape == subject.t1.data.shape


def _same_batch(batch_size: int = 6) -> tio.SubjectsBatch:
    data = torch.rand(1, 12, 12, 12)
    return tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data.clone())) for _ in range(batch_size)])


def test_per_instance_differs_across_batch():
    torch.manual_seed(0)
    batch = _same_batch()
    result = tio.Ghosting(intensity=(0.5, 1.0))(batch)
    params = result.applied_transforms[-1].params
    assert "_batched_keys" in params
    assert len(params["intensity"]) == batch.batch_size
    assert not torch.allclose(result.t1.data[0], result.t1.data[1])


def test_per_instance_false_is_shared():
    torch.manual_seed(0)
    result = tio.Ghosting(intensity=(0.5, 1.0), per_instance=False)(_same_batch())
    torch.testing.assert_close(result.t1.data[0], result.t1.data[1])


def test_single_subject_keeps_scalar_params():
    subject = tio.Subject(t1=tio.ScalarImage(torch.rand(1, 12, 12, 12)))
    result = tio.Ghosting(intensity=(0.5, 1.0))(subject)
    assert "_batched_keys" not in result.applied_transforms[-1].params


# ---- the reference's Ghosting cases of test_vectorization.py and test_per_instance.py -------------

def test_vectorized_matches_per_element():
    torch.manual_seed(0)
    assert_vectorized(tio.Ghosting(num_ghosts=(2, 5), intensity=(0.5, 1.0)), _vectorization_batch())


def test_vectorized_matches_per_element_with_gating():
    torch.manual_seed(0)
    assert_vectorized(tio.Ghosting(num_ghosts=4, intensity=1.0, p=0.5), _vectorization_batch(batch_size=6))


def test_preserves_float64():
    torch.manual_seed(0)
    data = (torch.rand(1, 8, 8, 8) + 0.5).to(torch.float64)
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data.clone())) for _ in range(8)])
    result = tio.Ghosting(num_ghosts=4, intensity=1.0, p=0.5)(batch)
    assert result.t1.data.dtype == torch.float64
