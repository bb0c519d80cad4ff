"""Motion on the GPU: the fixtures of tests/golden/generate_motion.py, every image dtype against a
float64 one-axis identity and against the reference's op sequence on the same CUDA tensors,
inactive and non-finite rows, 32 x 1 x 256^3 batches, pipelines, host batches streamed through a
Compose, the reference's own Motion tests, host syncs and launch counts."""

from __future__ import annotations

import json
import subprocess
import sys
import warnings
import zlib
from pathlib import Path

import numpy as np
import pytest
import torch

import motion_cases as mc
import torchio_b200 as tio
from test_gpu_vectorization import _batch as _vectorization_batch
from test_gpu_vectorization import assert_vectorized
from torchio_b200 import ops
from torchio_b200.transforms.motion import motion_theta

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
CASES = mc.CASES


def _batch(data: torch.Tensor, seg: torch.Tensor | None = None) -> tio.SubjectsBatch:
    subjects = []
    for b in range(data.shape[0]):
        images = {"t1": tio.ScalarImage(data[b])}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b])
        subjects.append(tio.Subject(**images))
    return tio.SubjectsBatch.from_subjects(subjects)


def _check_close(got: torch.Tensor, ref: torch.Tensor, exact: torch.Tensor | None = None, rel: float = 1e-4) -> float:
    """Within rel of the reference's range (floats; plus one unit in the last place of fp16 / bf16),
    within 1 (integers where the float value, ``exact`` when given, lies inside the dtype's range:
    the cast of a value outside it is not pinned); NaN positions equal.  Returns the largest
    difference (over the range for floats)."""
    assert got.dtype == ref.dtype and got.shape == ref.shape
    g, r = got.double(), ref.double().to(got.device)
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
        exact = exact.to(r.device)
        inside = ok & (exact > info.min + 1) & (exact < info.max - 1)
    diff = float((g[inside] - r[inside]).abs().max()) if bool(inside.any()) else 0.0
    assert diff <= 1
    return diff


def _check_one_axis(got: torch.Tensor, x: torch.Tensor, params: dict) -> float:
    """``got`` against `motion_cases.one_axis` of float(x) within `motion_cases.error_bound` (plus
    the output's rounding); integers within 1 of the truncated float64 value.  Returns the largest
    difference over the bound (floats) or in units (integers)."""
    xf = x.float().double()
    want = mc.one_axis(xf, params)
    assert torch.equal(torch.isnan(got), torch.isnan(want)), "NaN positions differ"
    ok = ~torch.isnan(want)
    bound = mc.error_bound(xf, params)
    g, w, bound = got.double()[ok], want[ok], bound[ok]
    if got.dtype.is_floating_point:
        ulp = {torch.float16: 2.0**-10, torch.bfloat16: 2.0**-7}.get(got.dtype, 0.0)
        excess = (g - w).abs() - bound - ulp * w.abs()
        assert float(excess.max()) <= 0, f"over the bound by {float(excess.max())}"
        return float(((g - w).abs() / (bound + 1e-30)).max())
    info = torch.iinfo(got.dtype)
    inside = (w > info.min) & (w < info.max)
    diff = float((g - torch.trunc(w)).abs()[inside].max()) if bool(inside.any()) else 0.0
    assert diff <= 1
    return diff


def _run_ops(data: torch.Tensor, params: dict) -> torch.Tensor:
    transforms = mc.per_element(params, data.shape[0])
    return ops.motion(data, motion_theta(transforms, data.shape[2:]), np.array([bool(t) for t in transforms]))


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_are_reproduced_on_the_device(name):
    case = CASES[name]
    fx = mc.load_fixture(name)
    data, seg = mc.scalar_image(case), mc.label_map(case)
    if "error" in fx and "hydra" not in fx:
        with pytest.raises(ValueError, match=fx["error"]["message"]):
            tio.Motion(**case["kwargs"])
        return
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = tio.Motion(**case["kwargs"])
        if case.get("compose"):
            transform = tio.Compose([transform, tio.Ghosting(**case["ghosting"]), tio.BiasField(**case["bias"])])
    torch.manual_seed(mc.seed(case))
    cuda = data.cuda()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        if "error" in fx:
            with pytest.raises(ValueError) as info:
                transform(_batch(cuda))
            assert str(info.value) == fx["error"]["message"]
            return
        out = transform(_batch(cuda, None if seg is None else seg.cuda()))
    assert [str(w.message) for w in caught] == fx["warnings"]
    history = [{"name": t.name, "params": t.params} for t in out.applied_transforms]
    assert json.loads(json.dumps(history)) == fx["history"]
    got = out.images["t1"].data
    assert str(got.dtype) == fx["dtype"] and got.is_cuda
    if seg is not None:
        assert torch.equal(out.images["seg"].data.cpu(), seg)
    want = torch.from_numpy(mc.as_float64(fx["out_t1"], case["dtype"])).to(case["dtype"])
    if not fx["history"]:
        assert np.array_equal(mc.as_stored(got), fx["out_t1"], equal_nan=True)
        return
    if case.get("compose"):
        _check_close(got.cpu(), want)
        return
    params = fx["history"][0]["params"]
    _check_close(got.cpu(), want, mc.one_axis(data.double(), params))
    _check_one_axis(got, cuda, params)


SHAPES = [(37, 29, 23), (64, 48, 40), (3, 20, 16), (12, 1, 10)]


def _values(shape, dtype, key) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(repr(key).encode()))
    if dtype.is_floating_point:
        return (torch.randn(shape, generator=g, device="cuda") * 100 + 50).to(dtype)
    info = torch.iinfo(dtype)
    lo, hi = max(-1000.0, 0.4 * info.min), min(1000.0, 0.4 * info.max)
    if dtype == torch.uint8:
        lo, hi = 60.0, 200.0
    return (torch.rand(shape, generator=g, device="cuda") * (hi - lo) + lo).round().to(dtype)


def _params(mode: str, batch: int, n: int = 2) -> dict:
    rng = np.random.default_rng(zlib.crc32(f"{mode}{batch}{n}".encode()))

    def draw():
        return [{"degrees": tuple(float(v) for v in rng.uniform(-12, 12, 3)),
                 "translation": tuple(float(v) for v in rng.uniform(-4, 4, 3))} for _ in range(n)]

    if mode == "shared":
        return {"transforms": draw()}
    transforms = [draw() for _ in range(batch)]
    if mode == "gated":
        transforms[0] = []
    return {"transforms": transforms, "_batched_keys": ["transforms"]}


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("batch,mode", [(1, "shared"), (1, "each"), (3, "shared"), (3, "each"), (3, "gated")],
                         ids=lambda v: str(v))
@pytest.mark.parametrize("dtype", mc.DTYPES, ids=mc.SHORT.get)
def test_every_dtype_mode_and_shape(dtype, batch, mode, shape):
    data = _values((batch, 2, *shape), dtype, (mc.SHORT[dtype], batch, mode, shape))
    params = _params(mode, batch)
    source = data.clone()
    got = _run_ops(data, params)
    assert torch.equal(data, source)  # out of place
    _check_close(got, mc.reference_ops(source, params), mc.one_axis(source.float().double(), params))
    _check_one_axis(got, source, params)


def test_inactive_rows_keep_their_bits():
    shape = (4, 2, 20, 18, 16)
    data = torch.randint(-2**31, 2**31 - 1, shape, device="cuda", dtype=torch.int32).view(torch.float32)
    data[0] = torch.randn(2, 20, 18, 16, device="cuda")
    data[2] = torch.randn(2, 20, 18, 16, device="cuda")
    params = _params("each", 4)
    params["transforms"][1] = []
    params["transforms"][3] = []
    got = _run_ops(data, params)
    for b in (1, 3):
        assert torch.equal(got[b].view(torch.int32), data[b].view(torch.int32))
    for b in (0, 2):
        assert not torch.equal(got[b], data[b])


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.float64], ids=str)
def test_non_finite_rows_become_nan_and_leave_their_neighbours(dtype):
    data = (torch.randn(2, 3, 24, 20, 16, device="cuda") * 10).to(dtype)
    data[0, 1, 5, 6, 7] = float("nan")
    data[1, 2, 0, 0, 0] = float("inf")
    data[1, 0, 23, 19, 15] = float("-inf")
    params = _params("each", 2)
    ref = mc.reference_ops(data, params)
    got = _run_ops(data, params)
    for b, c in [(0, 1), (1, 2), (1, 0)]:
        assert bool(torch.isnan(got[b, c]).all())
        print(f"reference on CUDA, row ({b}, {c}): all NaN {bool(torch.isnan(ref[b, c]).all())}")
    for b, c in [(0, 0), (0, 2), (1, 1)]:
        assert not bool(torch.isnan(got[b, c]).any())
        _check_close(got[b, c], ref[b, c])


def test_a_storage_offset_view():
    base = torch.randn(1 + 3 * 2 * 30 * 20 * 10, device="cuda")
    data = base[1:].view(3, 2, 30, 20, 10)
    assert data.storage_offset() == 1 and data.is_contiguous()
    source, before = data.clone(), base.clone()
    torch.manual_seed(3)
    out = tio.Motion(degrees=(-10, 10), translation=(-3, 3), copy=False)(_batch(data))
    params = out.applied_transforms[-1].params
    _check_close(out.images["t1"].data, mc.reference_ops(source, params))
    assert torch.equal(base, before)  # the caller's tensor is never written


def test_no_host_sync_on_a_large_cuda_batch():
    data = torch.randn(32, 1, 256, 256, 256, device="cuda")
    batch = _batch(data)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            tio.Motion(degrees=(-10, 10), translation=(-5, 5), copy=False)(batch)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    flagged = [str(w.message) for w in caught
               if "synchroniz" in str(w.message).lower() and "prototype feature" not in str(w.message)]
    assert flagged == []
    del data, batch
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", [torch.float32, torch.int16], ids=str)
def test_a_32_x_256_cubed_batch_on_every_voxel(dtype):
    g = torch.Generator(device="cuda").manual_seed(7)
    data = (torch.randn(32, 1, 256, 256, 256, generator=g, device="cuda") * 300).to(dtype)
    params = _params("each", 32)
    got = _run_ops(data, params)
    worst_ref, worst_bound = 0.0, 0.0
    for b0 in range(0, 32, 4):
        chunk = {**params, "transforms": params["transforms"][b0:b0 + 4]}
        x = data[b0:b0 + 4]
        exact = mc.one_axis(x.float().double(), chunk)
        worst_ref = max(worst_ref, _check_close(got[b0:b0 + 4], mc.reference_ops(x, chunk), exact))
        del exact
        worst_bound = max(worst_bound, _check_one_axis(got[b0:b0 + 4], x, chunk))
        torch.cuda.empty_cache()
    print(f"{dtype}: largest difference from the reference's op sequence {worst_ref:.3e}"
          f" ({'of range' if dtype.is_floating_point else 'units'}), from float64"
          f" {worst_bound:.3e} ({'of the bound' if dtype.is_floating_point else 'units'})")
    del data, got
    torch.cuda.empty_cache()


def _pipeline():
    return [tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.Motion(degrees=(-8, 8), translation=(-3, 3)),
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
        return [tio.ZNormalization(), tio.Motion(degrees=(-10, 10), translation=(-3, 3), p=0.7)]

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


def test_a_first_axis_longer_than_4096_is_refused():
    data = torch.rand(1, 1, 4097, 2, 3, device="cuda")
    with pytest.raises(NotImplementedError, match="longer than 4096"):
        tio.Motion()(_batch(data))
    out = tio.Motion()(_batch(data.permute(0, 1, 4, 3, 2).contiguous()))  # J and K are not bounded
    assert out.images["t1"].data.shape == (1, 1, 3, 2, 4097)


# ---- the reference's tests/test_motion.py --------------------------------------------------------

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
    result = tio.Motion(degrees=15, translation=10)(subject)
    assert not torch.allclose(result.t1.data.cpu(), original)


def test_num_transforms_validation():
    with pytest.raises(ValueError, match="num_transforms"):
        tio.Motion(num_transforms=0)


def test_leaves_labels_unchanged():
    subject = _subject()
    original_seg = subject.seg.data.clone()
    result = tio.Motion()(subject)
    torch.testing.assert_close(result.seg.data.cpu(), original_seg)


def test_preserves_shape():
    subject = _subject(with_label=False)
    assert tio.Motion()(subject).t1.data.shape == subject.t1.data.shape


def test_single_transform():
    subject = _subject(with_label=False)
    assert tio.Motion(num_transforms=1)(subject).t1.data.shape == subject.t1.data.shape


def _same_batch(batch_size: int = 5) -> tio.SubjectsBatch:
    data = torch.rand(1, 12, 12, 12)
    return tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data.clone())) for _ in range(batch_size)])


def test_per_instance_differs_across_batch():
    torch.manual_seed(0)
    batch = _same_batch()
    result = tio.Motion(degrees=(5, 15), translation=(5, 15), num_transforms=2)(batch)
    params = result.applied_transforms[-1].params
    assert "_batched_keys" in params
    assert len(params["transforms"]) == batch.batch_size
    assert not torch.allclose(result.t1.data[0], result.t1.data[1])


def test_per_instance_false_is_shared():
    torch.manual_seed(0)
    transform = tio.Motion(degrees=(5, 15), translation=(5, 15), num_transforms=2, per_instance=False)
    result = transform(_same_batch())
    torch.testing.assert_close(result.t1.data[0], result.t1.data[1])


def test_single_subject_keeps_scalar_params():
    subject = tio.Subject(t1=tio.ScalarImage(torch.rand(1, 12, 12, 12)))
    result = tio.Motion(degrees=15, translation=10)(subject)
    assert "_batched_keys" not in result.applied_transforms[-1].params


def test_too_many_transforms_for_first_axis_raises():
    subject = tio.Subject(t1=tio.ScalarImage(torch.rand(1, 2, 8, 8)))
    with pytest.raises(ValueError, match="motion segments"):
        tio.Motion(degrees=5, translation=5, num_transforms=4)(subject)


# ---- the reference's Motion cases of test_vectorization.py and test_per_instance.py --------------

def test_vectorized_matches_per_element():
    torch.manual_seed(0)
    assert_vectorized(tio.Motion(degrees=10.0, translation=10.0, num_transforms=2), _vectorization_batch())


def test_vectorized_matches_per_element_with_gating():
    torch.manual_seed(0)
    assert_vectorized(tio.Motion(degrees=10.0, translation=10.0, num_transforms=2, p=0.5),
                      _vectorization_batch(batch_size=6))


def test_preserves_float64():
    torch.manual_seed(0)
    data = (torch.rand(1, 8, 8, 8) + 0.5).to(torch.float64)
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data.clone())) for _ in range(8)])
    result = tio.Motion(degrees=10.0, translation=10.0, num_transforms=2, p=0.5)(batch)
    assert result.t1.data.dtype == torch.float64


# ---- launches -------------------------------------------------------------------------------------

def _launch_cases():
    x = torch.randn(3, 2, 24, 20, 16, device="cuda")
    shared, gated = _params("shared", 3), _params("gated", 3)
    return {"motion_shared": lambda: _run_ops(x, shared), "motion_gated": lambda: _run_ops(x, gated)}


def count_every_case(out_path: str) -> None:
    """{case: [ops.launches() delta, the library's kernels in a CUDA trace]} of every case, as JSON."""
    out = Path(out_path)
    trace = out.with_suffix(".trace.json")
    results = {}
    for name, call in _launch_cases().items():
        call()  # warm-up: module load
        torch.cuda.synchronize()
        before = ops.launches()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        counted = ops.launches() - before
        prof.export_chrome_trace(str(trace))
        events = json.loads(trace.read_text())["traceEvents"]
        results[name] = [counted, sum(1 for e in events if e.get("cat") == "kernel" and "tio::" in e.get("name", ""))]
    out.write_text(json.dumps(results))


def test_launch_count_equals_the_kernels_in_a_trace(tmp_path):
    """Traced in a process of its own, as tests/test_launch_count.py does."""
    out = tmp_path / "counts.json"
    code = (f"import sys; sys.path[:0] = {[str(ROOT), str(ROOT / 'tests')]!r}; "
            f"import test_gpu_motion; test_gpu_motion.count_every_case({str(out)!r})")
    subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], check=True)
    for name, (counted, traced) in json.loads(out.read_text()).items():
        assert traced == 3 and counted == traced, name  # the table upload, the motion pass, the NaN pass
