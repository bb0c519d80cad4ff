"""Spike on the GPU: the fixtures of tests/golden/generate_spike.py, the reference's op sequence on the
same CUDA tensors for every image dtype, the spectrum peak against torch.fft, gating, batches past
2**31 elements, host batches streamed through a Compose, and the reference's own Spike tests."""

from __future__ import annotations

import warnings
import zlib

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import ops
from torchio_b200.transforms.spike import spike_table

import spike_cases as sc

pytestmark = pytest.mark.gpu

CASES = sc.CASES


def _batch(data: torch.Tensor, seg: torch.Tensor | None = None) -> tio.SubjectsBatch:
    subjects = []
    for b in range(data.shape[0]):
        images = {"t1": tio.ScalarImage(data[b])}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b])
        subjects.append(tio.Subject(**images))
    return tio.SubjectsBatch.from_subjects(subjects)


def _params(out) -> dict | None:
    history = out.applied_transforms
    return history[-1].params if history else None


def _check_against_reference(got: torch.Tensor, data: torch.Tensor, params: dict) -> None:
    """Within 1e-4 of the output's range of the reference's CUDA op sequence (floats; plus one unit
    in the last place of fp16 / bf16, where both round an fp32 value), within 1 (integers inside
    the dtype's range); NaN positions equal."""
    ref = sc.reference_ops(data, params)
    assert got.dtype == ref.dtype and got.shape == ref.shape
    g, r = got.double(), ref.double()
    assert torch.equal(torch.isnan(g), torch.isnan(r))
    ok = ~torch.isnan(r)
    if got.dtype.is_floating_point:
        finite = r[ok & torch.isfinite(r)]
        span = float(finite.max() - finite.min()) if finite.numel() else 1.0
        ulp = {torch.float16: 2.0**-10, torch.bfloat16: 2.0**-7}.get(got.dtype, 0.0)
        both = ok & torch.isfinite(r)
        assert bool(((g[both] - r[both]).abs() <= 1e-4 * span + ulp * r[both].abs()).all())
        assert torch.equal(g[ok & ~torch.isfinite(r)], r[ok & ~torch.isfinite(r)])
        return
    info = torch.iinfo(got.dtype)
    inside = ok & (r > info.min) & (r < info.max)
    assert float((g[inside] - r[inside]).abs().max()) <= 1


def _run(transform, data, seg=None):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return transform(_batch(data, seg))


@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_are_reproduced_on_the_device(name):
    case = CASES[name]
    fx = sc.load_fixture(name)
    data, seg = sc.scalar_image(case), sc.label_map(case)
    if "error" in fx:
        with pytest.raises(ValueError, match=fx["error"]["message"]):
            tio.Spike(**case["kwargs"])
        return
    torch.manual_seed(sc.seed(case))
    out = _run(tio.Spike(**case["kwargs"]), data.cuda(), None if seg is None else seg.cuda())
    assert [{"name": t.name, "params": t.params} for t in out.applied_transforms] == fx["history"]
    got = out.images["t1"].data
    assert str(got.dtype) == fx["dtype"] and got.is_cuda
    if seg is not None:
        assert torch.equal(out.images["seg"].data.cpu(), seg)
    if not fx["history"] or "t1" in case["kwargs"].get("exclude", []):
        assert np.array_equal(sc.as_stored(got), fx["out_t1"], equal_nan=True)
        return
    params = fx["history"][0]["params"]
    sc.check_against_oracle(sc.as_float64(sc.as_stored(got), case["dtype"]), data.double().numpy(), params,
                            case["dtype"])
    _check_against_reference(got, data.cuda(), params)


SHAPES = [(23, 19, 17), (1, 37, 29), (181, 217, 181), (4096, 3, 2)]


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("kind", ["signed", "nonneg"])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("dtype", sc.DTYPES, ids=sc.SHORT.get)
def test_every_dtype_follows_the_reference_op_sequence(dtype, batch, kind, shape):
    if kind == "signed" and dtype == torch.uint8:
        kind = "nonneg"
    rng = np.random.default_rng(zlib.crc32(repr((sc.SHORT[dtype], batch, kind, shape)).encode()))
    data = sc.random_values(rng, (batch, 1, *shape), dtype, kind).cuda()
    intensity = (1, 3) if dtype.is_floating_point else (0.01, 0.05)
    torch.manual_seed(batch + len(shape))
    source = data.clone()
    out = _run(tio.Spike(num_spikes=(1, 3), intensity=intensity), data)
    got = out.images["t1"].data
    assert torch.equal(data, source)  # copy=True: the caller's tensor is untouched
    _check_against_reference(got, source, _params(out))
    if shape[0] * shape[1] * shape[2] <= 10000:
        sc.check_against_oracle(got.double().cpu().numpy(), source.double().cpu().numpy(), _params(out), dtype)


@pytest.mark.parametrize("shape", [(32, 31, 30), (181, 217, 181), (1, 64, 45), (4096, 2, 3), (5, 4096, 1)],
                         ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", [torch.float32, torch.int16, torch.bfloat16], ids=str)
def test_spectrum_peak_and_sum(dtype, shape):
    g = torch.Generator(device="cuda").manual_seed(3)
    signed = (torch.randn(2, 2, *shape, generator=g, device="cuda") * 100).to(dtype)
    nonneg = signed.abs()
    data = torch.cat([signed, nonneg])  # elements 0, 1 signed, 2, 3 non-negative
    intensity = torch.ones(4, dtype=torch.float32, device="cuda")
    total, flags = ops.spike_stats(data, intensity)
    peak = ops.spectrum_peak(data, intensity, flags, workspace_bytes=shape[0] * shape[1] * (shape[2] // 2 + 1) * 8)
    x = data.float()
    assert flags.tolist() == [1, 1, 1, 1, 0, 0, 0, 0]
    assert torch.allclose(total, x.double().sum(dim=(2, 3, 4)).reshape(-1), rtol=1e-12, atol=0)
    want = torch.fft.rfftn(x[:2].double(), dim=(-3, -2, -1)).abs().amax(dim=(-3, -2, -1)).reshape(-1)
    assert torch.allclose(peak[:4].double(), want, rtol=1e-5, atol=0)
    assert peak[4:].tolist() == [0.0] * 4
    nonneg_peak = torch.fft.fftn(x[2:], dim=(-3, -2, -1)).abs().amax(dim=(-3, -2, -1)).reshape(-1).double()
    assert torch.allclose(total[4:], nonneg_peak, rtol=1e-5, atol=0)


def test_stats_flags_and_inactive_rows():
    data = torch.rand(3, 2, 6, 5, 4, device="cuda")
    data[0, 1, 0, 0, 0] = float("nan")
    data[1, 0, 1, 1, 1] = -0.0
    data[1, 1, 1, 1, 1] = -1.0
    data[2, 0, 2, 2, 2] = float("-inf")
    total, flags = ops.spike_stats(data, torch.tensor([1.0, 2.0, 0.0], device="cuda"))
    assert flags.tolist() == [0, 2, 0, 1, 0, 0]
    assert total[4:].tolist() == [0.0, 0.0]
    again, _ = ops.spike_stats(data, torch.tensor([1.0, 2.0, 0.0], device="cuda"))
    assert torch.equal(total[~torch.isnan(total)], again[~torch.isnan(again)])  # same bits every call


def test_a_batch_mixing_signed_and_non_negative_elements():
    g = torch.Generator(device="cuda").manual_seed(8)
    data = torch.randn(4, 2, 40, 36, 30, generator=g, device="cuda") * 50
    data[1] = data[1].abs()
    data[3, 0] = data[3, 0].abs()
    torch.manual_seed(2)
    out = _run(tio.Spike(num_spikes=(1, 5), intensity=(1, 3)), data)
    _check_against_reference(out.images["t1"].data, data, _params(out))
    sc.check_against_oracle(out.images["t1"].data.double().cpu().numpy(), data.double().cpu().numpy(), _params(out),
                            torch.float32)


@pytest.mark.parametrize("dtype", [torch.float32, torch.uint8, torch.bfloat16], ids=str)
def test_gated_out_elements_keep_their_bits(dtype):
    data = (torch.rand(8, 1, 20, 18, 16, device="cuda") * 200).to(dtype)
    data[2, 0, 0, 0, 0] = 0 if not dtype.is_floating_point else float("nan")
    torch.manual_seed(6)
    out = _run(tio.Spike(intensity=(1, 3), p=0.5), data)
    keep = _params(out)["_keep"]
    assert 0 < sum(keep) < 8
    got = out.images["t1"].data
    for b, kept in enumerate(keep):
        if not kept:
            assert torch.equal(got[b].view(torch.uint8), data[b].view(torch.uint8))
        else:
            assert not torch.equal(got[b], data[b])


def test_shared_intensity_zero_returns_the_same_tensor():
    data = torch.rand(3, 1, 8, 8, 8, device="cuda")
    batch = _batch(data)
    before = batch.images["t1"].data
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        tio.Spike(intensity=0.0, per_instance=False, copy=False)(batch)
    assert batch.images["t1"].data is before


def test_no_host_sync_on_a_cuda_batch():
    data = torch.rand(4, 1, 64, 64, 64, device="cuda") - 0.5
    data[1] = data[1].abs()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = tio.Spike(num_spikes=(1, 3), intensity=(1, 3))(_batch(data))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _check_against_reference(out.images["t1"].data, data, _params(out))


def _element_by_element(data, table, ratio):
    for b in range(data.shape[0]):
        ops.spike(data[b:b + 1], table[b:b + 1], ratio[b:b + 1])


@pytest.mark.parametrize("dtype,kind", [(torch.uint8, "nonneg"), (torch.int8, "signed")], ids=["u8_sum", "i8_fft"])
def test_past_2_31_elements_equals_small_batches(dtype, kind):
    shape = (9, 1, 640, 640, 640)  # 2.36e9 elements
    assert np.prod(shape) > 2**31
    g = torch.Generator(device="cuda").manual_seed(4)
    if kind == "nonneg":
        data = torch.randint(0, 200, shape, generator=g, device="cuda", dtype=dtype)
    else:
        data = torch.randint(-100, 100, shape, generator=g, device="cuda", dtype=dtype)
    rows = [[[0.1 * b, 0.3, 0.7], [0.5, 0.25 * (b % 4), 0.9]] for b in range(9)]
    table, ratio = spike_table(rows, [0.02 + 0.005 * b for b in range(9)], shape[2:])
    ratio[4] = 0.0  # one element not active
    source = data[[0, 4, 8]].clone()
    ops.spike(data, table, ratio)
    small = source.clone()
    _element_by_element(small, table[[0, 4, 8]], ratio[[0, 4, 8]])
    got = data[[0, 4, 8]]
    assert torch.equal(got[1], source[1])
    diff = (got.int() - small.int()).abs()
    assert int(diff.max()) <= 1 and float((diff > 0).double().mean()) < 1e-6
    assert not torch.equal(got[2], source[2])
    del data, got, small, source
    torch.cuda.empty_cache()


def test_compose_stream_on_a_host_batch_equals_the_transforms_one_by_one():
    g = torch.Generator().manual_seed(21)
    batches = [(torch.randn(6, 1, 24, 22, 20, generator=g) * 100 + 50) for _ in range(3)]
    pipeline = tio.Compose([tio.ZNormalization(), tio.Spike(num_spikes=(1, 3), intensity=(1, 3))])
    pipeline.chunk_size = 2
    torch.manual_seed(17)
    streamed = list(pipeline.stream(_batch(b) for b in batches))
    torch.manual_seed(17)
    for data, out in zip(batches, streamed, strict=True):
        step = _batch(data)
        for t in (tio.ZNormalization(), tio.Spike(num_spikes=(1, 3), intensity=(1, 3))):
            step = t(step)
        assert out.images["t1"].data.device.type == "cpu"
        assert [t.name for t in out.applied_transforms] == [t.name for t in step.applied_transforms]
        assert _params(out) == _params(step)
        torch.testing.assert_close(out.images["t1"].data, step.images["t1"].data, rtol=1e-5, atol=1e-5)


def test_axis_longer_than_4096_is_refused():
    data = torch.rand(1, 1, 4097, 2, 1, device="cuda")
    with pytest.raises(NotImplementedError, match="longer than 4096"):
        tio.Spike(intensity=2.0)(_batch(data))


# ---- the reference's tests/test_spike.py --------------------------------------------------------

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
    result = tio.Spike(num_spikes=3, intensity=2.0)(subject)
    assert not torch.allclose(result.t1.data, original)


def test_zero_intensity_is_identity():
    subject = _subject(with_label=False)
    original = subject.t1.data.clone()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        result = tio.Spike(intensity=0.0)(subject)
    torch.testing.assert_close(result.t1.data, original)


def test_leaves_labels_unchanged():
    subject = _subject()
    original_seg = subject.seg.data.clone()
    result = tio.Spike(num_spikes=3, intensity=2.0)(subject)
    torch.testing.assert_close(result.seg.data, original_seg)


def test_single_spike():
    subject = _subject(with_label=False)
    original = subject.t1.data.clone()
    result = tio.Spike(num_spikes=1, intensity=1.0)(subject)
    assert not torch.allclose(result.t1.data, original)


def _same_batch(batch_size: int = 6) -> tio.SubjectsBatch:
    data = torch.rand(1, 12, 12, 12)
    return tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data.clone())) for _ in range(batch_size)])


def test_per_instance_differs_across_batch():
    torch.manual_seed(0)
    batch = _same_batch()
    result = tio.Spike(intensity=(1.0, 3.0))(batch)
    params = result.applied_transforms[-1].params
    assert "_batched_keys" in params
    assert len(params["intensity"]) == batch.batch_size
    assert not torch.allclose(result.t1.data[0], result.t1.data[1])


def test_per_instance_false_is_shared():
    torch.manual_seed(0)
    result = tio.Spike(intensity=(1.0, 3.0), per_instance=False)(_same_batch())
    torch.testing.assert_close(result.t1.data[0], result.t1.data[1])


def test_single_subject_keeps_scalar_params():
    subject = tio.Subject(t1=tio.ScalarImage(torch.rand(1, 12, 12, 12)))
    result = tio.Spike(intensity=(1.0, 3.0))(subject)
    assert "_batched_keys" not in result.applied_transforms[-1].params
