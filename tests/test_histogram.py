"""HistogramStandardization, ZNormalization and compute_histogram_landmarks against the reference:
CPU checks of the host percentile restatement, constructors and fixtures; GPU checks of the
batched select, the device tables and the map, bit for bit against the reference's op sequence on
the same CUDA tensors and against the fixtures of tests/golden/generate_histogram.py."""

from __future__ import annotations

import builtins
import hashlib

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import ops
from torchio_b200.transforms import compute_histogram_landmarks
from torchio_b200.transforms.histogram import percentiles_from_neighbours

import histogram_cases as hc

CASES = {c["name"]: c for c in hc.HIST_CASES}
LM_CASES = {c["name"]: c for c in hc.LANDMARK_CASES}
HOST_DTYPES = [torch.float32, torch.float16, torch.uint8, torch.int8, torch.int16]
NUMPY = {torch.float32: np.float32, torch.float16: np.float16, torch.uint8: np.uint8, torch.int8: np.int8,
         torch.int16: np.int16}


def _host_neighbours(x: np.ndarray, qs):
    s = np.sort(x.astype(np.float32).reshape(-1))
    n = s.size
    vals, weights = [], []
    for q in qs:
        index = q * (n - 1)
        lower = int(np.floor(index))
        vals += [s[lower], s[min(lower + 1, n - 1)]]
        weights.append(index - lower)
    return np.array(vals, dtype=np.float32), np.array(weights)


def _same(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


# ---- CPU ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", HOST_DTYPES, ids=str)
def test_host_percentile_restatement_equals_np_percentile(dtype):
    rng = np.random.default_rng(7)
    qs_list = [hc.DEFAULT_QUANTILES, hc.quantiles_for((0.05, 0.95)), (0.0, 0.37, 1.0)]
    for trial in range(300):
        n = int(rng.integers(1, 5001))
        if dtype.is_floating_point:
            x = rng.standard_normal(n) * 10 ** rng.uniform(-3, 4)
        else:
            info = np.iinfo(NUMPY[dtype])
            x = rng.integers(info.min, info.max + 1, n)
        if trial % 3 == 0:
            x[rng.random(n) < 0.6] = 0
        x = x.astype(NUMPY[dtype])
        qs = qs_list[trial % 3]
        pct = [100.0 * q for q in qs]
        vals, weights = _host_neighbours(x, np.asarray(pct) / 100.0)
        got = percentiles_from_neighbours(vals, weights, False, dtype)
        assert _same(got, np.percentile(x, pct)), (dtype, n)


def test_fixtures_regenerate_from_the_cases_file():
    for case in hc.HIST_CASES:
        fx = hc.load_fixture(case["name"])
        if "error" in fx:
            assert case.get("landmark_count") is not None
            continue
        data = hc.scalar_image(case)
        expected = fx["out_t1"]
        applied = fx["history"] != [] and "exclude" not in case.get("kwargs", {})
        got = hc.reference_output(data, hc.landmarks(case), hc.case_cutoff(case)) if applied else data
        got = got.view(torch.int16) if got.dtype == torch.bfloat16 else got
        assert _same(got.numpy(), expected), case["name"]
        assert np.array_equal(fx["out_seg"], hc.label_map(case).numpy())
    for case in hc.LANDMARK_CASES:
        fx = hc.load_fixture(case["name"])
        kwargs = {k: case[k] for k in ("quantiles", "cutoff") if k in case}
        if case.get("masked"):
            kwargs["masking_method"] = hc.positive_mask
        if "error" in fx:
            continue
        got = hc.reference_landmarks(hc.training_images(case), **kwargs)
        assert _same(got.numpy(), fx["landmarks"]), case["name"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_repr_hydra_and_history_match_the_reference(name):
    case = CASES[name]
    fx = hc.load_fixture(name)
    transform = tio.HistogramStandardization(hc.landmarks(case), cutoff=hc.case_cutoff(case), **case.get("kwargs", {}))
    assert repr(transform) == fx["repr"]
    assert transform.to_hydra() == fx["hydra"]
    if "history" in fx and fx["history"]:
        assert fx["history"] == [{"name": "HistogramStandardization", "params": {}}]


def test_aliases_and_exports():
    assert tio.ZNormalization is tio.Standardize
    assert tio.HistogramStandardization is tio.transforms.HistogramStandardization
    assert callable(compute_histogram_landmarks)


def test_landmark_loaders(tmp_path):
    lm = torch.linspace(0, 100, 13)
    np.save(tmp_path / "lm.npy", lm.double().numpy())
    torch.save(lm, tmp_path / "lm.pt")
    torch.save({"a": lm}, tmp_path / "bad.pth")
    assert torch.equal(tio.HistogramStandardization(tmp_path / "lm.npy").landmarks, lm)
    assert torch.equal(tio.HistogramStandardization(str(tmp_path / "lm.pt")).landmarks, lm)
    assert tio.HistogramStandardization(lm.double()).landmarks.dtype == torch.float32
    with pytest.raises(TypeError, match="Expected a Tensor in .*bad.pth, got dict"):
        tio.HistogramStandardization(tmp_path / "bad.pth")
    with pytest.raises(ValueError, match="Unsupported landmarks file extension: .txt"):
        tio.HistogramStandardization(tmp_path / "lm.txt")


@pytest.mark.parametrize("name", [n for n in sorted(LM_CASES) if "error" in n])
def test_landmark_validation_errors(name):
    case = LM_CASES[name]
    fx = hc.load_fixture(name)
    kwargs = {k: case[k] for k in ("quantiles", "cutoff") if k in case}
    images = [tio.ScalarImage(t) for t in hc.training_images(case)]
    with pytest.raises(getattr(builtins, fx["error"]["type"])) as info:
        compute_histogram_landmarks(images, **kwargs)
    assert str(info.value) == fx["error"]["message"]


def test_landmarks_refuse_training_dtypes_fp32_does_not_hold():
    for dtype in (torch.int32, torch.int64, torch.float64):
        with pytest.raises(NotImplementedError, match=str(dtype)):
            compute_histogram_landmarks([tio.ScalarImage(torch.zeros(1, 2, 2, 2, dtype=dtype))])


# ---- GPU ----------------------------------------------------------------------------------------

def _run(case, data: torch.Tensor, **overrides) -> torch.Tensor:
    subjects = [tio.Subject(t1=tio.ScalarImage(data[b]), seg=tio.LabelMap(hc.label_map(case)[b].to(data.device)))
                for b in range(data.shape[0])]
    batch = tio.SubjectsBatch.from_subjects(subjects)
    kwargs = {**case.get("kwargs", {}), **overrides}
    out = tio.HistogramStandardization(hc.landmarks(case), cutoff=hc.case_cutoff(case), **kwargs)(batch)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_outputs_equal_the_op_sequence_on_cuda(name):
    case = CASES[name]
    data = hc.scalar_image(case).cuda()
    if case.get("landmark_count"):
        with pytest.raises(ValueError, match=r"Number of landmarks \(15\) does not match .* \(13\)"):
            _run(case, data)
        return
    out = _run(case, data)
    got = out.images["t1"].data
    applied = case.get("kwargs", {}).get("p", 1.0) > 0 and "exclude" not in case.get("kwargs", {})
    expected = hc.reference_output(data, hc.landmarks(case), hc.case_cutoff(case)) if applied else data
    assert got.dtype == data.dtype
    assert _same(got.cpu().view(torch.int16) if got.dtype == torch.bfloat16 else got.cpu(),
                 expected.cpu().view(torch.int16) if expected.dtype == torch.bfloat16 else expected.cpu())
    assert torch.equal(out.images["seg"].data.cpu(), hc.label_map(case))
    assert [t.params for t in out.applied_transforms] == ([{}] if case.get("kwargs", {}).get("p", 1.0) > 0 else [])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_device_tables_equal_the_op_sequence(name):
    case = CASES[name]
    if case.get("landmark_count"):
        return
    data = hc.scalar_image(case).cuda()
    qs = np.asarray([100.0 * q for q in hc.quantiles_for(hc.case_cutoff(case))]) / 100.0
    vals, w, _, nan = ops.quantiles_batched(data, qs)
    tables = ops.histogram_tables(vals, w, nan, hc.landmarks(case).cuda()).cpu()
    m = len(qs)
    for b in range(data.shape[0]):
        _, s, c, e = hc.element_tables(data[b], hc.landmarks(case), hc.case_cutoff(case))
        assert _same(tables[b, : m - 1], s.cpu()), (name, b)
        assert _same(tables[b, m - 1: 2 * (m - 1)], c.cpu()), (name, b)
        assert _same(tables[b, 2 * (m - 1): 2 * (m - 1) + m - 2], e.cpu()), (name, b)


@pytest.mark.gpu
def test_nan_voxels_bucket_like_aten():
    edges = torch.tensor([0.1, 0.2, 0.9], device="cuda")
    assert torch.bucketize(torch.tensor([float("nan")], device="cuda"), edges).item() == 3
    case = CASES["histstd_b3_c1_f32_nonfinite"]
    data = hc.scalar_image(case).cuda()
    got = _run(case, data).images["t1"].data
    assert bool(torch.isnan(got[0]).all())
    assert not bool(torch.isnan(got[1:]).any())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_outputs_match_the_reference_fixtures(name):
    case = CASES[name]
    fx = hc.load_fixture(name)
    data = hc.scalar_image(case).cuda()
    if "error" in fx:
        with pytest.raises(ValueError, match=r"Number of landmarks"):
            _run(case, data)
        return
    got = _run(case, data).images["t1"].data.cpu()
    got = got.view(torch.int16) if got.dtype == torch.bfloat16 else got
    expected = fx["out_t1"]
    differ = ~((got.numpy() == expected) | (np.isnan(got.numpy().astype(np.float64)) & np.isnan(expected.astype(np.float64))))
    if case["dtype"] == torch.float32 or not differ.any():
        assert not differ.any(), name
        return
    # the reference's CPU and CUDA casts of out-of-range fp32 results differ; nothing else may
    ref32 = hc.reference_output(data.float(), hc.landmarks(case), hc.case_cutoff(case)).cpu().numpy()
    info = np.iinfo(np.dtype(str(case["dtype"]).split(".")[1]))
    print(f"{name}: {int(differ.sum())} voxels differ from the CPU fixture, all out of {case['dtype']} range")
    assert np.all((ref32[differ] < info.min) | (ref32[differ] > info.max))


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in sorted(LM_CASES) if "error" not in n])
def test_compute_histogram_landmarks_equals_the_fixtures(name):
    case = LM_CASES[name]
    kwargs = {k: case[k] for k in ("quantiles", "cutoff") if k in case}
    if case.get("masked"):
        kwargs["masking_method"] = hc.positive_mask
    got = compute_histogram_landmarks([tio.ScalarImage(t) for t in hc.training_images(case)], **kwargs)
    assert got.dtype == torch.float32 and got.device.type == "cpu"
    assert _same(got.numpy(), hc.load_fixture(name)["landmarks"])


@pytest.mark.gpu
def test_batched_select_ranks_and_masks_at_b32():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(32, 1, 24, 20, 17, generator=g)
    x[5] = 3.25  # all equal
    qs = [0.0, 1.0, 0.5]
    vals, w, count, nan = ops.quantiles_batched(x.cuda(), qs)
    vals = vals.cpu()
    flat = x.view(32, -1)
    assert torch.equal(vals[:, 0], flat.min(1).values) and torch.equal(vals[:, 2], flat.max(1).values)
    assert bool((vals[5] == 3.25).all())
    for b in (0, 17, 31):
        s = flat[b].sort().values
        n = s.numel()
        lower = int(np.floor(0.5 * (n - 1)))
        assert vals[b, 4].item() == s[lower].item() and vals[b, 5].item() == s[lower + 1].item()
    assert bool((count.cpu() == flat.shape[1]).all()) and not bool(nan.any())
    mask = x > 0.3
    vals_m, _, count_m, _ = ops.quantiles_batched(x.cuda(), qs, mask.cuda())
    assert torch.equal(count_m.cpu(), mask.view(32, -1).sum(1).double())
    for b in (0, 31):
        sel = flat[b][mask.view(32, -1)[b]]
        assert vals_m[b, 0].item() == sel.min().item() and vals_m[b, 2].item() == sel.max().item()
    # more quantiles than one round holds
    many = np.linspace(0, 1, 40)
    vals_many, _, _, _ = ops.quantiles_batched(x[:2].cuda(), many)
    s = flat[1].sort().values
    idx = np.floor(many * (s.numel() - 1)).astype(np.int64)
    assert torch.equal(vals_many.cpu()[1, 0::2], s[idx])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.int16], ids=str)
def test_full_size_batch_equals_the_op_sequence(dtype):
    g = torch.Generator().manual_seed(11)
    x = torch.randn(32, 1, 256, 256, 256, generator=g).mul_(300)
    x[torch.rand(x.shape, generator=g) < 0.6] = 0
    data = x.to(dtype).cuda()
    del x
    lm = torch.linspace(0, 100, 13)
    expected = hc.reference_output(data, lm, (0.01, 0.99))
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data[b])) for b in range(32)])
    got = tio.HistogramStandardization(lm, copy=False)(batch).images["t1"].data
    print(dtype, "sha256", hashlib.sha256(got.cpu().numpy().tobytes()).hexdigest())
    assert torch.equal(got, expected)


@pytest.mark.gpu
def test_host_batch_streams_in_slices_like_the_one_shot_run():
    case = dict(CASES["histstd_b3_c2_f32"], batch=8, seed=470)
    data = hc.scalar_image(case)
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data[b])) for b in range(8)])
    one_shot = tio.HistogramStandardization(hc.landmarks(case))(batch).images["t1"].data
    pipeline = tio.Compose([tio.HistogramStandardization(hc.landmarks(case))])
    pipeline.chunk_size = 3
    streamed = pipeline(batch).images["t1"].data
    assert streamed.device.type == "cpu"
    assert torch.equal(streamed, one_shot)
    assert torch.equal(one_shot, hc.reference_output(data, hc.landmarks(case), (0.01, 0.99)))


@pytest.mark.gpu
def test_pipeline_with_znormalization():
    case = CASES["histstd_b3_c2_f32"]
    data = hc.scalar_image(case).cuda()
    seg = (data > 0).to(torch.int16)
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data[b]), seg=tio.LabelMap(seg[b]))
                                             for b in range(3)])
    out = tio.Compose([tio.HistogramStandardization(hc.landmarks(case)),
                       tio.ZNormalization(masking_method="seg")])(batch)
    step1 = hc.reference_output(data, hc.landmarks(case), (0.01, 0.99))
    sel = step1[0][seg[0].bool()]
    # Standardize's statistics are fp64 sums rounded to fp32, equal to torch's fp32 mean / std to
    # fp32 rounding (DESIGN §3)
    torch.testing.assert_close(out.images["t1"].data, (step1 - sel.mean()) / sel.std(), rtol=1e-5, atol=1e-5)
    assert [t.name for t in out.applied_transforms] == ["HistogramStandardization", "Standardize"]
