"""Standardize / Normalize (SURVEY §8 f-3) on the GPU against the unmodified reference's fixtures:
the statistics kernels (tio_moments, tio_quantiles) must reproduce the params the reference
recorded — quantiles exactly (order statistics + the same fp32 lerp), moments to fp32 rounding —
and tio_rescale must reproduce its outputs bit for bit given those params."""

import json
import warnings

import numpy as np
import pytest
import torch

from golden_cases import CASES_BY_NAME, STAT_CASES
from util import load_golden, make_product_transform, product_batch, product_replay, report

pytestmark = pytest.mark.gpu
NAMES = [c["name"] for c in STAT_CASES]


@pytest.mark.parametrize("name", NAMES)
def test_replay_of_reference_params_is_bit_exact(name):
    """Recorded params through tio_rescale == the reference's elementwise ops, bit for bit
    (sub, div, mul, add each rounded to fp32; clamp first)."""
    _, images, history, expected, _ = load_golden(name)
    out = product_replay(product_batch(images, device="cuda"), history)
    for n, exp in expected.items():
        got = out.images[n].data.cpu()
        assert got.dtype == exp.dtype
        assert torch.equal(got, exp), (n, report(got, exp))


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_public_call_derives_the_reference_params(name, device):
    """Sampling + statistics of batch element 0 (masked, percentiles, explicit ranges) through the
    public call with the reference's seed; host-resident batches stage sample 0 for the kernels."""
    case = CASES_BY_NAME[name]
    _, images, history, expected, _ = load_golden(name)
    transform = make_product_transform(case["transform"])
    torch.manual_seed(case["seed"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = transform(product_batch(images, device=None if device == "cpu" else "cuda"))
    mine = json.loads(json.dumps(out.applied_transforms[0].params))
    want = history[0]["params"]
    assert set(mine) == set(want)
    for key in want:
        if key == "stats":  # (mean, std): fp64 sums here, fp32 cascade sums in the reference
            for img, (mean, std) in want[key].items():
                assert mine[key][img][0] == pytest.approx(mean, rel=2e-6, abs=1e-7)
                assert mine[key][img][1] == pytest.approx(std, rel=2e-6)
        elif key == "in_ranges":  # order statistics: exact
            assert mine[key] == want[key]
        else:
            assert mine[key] == want[key], key
    for n, exp in expected.items():
        got = out.images[n].data.cpu()
        rng = float(exp.float().max() - exp.float().min()) or 1.0
        assert float((got.float() - exp.float()).abs().max()) <= 1e-5 * rng, n


def test_quantile_select_and_moments_match_torch_on_a_large_volume():
    """128^3 x 2 channels (4.2M values): every order statistic the reference would read, and the
    moments, vs torch on the host; ties, signed zeros, masks."""
    from torchio_b200 import ops

    g = torch.Generator().manual_seed(12)
    x = torch.randn((2, 128, 128, 128), generator=g) * 3 - 1
    x[0, :4] = 0.0
    x[1, 5, 5, :5] = -0.0
    mask = torch.rand((1, 128, 128, 128), generator=g) > 0.6
    flat = x.reshape(-1)
    for m, values in ((None, flat), (mask, x[mask.expand_as(x)])):
        qs = [0.005, 0.995]
        vals, weights, count = ops.quantile_neighbours(x.cuda(), qs, None if m is None else m.cuda())
        assert count == values.numel()
        for t, q in enumerate(qs):
            index = q * (values.numel() - 1)
            lower = int(np.floor(index))
            want_lo = float(torch.kthvalue(values, lower + 1).values)
            want_hi = float(torch.kthvalue(values, min(lower + 2, values.numel())).values)
            assert vals[2 * t] == want_lo and vals[2 * t + 1] == want_hi
            assert weights[t] == pytest.approx(index - lower, abs=1e-9)
        s, dev, n = ops.moments(x.cuda(), None if m is None else m.cuda())
        assert n == values.numel()
        assert s / n == pytest.approx(float(values.double().mean()), rel=1e-12, abs=1e-12)
        # the second value is the sum of squared deviations from the mean, with no raw-moment cancellation
        assert dev / (n - 1) == pytest.approx(float(values.double().var()), rel=1e-12)
    v, w, c = ops.quantile_neighbours(x.cuda(), [0.0, 1.0])
    assert v[0] == float(flat.min()) and v[2] == float(flat.max()) and w == [0.0, 0.0]


def test_standardize_and_normalize_invert():
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(3)
    x = torch.rand((3, 1, 20, 24, 16), generator=g) * 5 - 2
    batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(x.cuda(), [tio.AffineMatrix() for _ in range(3)])})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for t in (tio.Standardize(), tio.Normalize(out_min=(-1.0, 0.0), out_max=(0.5, 1.0))):
            torch.manual_seed(4)
            out = t(batch)
            back = out.apply_inverse_transform()
            # (Normalize clips to the range of sample 0: only that element is guaranteed to come back)
            rows = slice(0, 1) if isinstance(t, tio.Normalize) else slice(None)
            assert float((back.images["t1"].data.cpu()[rows] - x[rows]).abs().max()) <= 5e-6 * 7
        out = tio.Standardize()(batch)
        y = out.images["t1"].data[0]
        assert abs(float(y.mean())) < 1e-5 and abs(float(y.std()) - 1) < 1e-5
