"""B-spline orders 2-7 on the GPU: the reference's fixtures, accuracy against the float64
restatement, the exact cases (mask, passthrough, short axes, NaN), the public paths and the launch
counts."""

from __future__ import annotations

import numpy as np
import pytest
import torch

import bspline_cases as bc
import torchio_b200 as tio
from torchio_b200 import ops

pytestmark = pytest.mark.gpu


def _batch(data, seg=None):
    subjects = []
    for b in range(data.shape[0]):
        images = {"t1": tio.ScalarImage(data[b])}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b])
        subjects.append(tio.Subject(**images))
    return tio.SubjectsBatch.from_subjects(subjects)


def _tolerance(order) -> float:
    """Share of the output's range: fp32 error of the prefilter grows with its gain (2, 3, 4.8, 7.5,
    11.8, 18.5 per axis for orders 2-7); 64 roundings of 2^-24 amplified by the three axes' gains
    bound the orders 6-7."""
    gain = {2: 2.0, 3: 3.0, 4: 4.8, 5: 7.5, 6: 11.8, 7: 18.5}[order]
    return 1e-4 if order <= 5 else 64 * 2.0**-24 * gain**3


@pytest.mark.parametrize("name", list(bc.CASES))
def test_fixture(name):
    case = bc.CASES[name]
    fx = bc.load_fixture(name)
    t1, seg = bc.scalar_image(case), bc.label_map(case)
    transform = getattr(tio, case["transform"])(**case["kwargs"])
    torch.manual_seed(bc.seed(case))
    out = transform(_batch(t1.cuda(), None if seg is None else seg.cuda()))
    for key in ("t1", "seg") if seg is not None else ("t1",):
        got = out.images[key].data
        assert got.is_cuda and str(got.dtype) == bc.dtype_of(fx, key)
        got = got.cpu().numpy()
        want = fx[f"out_{key}"]
        assert got.shape == want.shape
        affines = np.stack([a.numpy() for a in out.images[key].affines])
        np.testing.assert_allclose(affines, fx[f"affines_{key}"], rtol=1e-6, atol=1e-6)
        kwargs = case["kwargs"]
        order_name = kwargs.get("image_interpolation", "linear") if key == "t1" else kwargs["label_interpolation"]
        if order_name == "label":
            if want.shape[1] == 1:  # argmax of fp32 channels: ties may break differently, rarely
                assert np.mean(got != want) < 0.01
            else:
                np.testing.assert_allclose(got, want, atol=1e-4)
            continue
        if order_name in ("nearest", "linear"):  # K1: the reference's own coordinate noise
            span = max(float(np.ptp(want)), 1e-6)
            assert np.max(np.abs(got.astype(np.float64) - want)) <= 1e-4 * span
            continue
        order = {**{v: k for k, v in bc.NAMES.items()}, **{o: o for o in bc.ORDERS}}[order_name]
        if np.issubdtype(want.dtype, np.integer):
            exact = bc.replay(case, exact=True)[key]["data"].numpy()
            _assert_integer_exact(got, want, exact, order)
        else:
            span = max(float(np.ptp(want)), 1e-6)
            assert np.max(np.abs(got.astype(np.float64) - want)) <= _tolerance(order) * span


def _assert_integer_exact(got, want, exact, order):
    """Integer outputs truncate the fp32 spline value: within 1 of the reference everywhere, and
    equal wherever the float64 value is further from an integer than 1e-3 or the fp32 error bound
    (8 roundings of 2^-24 of the largest value, amplified by the three axes' prefilter gains)."""
    gain = {2: 2.0, 3: 3.0, 4: 4.8, 5: 7.5, 6: 11.8, 7: 18.5}[order]
    thr = max(1e-3, 8 * 2.0**-24 * gain**3 * float(np.max(np.abs(exact))))
    diff = got.astype(np.int64) - want.astype(np.int64)
    assert np.max(np.abs(diff)) <= 1
    away = np.abs(exact - np.round(exact)) > thr
    assert away.mean() > 0.5, away.mean()
    bad = away & (diff != 0)
    assert not bad.any(), (int(bad.sum()), exact[bad][:5], got[bad][:5], want[bad][:5])


def _affine_points(mat, shape):
    """The kernel's fp32 coordinate chain (affine_row) for a matrix-only element, on the host."""
    i, j, k = np.meshgrid(*(np.arange(n, dtype=np.float32) for n in shape), indexing="ij")
    m = mat.astype(np.float32)
    rows = []
    for ax in range(3):
        r = m[ax]
        acc = np.float32(i * r[0])
        acc = (j.astype(np.float64) * r[1] + acc).astype(np.float32)
        acc = (k.astype(np.float64) * r[2] + acc).astype(np.float32)
        acc = (acc + r[3]).astype(np.float32)
        rows.append(acc)
    return np.stack(rows, axis=-1).astype(np.float64)


def _mats(batch, shape, seed, scale=0.12):
    rng = np.random.default_rng(seed)
    c = (np.asarray(shape) - 1) / 2
    out = []
    for _ in range(batch):
        a = np.eye(3) + rng.uniform(-scale, scale, size=(3, 3))
        t = c - a @ c + rng.uniform(-1, 1, size=3)
        out.append(np.concatenate([a, t[:, None]], axis=1))
    return np.stack(out).astype(np.float32)


def _pull(data, mats, order, flags=None, out_shape=None):
    mat = torch.from_numpy(mats.reshape(len(mats), 12)).cuda()
    coeff = ops.bspline_prefilter(data, order, flags)
    return ops.bspline_resample(coeff, data, mat, None, flags, (1, 1, 1), (1, 1, 1), affine_first=True,
                                order=order, out_shape=out_shape)


@pytest.mark.parametrize("kind", ["noise", "smooth", "checkerboard"])
@pytest.mark.parametrize("order", bc.ORDERS)
def test_accuracy_against_float64(order, kind):
    shape = (64, 64, 64)
    g = torch.Generator().manual_seed(order)
    if kind == "noise":
        x = torch.randn(2, 1, *shape, generator=g, dtype=torch.float64)
    elif kind == "smooth":
        i, j, k = torch.meshgrid(*(torch.arange(n, dtype=torch.float64) for n in shape), indexing="ij")
        x = (torch.sin(i / 5) * torch.cos(j / 7) + torch.sin(k / 3))[None, None].repeat(2, 1, 1, 1, 1)
    else:
        i, j, k = torch.meshgrid(*(torch.arange(n) for n in shape), indexing="ij")
        x = ((i + j + k) % 2).double()[None, None].repeat(2, 1, 1, 1, 1)
    x32 = x.float()
    mats = _mats(2, shape, order)
    got = _pull(x32.cuda(), mats, order).cpu().numpy().astype(np.float64)
    hi = np.asarray(shape) - 1 + 0.05
    for b in range(2):
        pts = _affine_points(mats[b], shape)
        want = bc.reference_pull(x32[b].double().numpy(), pts, order)
        # the host restates the kernel's fp32 coordinate chain up to double rounding: leave the
        # voxels within 1e-3 of the mask's edges to test_mask_bounds_are_strict
        clear = np.all((np.abs(pts + 0.05) > 1e-3) & (np.abs(pts - hi) > 1e-3), axis=-1)
        span = float(np.ptp(want))
        err = np.abs(got[b] - want)[0][clear]
        assert np.max(err) <= _tolerance(order) * span, (np.max(err), np.unravel_index(
            np.argmax(np.abs(got[b] - want)[0] * clear), shape))
        inside = np.all((pts > -0.05) & (pts < hi), axis=-1)
        assert np.all(got[b][0][~inside & clear] == 0)


def test_mask_bounds_are_strict():
    shape = (6, 6, 6)
    data = torch.ones(1, 1, *shape, device="cuda")
    # translations putting the first / last planes on -0.05 and n - 1 + 0.05 (inclusive: masked)
    for shift, expect in ((-0.05, 0.0), (-0.0498, 1.0), (0.05, 0.0), (0.0498, 1.0)):
        m = np.concatenate([np.eye(3), [[shift], [0], [0]]], axis=1)[None].astype(np.float32)
        got = _pull(data, m, 3).cpu().numpy()[0, 0]
        plane = got[0] if shift < 0 else got[-1]
        assert np.all(plane == np.float32(expect)), (shift, plane.min(), plane.max())


def test_u8_overshoot_truncates_like_the_reference():
    """Cubic overshoot of 0 / 255 blocks leaves [0, 255]; the cast truncates it as the reference's
    Tensor.to(uint8) does, exactly away from integers."""
    case = bc.CASES["bspline_cubic_uint8"]
    want = bc.load_fixture("bspline_cubic_uint8")["out_t1"]
    exact = bc.replay(case, exact=True)["t1"]["data"].numpy()
    assert (exact < -0.5).any() and (exact > 255.5).any()
    torch.manual_seed(bc.seed(case))
    out = tio.Affine(**case["kwargs"])(_batch(bc.scalar_image(case).cuda())).images["t1"].data.cpu().numpy()
    _assert_integer_exact(out, want, exact, 3)


@pytest.mark.parametrize("shape", [(1, 5, 6), (2, 3, 7), (3, 1, 2), (2, 2, 1), (1, 1, 1), (1, 2, 2100)])
@pytest.mark.parametrize("order", [3, 7])
def test_short_axes(shape, order):
    x = torch.randn(2, 2, *shape, generator=torch.Generator().manual_seed(3))
    mats = np.stack([np.concatenate([np.eye(3), np.full((3, 1), 0.02)], axis=1)] * 2).astype(np.float32)
    mats[1, :, 3] = -0.03
    got = _pull(x.cuda(), mats, order).cpu().numpy()
    for b in range(2):
        want = bc.reference_pull(x[b].double().numpy(), _affine_points(mats[b], shape), order)
        assert np.max(np.abs(got[b] - want)) <= _tolerance(order) * max(float(np.ptp(want)), 1.0)


def test_passthrough_rows_are_bit_exact_and_skip_the_prefilter():
    shape = (10, 9, 8)
    x = torch.randn(3, 2, *shape, device="cuda")
    flags = torch.tensor([0, ops.FLAG_PASSTHROUGH, 0], dtype=torch.uint8, device="cuda")
    coeff = x.clone()
    ops.bspline_prefilter(coeff, 5, flags, in_place=True)
    assert torch.equal(coeff[1], x[1]) and not torch.equal(coeff[0], x[0])
    got = _pull(x, _mats(3, shape, 0), 5, flags)
    assert torch.equal(got[1], x[1])


def test_nan_fills_the_volume_inside_the_mask():
    shape = (12, 11, 10)
    x = torch.randn(2, 2, *shape, device="cuda")
    x[0, 1, 5, 5, 5] = float("nan")
    mats = _mats(2, shape, 1, scale=0.05)
    got = _pull(x, mats, 3).cpu().numpy()
    pts = _affine_points(mats[0], shape)
    inside = np.all((pts > -0.05) & (pts < np.asarray(shape) - 1 + 0.05), axis=-1)
    assert np.all(np.isnan(got[0, 1][inside])) and np.all(got[0, 1][~inside] == 0)
    assert np.isfinite(got[0, 0]).all() and np.isfinite(got[1]).all()


def test_public_paths():
    shape = (16, 14, 12)
    x = torch.randn(2, 1, *shape, device="cuda")
    seg = (torch.rand(2, 1, *shape, device="cuda") * 3).to(torch.int16)
    kwargs = dict(degrees=10, image_interpolation="cubic", label_interpolation="label",
                  one_hot_label_interpolation="cubic")
    torch.manual_seed(5)
    alone = tio.Affine(**kwargs)(_batch(x, seg))
    torch.manual_seed(5)
    composed = tio.Compose([tio.Affine(**kwargs)])(_batch(x, seg))
    for key in ("t1", "seg"):
        assert torch.equal(alone.images[key].data, composed.images[key].data)
    back = composed.apply_inverse_transform()
    assert back.images["t1"].data.shape == x.shape and back.images["seg"].data.dtype == torch.int16
    torch.manual_seed(5)
    resampled = tio.Resample((2.0, 2.0, 2.0), image_interpolation="fifth")(_batch(x))
    assert resampled.images["t1"].data.shape[2:] == (8, 7, 6)


def test_stream_of_host_batches_matches_batch_by_batch():
    shape = (12, 10, 9)
    hosts = [_batch(torch.randn(2, 1, *shape, generator=torch.Generator().manual_seed(s))) for s in range(3)]
    transform = tio.Compose([tio.Affine(degrees=10, image_interpolation="quadratic")])
    torch.manual_seed(9)
    one_by_one = [transform(h).images["t1"].data.cpu() for h in hosts]
    torch.manual_seed(9)
    streamed = [out.images["t1"].data.cpu() for out in transform.stream(hosts)]
    for got, want in zip(streamed, one_by_one):
        assert torch.equal(got, want)


@pytest.mark.parametrize("shape,passes", [((12, 10, 9), 3), ((12, 10, 1), 2), ((1, 1, 9), 1), ((1, 1, 1), 1)])
def test_launch_counts(shape, passes):
    x = torch.randn(2, 1, *shape, device="cuda")
    mats = _mats(2, shape, 0)
    torch.cuda.synchronize()
    before = ops.launches()
    coeff = ops.bspline_prefilter(x, 3)
    assert ops.launches() - before == passes
    before = ops.launches()
    ops.bspline_resample(coeff, x, torch.from_numpy(mats.reshape(2, 12)).cuda(), None, None, (1, 1, 1),
                         (1, 1, 1), affine_first=True, order=3)
    assert ops.launches() - before == 1
