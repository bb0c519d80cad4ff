"""B-spline orders 2-7 on the GPU: the reference's fixtures within the per-voxel end-to-end bound of
tests/bspline_cases.py (label mode by its float64 margins), the exact cases (mask, passthrough,
NaN), the public paths and the launch counts.  Every kernel path against float64 is in
tests/test_gpu_bspline_paths.py."""

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
            if want.shape[1] == 1:
                _check_label_decisions(case, got, want)
            else:
                np.testing.assert_allclose(got, want, atol=1e-4)
            continue
        if order_name in ("nearest", "linear"):  # K1: the reference's own coordinate noise
            span = max(float(np.ptp(want)), 1e-6)
            assert np.max(np.abs(got.astype(np.float64) - want)) <= 1e-4 * span
            continue
        order = {**{v: k for k, v in bc.NAMES.items()}, **{o: o for o in bc.ORDERS}}[order_name]
        data = t1 if key == "t1" else seg
        if not bc.params_of(fx):  # every element gated out
            assert np.array_equal(got, data.numpy())
            continue
        (step,) = bc.params_of(fx)
        source, error = _antialiased(data, step["params"]) if kwargs.get("antialias") and key == "t1" else (None, None)
        ratio = bc.check_end_to_end(data, torch.from_numpy(got), step["params"], order, source, error)
        if got.dtype.kind == "f":
            print(f"[fixture {name} {key}] max |gpu - ref| / bound = {ratio:.3f}")
        else:  # most voxels must fall under the exact-equality rule, or it checks nothing
            assert ratio < 0.5, ratio
            print(f"[fixture {name} {key}] share within the bound of an integer = {ratio:.3f}")


def _antialiased(data, params):
    """The anti-alias blur of the reference (torch_port) and a bound on how far the GPU's blur of the
    same data may lie from it, gamma_m of the blur of |data|.  Per blurred axis of radius r, each side
    rounds its 2r+1 weights (x / sigma, the square, exp counted as 2, the sum of 2r+1 weights and the
    division: 2r + 5) and its sum of 2r+1 products (2r+1), all terms non-negative; m adds 4r + 6 per
    axis for the host and again for the device.  The factor 1 + 2^-10 covers the fp32 rounding of
    the blurred |data| itself."""
    from oracle import torch_port as tp

    a_out = np.asarray(params["target"]["affine"], dtype=np.float64)
    sp_in = np.asarray(tp.spacing_of(np.eye(4)))
    sigmas = tp.antialias_sigmas(np.asarray(tp.spacing_of(a_out)) / sp_in, sp_in)
    radii = [max(int(np.ceil(3 * s)), 1) for s in sigmas if s > 0]
    m = 2 * sum(4 * r + 6 for r in radii)
    blurred = tp.antialias(data.float(), np.eye(4), a_out)
    magnitude = tp.antialias(data.float().abs(), np.eye(4), a_out).double().numpy()
    return blurred, bc.gamma(m) * magnitude * (1 + 2.0**-10)


def _check_label_decisions(case, got, want):
    """Label mode at C = 1 (argmax over one-hot splines, pad where their sum is not > 0.5): every
    voxel whose |sum - 0.5| margin exceeds its bound, and, where the sum is above 0.5, whose top-two
    margin exceeds its bound too, equals the float64 decision; the others are counted, and each holds
    one of its near-tied labels."""
    seg = bc.label_map(case)
    (step,) = bc.params_of(bc.load_fixture(case["name"]))
    params = step["params"]
    order = {**{v: k for k, v in bc.NAMES.items()}}[params["one_hot_label_interpolation"]]
    labels = torch.unique(seg)
    onehot = (seg[:, 0][:, None] == labels.reshape(1, -1, 1, 1, 1)).float()
    q, out_shape, flags = bc.step_coords(params, seg.shape[0], tuple(seg.shape[2:]))
    pad = float(params["default_pad_label"])
    undecided = 0
    for e in range(seg.shape[0]):
        value, bound, _ = bc.end_to_end(onehot[e].double().numpy(), q[e].reshape(-1, 3), order)
        n = value.shape[0]
        total = value.sum(axis=0)
        total_bound = bound.sum(axis=0) + bc.gamma(n) * np.abs(value).sum(axis=0)
        top = np.argsort(-value, axis=0, kind="stable")
        v1 = np.take_along_axis(value, top[:1], 0)[0]
        v2 = np.take_along_axis(value, top[1:2], 0)[0] if n > 1 else np.full_like(v1, -np.inf)
        b1 = np.take_along_axis(bound, top[:1], 0)[0]
        b2 = np.take_along_axis(bound, top[1:2], 0)[0] if n > 1 else np.zeros_like(v1)
        # the argmax matters only where the sum says "inside"
        decided = (np.abs(total - 0.5) > total_bound) & ((total < 0.5) | (v1 - v2 > b1 + b2))
        decision = np.where(total > 0.5, labels.numpy()[top[0]], pad)
        g = got[e, 0].reshape(-1).astype(np.float64)
        assert np.array_equal(g[decided], decision[decided]), int((g[decided] != decision[decided]).sum())
        near = value >= (v1 - b1)[None] - bound  # labels within the bounds of the top one
        allowed = [set(labels.numpy()[near[:, p]].tolist()) | ({pad} if abs(total[p] - 0.5) <= total_bound[p] else set())
                   for p in np.flatnonzero(~decided)]
        for p, ok in zip(np.flatnonzero(~decided), allowed):
            assert g[p] in ok, (p, g[p], ok)
        undecided += int((~decided).sum())
    print(f"[fixture {case['name']} label mode] {undecided} voxels within their bounds of a tie")


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
    out = tio.Affine(**case["kwargs"])(_batch(bc.scalar_image(case).cuda())).images["t1"].data.cpu()
    assert np.max(np.abs(out.numpy().astype(np.int64) - want.astype(np.int64))) <= 1
    (step,) = bc.params_of(bc.load_fixture("bspline_cubic_uint8"))
    near = bc.check_end_to_end(bc.scalar_image(case), out, step["params"], 3)
    assert near < 0.5, near  # most voxels fall under the exact-equality rule


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
