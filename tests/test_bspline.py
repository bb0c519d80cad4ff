"""B-spline orders 2-7 without a GPU: the float64 restatement of interpol.grid_pull against SciPy and
against its own defining properties, the fixtures' shape and dtype records, the constructors, and
the C entry points' argument checks."""

from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch
from scipy import ndimage

import bspline_cases as bc
import torchio_b200 as tio
from torchio_b200 import _native


def _points(shape, n, seed):
    rng = np.random.default_rng(seed)
    hi = np.asarray(shape, dtype=np.float64) - 1
    return rng.uniform(-0.049, hi + 0.049, size=(n, 3))  # within the 0.05 margin


@pytest.mark.parametrize("order", [2, 3, 4, 5])
@pytest.mark.parametrize("shape", [(9, 7, 6), (3, 2, 5), (1, 4, 3)])
def test_restatement_matches_scipy_reflect(order, shape):
    data = np.random.default_rng(order).standard_normal((1, *shape))
    pts = _points(shape, 300, order)
    ours = bc.reference_pull(data, pts, order)[0]
    scipy = ndimage.map_coordinates(data[0], pts.T, order=order, mode="reflect", prefilter=True)
    assert np.max(np.abs(ours - scipy)) < 1e-10


@pytest.mark.parametrize("order", [6, 7])
@pytest.mark.parametrize("shape", [(8, 5, 3), (2, 1, 4)])
def test_high_orders_interpolate_and_are_half_sample_symmetric(order, shape, monkeypatch):
    data = np.random.default_rng(order).standard_normal((2, *shape))
    grid = np.stack(np.meshgrid(*(np.arange(n, dtype=np.float64) for n in shape), indexing="ij"), axis=-1)
    assert np.allclose(bc.reference_pull(data, grid, order), data, atol=1e-10)
    monkeypatch.setattr(bc, "MARGIN", 10.0)  # evaluate outside the volume to see the boundary
    coeff = bc.coefficients(data, order)
    d = np.random.default_rng(1).uniform(0, 0.5, size=(50, 1)) * np.ones((1, 3))
    for centre in (-0.5, np.asarray(shape) - 0.5):
        a = bc.evaluate(coeff, centre + d, order)
        b = bc.evaluate(coeff, centre - d, order)
        assert np.allclose(a, b, atol=1e-10)


def test_restatement_refuses_other_arguments():
    x = torch.zeros(1, 1, 3, 3, 3)
    g = torch.zeros(1, 2, 2, 2, 3)
    with pytest.raises(NotImplementedError):
        bc.grid_pull(x, g, interpolation=3, bound="zero", extrapolate=False, prefilter=True)
    with pytest.raises(NotImplementedError):
        bc.grid_pull(x, g, interpolation=3, bound="dct2", extrapolate=True, prefilter=True)
    with pytest.raises(NotImplementedError):
        bc.grid_pull(x, g, interpolation=1, bound="dct2", extrapolate=False, prefilter=True)


def test_restatement_masks_outside_the_margin():
    data = np.ones((1, 4, 4, 4))
    pts = np.array([[-0.049, 0, 0], [-0.05, 0, 0], [3.049, 3, 3], [3.05, 3, 3], [np.nan, 1, 1]])
    assert bc.reference_pull(data, pts, 3)[0].tolist() == pytest.approx([1, 0, 1, 0, 0])


@pytest.mark.parametrize("name", list(bc.CASES))
def test_fixture_records_every_image(name):
    case = bc.CASES[name]
    fx = bc.load_fixture(name)
    t1 = bc.scalar_image(case)
    assert fx["out_t1"].shape[:2] == tuple(t1.shape[:2])
    assert bc.dtype_of(fx, "t1") == str(t1.dtype)
    assert fx["affines_t1"].shape == (bc.BATCH, 4, 4)
    assert np.isfinite(fx["out_t1"].astype(np.float64)).all()
    assert ("out_seg" in fx) == bool(case.get("seg"))
    assert all(t["name"] == case["transform"] for t in bc.params_of(fx))


@pytest.mark.parametrize("name", list(bc.CASES))
def test_replay_matches_every_fixture(name):
    """The reference's op sequence (torch_port's geometry + the restatement) reproduces each fixture:
    the same fp32 results, so equal to 2e-6 of the range for images (ATen's last ulp may differ
    across CPU builds) and exactly for integer and label outputs."""
    fx = bc.load_fixture(name)
    out = bc.replay(bc.CASES[name])
    for key, img in out.items():
        got, want = img["data"], torch.from_numpy(fx[f"out_{key}"])
        assert str(got.dtype) == bc.dtype_of(fx, key) and got.shape == want.shape
        if got.dtype.is_floating_point:
            span = float(want.double().max() - want.double().min()) or 1.0
            assert float((got.double() - want.double()).abs().max()) <= 2e-6 * span
        else:
            assert torch.equal(got, want)
        np.testing.assert_allclose(np.stack(img["affines"]), fx[f"affines_{key}"], atol=1e-12)


@pytest.mark.parametrize("order", bc.ORDERS)
def test_integer_orders_equal_their_names(order):
    by_int = tio.Affine(degrees=5, image_interpolation=order, label_interpolation=order,
                        one_hot_label_interpolation=order)
    by_name = tio.Affine(degrees=5, image_interpolation=bc.NAMES[order], label_interpolation=bc.NAMES[order],
                         one_hot_label_interpolation=bc.NAMES[order])
    for attr in ("image_interpolation", "label_interpolation", "one_hot_label_interpolation"):
        assert getattr(by_int, attr) == getattr(by_name, attr) == bc.NAMES[order]


def test_one_hot_label_mode_is_still_refused():
    with pytest.raises(ValueError, match="one_hot_label_interpolation"):
        tio.Affine(degrees=5, one_hot_label_interpolation="label")


def test_entry_points_refuse_bad_arguments_without_touching_the_gpu():
    lib = _native.lib()
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    sp = (ctypes.c_float * 3)(1, 1, 1)
    before = lib.tio_launch_count()
    refusals = [
        (("tio_bspline_prefilter", None, 0, p, None, 1, 1, 2, 2, 2, 3, None), "null"),
        (("tio_bspline_prefilter", p, 0, p + 64, None, 1, 1, 2, 2, 2, 1, None), "order"),
        (("tio_bspline_prefilter", p, 0, p + 64, None, 1, 1, 2, 2, 2, 8, None), "order"),
        (("tio_bspline_prefilter", p, 1, p, None, 1, 1, 2, 2, 2, 3, None), "alias"),
        (("tio_bspline_prefilter", p, 0, p + 4, None, 1, 1, 2, 2, 2, 3, None), "overlaps"),
        (("tio_bspline_resample", p, p + 64, p, 0, 1, 1, 2, 2, 2, 2, 2, 2, p + 128, None, None, 0, 0, 0,
          ctypes.addressof(sp), ctypes.addressof(sp), 1, 3, None), "alias coeff"),
        (("tio_bspline_resample", p, p + 64, p + 80, 0, 1, 1, 2, 2, 2, 2, 2, 2, p + 1024, None, None, 0, 0, 0,
          ctypes.addressof(sp), ctypes.addressof(sp), 1, 3, None), "alias src"),
        (("tio_bspline_resample", p, p + 64, p + 512, 0, 1, 1, 2, 2, 2, 2, 2, 2, p + 1024, None, None, 0, 0, 0,
          ctypes.addressof(sp), ctypes.addressof(sp), 1, 9, None), "order"),
        (("tio_bspline_resample", p, p + 64, p + 512, 0, 1, 1, 2, 2, 2, 2, 2, 2, None, None, None, 0, 0, 0,
          ctypes.addressof(sp), ctypes.addressof(sp), 1, 3, None), "null"),
    ]
    for args, message in refusals:
        with pytest.raises(RuntimeError, match=message):
            _native.call(*args)
    assert lib.tio_launch_count() == before
