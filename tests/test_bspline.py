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


# ---- the float64 references and bounds the GPU tests use ------------------------------------------

def _geometries():
    """(name, out_shape, mat, cp, flags, spacing_in, spacing_out, affine_first, (a_in, a_out, worlds, cps))"""
    from oracle import torch_port as tp

    fx = bc.load_fixture("bspline_affine_o3")
    (step,) = bc.params_of(fx)
    worlds = step["params"]["affine_matrix"]
    rng = np.random.default_rng(4)
    cp = rng.uniform(-2, 2, (2, 5, 6, 4, 3)).astype(np.float32)
    cp[:, :1] = cp[:, -1:] = 0
    a_in = np.diag([1.2, 0.9, 1.0, 1.0])
    a_out = np.diag([2.0, 1.5, 0.8, 1.0])
    a_out[:3, 3] = (0.4, -0.3, 0.2)
    tilt = np.eye(4)
    tilt[:3, :3] = tp.output_to_input_matrix(np.eye(4), np.eye(4), None)[:3, :3].numpy()
    tilt[0, 1] = 0.05
    return [
        ("golden_affine", bc.SHAPE, bc.SHAPE, np.eye(4), np.eye(4), worlds, [None] * len(worlds), True),
        ("elastic_affine_first", (13, 11, 9), (13, 11, 9), a_in, a_in, [tilt, None], list(cp), True),
        ("elastic_affine_last", (13, 11, 9), (13, 11, 9), a_in, a_in, [tilt, None], list(cp), False),
        ("target_space", (13, 11, 9), (7, 8, 12), a_in, a_out, [tilt, None], [None, None], True),
    ]


@pytest.mark.parametrize("geometry", _geometries(), ids=lambda g: g[0])
def test_sampling_coords_equal_torch_port(geometry):
    """The C oracle's coordinate export is the reference's sampling grid, bit for bit."""
    from oracle import c_port, torch_port as tp

    _, in_shape, out_shape, a_in, a_out, worlds, cps, affine_first = geometry
    mat = np.stack([tp.output_to_input_matrix(a_in, a_out, w)[:3].reshape(12).numpy() for w in worlds])
    flags = np.array([2 if c is not None else 0 for c in cps], np.uint8)
    cp = None if all(c is None for c in cps) else np.stack([np.zeros_like(cps[0]) if c is None else c for c in cps])
    q = c_port.sampling_coords(out_shape, mat, cp, flags, tp.spacing_of(a_in), tp.spacing_of(a_out),
                               affine_first=affine_first)
    for b, (w, c) in enumerate(zip(worlds, cps)):
        want = tp.sampling_grid(in_shape, a_in, out_shape, a_out, w, c, affine_first)
        assert torch.equal(q[b].view(torch.int32), want.contiguous().view(torch.int32))


@pytest.mark.parametrize("order", bc.ORDERS)
def test_banded_solve_equals_dense_and_scipy(order):
    rng = np.random.default_rng(order)
    for n in range(1, 201):
        x = rng.standard_normal((n, 2))
        dense = np.linalg.solve(bc.collocation(n, order), x) if n > 1 else x
        assert np.max(np.abs(bc.banded_coefficients(x, order) - dense)) <= 1e-12 * max(1.0, np.abs(dense).max())
    if order <= 5:
        x = rng.standard_normal(51199)
        want = ndimage.spline_filter1d(x, order=order, mode="reflect")
        assert np.max(np.abs(bc.banded_coefficients(x[:, None], order)[:, 0] - want)) <= 1e-10


def _float64_slack(c, E):
    """Float64's own rounding in prefilter64 (its fp32 bound E scaled by 2^-53 / 2^-24, doubled) and
    in the dense solve (well below 2^-44 of the coefficients for these sizes): the truncation term is
    attained on the alternating line, so the comparison needs them."""
    return 2.0**-28 * E + 2.0**-44 * np.max(np.abs(c))


@pytest.mark.parametrize("order", bc.ORDERS)
def test_prefilter64_is_the_collocation_solve_within_its_algorithmic_bound(order):
    """The documented algorithm with the kernel's fp32 poles, gain and horizons, in float64, against
    the dense solve: every n from 2 to 64 (both initial sums for every pole), longer axes, and 3-D."""
    rng = np.random.default_rng(10 + order)
    zs, _ = bc.kernel_poles(order)
    for z in zs:  # the host's logf may differ from the device's by an ulp: far from an integer either way
        assert 1e-3 < float(bc.horizon_quotient(z)) % 1 < 1 - 1e-3
    worst = 0.0
    for n in [*range(2, 65), 100, 200]:
        x = rng.standard_normal((n, 4))
        x[:, 3] = (np.arange(n) % 2) * 2.0 - 1.0  # the alternating line: the largest coefficients
        c, E, A = bc._pass(x, np.zeros_like(x), np.zeros_like(x), order)
        err = np.abs(c - np.linalg.solve(bc.collocation(n, order), x))
        bound = A + _float64_slack(c, E)
        assert np.all(err <= bound), (n, float(np.max(err / bound)))
        worst = max(worst, float(np.max(err / bound)))
    x = rng.standard_normal((2, 9, 70, 13))
    c, E, A = bc.prefilter64(x, order)
    assert np.all(np.abs(c - bc.coefficients(x, order)) <= A + _float64_slack(c, E))
    print(f"[prefilter64 o{order}] max |c64 - collocation| / A = {worst:.3f}")


def _mutation_inputs():
    from oracle import c_port

    i, j, k = np.meshgrid(*(np.arange(n, dtype=np.float64) for n in bc.SHAPE), indexing="ij")
    smooth = np.sin(i / 3) * np.cos(j / 4) + 0.5 * np.sin(k / 2)
    noise = np.random.default_rng(5).standard_normal(bc.SHAPE)
    rng = np.random.default_rng(6)
    c = (np.asarray(bc.SHAPE) - 1) / 2
    a = np.eye(3) + rng.uniform(-0.12, 0.12, (3, 3))
    mat = np.concatenate([a, (c - a @ c + rng.uniform(-1, 1, 3))[:, None]], axis=1).astype(np.float32)
    q = c_port.sampling_coords(bc.SHAPE, mat.reshape(1, 12), None, None, (1, 1, 1), (1, 1, 1),
                               affine_first=True)[0].numpy().reshape(-1, 3)
    return {"smooth": smooth, "noise": noise}, q


@pytest.mark.parametrize("order", bc.ORDERS)
def test_wrong_splines_leave_the_bound(order, monkeypatch):
    """Three deliberately wrong float64 splines each leave the end-to-end bound somewhere, on smooth
    and on noise input: the bounds are tight enough to see a subtly wrong kernel."""
    inputs, q = _mutation_inputs()
    for kind, x in inputs.items():
        x32 = x.astype(np.float32).astype(np.float64)[None]
        value, bound, inside = bc.end_to_end(x32, q, order)
        c = bc.prefilter64(x32, order)[0]
        shape = bc.SHAPE

        def leaves(v):
            return float(np.max(np.abs(v - value)[:, inside] / bound[:, inside]))

        with monkeypatch.context() as m:  # the smallest Cox-de Boor weight dropped
            cdb = bc.cox_de_boor
            m.setattr(bc, "cox_de_boor", lambda g, o: cdb(g, o) * (np.arange(o + 1) != 0))
            dropped = bc.tap_sums(q, order, shape, c)[0]
        with monkeypatch.context() as m:  # the outermost tap folded as dct1 (-1 -> 1, n -> n - 2)
            fold = bc.fold
            m.setattr(bc, "fold", lambda t, n: np.where(t == -1, 1 % n, np.where(t == n, max(n - 2, 0),
                                                                                  fold(t, n))))
            dct1_tap = bc.tap_sums(q, order, shape, c)[0]
        mirrored = bc.tap_sums(q, order, shape, bc.prefilter64(x32, order, mirror="dct1")[0])[0]
        ratios = [leaves(dropped), leaves(dct1_tap), leaves(mirrored)]
        print(f"[mutations o{order} {kind}] largest |wrong - right| / bound: " + ", ".join(f"{r:.3g}" for r in ratios))
        assert min(ratios) > 1, ratios
