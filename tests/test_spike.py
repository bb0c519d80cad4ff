"""Spike against the reference on CPU: params, history, warnings, repr, to_hydra and errors equal the
fixtures of tests/golden/generate_spike.py; a float64 oracle of the plane-wave identity regenerates
every fixture's voxels and agrees with a float64 FFT evaluation of the reference's steps; the C
entry points check their arguments before any launch."""

from __future__ import annotations

import ctypes
import json
import warnings

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import _native
from torchio_b200.transforms.spike import spike_frequencies, spike_table

import spike_cases as sc

CASES = sc.CASES
OK_CASES = sorted(n for n in CASES if "error" not in n)


def _batch(data: torch.Tensor, seg: torch.Tensor | None) -> tio.SubjectsBatch:
    subjects = []
    for b in range(data.shape[0]):
        images = {"t1": tio.ScalarImage(data[b])}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b])
        subjects.append(tio.Subject(**images))
    return tio.SubjectsBatch.from_subjects(subjects)


def _json(obj):
    return json.loads(json.dumps(obj))


def _sampled_params(transform, batch):
    """The gate draw and make_params of Transform._forward_batch, without applying."""
    if not transform._per_instance_p_active(batch) and torch.rand(1).item() >= transform.p:
        return None
    return transform.make_params(batch)


@pytest.mark.parametrize("name", OK_CASES)
def test_float64_oracle_regenerates_the_fixtures(name):
    case = CASES[name]
    fx = sc.load_fixture(name)
    data = sc.scalar_image(case)
    assert fx["dtype"] == str(data.dtype)
    got = sc.as_float64(fx["out_t1"], case["dtype"])
    history = fx["history"]
    if not history or "t1" in case["kwargs"].get("exclude", []):
        assert np.array_equal(got, data.double().numpy(), equal_nan=True)
        return
    sc.check_against_oracle(got, data.double().numpy(), history[0]["params"], case["dtype"])
    if "seg" in fx:
        assert np.array_equal(fx["out_seg"], sc.label_map(case).numpy())


@pytest.mark.parametrize("name", [n for n in OK_CASES if "nonfinite" not in n])
def test_closed_form_equals_the_reference_steps_in_float64(name):
    case = CASES[name]
    fx = sc.load_fixture(name)
    if not fx["history"]:
        return
    params = fx["history"][0]["params"]
    x = sc.scalar_image(case).double().numpy()
    want = sc.fft_steps(x, params)
    got, _ = sc.closed_form(x, params)
    assert np.abs(got - want).max() <= 1e-9 * (np.abs(want).max() + 1.0)


def test_sum_is_the_spectrum_peak_of_a_non_negative_volume():
    rng = np.random.default_rng(5)
    for shape in [(7, 6, 5), (16, 9, 11), (1, 8, 13)]:
        x = rng.uniform(0, 100, shape)
        x[rng.random(shape) < 0.5] = 0
        peak = np.abs(np.fft.fftn(x)).max()
        assert abs(peak - x.sum()) <= 1e-12 * x.sum()
        signed = x - 50
        assert np.abs(np.fft.rfftn(signed)).max() == pytest.approx(np.abs(np.fft.fftn(signed)).max(), rel=1e-12)


@pytest.mark.parametrize("name", sorted(CASES))
def test_params_history_and_warnings_equal_the_fixtures_sequentially_and_in_a_compose_plan(name):
    case = CASES[name]
    fx = sc.load_fixture(name)
    data, seg = sc.scalar_image(case), sc.label_map(case)
    if "error" in fx:
        with pytest.raises(ValueError) as info:
            tio.Spike(**case["kwargs"])
        assert type(info.value).__name__ == fx["error"]["type"] and str(info.value) == fx["error"]["message"]
        return
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        tio.Spike(**case["kwargs"])
    assert [str(w.message) for w in caught] == fx["init_warnings"]
    for planned in (False, True):
        batch = _batch(data, seg)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            transform = tio.Spike(**case["kwargs"])
        torch.manual_seed(sc.seed(case))
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            if planned:
                applied = tio.Compose([transform])._plan(batch)[0][1]
                params = applied[0][1] if applied else None
            else:
                params = _sampled_params(transform, batch)
        recorded = [] if params is None or (params.get("_keep") is not None and not any(params["_keep"])) else \
            [{"name": "Spike", "params": _json(params)}]
        assert recorded == fx["history"]
        assert [str(w.message) for w in caught] == fx["warnings"]


@pytest.mark.parametrize("name", OK_CASES)
def test_repr_and_hydra_equal_the_fixtures(name):
    fx = sc.load_fixture(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = tio.Spike(**CASES[name]["kwargs"])
    assert repr(transform) == fx["repr"]
    assert _json(transform.to_hydra()) == fx["hydra"]


def test_flags_chunks_and_inverse():
    transform = tio.Spike(intensity=(1, 3))
    assert transform.supports_per_instance_params and transform.supports_per_instance_p
    batch = _batch(sc.scalar_image(CASES["spike_b3_f32"]), None)
    assert transform.supports_chunks(batch)
    assert not transform.invertible
    record = tio.AppliedTransform(name="Spike", params={"positions": [[0.1, 0.2, 0.3]], "intensity": 2.0})
    with pytest.warns(UserWarning, match="Spike is not invertible, skipping"):
        inverse = tio.get_inverse_transform([record])
    assert len(inverse) == 0


def test_frequencies_and_tables():
    # fftshift index int(p * n) % n, then back by n // 2
    assert spike_frequencies([[0.0, 0.5, 0.99]], (4, 5, 1)) == [(2, 0, 0)]
    assert spike_frequencies([[0.5, 0.6, 0.25]], (4, 5, 8)) == [(0, 1, 6)]
    rows = [[[0.1, 0.2, 0.3], [0.5, 0.5, 0.5]], [], [[0.9, 0.0, 0.4]]]
    table, ratio = spike_table(rows, [2.0, 0.0, 1.5], (10, 10, 10))
    assert table.shape == (3, 2, 4) and table.dtype == np.int32
    assert table[0].tolist() == [[6, 7, 8, 1], [0, 0, 0, 1]]
    assert table[1].tolist() == [[0, 0, 0, 0]] * 2
    assert table[2].tolist() == [[4, 5, 9, 1], [0, 0, 0, 0]]
    assert ratio.tolist() == [2.0, 0.0, 1.5]
    table, ratio = spike_table([[[0.1, 0.2, 0.3]]], [0.0], (10, 10, 10))
    assert not ratio.any() and not table[..., 3].any()


def test_entry_points_reject_bad_arguments_without_touching_a_gpu():
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    ws = _native.lib().tio_spike_stats_workspace_bytes(2)
    assert ws >= 2 * 1024 * 12
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_spike_stats", None, 0, 1, 2, 8, p, p, p, p, ws, None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_spike_stats", p, 0, 0, 2, 8, p, p, p, p, ws, None)
    with pytest.raises(RuntimeError, match="unknown dtype 9"):
        _native.call("tio_spike_stats", p, 9, 1, 2, 8, p, p, p, p, ws, None)
    with pytest.raises(RuntimeError, match="workspace"):
        _native.call("tio_spike_stats", p, 0, 1, 2, 8, p, p, p, p, ws - 1, None)
    with pytest.raises(RuntimeError, match="at most 65535"):
        _native.call("tio_spike_stats", p, 0, 65536, 1, 8, p, p, p, p, 1 << 40, None)
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_spectrum_peak", p, 0, 1, 1, 4, 4, 4, p, None, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="axis of 4097 points, at most 4096"):
        _native.call("tio_spectrum_peak", p, 0, 1, 1, 4, 4097, 4, p, p, p, p, 1 << 40, None)
    with pytest.raises(RuntimeError, match="one row needs 768"):
        _native.call("tio_spectrum_peak", p, 0, 1, 1, 4, 8, 4, p, p, p, p, 767, None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_spectrum_peak", p, 0, 1, 1, 4, 0, 4, p, p, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_spike", p, 0, 1, 1, 4, 4, 4, None, 1, p, p, p, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="1 spikes|-1 spikes|0 spikes"):
        _native.call("tio_spike", p, 0, 1, 1, 4, 4, 4, p, 0, p, p, p, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="tables of 191 bytes, 192 needed"):
        _native.call("tio_spike", p, 0, 2, 1, 4, 4, 4, p, 1, p, p, p, p, p, 191, None)
    with pytest.raises(RuntimeError, match="unknown dtype"):
        _native.call("tio_spike", p, 12, 1, 1, 4, 4, 4, p, 1, p, p, p, p, p, 1 << 20, None)
