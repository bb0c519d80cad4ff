"""Ghosting against the reference on CPU: the restated op sequence regenerates every fixture of
tests/golden/generate_ghosting.py bit for bit, a float64 one-axis filter matches them within fp32
rounding, params, history, warnings, repr, to_hydra and errors equal them, the host filter table is
the reference's mask, and the C entry point checks its arguments before any launch."""

from __future__ import annotations

import copy
import ctypes
import json
import warnings

import numpy as np
import pytest
import torch

import ghosting_cases as gc
import spike_cases as sc
import torchio_b200 as tio
from oracle import torch_port
from torchio_b200 import _native, ops
from torchio_b200.transforms.ghosting import ghosting_filter, ghosting_table

CASES = gc.CASES
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


def _make(case):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ghosting = tio.Ghosting(**case["kwargs"])
        if not case.get("compose"):
            return ghosting
        return tio.Compose([tio.Spike(**case["spike"]), ghosting, tio.BiasField(**case["bias"])])


def replay(data: torch.Tensor, history) -> torch.Tensor:
    """The fixture's history replayed through the reference's op sequences on ``data`` (any device)."""
    for entry in history:
        if entry["name"] == "Ghosting":
            data = gc.reference_ops(data, entry["params"])
        elif entry["name"] == "Spike":
            data = sc.reference_ops(data, entry["params"])
        else:
            images = {"t1": {"kind": "scalar", "data": data, "affines": [np.eye(4)] * data.shape[0]}}
            torch_port.bias_field(images, copy.deepcopy(entry["params"]))
            data = images["t1"]["data"]
    return data


@pytest.mark.parametrize("name", OK_CASES)
def test_reference_op_sequence_regenerates_the_fixtures_bit_for_bit(name):
    case = CASES[name]
    fx = gc.load_fixture(name)
    torch.set_num_threads(1)
    got = replay(gc.scalar_image(case), fx["history"])
    assert str(got.dtype) == fx["dtype"]
    assert np.array_equal(gc.as_stored(got), fx["out_t1"], equal_nan=True)
    if "seg" in fx:
        assert np.array_equal(fx["out_seg"], gc.label_map(case).numpy())


@pytest.mark.parametrize("name", [n for n in OK_CASES if "compose" not in n])
def test_float64_one_axis_filter_matches_the_fixtures(name):
    case = CASES[name]
    fx = gc.load_fixture(name)
    data = gc.scalar_image(case)
    got = gc.as_float64(fx["out_t1"], case["dtype"])
    if not fx["history"]:
        assert np.array_equal(got, data.double().numpy(), equal_nan=True)
        return
    gc.check_against_oracle(got, data.double().numpy(), fx["history"][0]["params"], case["dtype"])


def test_one_axis_filter_equals_the_reference_steps_in_float64():
    rng = np.random.default_rng(3)
    for shape, axis, ghosts, restore in [((37, 29, 23), 0, 5, 0.0), ((16, 20, 24), 1, 40, 0.2),
                                         ((8, 8, 33), 2, 3, 1.5), ((1, 8, 8), 0, 2, 0.25)]:
        x = rng.standard_normal((1, 1, *shape))
        params = {"num_ghosts": ghosts, "axis": axis, "intensity": 0.7, "restore": restore}
        n = shape[axis]
        mask = gc.line_mask(n, ghosts, 0.7, restore).double().numpy()
        view = [1, 1, 1, 1, 1]
        view[2 + axis] = n
        dims = (-3, -2, -1)
        steps = np.fft.ifftn(np.fft.ifftshift(np.fft.fftshift(np.fft.fftn(x, axes=dims), axes=dims) * mask.reshape(view),
                                              axes=dims), axes=dims).real
        assert np.abs(gc.one_axis(x, params) - steps).max() <= 1e-12 * np.abs(x).max()


@pytest.mark.parametrize("name", sorted(CASES))
def test_params_history_and_warnings_equal_the_fixtures_sequentially_and_in_a_compose_plan(name):
    case = CASES[name]
    fx = gc.load_fixture(name)
    data, seg = gc.scalar_image(case), gc.label_map(case)
    if "error" in fx:
        with pytest.raises(ValueError) as info:
            tio.Ghosting(**case["kwargs"])
        assert type(info.value).__name__ == fx["error"]["type"] and str(info.value) == fx["error"]["message"]
        return
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        _make(case) if case.get("compose") else tio.Ghosting(**case["kwargs"])
    assert [str(w.message) for w in caught] == fx["init_warnings"]
    for planned in (False, True) if not case.get("compose") else (True,):
        batch = _batch(data, seg)
        transform = _make(case)
        torch.manual_seed(gc.seed(case))
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            if planned:
                recorded = _planned_history(transform if case.get("compose") else tio.Compose([transform]), batch)
            else:
                params = None if not transform._per_instance_p_active(batch) and torch.rand(1).item() >= transform.p \
                    else transform.make_params(batch)
                recorded = [] if params is None or (params.get("_keep") is not None and not any(params["_keep"])) \
                    else [{"name": "Ghosting", "params": _json(params)}]
        assert recorded == fx["history"]
        assert [str(w.message) for w in caught] == fx["warnings"]


def _planned_history(pipeline, batch) -> list[dict]:
    return [{"name": type(child).__name__, "params": _json(params)}
            for _, applied in pipeline._plan(batch) for child, params in applied
            if params.get("_keep") is None or any(params["_keep"])]


@pytest.mark.parametrize("name", OK_CASES)
def test_repr_and_hydra_equal_the_fixtures(name):
    fx = gc.load_fixture(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = tio.Ghosting(**CASES[name]["kwargs"])
    assert repr(transform) == fx["repr"]
    assert _json(transform.to_hydra()) == fx["hydra"]


def test_flags_chunks_and_inverse():
    transform = tio.Ghosting(intensity=(0.5, 1))
    assert transform.supports_per_instance_params and transform.supports_per_instance_p
    batch = _batch(gc.scalar_image(CASES["ghosting_b3_f32"]), None)
    assert transform.supports_chunks(batch)
    assert not transform.invertible
    record = tio.AppliedTransform(name="Ghosting", params={"num_ghosts": 4, "axis": 0, "intensity": 0.5,
                                                           "restore": 0.0})
    with pytest.warns(UserWarning, match="Ghosting is not invertible, skipping"):
        inverse = tio.get_inverse_transform([record])
    assert len(inverse) == 0


@pytest.mark.parametrize("restore", [0.0, 0.1, 0.25, 0.5, 0.99, 1.0, 1.5, 2.5])
def test_filter_table_is_the_reference_mask_bit_for_bit(restore):
    for n in range(1, 301):
        for ghosts in (1, 2, 3, 4, 5, 7, 10, 40, n, n + 1):
            for strength in (0.5, 1.0, 1.3, 0.1234567):
                want = np.fft.ifftshift(gc.line_mask(n, ghosts, strength, restore).numpy())
                got = ghosting_filter(n, ghosts, strength, restore)
                assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
                    (n, ghosts, strength, restore)


def test_table_rows_axes_and_activity():
    table, axis, active = ghosting_table([4, 0, 2, 3], [0, 1, 2, 1], [0.5, 0.8, 0.0, 1.0], 0.0, (8, 6, 5))
    assert table.shape == (4, 8) and table.dtype == np.float32
    assert axis.tolist() == [0, 1, 2, 1] and active.tolist() == [True, False, False, True]
    assert np.array_equal(table[0], ghosting_filter(8, 4, 0.5, 0.0))
    assert np.array_equal(table[3, :6], ghosting_filter(6, 3, 1.0, 0.0)) and not table[3, 6:].any()
    assert not table[1].any() and not table[2].any()
    _, _, active = ghosting_table([4], [5], [0.0], 0.0, (8, 6, 5))  # not active: the axis is not looked at
    assert not active.any()
    with pytest.raises(ValueError, match="not a spatial axis"):
        ghosting_table([4], [3], [0.5], 0.0, (8, 6, 5))


def test_ops_rejects_bad_input_before_touching_a_gpu():
    with pytest.raises(RuntimeError, match="expected a CUDA tensor"):
        ops.ghosting(torch.zeros(1, 1, 4, 4, 4), np.ones((1, 4), np.float32), [0], [True])


def test_entry_point_rejects_bad_arguments_without_touching_a_gpu():
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)

    def call(data=p, dtype=0, B=1, C=1, I=4, J=4, K=4, table=p, n_max=4, axis=p, active=p, axes=1, flags=p):
        _native.call("tio_ghosting", data, dtype, B, C, I, J, K, table, n_max, axis, active, axes, flags, None)

    for missing in ("data", "table", "axis", "active", "flags"):
        with pytest.raises(RuntimeError, match="null pointer"):
            call(**{missing: None})
    with pytest.raises(RuntimeError, match="bad shape"):
        call(J=0)
    with pytest.raises(RuntimeError, match="at most 65535"):
        call(B=65536)
    with pytest.raises(RuntimeError, match="axis outside 0..2"):
        call(axes=0)
    with pytest.raises(RuntimeError, match="axis outside 0..2"):
        call(axes=8)
    with pytest.raises(RuntimeError, match="unknown dtype 9"):
        call(dtype=9)
    with pytest.raises(RuntimeError, match="axis 1 of 4097 points, at most 4096"):
        call(J=4097, n_max=5000, axes=2)
    with pytest.raises(RuntimeError, match="table rows of 4 entries, axis 2 has 5 points"):
        call(K=5, axes=4)
    with pytest.raises(RuntimeError, match="blocks along axis 2"):
        call(I=1 << 20, J=1 << 16, K=4, axes=4)
