"""Motion against the reference on CPU: the restated op sequence regenerates every fixture of
tests/golden/generate_motion.py bit for bit, a float64 one-axis identity matches them within fp32
rounding, the host affine matrices are the reference's bit for bit, params, RNG use, history,
warnings, repr, to_hydra and errors equal them, and the C entry point checks its arguments before
any launch."""

from __future__ import annotations

import copy
import ctypes
import json
import warnings

import numpy as np
import pytest
import torch

import ghosting_cases as gc
import motion_cases as mc
import torchio_b200 as tio
from oracle import torch_port
from torchio_b200 import _native, ops
from torchio_b200.transforms.motion import motion_theta

CASES = mc.CASES
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
        motion = tio.Motion(**case["kwargs"])
        if not case.get("compose"):
            return motion
        return tio.Compose([motion, tio.Ghosting(**case["ghosting"]), tio.BiasField(**case["bias"])])


def replay(data: torch.Tensor, history) -> torch.Tensor:
    """The fixture's history replayed through the reference's op sequences on ``data`` (any device)."""
    for entry in history:
        if entry["name"] == "Motion":
            data = mc.reference_ops(data, entry["params"])
        elif entry["name"] == "Ghosting":
            data = gc.reference_ops(data, entry["params"])
        else:
            images = {"t1": {"kind": "scalar", "data": data, "affines": [np.eye(4)] * data.shape[0]}}
            torch_port.bias_field(images, copy.deepcopy(entry["params"]))
            data = images["t1"]["data"]
    return data


@pytest.mark.parametrize("name", OK_CASES)
def test_reference_op_sequence_regenerates_the_fixtures_bit_for_bit(name):
    case = CASES[name]
    fx = mc.load_fixture(name)
    torch.set_num_threads(1)
    got = replay(mc.scalar_image(case), fx["history"])
    assert str(got.dtype) == fx["dtype"]
    assert np.array_equal(mc.as_stored(got), fx["out_t1"], equal_nan=True)
    if "seg" in fx:
        assert np.array_equal(fx["out_seg"], mc.label_map(case).numpy())


@pytest.mark.parametrize("name", [n for n in OK_CASES if "compose" not in n])
def test_float64_one_axis_identity_matches_the_fixtures(name):
    case = CASES[name]
    fx = mc.load_fixture(name)
    data = mc.scalar_image(case)
    got = mc.as_float64(fx["out_t1"], case["dtype"])
    if not fx["history"]:
        assert np.array_equal(got, data.double().numpy(), equal_nan=True)
        return
    mc.check_against_oracle(got, data.double().numpy(), fx["history"][0]["params"], case["dtype"])


def test_one_axis_identity_equals_the_reference_steps_in_float64():
    """The splice of whole 3-D spectra equals the one-axis filter sum in float64."""
    rng = np.random.default_rng(5)
    for shape, n in [((20, 14, 11), 3), ((7, 6, 5), 2), ((3, 4, 4), 2), ((12, 1, 9), 1)]:
        x = torch.from_numpy(rng.standard_normal((2, 2, *shape)))
        transforms = [[{"degrees": tuple(rng.uniform(-10, 10, 3)), "translation": tuple(rng.uniform(-3, 3, 3))}
                       for _ in range(n)] for _ in range(2)]
        params = {"transforms": transforms, "_batched_keys": ["transforms"]}
        dims = (-3, -2, -1)
        spectrum = torch.fft.fftn(x, dim=dims)
        for s, theta in enumerate(mc.thetas(transforms, shape), start=1):
            start, end = mc.bounds(s, n + 1, shape[0])
            spectrum[:, :, start:end] = torch.fft.fftn(mc.moved(x, theta.double()), dim=dims)[:, :, start:end]
        steps = torch.fft.ifftn(spectrum, dim=dims).real
        assert float((mc.one_axis(x, params) - steps).abs().max()) <= 1e-12 * float(x.abs().max())


@pytest.mark.parametrize("name", [n for n in OK_CASES if "theta" in mc.load_fixture(n)])
def test_host_affine_matrices_are_the_reference_bit_for_bit(name):
    fx = mc.load_fixture(name)
    entry = next(e for e in fx["history"] if e["name"] == "Motion")
    case = CASES[name]
    got = motion_theta(mc.per_element(entry["params"], case["batch"]), case["shape"])
    want = fx["theta"]  # (N, B, 3, 4) from the reference's _affine_matrices
    assert got.dtype == np.float32
    assert np.array_equal(got.view(np.uint32), want.transpose(1, 0, 2, 3).reshape(got.shape).view(np.uint32))


@pytest.mark.parametrize("name", sorted(CASES))
def test_params_history_and_warnings_equal_the_fixtures_sequentially_and_in_a_compose_plan(name):
    case = CASES[name]
    fx = mc.load_fixture(name)
    data, seg = mc.scalar_image(case), mc.label_map(case)
    if "error" in fx and "hydra" not in fx:  # raised by the constructor
        with pytest.raises(ValueError) as info:
            tio.Motion(**case["kwargs"])
        assert type(info.value).__name__ == fx["error"]["type"] and str(info.value) == fx["error"]["message"]
        return
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        _make(case)
    if "init_warnings" in fx:
        assert [str(w.message) for w in caught] == fx["init_warnings"]
    if "error" in fx:  # raised by the call, after the params were drawn, before any voxel moves
        transform, batch = _make(case), _batch(data, seg)
        torch.manual_seed(mc.seed(case))
        torch.rand(1)
        with pytest.raises(ValueError) as info:
            transform.apply_transform(batch, transform.make_params(batch))
        assert str(info.value) == fx["error"]["message"]
        return
    for planned in (False, True) if not case.get("compose") else (True,):
        batch = _batch(data, seg)
        transform = _make(case)
        torch.manual_seed(mc.seed(case))
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            if planned:
                recorded = _planned_history(transform if case.get("compose") else tio.Compose([transform]), batch)
            else:
                params = None if not transform._per_instance_p_active(batch) and torch.rand(1).item() >= transform.p \
                    else transform.make_params(batch)
                recorded = [] if params is None or (params.get("_keep") is not None and not any(params["_keep"])) \
                    else [{"name": "Motion", "params": _json(params)}]
        assert recorded == fx["history"]
        # the call's own warnings (affine_grid's on a unit-size axis) are checked on the GPU
        assert [str(w.message) for w in caught] == [w for w in fx["warnings"] if "affine_grid" not in w]


def _planned_history(pipeline, batch) -> list[dict]:
    return [{"name": type(child).__name__, "params": _json(params)}
            for _, applied in pipeline._plan(batch) for child, params in applied
            if params.get("_keep") is None or any(params["_keep"])]


@pytest.mark.parametrize("name", sorted(n for n in CASES if "hydra" in mc.load_fixture(n)))
def test_repr_and_hydra_equal_the_fixtures(name):
    fx = mc.load_fixture(name)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = tio.Motion(**CASES[name]["kwargs"])
    assert repr(transform) == fx["repr"]
    assert _json(transform.to_hydra()) == fx["hydra"]


def test_scalar_ranges_draw_nothing_and_ranges_draw_degrees_then_translation_per_segment():
    batch = _batch(torch.zeros(3, 1, 6, 6, 6), None)
    torch.manual_seed(0)
    state = torch.get_rng_state()
    params = tio.Motion(degrees=7, translation=2, num_transforms=3).make_params(batch)
    assert torch.equal(torch.get_rng_state(), state)
    assert params["transforms"] == [[{"degrees": (7.0, 7.0, 7.0), "translation": (2.0, 2.0, 2.0)}] * 3] * 3
    torch.manual_seed(1)
    params = tio.Motion(degrees=(-5, 5), translation=(-1, 1), num_transforms=2, p=0.5).make_params(batch)
    torch.manual_seed(1)
    keep = torch.rand(3) < 0.5
    for e in range(3):
        if not keep[e]:
            assert params["transforms"][e] == []
            continue
        for segment in params["transforms"][e]:
            degrees = tuple(torch.empty(1).uniform_(-5.0, 5.0).item() for _ in range(3))
            translation = tuple(torch.empty(1).uniform_(-1.0, 1.0).item() for _ in range(3))
            assert segment == {"degrees": degrees, "translation": translation}


def test_flags_chunks_and_inverse():
    transform = tio.Motion()
    assert transform.supports_per_instance_params and transform.supports_per_instance_p
    assert transform.supports_chunks(_batch(mc.scalar_image(CASES["motion_b3_f32"]), None))
    assert not transform.invertible
    record = tio.AppliedTransform(name="Motion", params={"transforms": [
        {"degrees": (1.0, 2.0, 3.0), "translation": (0.0, 0.0, 1.0)}]})
    with pytest.warns(UserWarning, match="Motion is not invertible, skipping"):
        inverse = tio.get_inverse_transform([record])
    assert len(inverse) == 0


def test_hand_made_params_are_checked_like_the_reference():
    transform = tio.Motion()
    batch = _batch(torch.zeros(3, 1, 8, 8, 8), None)
    one = [{"degrees": (1.0, 1.0, 1.0), "translation": (0.0, 0.0, 0.0)}]
    with pytest.raises(ValueError, match="Expected 3 motion parameter lists, got 2"):
        transform.apply_transform(batch, {"transforms": [one, one], "_batched_keys": ["transforms"]})
    with pytest.raises(ValueError, match=r"Expected uniform motion transform counts, got \[1, 2\]"):
        transform.apply_transform(batch, {"transforms": [one, one * 2, []], "_batched_keys": ["transforms"]})
    before = batch.images["t1"].data
    transform.apply_transform(batch, {"transforms": [[], [], []], "_batched_keys": ["transforms"]})
    assert batch.images["t1"].data is before  # nothing active: the data itself, as in the reference
    tiny = _batch(torch.zeros(3, 1, 1, 8, 8), None)
    tiny_before = tiny.images["t1"].data
    transform.apply_transform(tiny, {"transforms": [[], [], []], "_batched_keys": ["transforms"]})  # no error
    assert tiny.images["t1"].data is tiny_before


def test_ops_rejects_bad_input_before_touching_a_gpu():
    with pytest.raises(RuntimeError, match="expected a CUDA tensor"):
        ops.motion(torch.zeros(1, 1, 4, 4, 4), np.zeros((1, 1, 12), np.float32), [True])


def test_entry_point_rejects_bad_arguments_without_launching():
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    q = p + (1 << 15)

    def call(src=p, dst=q, dtype=0, B=1, C=1, I=4, J=4, K=4, segments=3, theta=p, active=p, flags=p):
        _native.call("tio_motion", src, dst, dtype, B, C, I, J, K, segments, theta, active, flags, None)

    before = ops.launches()
    for missing in ("src", "dst", "theta", "active", "flags"):
        with pytest.raises(RuntimeError, match="null pointer"):
            call(**{missing: None})
    with pytest.raises(RuntimeError, match="bad shape"):
        call(K=0)
    with pytest.raises(RuntimeError, match="at most 65535"):
        call(B=65536)
    with pytest.raises(RuntimeError, match="unknown dtype 9"):
        call(dtype=9)
    with pytest.raises(RuntimeError, match="first axis of 4097 points, at most 4096"):
        call(I=4097)
    with pytest.raises(RuntimeError, match="5 segments for a first axis of 4 points"):
        call(segments=5)
    with pytest.raises(RuntimeError, match="1 segments"):
        call(segments=1)
    with pytest.raises(RuntimeError, match="in and out overlap"):
        call(dst=p + 16)
    with pytest.raises(RuntimeError, match="in and out overlap"):
        call(dst=p - 8, dtype=5)  # 8-byte elements: 64 bytes from p - 8 cover p
    with pytest.raises(RuntimeError, match="blocks per row"):
        call(I=2, J=1 << 20, K=1 << 16, segments=2, dst=p + (1 << 62))
    assert ops.launches() == before
