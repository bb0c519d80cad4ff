"""Clamp, Mask and Swap against the reference: CPU checks of the fixtures, params, history,
constructors and the C entry points' argument checks; GPU checks, bit for bit, against the
reference's op sequences on the same CUDA tensors and against the fixtures of
tests/golden/generate_intensity_utilities.py."""

from __future__ import annotations

import builtins
import ctypes
import hashlib
import json
import warnings

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import _native, ops
from torchio_b200.transforms.clamp_mask_swap import clamp_bounds, swap_table, where_outside

import intensity_utility_cases as iu

CASES = iu.CASES
OK_CASES = sorted(n for n in CASES if "error" not in n)


def _batch(case, data: torch.Tensor, seg: torch.Tensor | None) -> tio.SubjectsBatch:
    subjects = []
    for b in range(data.shape[0]):
        images = {"t1": tio.ScalarImage(data[b])}
        if seg is not None:
            images["seg"] = tio.LabelMap(seg[b])
        subjects.append(tio.Subject(**images))
    return tio.SubjectsBatch.from_subjects(subjects)


def _transform(case, **overrides):
    return getattr(tio, iu.transform_name(case))(**{**case["kwargs"], **overrides})


def _json(obj):
    return json.loads(json.dumps(obj))


def _same(a, b) -> bool:
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if a.dtype.kind == "f":
        return bool(np.all((a.view(f"u{a.itemsize}") == b.view(f"u{b.itemsize}")) | (np.isnan(a) & np.isnan(b))))
    return bool(np.array_equal(a, b))


def _sampled_params(transform, batch):
    """The gate draw and make_params of Transform._forward_batch, without applying."""
    if not transform._per_instance_p_active(batch) and torch.rand(1).item() >= transform.p:
        return None
    return transform.make_params(batch)


# ---- CPU ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", OK_CASES)
def test_op_sequences_regenerate_the_fixtures(name):
    case = CASES[name]
    fx = iu.load_fixture(name)
    data, seg = iu.scalar_image(case), iu.label_map(case)
    params = fx["history"][0]["params"] if fx["history"] else None
    expected = data if params is None else iu.reference_output(case, data, seg, params)
    assert str(expected.dtype) == fx["dtype"]
    assert _same(iu.as_stored(expected), fx["out_t1"]), name
    if seg is not None:
        assert _same(iu.as_stored(seg), fx["out_seg"])


@pytest.mark.parametrize("name", sorted(n for n in CASES if n != "clamp_error_init"))
def test_params_and_history_equal_the_fixtures_sequentially_and_in_a_compose_plan(name):
    case = CASES[name]
    fx = iu.load_fixture(name)
    data, seg = iu.scalar_image(case), iu.label_map(case)
    for planned in (False, True):
        batch = _batch(case, data, seg)
        transform = _transform(case)
        torch.manual_seed(iu.seed(case))
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            if name == "swap_error_too_large":
                with pytest.raises(ValueError) as info:
                    _sampled_params(transform, batch)
                assert str(info.value) == fx["error"]["message"]
                continue
            if planned:
                applied = tio.Compose([transform])._plan(batch)[0][1]
                params = applied[0][1] if applied else None
            else:
                params = _sampled_params(transform, batch)
        if "history" in fx:
            assert ([] if params is None else [{"name": iu.transform_name(case), "params": _json(params)}]) == fx["history"]
            assert [str(w.message) for w in caught] == fx["warnings"]


@pytest.mark.parametrize("name", [n for n in OK_CASES if not callable(CASES[n]["kwargs"].get("masking_method"))])
def test_repr_and_hydra_equal_the_fixtures(name):
    case = CASES[name]
    fx = iu.load_fixture(name)
    transform = _transform(case)
    assert repr(transform) == fx["repr"]
    assert _json(transform.to_hydra()) == fx["hydra"]


def test_constructor_errors_match_the_reference():
    fx = iu.load_fixture("clamp_error_init")
    with pytest.raises(ValueError) as info:
        tio.Clamp(out_min=5.0, out_max=1.0)
    assert str(info.value) == fx["error"]["message"]
    with pytest.raises(ValueError, match="Value must be non-negative"):
        tio.Swap(num_iterations=(-1, 3))
    assert tio.Swap(patch_size=4).patch_size == (4, 4, 4)


@pytest.mark.parametrize("name", ["clamp_error_none_f32", "clamp_error_u8_max_300", "mask_error_u8_300",
                                  "mask_error_missing_key", "mask_error_not_label_map"])
def test_host_side_errors_equal_the_fixtures(name):
    case = CASES[name]
    fx = iu.load_fixture(name)
    batch = _batch(case, iu.scalar_image(case), iu.label_map(case))
    transform = _transform(case)
    with pytest.raises(getattr(builtins, fx["error"]["type"])) as info:
        if name.startswith("clamp"):
            clamp_bounds(case["dtype"], transform.out_min, transform.out_max)
        elif name == "mask_error_u8_300":
            where_outside(case["dtype"], transform.outside_value)
        else:
            transform._resolve_mask(batch)
    assert str(info.value) == fx["error"]["message"]


def test_mask_refuses_a_masking_method_of_another_type():
    batch = _batch(CASES["mask_key_f32"], iu.scalar_image(CASES["mask_key_f32"]), iu.label_map(CASES["mask_key_f32"]))
    with pytest.raises(TypeError, match="masking_method must be a str or callable, got <class 'int'>"):
        tio.Mask(masking_method=3)._resolve_mask(batch)


def test_bounds_and_outside_values_follow_torch_promotion():
    lo, hi = clamp_bounds(torch.int16, -20.5, None)
    assert lo.dtype == torch.float32 and lo.item() == -20.5 and hi is None
    lo, _ = clamp_bounds(torch.uint8, -1, None)
    assert lo.dtype == torch.uint8 and lo.item() == 255
    _, hi = clamp_bounds(torch.float16, None, 100.3)
    assert hi.dtype == torch.float16 and hi.item() == torch.tensor(100.3).half().item()
    assert where_outside(torch.int16, 0.0).dtype == torch.float32
    assert where_outside(torch.int16, -5).dtype == torch.int16
    assert where_outside(torch.float16, 0.0).dtype == torch.float16


def test_chunk_support():
    batch = _batch(CASES["mask_key_f32"], iu.scalar_image(CASES["mask_key_f32"]), iu.label_map(CASES["mask_key_f32"]))
    assert tio.Clamp(out_min=0).supports_chunks(batch)
    assert tio.Swap().supports_chunks(batch)
    assert not tio.Mask(masking_method="seg").supports_chunks(batch)


def test_swap_table_marks_overlaps_and_pads_with_no_ops():
    rows = [[((0, 0, 0), (5, 5, 5)), ((0, 0, 0), (2, 2, 2))], []]
    table = swap_table(rows, (3, 3, 3))
    assert table.shape == (2, 2, 8) and table.dtype == np.int32
    assert table[0, :, 6].tolist() == [ops.SWAP_EXCHANGE, ops.SWAP_STAGED]
    assert table[0, 0, :6].tolist() == [0, 0, 0, 5, 5, 5]
    assert table[1, :, 6].tolist() == [ops.SWAP_NOOP] * 2


def test_entry_points_reject_bad_arguments_without_touching_a_gpu():
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    value = ctypes.c_float(1.0)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_clamp", None, p, 0, 0, 4, ctypes.addressof(value), None, None)
    with pytest.raises(RuntimeError, match="no bound"):
        _native.call("tio_clamp", p, p, 0, 0, 4, None, None, None)
    with pytest.raises(RuntimeError, match="cannot give"):
        _native.call("tio_clamp", p, p + 64, 0, 3, 4, ctypes.addressof(value), None, None)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_mask", None, 1, 1, None, -1, p, 0, p, 0, 1, 1, 8, ctypes.addressof(value), None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_mask", p, 1, 3, None, -1, p, 0, p, 0, 1, 2, 8, ctypes.addressof(value), None)
    with pytest.raises(RuntimeError, match="in place"):
        _native.call("tio_mask", p, 1, 1, None, -1, p, 0, p + 64, 0, 1, 1, 8, ctypes.addressof(value), None)

    def swap(table, elem=4, patch=(2, 2, 2), dev=p, stage=None):
        table = np.ascontiguousarray(table, dtype=np.int32)
        _native.call("tio_swap_patches", p, elem, 1, 1, 4, 4, 4, *patch, table.ctypes.data, table.shape[0],
                     table.shape[1], dev, stage, None)

    good = np.array([[[0, 0, 0, 2, 2, 2, 0, 0]]])
    with pytest.raises(RuntimeError, match="null"):
        swap(good, dev=None)
    with pytest.raises(RuntimeError, match="element size 3"):
        swap(good, elem=3)
    with pytest.raises(RuntimeError, match="does not fit"):
        swap(good, patch=(5, 2, 2))
    with pytest.raises(RuntimeError, match="patch at 3 on axis 1 does not fit in 4"):
        swap(np.array([[[0, 0, 0, 2, 3, 2, 0, 0]]]))
    with pytest.raises(RuntimeError, match="does not fit"):
        swap(np.array([[[-1, 0, 0, 2, 2, 2, 0, 0]]]))
    with pytest.raises(RuntimeError, match="overlapping pair marked as an exchange"):
        swap(np.array([[[0, 0, 0, 1, 1, 1, 0, 0]]]))
    with pytest.raises(RuntimeError, match="staging buffer"):
        swap(np.array([[[0, 0, 0, 1, 1, 1, 1, 0]]]))
    with pytest.raises(RuntimeError, match="step kind 5"):
        swap(np.array([[[0, 0, 0, 2, 2, 2, 5, 0]]]))


# ---- GPU ----------------------------------------------------------------------------------------

def _run(case, data, seg, **overrides):
    torch.manual_seed(iu.seed(case))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return _transform(case, **overrides)(_batch(case, data, seg))


def _expected(case, data, seg, out):
    history = out.applied_transforms
    if not history:
        return data
    return iu.reference_output(case, data, seg, _json(history[0].params))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_are_reproduced_on_the_device(name):
    case = CASES[name]
    fx = iu.load_fixture(name)
    data, seg = iu.scalar_image(case), iu.label_map(case)
    if "error" in fx:
        with pytest.raises(getattr(builtins, fx["error"]["type"])) as info:
            _run(case, data.cuda(), None if seg is None else seg.cuda())
        assert str(info.value) == fx["error"]["message"]
        return
    out = _run(case, data.cuda(), None if seg is None else seg.cuda())
    got = out.images["t1"].data
    assert str(got.dtype) == fx["dtype"]
    assert [{"name": t.name, "params": _json(t.params)} for t in out.applied_transforms] == fx["history"]
    if seg is not None:
        assert _same(iu.as_stored(out.images["seg"].data), iu.as_stored(seg))
    cuda_ref = _expected(case, data.cuda(), None if seg is None else seg.cuda(), out)
    assert _same(iu.as_stored(got), iu.as_stored(cuda_ref)), name
    if not _same(iu.as_stored(got), fx["out_t1"]):
        a, b = iu.as_stored(got), fx["out_t1"]
        differ = a.view(f"u{a.itemsize}") != b.view(f"u{b.itemsize}")
        print(f"{name}: {int(differ.sum())} voxels differ between the reference on CPU and on CUDA;"
              f" CPU {b[differ][:4].tolist()}, CUDA {a[differ][:4].tolist()}")
        # the only difference allowed: which zero a clamp at a signed zero keeps
        assert name.startswith("clamp_nonfinite") and np.all(a[differ] == 0) and np.all(b[differ] == 0)


def _odd_inputs(dtype, batch, misaligned, seed):
    rng = np.random.default_rng(seed)
    shape = (batch, 1, 37, 29, 23)
    data = iu.random_values(rng, shape, dtype, "nonfinite" if dtype.is_floating_point else "background").cuda()
    seg = torch.as_tensor(rng.integers(0, 4, shape), dtype=torch.int16).cuda()
    if misaligned:
        flat = torch.empty(data.numel() + 1, dtype=dtype, device="cuda")
        flat[1:] = data.reshape(-1)
        data = flat[1:].view(shape)
        assert data.storage_offset() == 1
    return data, seg


@pytest.mark.gpu
@pytest.mark.parametrize("misaligned", [False, True], ids=["aligned", "offset1"])
@pytest.mark.parametrize("per_instance", [True, False], ids=["per_instance", "shared"])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("dtype", iu.DTYPES, ids=iu.SHORT.get)
@pytest.mark.parametrize("kind", ["Clamp", "Mask", "Swap"])
def test_every_dtype_equals_the_op_sequence_on_an_odd_shape(kind, dtype, batch, per_instance, misaligned):
    data, seg = _odd_inputs(dtype, batch, misaligned, seed=7 + batch)
    kwargs = {"Clamp": dict(out_min=10, out_max=100.5), "Mask": dict(masking_method="seg", labels=[1, 2]),
              "Swap": dict(patch_size=(7, 5, 3), num_iterations=(20, 40), p=0.7)}[kind]
    case = {"name": f"{kind.lower()}_odd", "kwargs": kwargs}
    torch.manual_seed(batch + 31)
    source = data.clone()
    out = getattr(tio, kind)(per_instance=per_instance, **kwargs)(_batch(case, data, seg))
    got = out.images["t1"].data
    expected = _expected(case, source, seg, out)
    assert got.dtype == expected.dtype and got.device == expected.device
    assert _same(iu.as_stored(got), iu.as_stored(expected))
    assert torch.equal(out.images["seg"].data, seg)
    assert _same(iu.as_stored(data), iu.as_stored(source))  # copy=True: the caller's tensor is untouched


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", iu.DTYPES, ids=iu.SHORT.get)
def test_clamp_edge_values_follow_torch_on_cuda(dtype):
    special = [0.0, -0.0, 1.0, -1.0, 0.1, 100.3, 65504.0, 1e30, -1e30, float("inf"), float("-inf"), float("nan")]
    x = torch.tensor(special * 7, dtype=torch.float64)
    x = (x if dtype.is_floating_point else x.nan_to_num(0.0, 1e3, -1e3).clamp(-100, 100)).to(dtype).cuda()
    x = x.reshape(1, 1, 7, 12, 1)
    bounds = [(0.1, 100.3), (-0.0, None), (0.0, None), (None, -0.0), (10, 100), (-1, None), (float("nan"), 1.0),
              (None, float("nan")), (1e-8, 1e-7)]
    for out_min, out_max in bounds:
        try:
            expected = x.clamp(min=out_min, max=out_max)
        except RuntimeError as exc:
            with pytest.raises(RuntimeError, match=str(exc).split(":")[0]):
                tio.Clamp(out_min=out_min, out_max=out_max)(x[0])
            continue
        got = tio.Clamp(out_min=out_min, out_max=out_max)(x[0])[None]
        assert got.dtype == expected.dtype, (out_min, out_max)
        assert _same(iu.as_stored(got), iu.as_stored(expected)), (dtype, out_min, out_max)


@pytest.mark.gpu
def test_mask_shapes_and_errors_follow_torch():
    case = {"name": "mask_shapes", "kwargs": {}}
    data = torch.randn(2, 2, 6, 5, 4, device="cuda")
    seg = torch.randint(0, 3, (2, 1, 6, 5, 4), dtype=torch.int16, device="cuda")
    batch = _batch(case, data, seg)
    # a callable whose mask broadcasts along a spatial axis
    got = tio.Mask(masking_method=lambda x: x[:1, :1] > 0)(batch).images["t1"].data
    assert torch.equal(got, torch.where((data[0, :1, :1] > 0).expand_as(data), data, 0.0))
    with pytest.raises(RuntimeError) as ours:
        tio.Mask(masking_method=lambda x: torch.ones(3, 6, 5, 4, dtype=torch.bool, device=x.device))(batch)
    with pytest.raises(RuntimeError) as theirs:
        torch.ones(3, 6, 5, 4, dtype=torch.bool, device="cuda").expand_as(data)
    assert str(ours.value) == str(theirs.value)
    with pytest.raises(RuntimeError) as theirs:
        torch.where(seg[0].bool().expand_as(seg), seg.to(torch.uint8), 300)
    with pytest.raises(RuntimeError) as ours:
        tio.Mask(masking_method="seg", outside_value=300)(_batch(case, data.to(torch.uint8), seg))
    assert str(ours.value) == str(theirs.value)


@pytest.mark.gpu
def test_swap_with_1000_iterations_and_a_fully_overlapping_list():
    g = torch.Generator().manual_seed(3)
    data = torch.randn(4, 2, 20, 18, 16, generator=g).cuda()
    case = {"name": "swap_long", "kwargs": dict(patch_size=(5, 4, 3), num_iterations=1000)}
    torch.manual_seed(9)
    out = tio.Swap(**case["kwargs"])(_batch(case, data, None))
    assert torch.equal(out.images["t1"].data, _expected(case, data, None, out))
    locations = [((i % 3, (2 * i) % 3, 0), ((i + 1) % 3, i % 2, 1)) for i in range(300)]
    for per_instance in (False, True):
        params = {"locations": [locations] * 4 if per_instance else locations}
        if per_instance:
            params["_batched_keys"] = ["locations"]
        sub = _batch(case, data.clone(), None)
        tio.Swap(patch_size=(8, 8, 8)).apply_transform(sub, params)
        table = swap_table(params["locations"] if per_instance else [locations], (8, 8, 8))
        assert bool((table[..., 6] == ops.SWAP_STAGED).all())
        assert torch.equal(sub.images["t1"].data, iu.swap_reference(data, params["locations"], (8, 8, 8), per_instance))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.int16], ids=str)
@pytest.mark.parametrize("kind", ["Clamp", "Mask", "Swap"])
def test_full_size_batch_equals_the_op_sequence(kind, dtype):
    g = torch.Generator(device="cuda").manual_seed(11)
    data = (torch.randn(32, 1, 256, 256, 256, generator=g, device="cuda") * 300).to(dtype)
    seg = (torch.rand(1, 1, 256, 256, 256, generator=g, device="cuda") * 2.5).to(torch.int16).expand(32, -1, -1, -1, -1)
    kwargs = {"Clamp": dict(out_min=-50, out_max=200), "Mask": dict(masking_method="seg"), "Swap": dict()}[kind]
    case = {"name": kind.lower(), "kwargs": kwargs}
    torch.manual_seed(5)
    source = data.clone()
    out = getattr(tio, kind)(copy=False, **kwargs)(_batch(case, data, seg))
    got = out.images["t1"].data
    expected = _expected(case, source, seg, out)
    print(kind, dtype, got.dtype, "sha256", hashlib.sha256(got.cpu().numpy().tobytes()).hexdigest())
    assert got.dtype == expected.dtype and torch.equal(got, expected)


@pytest.mark.gpu
def test_compose_equals_the_transforms_one_by_one():
    g = torch.Generator().manual_seed(21)
    data = (torch.randn(3, 1, 24, 22, 20, generator=g) * 100).cuda()
    seg = (torch.rand(3, 1, 24, 22, 20, generator=g) * 3).to(torch.int16).cuda()
    transforms = lambda: [tio.Affine(degrees=10), tio.Clamp(out_min=-150, out_max=150),  # noqa: E731
                          tio.Mask(masking_method="seg", labels=[1, 2]), tio.BiasField(std=0.3),
                          tio.Blur(std=(0.5, 1.5)), tio.Noise(std=(0, 5)), tio.Gamma(log_gamma=(-0.2, 0.2)),
                          tio.Swap(patch_size=5, num_iterations=20)]
    case = {"name": "compose", "kwargs": {}}
    torch.manual_seed(17)
    composed = tio.Compose(transforms())(_batch(case, data, seg))
    torch.manual_seed(17)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        step = _batch(case, data, seg)
        for t in transforms():
            step = t(step)
    assert [t.name for t in composed.applied_transforms] == [t.name for t in step.applied_transforms]
    assert torch.equal(composed.images["t1"].data, step.images["t1"].data)
    assert torch.equal(composed.images["seg"].data, step.images["seg"].data)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["Clamp", "Swap", "Mask"])
def test_host_batches_stay_on_the_host_and_stream_in_slices(kind):
    g = torch.Generator().manual_seed(23)
    data = (torch.randn(7, 1, 16, 15, 14, generator=g) * 100).to(torch.int16)
    seg = (torch.rand(7, 1, 16, 15, 14, generator=g) * 3).to(torch.int16)
    kwargs = {"Clamp": dict(out_min=-20, out_max=40.5), "Mask": dict(masking_method="seg"),
              "Swap": dict(patch_size=4, num_iterations=(5, 15), p=0.6)}[kind]
    case = {"name": kind.lower(), "kwargs": kwargs}
    torch.manual_seed(4)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        plain = getattr(tio, kind)(**kwargs)(_batch(case, data, seg))
        pipeline = tio.Compose([getattr(tio, kind)(**kwargs)])
        pipeline.chunk_size = 3
        torch.manual_seed(4)
        streamed = pipeline(_batch(case, data, seg))
    assert plain.images["t1"].data.device.type == "cpu"
    assert streamed.images["t1"].data.device.type == "cpu"
    assert torch.equal(plain.images["t1"].data, _expected(case, data, seg, plain))
    assert torch.equal(streamed.images["t1"].data, plain.images["t1"].data)
    assert _json([t.params for t in streamed.applied_transforms]) == _json([t.params for t in plain.applied_transforms])
    assert (pipeline._chunk_size(_batch(case, data, seg)) > 0) == (kind != "Mask")
