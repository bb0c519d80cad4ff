"""Label-map utilities (RemapLabels, RemoveLabels, SequentialLabels, OneHot, Contour and the
inverses): params, history, tables and errors against the reference's fixtures (CPU), and the
kernels bit for bit against the fixtures and the reference's op sequences on the same CUDA tensors
(GPU)."""

from __future__ import annotations

import hashlib
import json
import warnings

import numpy as np
import pytest
import torch

import label_map_cases as ref
from label_map_cases import LABEL_CASES, affines, label_map, load_fixture, scalar_image

CASES = {c["name"]: c for c in LABEL_CASES}
CASE_NAMES = list(CASES)
DTYPES = [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float32]


def _batch(case, labels=None, device=None):
    import torchio_b200 as tio

    seg = label_map(case) if labels is None else labels
    t1 = scalar_image(case)
    if device is not None:
        seg, t1 = seg.to(device), t1.to(device)
    aff = [tio.AffineMatrix(a) for a in affines(case)]
    return tio.SubjectsBatch({"seg": tio.ImagesBatch(seg, aff, image_class=tio.LabelMap),
                              "t1": tio.ImagesBatch(t1, [a.clone() for a in aff], image_class=tio.ScalarImage)})


def _transform(case):
    import torchio_b200 as tio

    children = [getattr(tio, name)(**kwargs) for name, kwargs in case["transforms"]]
    return children[0] if len(children) == 1 else tio.Compose(children)


def _history(batch):
    return json.dumps([{"name": t.name, "params": t.params} for t in batch.applied_transforms])


def _same(a: torch.Tensor, b: torch.Tensor) -> bool:
    """Equal dtype, shape and bits (NaN payloads and the sign of zero included)."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


# ---- CPU ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", CASE_NAMES)
def test_op_sequence_regenerates_the_fixture(name):
    """The restated op sequence is the reference: output, inverse, history and errors."""
    case = CASES[name]
    fixture = load_fixture(name)
    if "error" in fixture:
        with pytest.raises(RuntimeError, match=f"^{fixture['error']['message']}$"):
            ref.reference_output(case, label_map(case))
        return
    if "inv_error" in fixture:
        with pytest.raises(RuntimeError, match=f"^{fixture['inv_error']['message']}$"):
            ref.reference_output(case, label_map(case))
        out = label_map(case)
        for name_, kwargs in case["transforms"]:
            params = {"remapping": kwargs["remapping"]}
            out = ref.apply(name_, kwargs, params, out)
        assert _same(out, fixture["out_seg"])
        return
    out, undone, history = ref.reference_output(case, label_map(case))
    assert _same(out, fixture["out_seg"])
    if "inv_seg" in fixture:
        assert _same(undone, fixture["inv_seg"])
    assert json.dumps([{"name": n, "params": p} for n, p in history]) == json.dumps(fixture["history"])


@pytest.mark.parametrize("name", CASE_NAMES)
def test_params_match_the_reference(name):
    """make_params on the host batch (a Compose: each child on the map its predecessors left)."""
    case = CASES[name]
    fixture = load_fixture(name)
    if "error" in fixture:
        return
    data = label_map(case)
    records = []
    for child_name, kwargs in case["transforms"]:
        import torchio_b200 as tio

        child = getattr(tio, child_name)(**kwargs)
        batch = _batch(case, labels=data)
        params = child.make_params(batch)
        records.append({"name": child_name, "params": params})
        data = ref.apply(child_name, kwargs, params, data)
    assert json.dumps(records) == json.dumps(fixture["history"])


KEYS_AND_VALUES = [0, 1, -1, 2, 7, 127, 128, -128, -129, 200, 255, 256, 257, 300, 4464, 32767, 32768, 70000,
                   -70000, 2**24, 2**24 + 1, 2**31 - 1, 2**31, 2**40, 1.5, -56.5, 2.0, -0.0, 0.0, float("nan"),
                   float("inf"), 1e10]


@pytest.mark.parametrize("dtype", DTYPES)
def test_table_builder_agrees_with_torch_compare_and_assign(dtype):
    """For each (key, value): the table of one pair, applied by plain lookup to every value of a
    probe map, equals ``out[probe == key] = value``, or both raise the same error."""
    from torchio_b200 import tables

    if dtype.is_floating_point:
        probe = torch.tensor([v for v in KEYS_AND_VALUES if not isinstance(v, float) or v == v] + [float("nan")],
                             dtype=torch.float64).to(dtype)
    else:
        info = torch.iinfo(dtype)
        probe = torch.tensor(sorted({max(info.min, min(info.max, int(v))) for v in KEYS_AND_VALUES
                                     if not isinstance(v, float) or abs(v) < 2**62} | {info.min, info.max}),
                             dtype=torch.int64).to(dtype)
    checked = 0
    for key in KEYS_AND_VALUES:
        for value in (3, -1, 300, 70000, 2.7, -0.0):
            try:
                want = ref.remap(probe, {key: value})
            except RuntimeError as exc:
                with pytest.raises(RuntimeError, match=str(exc)):
                    tables.label_lut([(key, value)], dtype, "cpu")
                continue
            keys, values = tables.label_lut([(key, value)], dtype, "cpu")
            got = probe.clone()
            for i, v in enumerate(probe.tolist()):
                hits = [j for j, k in enumerate(keys.tolist()) if k == v]
                if hits:
                    got[i] = torch.from_numpy(values[hits[-1]:hits[-1] + 1])[0]
            assert _same(got, want), (key, value)
            checked += 1
    assert checked > 50


def test_later_pairs_override_earlier_ones_with_the_same_stored_key():
    from torchio_b200 import tables

    keys, values = tables.label_lut([(1, 2), (2, 1), (257, 9)], torch.uint8, "cpu")
    assert keys.tolist() == [1, 2] and values.tolist() == [9, 1]
    keys, values = tables.label_lut([(-0.0, 3), (0, 4), (float("nan"), 5)], torch.float32, "cpu")
    assert keys.tolist() == [0.0] and not np.signbit(keys[0]) and values.tolist() == [4.0]
    keys, values = tables.label_lut([], torch.int16, "cpu")
    assert keys.dtype == np.int64 and values.dtype == np.int16 and keys.size == 0


def test_constructors_repr_hydra_and_inverse_names():
    import torchio_b200 as tio
    from torchio_b200.transforms.base import _TRANSFORM_REGISTRY

    with pytest.raises(TypeError):
        tio.RemoveLabels(3)
    with pytest.raises(TypeError):
        tio.OneHot(5)  # keyword-only, as in the reference
    with pytest.raises(ValueError, match="Probability"):
        tio.Contour(p=2)
    assert repr(tio.RemapLabels({1: 2})) == "RemapLabels(remapping={1: 2})"
    assert repr(tio.RemoveLabels([3], background_label=1)) == "RemoveLabels(labels=[3], background_label=1)"
    assert repr(tio.OneHot()) == "OneHot()" and repr(tio.OneHot(num_classes=4)) == "OneHot(num_classes=4)"
    assert tio.SequentialLabels().to_hydra() == {"_target_": "torchio.SequentialLabels"}
    assert tio.RemoveLabels([3, 4]).to_hydra() == {"_target_": "torchio.RemoveLabels", "labels": [3, 4]}
    assert type(tio.RemapLabels({1: 2, 3: 4}).inverse({"remapping": {1: 2, 3: 4}})).__name__ == "RemapLabels"
    assert tio.RemapLabels({}).inverse({"remapping": {1: 2, 3: 4}}).remapping == {2: 1, 4: 3}
    assert type(tio.SequentialLabels().inverse({"remappings": {}})).__name__ == "_SequentialLabelsInverse"
    assert type(tio.OneHot().inverse({"num_classes": -1})).__name__ == "_OneHotInverse"
    for name in ("RemapLabels", "RemoveLabels", "SequentialLabels", "OneHot", "Contour", "_SequentialLabelsInverse",
                 "_OneHotInverse"):
        assert name in _TRANSFORM_REGISTRY
    assert not tio.RemoveLabels([1]).invertible and not tio.Contour().invertible


def test_onehot_range_errors_are_raised_before_the_one_hot_launch(monkeypatch):
    import torchio_b200 as tio
    from torchio_b200 import ops

    launched = []
    monkeypatch.setattr(ops, "onehot_classes", lambda data, k: launched.append(k) or data)
    case = CASES["label_onehot_auto_i64"]
    for (lo, hi), num_classes, message in [((-1, 3), -1, "non-negative"), ((-1, 3), 9, "non-negative"),
                                           ((0, 3), 3, "smaller than num_classes"),
                                           ((0, 0), 0, "smaller than num_classes")]:
        monkeypatch.setattr(ops, "label_range", lambda data, r=(lo, hi): r)
        with pytest.raises(RuntimeError, match=message):
            tio.OneHot(num_classes=num_classes).apply_transform(_batch(case), {"num_classes": num_classes})
    assert launched == []
    monkeypatch.setattr(ops, "label_range", lambda data: (0, 4))
    tio.OneHot().apply_transform(_batch(case), {"num_classes": -1})
    assert launched == [5]


def test_which_transforms_stream_in_slices():
    import torchio_b200 as tio
    from torchio_b200.transforms.label import _OneHotInverse, _SequentialLabelsInverse

    batch = _batch(CASES["label_remap_swap_i16"])
    assert tio.RemapLabels({1: 2}).supports_chunks(batch)
    assert tio.RemoveLabels([1]).supports_chunks(batch)
    assert tio.Contour().supports_chunks(batch)
    assert tio.OneHot(num_classes=4).supports_chunks(batch)
    assert not tio.OneHot().supports_chunks(batch)
    assert not tio.SequentialLabels().supports_chunks(batch)
    assert _SequentialLabelsInverse(remappings={}).supports_chunks(batch)
    assert _OneHotInverse().supports_chunks(batch)


# ---- GPU ----------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_fixture_bit_for_bit_on_the_device(name):
    case = CASES[name]
    fixture = load_fixture(name)
    batch = _batch(case, device="cuda")
    torch.manual_seed(case["seed"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if "error" in fixture:
            with pytest.raises(RuntimeError, match=f"^{fixture['error']['message']}$"):
                _transform(case)(batch)
            return
        out = _transform(case)(batch)
        assert _same(out.images["seg"].data, fixture["out_seg"])
        assert out.images["seg"].data.is_cuda
        assert _same(out.images["t1"].data, fixture["out_t1"])  # ScalarImages are untouched
        assert _history(out) == json.dumps(fixture["history"])
        if "inv_error" in fixture:
            with pytest.raises(RuntimeError, match=f"^{fixture['inv_error']['message']}$"):
                out.apply_inverse_transform()
        elif "inv_seg" in fixture:
            assert _same(out.apply_inverse_transform().images["seg"].data, fixture["inv_seg"])


def _random_map(dtype, batch_size, channels, shape, seed, low=-3, high=9):
    g = torch.Generator().manual_seed(seed)
    low = 0 if dtype == torch.uint8 else low
    data = torch.randint(low, high, (batch_size, channels, *shape), generator=g)
    data[:, :, 1::5] = data[:, :, 1::5] // 4  # blocks of equal labels for the contour
    data = data.to(dtype)
    if dtype == torch.float32:
        data[:, :, ::4, 1] += 0.5
    return data


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_equals_the_op_sequence_on_cuda(dtype, batch_size):
    """Every transform and inverse on odd-shaped one- and two-channel maps, against the reference's
    op sequence on the same CUDA tensors."""
    import torchio_b200 as tio

    for channels, shape in ((1, (19, 23, 17)), (2, (9, 70, 13))):
        data = _random_map(dtype, batch_size, channels, shape, seed=channels * 10 + batch_size).cuda()
        aff = [tio.AffineMatrix(np.eye(4))] * batch_size

        def run(transform, x=data):
            batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(x.clone(), list(aff), image_class=tio.LabelMap)})
            return transform(batch).images["seg"].data

        remapping = {1: 5, 5: 1, 2: 0, -2: 7, 8: 3, 300: 2}
        assert _same(run(tio.RemapLabels(remapping)), ref.remap(data, remapping))
        assert _same(run(tio.RemoveLabels([0, 3, -3], background_label=4)), ref.remove(data, [0, 3, -3], 4))
        table = ref.sequential_params(data)
        assert _same(run(tio.SequentialLabels()), ref.renumber(data, table))
        assert _same(run(tio.Contour()), ref.contour(data))
        classes = (data.abs() if dtype != torch.uint8 else data)
        assert _same(run(tio.OneHot(), classes), ref.one_hot(classes, -1))
        assert _same(run(tio.OneHot(num_classes=12), classes), ref.one_hot(classes, 12))
        encoded = ref.one_hot(classes, -1)
        scores = encoded * torch.rand(encoded.shape, device="cuda")  # ties (zeros) and distinct maxima
        from torchio_b200.transforms.label import _OneHotInverse

        assert _same(run(_OneHotInverse(), scores), ref.one_hot_inverse(scores))
        assert _same(run(_OneHotInverse(), data), ref.one_hot_inverse(data))


@pytest.mark.gpu
def test_onehot_classes_the_dtype_cannot_hold_are_zero_channels():
    import torchio_b200 as tio

    data = torch.tensor([0, 1, 255, 0, 4, 255], dtype=torch.uint8).reshape(1, 1, 1, 2, 3).cuda()
    batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(data, [tio.AffineMatrix(np.eye(4))], image_class=tio.LabelMap)})
    out = tio.OneHot(num_classes=300)(batch).images["seg"].data
    assert _same(out, ref.one_hot(data, 300))
    assert out.shape[1] == 300 and not out[:, 256:].any() and int(out[:, 0].sum()) == 2


@pytest.mark.gpu
def test_channel_argmax_takes_the_first_maximum_and_nan():
    from torchio_b200 import ops

    nan = float("nan")
    rows = [[1, 3, 3, 0], [nan, 5, nan, 1], [2, nan, 9, nan], [-1, -1, -1, -1], [0, -0.0, 0, 1]]
    data = torch.tensor(rows, dtype=torch.float32).T.reshape(1, 4, 5, 1, 1).cuda()
    assert _same(ops.channel_argmax(data), data.argmax(dim=1, keepdim=True).float())
    assert ops.channel_argmax(data).flatten().tolist() == [1, 0, 1, 0, 3]
    # 4 voxels per thread (vox % 4 == 0): ties, NaN and -0 in every dtype
    g = torch.Generator().manual_seed(9)
    for dtype in DTYPES:
        scores = torch.randint(-2, 3, (2, 5, 8, 4, 4), generator=g).to(dtype)
        if dtype == torch.float32:
            scores[:, 2, ::3] = nan
            scores[:, 1, 1::5] = -0.0
        scores = scores.cuda()
        assert _same(ops.channel_argmax(scores), scores.argmax(dim=1, keepdim=True).float()), dtype


@pytest.mark.gpu
def test_lookup_tables_larger_than_shared_memory_and_misaligned_views():
    """A table of 5000 keys is searched in global memory; a map starting 2 bytes past an aligned
    address takes the scalar path; both equal the op sequence."""
    import torchio_b200 as tio
    from torchio_b200 import ops, tables

    g = torch.Generator().manual_seed(3)
    data = torch.randint(-6000, 6000, (2, 1, 21, 22, 23), generator=g).to(torch.int32).cuda()
    remapping = {k: (k * 7) % 6000 for k in range(-5000, 5000, 2)}
    batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(data.clone(), [tio.AffineMatrix(np.eye(4))] * 2,
                                                       image_class=tio.LabelMap)})
    assert _same(tio.RemapLabels(remapping)(batch).images["seg"].data, ref.remap(data, remapping))
    flat = data.to(torch.int16).flatten()
    view = flat[1:1 + 5 * 7 * 9].reshape(1, 1, 5, 7, 9)  # 2 bytes past the allocation
    small = {1: 2, 2: -1, -5: 300}
    keys, values = tables.label_lut(list(small.items()), torch.int16, "cuda")
    got = ops.label_lut(view, keys, values, identity=True)
    assert _same(got, ref.remap(view, small))


def _full_int16_batch():
    labels = torch.empty((32, 1, 256, 256, 256), dtype=torch.int16, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(11)
    coarse = torch.randint(0, 120, (32, 1, 64, 64, 64), generator=g, device="cuda", dtype=torch.int16)
    labels.copy_(coarse.repeat_interleave(4, 2).repeat_interleave(4, 3).repeat_interleave(4, 4))
    return labels


@pytest.mark.gpu
def test_full_size_int16_batch_every_voxel():
    """32 x 1 x 256^3 int16: RemapLabels with 100 entries, SequentialLabels and Contour."""
    import torchio_b200 as tio

    labels = _full_int16_batch()
    aff = [tio.AffineMatrix(np.eye(4))] * 32
    remapping = {k: (k * 37 + 5) % 100 for k in range(100)}
    for name, transform, want in [
            ("RemapLabels", tio.RemapLabels(remapping, copy=False), lambda: ref.remap(labels, remapping)),
            ("SequentialLabels", tio.SequentialLabels(copy=False),
             lambda: ref.renumber(labels, ref.sequential_params(labels))),
            ("Contour", tio.Contour(copy=False), lambda: ref.contour(labels))]:
        batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(labels, list(aff), image_class=tio.LabelMap)})
        ours = transform(batch).images["seg"].data
        expected = want()
        equal = _same(ours, expected)
        digest = hashlib.sha256(ours.cpu().numpy().tobytes()).hexdigest()
        print(f"{name} 32x256^3 int16: sha256 {digest}, bit-identical={equal}")
        assert equal
        del ours, expected


@pytest.mark.gpu
def test_onehot_full_size():
    """4 x 1 x 256^3 with 16 classes (int16 and fp32 maps), and the inverse restores the map."""
    import torchio_b200 as tio

    g = torch.Generator(device="cuda").manual_seed(5)
    for dtype in (torch.int16, torch.float32):
        labels = torch.randint(0, 16, (4, 1, 256, 256, 256), generator=g, device="cuda").to(dtype)
        batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(labels, [tio.AffineMatrix(np.eye(4))] * 4,
                                                           image_class=tio.LabelMap)})
        out = tio.OneHot()(batch)
        ours = out.images["seg"].data
        assert _same(ours, ref.one_hot(labels, -1))
        digest = hashlib.sha256(ours.cpu().numpy().tobytes()).hexdigest()
        print(f"OneHot 4x256^3 {dtype} 16 classes: sha256 {digest}")
        del ours
        assert _same(out.apply_inverse_transform().images["seg"].data, labels.float())


def _chain_batch(device="cuda"):
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(21)
    labels = torch.randint(0, 6, (3, 1, 32, 28, 24), generator=g).to(torch.int16)
    t1 = torch.rand((3, 1, 32, 28, 24), generator=g)
    if device is not None:
        labels, t1 = labels.to(device), t1.to(device)
    affine = [tio.AffineMatrix(np.diag([1.0, 1.0, 1.2, 1.0])) for _ in range(3)]
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(t1, affine, image_class=tio.ScalarImage),
                              "seg": tio.ImagesBatch(labels, [a.clone() for a in affine], image_class=tio.LabelMap)})


@pytest.mark.gpu
def test_compose_with_affine_and_labels_to_image_equals_one_by_one():
    import torchio_b200 as tio

    def chain():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return [tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.LabelsToImage("seg"),
                    tio.RemapLabels({1: 2, 2: 1, 5: 0}), tio.OneHot()]

    torch.manual_seed(31)
    torch.cuda.manual_seed(32)
    batch = _chain_batch()
    for transform in chain():
        batch = transform(batch)
    torch.manual_seed(31)
    torch.cuda.manual_seed(32)
    composed = tio.Compose(chain())(_chain_batch())
    for name in ("t1", "seg", "image_from_labels"):
        assert _same(composed.images[name].data, batch.images[name].data), name
    assert composed.images["seg"].data.shape[1] == 5  # labels 0..5 with 5 merged into 0
    assert _history(composed) == _history(batch)


@pytest.mark.gpu
def test_host_batch_comes_back_on_the_host_and_streams_like_the_plain_call():
    import torchio_b200 as tio

    def chain():
        return [tio.RemapLabels({1: 3, 3: 1}), tio.RemoveLabels([4]), tio.Contour()]

    on_device = tio.Compose(chain())(_chain_batch())
    one_shot = tio.Compose(chain())
    one_shot.chunk_size = 0
    plain = one_shot(_chain_batch(device=None))
    streamed_pipe = tio.Compose(chain())
    streamed_pipe.chunk_size = 1
    assert streamed_pipe._chunk_size(_chain_batch(device=None)) == 1
    streamed = list(streamed_pipe.stream([_chain_batch(device=None), _chain_batch(device=None)]))
    for out in (plain, *streamed):
        for name in ("t1", "seg"):
            assert out.images[name].data.device.type == "cpu"
            assert _same(out.images[name].data, on_device.images[name].data), name
        assert _history(out) == _history(on_device)
    onehot = tio.OneHot(num_classes=8)(_chain_batch(device=None))
    assert onehot.images["seg"].data.device.type == "cpu"
    assert _same(onehot.images["seg"].data, ref.one_hot(_chain_batch(device=None).images["seg"].data, 8))
