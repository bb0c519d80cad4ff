"""KeepLargestComponent: the op sequence and the C oracle's labeller against the reference's fixtures
and scipy (CPU), and the union-find kernels bit for bit against the fixtures, the reference's op
sequence on the same CUDA tensors and the C oracle's component roots (GPU)."""

from __future__ import annotations

import ctypes
import hashlib
import json
import warnings

import numpy as np
import pytest
import torch

import keep_largest_cases as ref
from keep_largest_cases import CASES_BY_NAME, affines, label_map, load_fixture, scalar_image

CASE_NAMES = list(CASES_BY_NAME)
DTYPES = [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float32]
LABELLERS = {"scipy": ref.scipy_labeller, "c": ref.c_labeller}
_ERRORS = {"RuntimeError": RuntimeError, "ValueError": ValueError, "OverflowError": OverflowError}


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


def _raises(error):
    return pytest.raises(_ERRORS[error["type"]], match=f"^{error['message']}$")


# ---- CPU ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("labeller", list(LABELLERS))
@pytest.mark.parametrize("name", CASE_NAMES)
def test_op_sequence_regenerates_the_fixture(name, labeller):
    """The restated op sequence with either labeller is the reference: output, history, errors."""
    if labeller == "scipy":
        pytest.importorskip("scipy")
    case = CASES_BY_NAME[name]
    fixture = load_fixture(name)
    if "error" in fixture:
        with _raises(fixture["error"]):
            ref.reference_output(case, label_map(case), LABELLERS[labeller])
        return
    if not fixture["history"]:  # the p < 1 coin came up tails: untouched
        assert _same(fixture["out_seg"], label_map(case))
    else:
        out, history = ref.reference_output(case, label_map(case), LABELLERS[labeller])
        assert _same(out, fixture["out_seg"])
        assert json.dumps(history) == json.dumps(fixture["history"])
    assert _same(fixture["out_t1"], scalar_image(case))  # ScalarImages are untouched


@pytest.mark.parametrize("name", CASE_NAMES)
def test_params_match_the_reference(name):
    """make_params on the host batch, alone and as a child of the case's Compose plan."""
    import torchio_b200 as tio

    case = CASES_BY_NAME[name]
    fixture = load_fixture(name)
    if "error" in fixture or not fixture["history"]:
        return
    data = label_map(case)
    records = []
    for child_name, kwargs in case["transforms"]:
        child = getattr(tio, child_name)(**kwargs)
        params = child.make_params(_batch(case, labels=data))
        records.append({"name": child_name, "params": params})
        data, _ = ref.reference_output(dict(case, transforms=[(child_name, kwargs)]), data, ref.c_labeller)
    assert json.dumps(records) == json.dumps(fixture["history"])


def test_constructor_repr_and_hydra_match_the_reference():
    import torchio_b200 as tio
    from torchio_b200.transforms.base import _TRANSFORM_REGISTRY

    assert repr(tio.KeepLargestComponent()) == "KeepLargestComponent()"
    t = tio.KeepLargestComponent(labels=(3,), background_label=-1, fully_connected=False, p=0.5)
    assert repr(t) == "KeepLargestComponent(labels=[3], background_label=-1, fully_connected=False, p=0.5)"
    assert t.to_hydra() == {"_target_": "torchio.KeepLargestComponent", "labels": [3], "background_label": -1,
                            "fully_connected": False, "p": 0.5}
    assert tio.KeepLargestComponent(labels=[1, 2]).to_hydra() == {"_target_": "torchio.KeepLargestComponent",
                                                                  "labels": [1, 2]}
    with pytest.raises(TypeError):
        tio.KeepLargestComponent([1], 0)  # background_label is keyword-only
    assert not t.invertible and "KeepLargestComponent" in _TRANSFORM_REGISTRY
    assert t.make_params(None) == {} and t.supports_chunks(None)
    assert tio.transforms.KeepLargestComponent is tio.KeepLargestComponent


def test_entry_points_refuse_bad_arguments_without_touching_the_gpu():
    from torchio_b200 import _native

    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_components", None, 3, 1, 2, 2, 2, 1, None, 0, 0, 1, 1, p, p, p, None)
    with pytest.raises(RuntimeError, match="2\\^32"):
        _native.call("tio_components", p, 3, 1, 2048, 2048, 1024, 1, None, 0, 0, 1, 1, p, p, p, None)
    with pytest.raises(RuntimeError, match="mode"):
        _native.call("tio_components", p, 4, 1, 2, 2, 2, 1, None, 0, 0, 1, 1, p, p, p, None)  # int32 by value
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_components", p, 3, 70000, 2, 2, 2, 1, None, 0, 0, 1, 1, p, p, p, None)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_keep_largest", p, 3, 1, 8, 1, None, 0, 0, 1, p, p, p, None, None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_keep_largest", p, 3, 1, 2**32, 1, None, 0, 0, 1, p, p, p, p, None)
    with pytest.raises(RuntimeError, match="null"):
        _native.call("tio_component_roots", p, 4, 1, 8, None, p, p, None)


def test_ops_refuses_an_oversized_element_before_any_launch():
    from torchio_b200 import ops

    huge = torch.empty(1, dtype=torch.int16).as_strided((1, 1, 2048, 2048, 1024), (0, 0, 0, 0, 0))
    with pytest.raises(ValueError, match="2\\*\\*32"):
        ops.keep_largest(huge, None, 0, True)


def _random_components_map(rng, shape, n_labels, density):
    values = rng.integers(1, n_labels + 1, shape)
    return np.where(rng.random(shape) < density, values, 0)


@pytest.mark.parametrize("fully_connected", [False, True])
def test_oracle_labeller_equals_scipy_on_random_maps(fully_connected):
    """Same partition and roots as scipy.ndimage.label per label, near each connectivity's site
    percolation threshold (0.31 for 6, 0.10 for 26), on flat, odd and one-voxel-thick shapes."""
    pytest.importorskip("scipy")
    from scipy import ndimage

    from oracle import components as cc_oracle

    rng = np.random.default_rng(11 + fully_connected)
    threshold = 0.10 if fully_connected else 0.31
    structure = ndimage.generate_binary_structure(3, 3 if fully_connected else 1)
    shapes = [(1, 1, 40), (40, 1, 1), (1, 37, 1), (9, 8, 1), (13, 11, 7), (16, 16, 16), (5, 31, 9)]
    checked = 0
    for shape in shapes:
        for n_labels in range(1, 6):
            for scale in (0.8, 1.0, 1.25):
                values = _random_components_map(rng, shape, n_labels, min(1.0, threshold * n_labels * scale))
                data = torch.from_numpy(values.astype(np.int16))
                roots = cc_oracle.connected_components(data, data != 0, fully_connected).numpy()
                want = -np.ones(shape, dtype=np.int64)
                for label in range(1, n_labels + 1):
                    labelled, n = ndimage.label(values == label, structure=structure)
                    flat = labelled.reshape(-1)
                    for component in range(1, n + 1):
                        members = np.flatnonzero(flat == component)
                        want.reshape(-1)[members] = members.min()
                assert np.array_equal(roots, want), (shape, n_labels, scale)
                checked += 1
    assert checked == len(shapes) * 15


# ---- GPU ----------------------------------------------------------------------------------------


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_fixture_bit_for_bit_on_the_device(name):
    case = CASES_BY_NAME[name]
    fixture = load_fixture(name)
    batch = _batch(case, device="cuda")
    torch.manual_seed(case["seed"])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        if "error" in fixture:
            with _raises(fixture["error"]):
                _transform(case)(batch)
            return
        out = _transform(case)(batch)
    assert out.images["seg"].data.is_cuda
    assert _same(out.images["seg"].data, fixture["out_seg"])
    assert _same(out.images["t1"].data, fixture["out_t1"])
    assert _history(out) == json.dumps(fixture["history"])


def _odd_map(dtype, batch_size, shape, seed):
    g = torch.Generator().manual_seed(seed)
    coarse = torch.randint(-1 if dtype != torch.uint8 else 0, 5, (batch_size, 1, *((s + 2) // 3 for s in shape)),
                           generator=g)
    data = coarse.repeat_interleave(3, 2).repeat_interleave(3, 3).repeat_interleave(3, 4)
    data = data[:, :, :shape[0], :shape[1], :shape[2]].clone()
    salt = torch.rand(data.shape, generator=g) < 0.15
    data[salt] = torch.randint(0, 5, data.shape, generator=g)[salt]
    data = data.to(dtype)
    if dtype == torch.float32:
        data[:, :, ::4, 1] += 0.5
        data[:, :, 1::5, 2] = -0.0
    return data


@pytest.mark.gpu
@pytest.mark.parametrize("fully_connected", [True, False])
@pytest.mark.parametrize("batch_size", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_equals_the_op_sequence_on_cuda(dtype, batch_size, fully_connected):
    """Explicit labels and labels=None on odd shapes (tile remainders on every axis), and a view at
    storage offset 1, against the reference's op sequence on the same CUDA tensors."""
    import torchio_b200 as tio
    from torchio_b200 import ops

    for shape in ((19, 23, 37), (5, 9, 70)):
        data = _odd_map(dtype, batch_size, shape, seed=batch_size * 10 + len(shape)).cuda()
        aff = [tio.AffineMatrix(np.eye(4))] * batch_size
        for labels, background in ((None, 0), ([1, 3, 300], 0), ([2, 0], -1), (None, 2)):
            transform = tio.KeepLargestComponent(labels=labels, background_label=background,
                                                 fully_connected=fully_connected)
            batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(data.clone(), list(aff), image_class=tio.LabelMap)})
            got = transform(batch).images["seg"].data
            want = ref.keep_largest(data.clone(), labels, background, fully_connected, ref.c_labeller)
            assert _same(got, want), (shape, labels, background)
    flat = data.flatten()
    view = flat[1:1 + batch_size * 7 * 9 * 11].reshape(batch_size, 1, 7, 9, 11)
    got, _ = ops.keep_largest(view.clone(), None, 0, fully_connected)
    assert _same(got, ref.keep_largest(view.clone(), None, 0, fully_connected, ref.c_labeller))
    shifted = view.clone()  # in place on a storage-offset-1 view of a larger tensor
    storage = torch.empty(shifted.numel() + 1, dtype=dtype, device="cuda")
    inplace = storage[1:].view(shifted.shape)
    inplace.copy_(shifted)
    out, _ = ops.keep_largest(inplace, None, 0, fully_connected)
    assert out.data_ptr() == inplace.data_ptr() and _same(inplace, got)


def _adversarial_volumes():
    rng = np.random.default_rng(5)
    vols = {}
    for fully, density in ((True, 0.10), (False, 0.31)):
        for n_labels in (1, 3):
            vols[f"threshold_{int(fully)}_{n_labels}"] = (
                _random_components_map(rng, (41, 35, 67), n_labels, density * n_labels), fully)
    serpentine = ref._serpentine((24, 24, 24)).numpy()
    vols["serpentine"] = (serpentine, False)
    i, j, k = np.meshgrid(*(np.arange(s) for s in (9, 10, 33)), indexing="ij")
    vols["checker_6"] = (1 + (i + j + k) % 2, False)
    vols["checker_26"] = (1 + (i + j + k) % 2, True)
    vols["one_label_everywhere"] = (np.ones((13, 17, 65), dtype=np.int64), True)
    vols["no_label"] = (np.zeros((13, 17, 65), dtype=np.int64), True)
    single = np.zeros((5, 9, 33), dtype=np.int64)
    single[4, 8, 32] = 1
    vols["single_voxel"] = (single, True)
    # components that cross every tile face, edge and corner (tiles are 4 x 8 x 32): diagonal and
    # axis-aligned lines through the tile boundaries
    lines = np.zeros((17, 25, 97), dtype=np.int64)
    for t in range(17):
        lines[t, (t * 3) % 25, (t * 11) % 97] = 2
        lines[t, 7, 31] = 1
        lines[t, 8, 32] = 1
        lines[t, t % 25, 63 + (t % 2)] = 3
    lines[3:5, 7:9, 31:33] = 4  # a 2 x 2 x 2 cube on a tile corner
    vols["tile_crossings_26"] = (lines, True)
    vols["tile_crossings_6"] = (lines, False)
    return vols


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(_adversarial_volumes()))
def test_roots_equal_the_oracle_roots(name):
    """The workspace's roots (labels=None) equal orc_connected_components' on every voxel."""
    from oracle import components as cc_oracle
    from torchio_b200 import ops

    values, fully = _adversarial_volumes()[name]
    for dtype in (torch.int16, torch.int32):
        data = torch.from_numpy(np.ascontiguousarray(values)).to(dtype)
        _, roots = ops.keep_largest(data[None, None].cuda(), None, 0, fully)
        want = cc_oracle.connected_components(data, data != 0, fully)
        got = roots[0].cpu().to(torch.int64) & 0xFFFFFFFF
        got = torch.where(got == 0xFFFFFFFF, torch.full_like(got, -1), got)
        assert torch.equal(got, want), (name, dtype)


@pytest.mark.gpu
def test_two_calls_are_bit_identical():
    from torchio_b200 import ops

    g = torch.Generator().manual_seed(4)
    data = torch.randint(0, 4, (3, 1, 64, 48, 80), generator=g).to(torch.int16).cuda()
    for fully in (True, False):
        a, ra = ops.keep_largest(data.clone(), None, 0, fully)
        b, rb = ops.keep_largest(data.clone(), None, 0, fully)
        assert _same(a, b) and _same(ra, rb)


def _full_int16_batch():
    """32 x 1 x 256^3: ~40 labels on a smooth (8-voxel blocks, shifted per element) map plus 1 % salt."""
    g = torch.Generator(device="cuda").manual_seed(17)
    coarse = torch.randint(0, 40, (32, 1, 33, 33, 33), generator=g, device="cuda", dtype=torch.int16)
    smooth = coarse.repeat_interleave(8, 2).repeat_interleave(8, 3).repeat_interleave(8, 4)
    labels = smooth[:, :, 3:259, 5:261, 1:257].contiguous()
    salt = torch.rand(labels.shape, generator=g, device="cuda") < 0.01
    noise = torch.randint(0, 40, labels.shape, generator=g, device="cuda", dtype=torch.int16)
    labels[salt] = noise[salt]
    return labels


@pytest.mark.gpu
def test_full_size_int16_batch_every_voxel():
    from oracle import components as cc_oracle
    from torchio_b200 import ops

    labels = _full_int16_batch()
    host = labels.cpu()
    fill = torch.zeros(1, dtype=torch.int16)
    for fully in (True, False):
        ours, roots = ops.keep_largest(labels.clone(), None, 0, fully)
        equal = roots_equal = True
        for e in range(host.shape[0]):  # one element at a time: the oracle's int64 roots are 128 MiB each
            want, want_roots = cc_oracle.keep_largest(host[e:e + 1, 0], host[e:e + 1, 0] != 0, fully, fill)
            equal &= _same(ours[e:e + 1, 0], want)
            roots_equal &= torch.equal(roots[e:e + 1].cpu().to(torch.int64), want_roots)
        digest = hashlib.sha256(ours.cpu().numpy().tobytes()).hexdigest()
        removed = int((ours != labels).sum())
        print(f"KeepLargestComponent 32x256^3 int16 fully_connected={fully}: sha256 {digest}, "
              f"{removed} voxels removed, bit-identical={equal}, roots equal={roots_equal}")
        assert equal and roots_equal
        del ours, roots


def _chain_batch(device="cuda"):
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(23)
    labels = torch.randint(0, 6, (3, 1, 32, 28, 24), generator=g).to(torch.int16)
    t1 = torch.rand((3, 1, 32, 28, 24), generator=g)
    if device is not None:
        labels, t1 = labels.to(device), t1.to(device)
    affine = [tio.AffineMatrix(np.diag([1.0, 1.0, 1.2, 1.0])) for _ in range(3)]
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(t1, affine, image_class=tio.ScalarImage),
                              "seg": tio.ImagesBatch(labels, [a.clone() for a in affine], image_class=tio.LabelMap)})


@pytest.mark.gpu
def test_compose_with_affine_remap_and_onehot_equals_one_by_one():
    import torchio_b200 as tio

    def chain():
        return [tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.RemapLabels({1: 2, 5: 0}),
                tio.KeepLargestComponent(fully_connected=False), tio.OneHot()]

    torch.manual_seed(41)
    batch = _chain_batch()
    for transform in chain():
        batch = transform(batch)
    torch.manual_seed(41)
    composed = tio.Compose(chain())(_chain_batch())
    for name in ("t1", "seg"):
        assert _same(composed.images[name].data, batch.images[name].data), name
    assert _history(composed) == _history(batch)


@pytest.mark.gpu
def test_host_batch_comes_back_on_the_host_and_streams_like_the_plain_call():
    import torchio_b200 as tio

    def chain():
        return [tio.RemapLabels({1: 3}), tio.KeepLargestComponent(labels=[3, 2, 4])]

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
    alone = tio.KeepLargestComponent()(_chain_batch(device=None))
    assert alone.images["seg"].data.device.type == "cpu"
    want = ref.keep_largest(_chain_batch(device=None).images["seg"].data.clone(), labeller=ref.c_labeller)
    assert _same(alone.images["seg"].data, want)
