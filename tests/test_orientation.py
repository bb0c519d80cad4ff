"""Reorient, Transpose, EnsureShapeMultiple, CopyAffine and ToReferenceSpace against the reference:
CPU checks of the fixtures (params, history, affines, repr, to_hydra, errors) and of `tio_permute`'s
argument checks; GPU checks, bit for bit, of every fixture and of `ops.permute` against
torch.flip(...).permute(...).contiguous() on the same CUDA tensors."""

from __future__ import annotations

import builtins
import ctypes
import itertools
import json
import re
import warnings

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import _native, ops
from torchio_b200.data import _axcodes2ornt, _inv_ornt_aff, _io_orientation, _ornt_transform
from torchio_b200.transforms.orientation import ornt_permutation

import orientation_cases as oc

CASES = oc.CASES
OK_CASES = sorted(n for n in CASES if "error" not in n)

PERMS = list(itertools.permutations(range(3)))
DTYPES = [torch.uint8, torch.int8, torch.bool, torch.int16, torch.float16, torch.bfloat16, torch.int32,
          torch.float32, torch.int64, torch.float64]
SHORT = {torch.uint8: "u8", torch.int8: "i8", torch.bool: "bool", torch.int16: "i16", torch.float16: "f16",
         torch.bfloat16: "bf16", torch.int32: "i32", torch.float32: "f32", torch.int64: "i64", torch.float64: "f64"}


def _json(obj):
    return json.loads(json.dumps(obj))


def _history(records):
    return [{"name": t.name, "params": _json(t.params)} for t in records]


def _names_and_params(history):
    return [{"name": r["name"], "params": r["params"]} for r in history]


def _sampled_params(transform, batch):
    if not transform._per_instance_p_active(batch) and torch.rand(1).item() >= transform.p:
        return None
    return transform.make_params(batch)


# ---- CPU ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", OK_CASES)
def test_numpy_oracle_regenerates_the_fixtures(name):
    """Voxels: np.flip then transpose from each recorded ornt; affines: the recorded ones."""
    case = CASES[name]
    fx = oc.load_fixture(name)
    images = oc.inputs(case)
    expected = oc.oracle_output(case, images, fx["history"])
    for key, (data, _) in expected.items():
        assert oc.same(oc.as_stored(data), fx[f"out_{key}"]), (name, key)


@pytest.mark.parametrize("name", sorted(n for n in CASES if CASES[n]["kind"] in ("Reorient", "Transpose", "CopyAffine",
                                                                                "ToReferenceSpace")
                                        and "error" not in n))
def test_params_history_and_affines_equal_the_fixtures_on_the_host(name):
    """Everything but the voxels, computed without a GPU: the sampled params (the gate draw and
    make_params) and the affines the transform writes, bit for bit."""
    case = CASES[name]
    fx = oc.load_fixture(name)
    batch = oc.batch(case, oc.inputs(case))
    transform = oc.transform(case)
    torch.manual_seed(oc.seed(case))
    params = _sampled_params(transform, batch)
    expected_history = _names_and_params(fx["history"])
    got = [] if params is None else [{"name": case["kind"], "params": _json(params)}]
    assert got == expected_history
    if params is None:
        return
    affines = oc.output_affines(case, batch, params)
    for key, matrices in affines.items():
        assert np.array_equal(np.stack(matrices), fx[f"affine_{key}"]), (name, key)


@pytest.mark.parametrize("name", sorted(n for n in OK_CASES if "hydra" in oc.load_fixture(n)))
def test_repr_and_hydra_equal_the_fixtures(name):
    case = CASES[name]
    fx = oc.load_fixture(name)
    transform = oc.transform(case)
    assert repr(transform) == fx["repr"]
    assert _json(transform.to_hydra()) == fx["hydra"]


@pytest.mark.parametrize("name", sorted(n for n in CASES if "error_init" in n))
def test_constructor_errors_equal_the_fixtures(name):
    fx = oc.load_fixture(name)
    with pytest.raises(getattr(builtins, fx["error"]["type"])) as info:
        oc.transform(CASES[name])
    # the message shows a set of letters, whose order depends on the interpreter's string hashing
    got, want = (re.sub(r"\{[^}]*\}", lambda m: str(sorted(m.group(0)[1:-1].split(", "))), text)
                 for text in (str(info.value), fx["error"]["message"]))
    assert got == want


def test_copy_affine_missing_target_equals_the_fixture():
    case = CASES["copy_affine_error_missing"]
    fx = oc.load_fixture("copy_affine_error_missing")
    batch = oc.batch(case, oc.inputs(case))
    with pytest.raises(KeyError) as info:
        oc.transform(case).apply_transform(batch, {})
    assert str(info.value) == fx["error"]["message"]


def test_from_tensor_equals_the_fixture():
    fx = oc.load_fixture("to_reference_space_from_tensor")
    image = tio.ToReferenceSpace.from_tensor(torch.zeros(8, 5, 6, 7), oc.reference_image())
    assert isinstance(image, tio.ScalarImage)
    assert np.array_equal(image.affine.numpy(), fx["affine"])


def test_nibabel_restatement_on_simple_affines():
    assert _io_orientation(np.diag([-2.0, 1, 3, 1])).tolist() == [[0.0, -1.0], [1.0, 1.0], [2.0, 1.0]]
    assert _axcodes2ornt("PSR").tolist() == [[1.0, -1.0], [2.0, 1.0], [0.0, 1.0]]
    ornt = _ornt_transform(_axcodes2ornt("RAS"), _axcodes2ornt("PSR"))
    assert ornt_permutation(ornt) == ((1, 2, 0), 0b010)  # P <- flipped A, S <- S, R <- R
    assert tio.AffineMatrix(np.eye(4)[:, [1, 2, 0, 3]]).orientation == ("A", "S", "R")
    # flipping an axis of length n about the centre moves voxel 0 to n - 1
    aff = _inv_ornt_aff(_axcodes2ornt("LAS"), (5, 6, 7))
    assert aff[0].tolist() == [-1.0, 0.0, 0.0, 4.0]


def test_streaming_is_refused():
    batch = oc.batch(CASES["reorient_lps_b3_f32"], oc.inputs(CASES["reorient_lps_b3_f32"]))
    reference = tio.ScalarImage(torch.zeros(1, 2, 2, 2))
    for transform in (tio.Reorient("LPS"), tio.Transpose(), tio.EnsureShapeMultiple(4), tio.CopyAffine("t1"),
                      tio.ToReferenceSpace(reference)):
        assert not transform.supports_chunks(batch)


def test_tio_permute_rejects_bad_arguments_without_touching_a_gpu():
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)

    def call(src=p, dst=p + 2048, elem=4, shape=(1, 1, 2, 3, 4), perm=(2, 1, 0), flips=0):
        _native.call("tio_permute", src, dst, elem, *shape, *perm, flips, None)

    with pytest.raises(RuntimeError, match="null"):
        call(src=None)
    with pytest.raises(RuntimeError, match="null"):
        call(dst=None)
    with pytest.raises(RuntimeError, match="overlap"):
        call(dst=p)
    with pytest.raises(RuntimeError, match="overlap"):
        call(dst=p + 8)
    with pytest.raises(RuntimeError, match="non-positive shape"):
        call(shape=(1, 1, 0, 3, 4))
    with pytest.raises(RuntimeError, match="non-positive shape"):
        call(shape=(-1, 1, 2, 3, 4))
    with pytest.raises(RuntimeError, match="element size 3"):
        call(elem=3)
    with pytest.raises(RuntimeError, match="not a permutation"):
        call(perm=(0, 0, 1))
    with pytest.raises(RuntimeError, match="not a permutation"):
        call(perm=(0, 1, 3))
    with pytest.raises(RuntimeError, match="not a permutation"):
        call(perm=(-1, 1, 2))
    with pytest.raises(RuntimeError, match="flip_bits 8"):
        call(flips=8)
    with pytest.raises(RuntimeError, match="flip_bits -1"):
        call(flips=-1)
    with pytest.raises(RuntimeError, match="identity permutation"):
        call(perm=(0, 1, 2), flips=1)
    with pytest.raises(RuntimeError, match="too many tiles"):
        call(shape=(1 << 20, 1 << 10, 1 << 10, 1, 1), elem=1, dst=p + (1 << 42), perm=(2, 1, 0))


# ---- GPU ----------------------------------------------------------------------------------------

def _reference_permute(x: torch.Tensor, perm, bits: int) -> torch.Tensor:
    for ax in range(3):
        if bits >> ax & 1:
            x = torch.flip(x, [ax + 2])
    return x.permute(0, 1, *(p + 2 for p in perm)).contiguous()


def _random(shape, dtype, seed=0) -> torch.Tensor:
    g = torch.Generator(device="cuda").manual_seed(seed)
    raw = torch.randint(-(1 << 62), 1 << 62, shape, dtype=torch.int64, device="cuda", generator=g)
    if dtype == torch.bool:
        return raw % 2 == 0
    size = torch.empty((), dtype=dtype).element_size()
    return raw.view(torch.uint8).reshape(*shape, 8)[..., :size].contiguous().view(dtype).reshape(shape)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.uint8) if t.dtype == torch.bool else t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32,
                                                                     8: torch.int64}[t.element_size()])


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(37, 29, 23), (5, 1, 70), (1, 131, 9), (66, 3, 1)],
                         ids=["odd", "j1", "i1", "k1"])
@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES, ids=SHORT.get)
def test_every_permutation_and_flip_equals_flip_then_permute(dtype, batch, shape):
    x = _random((batch, 2, *shape), dtype, seed=batch)
    for perm in PERMS:
        for bits in range(8):
            got = ops.permute(x, perm, bits)
            want = _reference_permute(x, perm, bits)
            assert got.shape == want.shape and got.dtype == want.dtype
            assert torch.equal(_bits(got), _bits(want)), (perm, bits)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.float32, torch.float64], ids=SHORT.get)
def test_tile_aligned_and_large_shapes(dtype):
    x = _random((2, 1, 128, 64, 256), dtype, seed=3)
    for perm in PERMS:
        for bits in (0, 5, 7):
            assert torch.equal(_bits(ops.permute(x, perm, bits)), _bits(_reference_permute(x, perm, bits)))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.float32, torch.int64], ids=SHORT.get)
def test_storage_offset_and_non_contiguous_views(dtype):
    base = _random((2 * 3 * 36 * 20 * 16 + 1,), dtype, seed=5)
    x = base[1:].view(2, 3, 36, 20, 16)
    assert x.storage_offset() == 1
    strided = _random((2, 3, 20, 36, 16), dtype, seed=6).transpose(2, 3)
    assert not strided.is_contiguous()
    for view in (x, strided, x[:, 1:2]):
        for perm in PERMS:
            got = ops.permute(view, perm, 6)
            assert torch.equal(_bits(got), _bits(_reference_permute(view, perm, 6))), perm


@pytest.mark.gpu
def test_identity_permutation():
    x = _random((3, 1, 9, 8, 7), torch.float32)
    assert ops.permute(x, (0, 1, 2), 0) is x
    for bits in range(1, 8):
        assert torch.equal(_bits(ops.permute(x, (0, 1, 2), bits)), _bits(_reference_permute(x, (0, 1, 2), bits)))


@pytest.mark.gpu
def test_uint8_past_two_to_the_31_elements():
    """2³¹ + 2²⁴ elements: every 64-bit offset of both paths (the tile kernel and the row kernel)."""
    shape = (1, 1, 2049, 1024, 1024)
    x = torch.empty(shape, dtype=torch.uint8, device="cuda")
    x.view(-1)[:] = (torch.arange(x.numel(), device="cuda", dtype=torch.int64) % 251).to(torch.uint8)
    for perm, bits in (((2, 1, 0), 5), ((1, 0, 2), 7)):
        got = ops.permute(x, perm, bits)
        want = _reference_permute(x, perm, bits)
        assert torch.equal(got, want), perm
        del got, want
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_fixtures_are_reproduced_on_the_device(name):
    case = CASES[name]
    fx = oc.load_fixture(name)
    if "error" in fx and "error_init" in name:
        return  # constructor errors: checked on the CPU
    images = {k: (v.cuda(), a) for k, (v, a) in oc.inputs(case).items()}
    batch = oc.batch(case, images)
    torch.manual_seed(oc.seed(case))
    if "error" in fx:
        with pytest.raises(getattr(builtins, fx["error"]["type"])) as info:
            oc.transform(case)(batch)
        assert str(info.value) == fx["error"]["message"]
        return
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        images, history = oc.apply(case, batch)
    assert _history(history) == _names_and_params(fx["history"])
    for key, ib in images.items():
        assert oc.same(oc.as_stored(ib[0]), fx[f"out_{key}"]), (name, key)
        assert np.array_equal(np.stack(ib[1]), fx[f"affine_{key}"]), (name, key)


@pytest.mark.gpu
@pytest.mark.parametrize("target", ["LPS", "SPL", "AIR", "ARS", "LAS", "RAS", "PSR", "ILA"])
def test_world_coordinates_are_kept_voxel_by_voxel(target):
    """Independent of the nibabel restatement: new_affine · o == old_affine · s(o) for sampled output
    voxels o, where s(o) is the input voxel whose value landed at o (the input holds its own index)."""
    shape = (1, 1, 13, 10, 7)
    index = torch.arange(int(np.prod(shape)), dtype=torch.int64).reshape(shape)
    old = oc.tilted_affine(0)
    batch = tio.SubjectsBatch({"t1": tio.ImagesBatch(index.cuda(), [tio.AffineMatrix(old)])})
    out = tio.Reorient(target)(batch)
    got = out.images["t1"].data.cpu()
    new = out.images["t1"].affines[0].numpy()
    assert "".join(out.images["t1"].affines[0].orientation) == target
    rng = np.random.default_rng(0)
    for _ in range(200):
        o = [int(rng.integers(0, n)) for n in got.shape[2:]]
        s = np.unravel_index(int(got[0, 0, o[0], o[1], o[2]]), shape[2:])
        world_new = new @ np.array([*o, 1.0])
        world_old = old @ np.array([*s, 1.0])
        assert np.allclose(world_new, world_old, rtol=0, atol=1e-9), (o, s)


@pytest.mark.gpu
@pytest.mark.parametrize("target", ["SPL", "LAS", "ARS", "RAS"])
def test_reorient_there_and_back_and_inverse(target):
    case = CASES["reorient_lps_b3_f32"]
    images = {k: (v.cuda(), a) for k, (v, a) in oc.inputs(case).items()}
    batch = oc.batch(case, images)
    original = {k: (ib.data.clone(), [a.numpy().copy() for a in ib.affines]) for k, ib in batch.images.items()}
    out = tio.Reorient(target)(batch)
    back = tio.Reorient(out.applied_transforms[0].params["original_orientation"])(out)
    inverted = tio.apply_inverse_transform(out)
    for result in (back, inverted):
        for key, (data, affines) in original.items():
            assert torch.equal(_bits(result.images[key].data), _bits(data))
            for got, want in zip(result.images[key].affines, affines, strict=True):
                assert np.allclose(got.numpy(), want, rtol=0, atol=1e-9)


@pytest.mark.gpu
def test_subject_inverse_of_reorient_and_transpose():
    data = torch.rand(1, 11, 9, 6)
    seg = (data * 4).to(torch.int16)
    affine = oc.tilted_affine(0)
    subject = tio.Subject(t1=tio.ScalarImage(data, affine=affine), seg=tio.LabelMap(seg, affine=affine))
    out = tio.Compose([tio.Reorient("SPL"), tio.Transpose()])(subject)
    assert not torch.equal(out["t1"].data, data)
    back = tio.apply_inverse_transform(out)
    assert torch.equal(back["t1"].data, data) and torch.equal(back["seg"].data, seg)
    assert np.allclose(back["t1"].affine.numpy(), affine, rtol=0, atol=1e-9)


@pytest.mark.gpu
def test_compose_on_a_host_batch_equals_sequential_application():
    """Reorient changes the orientation Flip resolves "L" from: the pipeline must not sample Flip on
    the batch as it entered."""
    subjects = [tio.Subject(t1=tio.ScalarImage(torch.rand(1, 12, 10, 8), affine=oc.tilted_affine(b)))
                for b in range(4)]
    batch = tio.SubjectsBatch.from_subjects(subjects)
    torch.manual_seed(1)
    composed = tio.Compose([tio.Reorient("LPS"), tio.Flip(axes="L")])(batch)
    torch.manual_seed(1)
    sequential = tio.Flip(axes="L")(tio.Reorient("LPS")(batch))
    assert not composed.images["t1"].data.is_cuda
    assert torch.equal(composed.images["t1"].data, sequential.images["t1"].data)
    assert _history(composed.applied_transforms) == _history(sequential.applied_transforms)
    # element 0 is LPS now, so "L" is its axis 0 (element 1 had another orientation to begin with)
    assert _history(composed.applied_transforms)[1]["params"]["axes"][0] == [0]


@pytest.mark.gpu
@pytest.mark.parametrize("device", ["cuda", "cpu"])
def test_preprocessing_chain(device):
    subjects = [tio.Subject(t1=tio.ScalarImage(torch.rand(1, 37, 29, 23), affine=oc.tilted_affine(0)),
                            seg=tio.LabelMap((torch.rand(1, 37, 29, 23) * 3).to(torch.int16),
                                             affine=oc.tilted_affine(0)))
                for _ in range(3)]
    batch = tio.SubjectsBatch.from_subjects(subjects).to(device)
    pipeline = tio.Compose([tio.Reorient("RAS"), tio.EnsureShapeMultiple(16), tio.Transpose(), tio.ZNormalization()])
    out = pipeline(batch)
    assert out.images["t1"].data.device.type == device
    assert all(n % 16 == 0 for n in out.images["t1"].data.shape[2:])
    assert [t.name for t in out.applied_transforms] == ["Reorient", "Pad", "EnsureShapeMultiple", "Transpose",
                                                        "Standardize"]
