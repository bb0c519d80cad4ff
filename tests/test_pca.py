"""PCA against the reference on CPU: the host algebra, fed float64 products G W and the sketch R drawn
from the CPU generator as the reference draws it, reproduces every fixture of
tests/golden/generate_pca.py up to each component's sign; params, history, ``repr``, ``to_hydra``,
errors and the generator's state after the call are the reference's; the C entry points check their
arguments before any launch."""

from __future__ import annotations

import ctypes
import json

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import _native
from torchio_b200.transforms.pca import fix_signs, lowrank_tall, lowrank_wide, projection

import pca_cases as pc

CASES = pc.CASES
ERROR_CASES = sorted(n for n in CASES if "error" in n or n == "pca_nan")
OK_CASES = sorted(n for n in CASES if n not in ERROR_CASES)


def host_pca(data: torch.Tensor, opts: dict) -> np.ndarray:
    """`transforms.pca.pca` with float64 numpy products in place of the GPU passes: the sketch from
    the CPU generator, the fp32-rounded channel means in the projection as `tio_pca_project` uses."""
    b, c = data.shape[:2]
    n = int(np.prod(data.shape[2:]))
    q = opts["q"]
    tall = n >= c
    r = torch.stack([torch.randn(c if tall else n, q, dtype=torch.float32) for _ in range(b)]).double().numpy()
    a = pc.centred(data)
    gram = pc.gram_of(a)
    s, v = lowrank_tall(r, gram) if tall else lowrank_wide(a, r)
    v = fix_signs(v)
    energy = np.einsum("bc,bc->b", v[:, :, 0], gram(v[:, :, :1])[:, :, 0])
    coef, offset = projection(s, v, energy, n, whiten=opts["whiten"], normalize=opts["normalize"],
                              values_range=opts["values_range"])
    x = data.float().reshape(b, c, -1).transpose(1, 2).numpy()
    mean32 = np.float32(x.astype(np.float64).mean(axis=1, keepdims=True))
    y = np.einsum("bnc,bcq->bqn", (x - mean32).astype(np.float64), coef) + offset
    if opts["clip"]:
        y = np.where(np.isnan(y), y, np.clip(y, 0.0, 1.0))
    return y.reshape(b, q, *data.shape[2:])


@pytest.mark.parametrize("name", [n for n in OK_CASES if not CASES[n].get("compose")])
def test_host_algebra_reproduces_the_fixture(name):
    case, fx = CASES[name], pc.load_fixture(name)
    opts = pc.options(case)
    inputs = pc.images(case)
    torch.manual_seed(pc.seed(case))
    gate = torch.rand(1).item()  # Transform.forward draws it even when p == 1
    if gate >= case["kwargs"].get("p", 1.0):
        assert fx["history"] == []
        for key, x in inputs.items():
            assert np.array_equal(fx[f"out_{key}"], pc.as_stored(x))
    else:
        for key in pc.transformed_names(case):
            got = host_pca(inputs[key], opts)
            assert fx["dtype"][key] == "torch.float32"
            err = pc.sign_errors(got, fx[f"out_{key}"], opts["values_range"], opts["clip"],
                                 shift="offset" in case)
            assert err.max() <= 1e-5, f"{key}: largest error {err.max():.3g} per component {err.max(axis=0)}"
        for key in set(inputs) - set(pc.transformed_names(case)):
            assert np.array_equal(fx[f"out_{key}"], pc.as_stored(inputs[key]))
    np.testing.assert_array_equal(torch.rand(4).numpy(), np.float32(fx["rng_after"]))


def test_offset_moves_each_component_by_a_constant_only():
    # the reference's fp32 channel mean of values near 10^4 is off by a few ulps (about 5e-4 each),
    # which shifts each unclipped component by a constant; everything else agrees to 1e-5
    case, fx = CASES["pca_offset"], pc.load_fixture("pca_offset")
    torch.manual_seed(pc.seed(case))
    torch.rand(1)
    got = host_pca(pc.images(case)["t1"], pc.options(case))
    plain = pc.sign_errors(got, fx["out_t1"], (-2.3, 2.3), False)
    assert plain.max() <= 2e-3


@pytest.mark.parametrize("name", ERROR_CASES)
def test_errors_equal_the_fixtures(name):
    case, fx = CASES[name], pc.load_fixture(name)
    want = fx["error"]
    if name == "pca_error_components":
        with pytest.raises(ValueError) as info:
            tio.PCA(**case["kwargs"])
        assert str(info.value) == want["message"]
        return
    data = pc.images(case)["t1"]
    if name == "pca_nan":  # the products of the NaN element are not finite
        a = pc.centred(data)
        r = np.random.default_rng(0).standard_normal((a.shape[0], a.shape[2], 3))
        assert want["type"] == "_LinAlgError"
        with pytest.raises(torch.linalg.LinAlgError) as info:
            lowrank_tall(r, pc.gram_of(a))
        assert str(info.value) == want["message"]
        return
    # the shape checks come before any device work
    assert want["type"] == "ValueError"
    transform = tio.PCA(**case["kwargs"])
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(data[0]))])
    with pytest.raises(ValueError) as info:
        transform.apply_transform(batch, {})
    assert str(info.value) == want["message"]


@pytest.mark.parametrize("name", sorted(n for n in CASES if n != "pca_error_components"))
def test_repr_and_hydra_equal_the_fixtures(name):
    fx = pc.load_fixture(name)
    transform = tio.PCA(**CASES[name]["kwargs"])
    assert repr(transform) == json.loads(json.dumps(fx["repr"]))
    assert json.loads(json.dumps(transform.to_hydra())) == fx["hydra"]


def test_history_and_flags():
    for name in OK_CASES:
        fx = pc.load_fixture(name)
        names = [h["name"] for h in fx["history"]]
        assert all(h["params"] == {} for h in fx["history"] if h["name"] == "PCA")
        assert names in ([], ["PCA"], ["Normalize", "PCA"]), name
    transform = tio.PCA()
    batch = tio.SubjectsBatch.from_subjects([tio.Subject(t1=tio.ScalarImage(torch.zeros(3, 2, 2, 2)))])
    assert transform.make_params(batch) == {}
    assert not transform.supports_chunks(batch)
    assert not transform.supports_per_instance_params and not transform.supports_per_instance_p
    assert not transform.invertible
    with pytest.warns(UserWarning, match="PCA is not invertible, skipping"):
        inverse = tio.get_inverse_transform([tio.AppliedTransform(name="PCA", params={})])
    assert len(inverse) == 0
    assert tio.transforms.PCA is tio.PCA


def test_orthonormalisation_is_the_qr_of_the_tall_matrix():
    rng = np.random.default_rng(5)
    a = rng.standard_normal((1, 300, 7)) * np.linspace(3, 1, 7)
    a -= a.mean(axis=1, keepdims=True)
    r = rng.standard_normal((1, 7, 3))
    s, v = lowrank_tall(r, pc.gram_of(a))
    # the same steps on the tall matrices
    basis = np.linalg.qr(a[0] @ r[0])[0]
    for _ in range(2):
        basis = np.linalg.qr(a[0].T @ basis)[0]
        basis = np.linalg.qr(a[0] @ basis)[0]
    _, s_ref, vh_ref = np.linalg.svd(basis.T @ a[0], full_matrices=False)
    np.testing.assert_allclose(s[0], s_ref, rtol=1e-12)
    np.testing.assert_allclose(np.abs(v[0]), np.abs(vh_ref.T), atol=1e-10)
    # q = C: the exact spectrum, whatever R
    s_full, v_full = lowrank_tall(rng.standard_normal((1, 7, 7)), pc.gram_of(a))
    np.testing.assert_allclose(s_full[0], np.linalg.svd(a[0], compute_uv=False), rtol=1e-10)
    flipped = fix_signs(-v_full)
    np.testing.assert_allclose(flipped, fix_signs(v_full))
    lead = np.take_along_axis(flipped, np.abs(flipped).argmax(axis=1)[:, None, :], axis=1)
    assert (lead > 0).all()


def test_sign_ties_go_to_the_lowest_channel():
    v = np.array([[[0.5, -0.5], [-0.5, 0.5], [0.5, 0.5], [-0.5, -0.5]]])
    out = fix_signs(v)
    assert np.array_equal(out[0, :, 0], v[0, :, 0])
    assert np.array_equal(out[0, :, 1], -v[0, :, 1])


def test_entry_points_reject_bad_arguments_without_touching_a_gpu():
    buf = ctypes.create_string_buffer(1 << 16)
    p = ctypes.addressof(buf)
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_pca_mean", None, 0, 1, 4, 512, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_pca_mean", p, 0, 1, 0, 512, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="unknown dtype 9"):
        _native.call("tio_pca_mean", p, 9, 1, 4, 512, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="at most 65535"):
        _native.call("tio_pca_gram_apply", p, 0, 65536, 4, 512, 3, p, p, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_pca_gram_apply", p, 0, 1, 4, 512, 3, p, None, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="0 columns, 1 to 6144"):
        _native.call("tio_pca_gram_apply", p, 0, 1, 4, 512, 0, p, p, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="6145 columns"):
        _native.call("tio_pca_gram_apply", p, 0, 1, 8000, 512, 6145, p, p, p, p, 1 << 20, None)
    with pytest.raises(RuntimeError, match="0 components"):
        _native.call("tio_pca_project", p, 0, 1, 4, 512, 0, p, p, ctypes.c_float(0.0), 1, p, None)
    with pytest.raises(RuntimeError, match="null pointer"):
        _native.call("tio_pca_project", p, 0, 1, 4, 512, 3, p, None, ctypes.c_float(0.0), 1, p, None)
    with pytest.raises(RuntimeError, match="bad shape"):
        _native.call("tio_pca_project", p, 0, 1, 4, -1, 3, p, p, ctypes.c_float(0.0), 1, p, None)
