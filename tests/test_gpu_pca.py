"""PCA on the GPU: the fixtures of tests/golden/generate_pca.py, the reference's op sequence on the
same CUDA tensors with the same seed, each kernel reduction against float64 torch, bit-stable reruns,
launch counts against a profiler trace, a 4 x 64 x 128^3 batch, and ports of the reference's
tests/test_pca.py."""

from __future__ import annotations

import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import ops

import pca_cases as pc

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
CASES = pc.CASES
ERROR_CASES = sorted(n for n in CASES if "error" in n or n == "pca_nan")
OK_CASES = sorted(n for n in CASES if n not in ERROR_CASES)


def _subjects(inputs: dict[str, torch.Tensor], device="cuda") -> tio.SubjectsBatch:
    b = next(iter(inputs.values())).shape[0]
    return tio.SubjectsBatch.from_subjects(
        [tio.Subject(**{k: tio.ScalarImage(v[e].to(device)) for k, v in inputs.items()}) for e in range(b)])


def _transform(case):
    pca = tio.PCA(**case["kwargs"])
    return tio.Compose([tio.Normalize(), pca]) if case.get("compose") else pca


@pytest.mark.parametrize("name", OK_CASES)
def test_fixture(name):
    """Every fixture whose spectrum has a gap at q (the result does not depend on the sketch) to 1e-5
    up to sign; the CUDA generator draws another sketch than the reference's CPU run did."""
    case, fx = CASES[name], pc.load_fixture(name)
    opts = pc.options(case)
    inputs = pc.images(case)
    reduced = inputs
    if case.get("compose"):  # the spectrum PCA sees is Normalize's output
        reduced = {k: v.data.cpu() for k, v in tio.Normalize()(_subjects(inputs)).images.items()}
    if not all(pc.spectral_gap(reduced[k], opts["q"]) for k in pc.transformed_names(case)):
        pytest.skip(f"{name}: no spectral gap at q = {opts['q']}, the components depend on the sketch")
    torch.manual_seed(pc.seed(case))
    out = _transform(case)(_subjects(inputs))
    assert [t.name for t in out.applied_transforms] == [h["name"] for h in fx["history"]]
    for key, x in inputs.items():
        got = out.images[key].data
        assert fx["dtype"][key] == str(got.dtype)
        if key not in pc.transformed_names(case) or not fx["history"]:
            assert np.array_equal(pc.as_stored(got), fx[f"out_{key}"])
            continue
        err = pc.sign_errors(got.cpu().numpy(), fx[f"out_{key}"], opts["values_range"], opts["clip"],
                             shift="offset" in case)
        assert err.max() <= 1e-5, f"{key}: largest error {err.max():.3g} per component {err.max(axis=0)}"


@pytest.mark.parametrize("name", ERROR_CASES)
def test_fixture_errors(name):
    case, fx = CASES[name], pc.load_fixture(name)
    want = fx["error"]
    exc = torch.linalg.LinAlgError if want["type"] == "_LinAlgError" else ValueError
    with pytest.raises(exc) as info:
        _transform(case)(_subjects(pc.images(case)))
    assert str(info.value) == want["message"]


@pytest.mark.parametrize("name", [n for n in OK_CASES if n != "pca_p05_gated"])
def test_reference_op_sequence_on_cuda(name):
    """Same CUDA tensors, same seed: the reference's op sequence draws the same sketches from the
    CUDA generator, so every component agrees to 1e-4 of the output range up to sign (the offset
    case up to a constant: the reference's fp32 channel means)."""
    case = CASES[name]
    opts = pc.options(case)
    inputs = {k: v.cuda() for k, v in pc.images(case).items()}
    if case.get("compose"):
        torch.manual_seed(pc.seed(case))
        inputs = {k: v.data for k, v in tio.Normalize()(_subjects(inputs)).images.items()}
    for key in pc.transformed_names(case):
        torch.manual_seed(pc.seed(case))
        want = pc.reference_ops(inputs[key], opts["q"], opts["whiten"], opts["normalize"], opts["values_range"],
                                opts["clip"])
        rng_want = torch.cuda.get_rng_state()
        torch.manual_seed(pc.seed(case))
        batch = _subjects({key: inputs[key]})
        got = tio.PCA(**{k: v for k, v in case["kwargs"].items() if k not in ("include", "exclude", "p")})(batch)
        assert torch.equal(torch.cuda.get_rng_state(), rng_want)
        err = pc.sign_errors(got.images[key].data.cpu().numpy(), want.cpu().numpy(), opts["values_range"],
                             opts["clip"], shift="offset" in case)
        assert err.max() <= 1e-4, f"{key}: largest error {err.max():.3g} per component {err.max(axis=0)}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.uint8, torch.int64])
@pytest.mark.parametrize("b,c,q,shape", [(2, 3, 3, (9, 17, 33)), (1, 64, 3, (16, 16, 16)), (2, 300, 7, (5, 6, 7)),
                                         (1, 300, 300, (4, 4, 4)), (1, 5000, 2, (3, 3, 3))])
def test_kernel_reductions_against_float64(b, c, q, shape, dtype):
    """Mean, G W and the projection against float64 torch on the same tensors.  Bounds: the mean
    within 1e-13 of max|x|; G W within 1e-12 of sum_v |d_v| (|d_v|^T |W|) (fp64 sums of at most a
    few thousand terms per partial); the projection within 2e-6 of sum_c |d_c| |coef_ck| (fp32)."""
    gen = torch.Generator().manual_seed(c * 7 + q)
    x = (torch.randn((b, c, *shape), generator=gen) * 40 + 100)
    x = (x.round().clamp(0, 255) if dtype == torch.uint8 else x.round() if not dtype.is_floating_point else x)
    x = x.to(dtype).cuda()
    xf = x.float().double().reshape(b, c, -1)
    workspace = ops.pca_workspace(x, q)
    mean = ops.pca_mean(x, workspace)
    want_mean = xf.mean(dim=2)
    assert (mean - want_mean).abs().max().item() <= 1e-13 * xf.abs().max().item()
    d = xf - mean[:, :, None]
    w = np.random.default_rng(q).standard_normal((b, c, q))
    got = ops.pca_gram_apply(x, mean, w, workspace)
    wt = torch.as_tensor(w, device="cuda")
    want = d @ (d.transpose(1, 2) @ wt)
    bound = d.abs() @ (d.abs().transpose(1, 2) @ wt.abs())
    assert ((got - want).abs() <= 1e-12 * bound).all()
    coef = np.random.default_rng(q + 1).standard_normal((b, c, q)).astype(np.float32)
    y = ops.pca_project(x, mean, coef, 0.25, False)
    d32 = (x.float().reshape(b, c, -1) - mean.float()[:, :, None]).double()
    ct = torch.as_tensor(coef, device="cuda").double()
    want_y = ct.transpose(1, 2) @ d32 + 0.25
    bound_y = ct.abs().transpose(1, 2) @ d32.abs()
    assert ((y.reshape(b, q, -1).double() - want_y).abs() <= 2e-6 * bound_y + 1e-7).all()
    clipped = ops.pca_project(x, mean, coef, 0.25, True)
    assert torch.equal(clipped, y.clamp(0, 1))


def test_reruns_are_bit_identical():
    x = torch.randn(2, 16, 64, 64, 64, device="cuda") * torch.linspace(3, 1, 16, device="cuda")[:, None, None, None]
    outs = []
    for _ in range(2):
        torch.manual_seed(5)
        outs.append(tio.PCA()(_subjects({"t1": x})).images["t1"].data)
    assert torch.equal(outs[0], outs[1])
    w = np.random.default_rng(0).standard_normal((2, 16, 3))
    ws = ops.pca_workspace(x, 3)
    mean = ops.pca_mean(x, ws)
    assert torch.equal(ops.pca_gram_apply(x, mean, w, ws), ops.pca_gram_apply(x, mean, w, ws))
    assert torch.equal(mean, ops.pca_mean(x, ws))


def test_nan_voxel_raises_as_the_reference_on_cpu():
    x = torch.randn(1, 4, 8, 8, 8, device="cuda")
    x[0, 2, 1, 2, 3] = float("nan")
    with pytest.raises(torch.linalg.LinAlgError, match="non-finite"):
        tio.PCA()(_subjects({"t1": x}))


def test_host_batch_draws_from_the_cpu_generator():
    x = pc.images(CASES["pca_flat"])["t1"]
    torch.manual_seed(11)
    torch.rand(1)
    want = pc.reference_ops(x, 3, True, True, (-2.3, 2.3), True)
    torch.manual_seed(11)
    got = tio.PCA()(_subjects({"t1": x}, device="cpu")).images["t1"].data
    assert got.device.type == "cpu"
    err = pc.sign_errors(got.numpy(), want.numpy(), (-2.3, 2.3), True)
    assert err.max() <= 1e-4


# ---- launch counts --------------------------------------------------------------------------------

def _launch_cases():
    x = torch.randn(3, 16, 12, 12, 12, device="cuda")
    wide = torch.randn(2, 16, 2, 2, 2, device="cuda")
    return {
        # mean, three G W passes and G v0 (each after the upload of its W), the coefficients' upload
        # and the projection
        "normalize": (11, lambda: tio.PCA()(_subjects({"t1": x}))),
        "no_normalize": (9, lambda: tio.PCA(normalize=False)(_subjects({"t1": x}))),
        # N < C: mean, the centred values through the projection kernel, the projection (two uploads)
        "wide": (5, lambda: tio.PCA()(_subjects({"t1": wide}))),
    }


def count_launch_cases(out_path: str) -> None:
    out = Path(out_path)
    trace = out.with_suffix(".trace.json")
    results = {}
    for name, (expected, call) in _launch_cases().items():
        call()
        torch.cuda.synchronize()
        before = ops.launches()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        counted = ops.launches() - before
        prof.export_chrome_trace(str(trace))
        events = json.loads(trace.read_text())["traceEvents"]
        kernels = [e["name"] for e in events if e.get("cat") == "kernel" and "tio::" in e.get("name", "")]
        results[name] = [expected, counted, len(kernels), sorted({k.split("<")[0] for k in kernels})]
    out.write_text(json.dumps(results))


def test_launch_count_equals_the_kernels_in_a_trace(tmp_path):
    out = tmp_path / "counts.json"
    code = (f"import sys; sys.path[:0] = {[str(ROOT), str(ROOT / 'tests')]!r}; "
            f"import test_gpu_pca; test_gpu_pca.count_launch_cases({str(out)!r})")
    subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], check=True)
    for name, (expected, counted, traced, kernels) in json.loads(out.read_text()).items():
        assert counted == traced == expected, (name, counted, traced, kernels)


# ---- scale ----------------------------------------------------------------------------------------

def test_4x64x128cubed_against_the_reference_op_sequence():
    gen = torch.Generator(device="cuda").manual_seed(3)
    scores = torch.randn(4, 64, 128 ** 3, device="cuda", generator=gen)
    sig = torch.cat([torch.tensor([8.0, 4.0, 2.0]), torch.full((61,), 0.1)]).cuda()
    u = torch.linalg.qr(torch.randn(4, 64, 64, device="cuda", generator=gen))[0]
    x = ((u * sig) @ scores + 50).reshape(4, 64, 128, 128, 128)
    del scores
    torch.manual_seed(21)
    want = pc.reference_ops(x, 3, True, True, (-2.3, 2.3), True)
    torch.manual_seed(21)
    got = tio.PCA()(_subjects({"t1": x})).images["t1"].data
    err = pc.sign_errors(got.cpu().numpy(), want.cpu().numpy(), (-2.3, 2.3), True)
    assert err.max() <= 1e-4, err


# ---- ports of the reference's tests/test_pca.py ---------------------------------------------------

def test_reduces_channels():
    result = tio.PCA(num_components=3)(tio.Subject(emb=tio.ScalarImage(torch.rand(8, 10, 10, 10).cuda())))
    assert result.emb.data.shape[0] == 3


def test_output_range():
    result = tio.PCA(num_components=3, clip=True)(tio.Subject(emb=tio.ScalarImage(torch.randn(16, 10, 10, 10).cuda())))
    assert result.emb.data.min() >= 0.0
    assert result.emb.data.max() <= 1.0


def test_too_few_channels_raises():
    with pytest.raises(ValueError, match="channels"):
        tio.PCA(num_components=5)(tio.Subject(emb=tio.ScalarImage(torch.rand(2, 10, 10, 10).cuda())))


def test_invalid_num_components_raises():
    with pytest.raises(ValueError, match="num_components"):
        tio.PCA(num_components=0)


def test_no_whitening():
    subject = tio.Subject(emb=tio.ScalarImage(torch.randn(8, 10, 10, 10).cuda()))
    result = tio.PCA(num_components=3, whiten=False, normalize=False)(subject)
    assert result.emb.data.shape[0] == 3
