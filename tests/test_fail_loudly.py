"""The product never falls back to a CPU path: without a CUDA device (this
container) every entry into the hot path raises, and nothing under oracle/ is
imported by the package."""

import subprocess
import sys
import warnings
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent

cpu_only = pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")


def _batch(b=2):
    import torchio_b200 as tio

    x = torch.rand((b, 1, 8, 8, 8))
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(b)])})


@cpu_only
@pytest.mark.parametrize("make", [
    lambda tio: tio.Affine(degrees=(-5, 5)), lambda tio: tio.ElasticDeformation(),
    lambda tio: tio.BiasField(), lambda tio: tio.Blur(std=(0.5, 1.0)), lambda tio: tio.Noise(std=0.1),
    lambda tio: tio.Gamma(log_gamma=(-0.2, 0.2)), lambda tio: tio.Flip(axes=0), lambda tio: tio.Pad(padding=1),
    lambda tio: tio.Crop(cropping=1), lambda tio: tio.CropOrPad(6),
    lambda tio: tio.Compose([tio.Affine(degrees=(-5, 5)), tio.Gamma(log_gamma=(-0.2, 0.2))]),
    lambda tio: tio.Standardize(), lambda tio: tio.Normalize(),
    lambda tio: tio.Pad(padding=1, padding_mode="median"), lambda tio: tio.Pad(padding=1, padding_mode="minimum"),
    lambda tio: tio.Affine(degrees=(-5, 5), default_pad_value="otsu"),
    lambda tio: tio.Resample(2, antialias=True),
], ids=["Affine", "Elastic", "BiasField", "Blur", "Noise", "Gamma", "Flip", "Pad", "Crop", "CropOrPad", "Compose",
        "Standardize", "Normalize", "PadMedian", "PadMinimum", "AffineOtsu", "ResampleAntialias"])
def test_transforms_raise_without_cuda(make):
    import torchio_b200 as tio

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        transform = make(tio)
        with pytest.raises(RuntimeError, match="CUDA"):
            transform(_batch())


@cpu_only
def test_label_partial_volume_raises_without_cuda():
    import torchio_b200 as tio

    lab = (torch.rand((2, 1, 8, 8, 8)) * 4).to(torch.int16)
    batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(lab, [tio.AffineMatrix() for _ in range(2)],
                                                      image_class=tio.LabelMap)})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for kwargs in ({}, {"antialias": True}):
            with pytest.raises(RuntimeError, match="CUDA"):
                tio.Spatial(degrees=(-5, 5), label_interpolation="label", copy=False, **kwargs)(batch)


def test_stream_validates_depth_before_touching_a_batch():
    import torchio_b200 as tio

    pipe = tio.Compose([], copy=False)
    with pytest.raises(ValueError, match="depth"):
        list(pipe.stream(iter([_batch()]), depth=-1))


@cpu_only
def test_stream_and_submit_raise_without_cuda():
    import torchio_b200 as tio

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipe = tio.Compose([tio.Gamma(log_gamma=(-0.2, 0.2))], copy=False)
        with pytest.raises(RuntimeError, match="CUDA"):
            pipe.submit(_batch())
        with pytest.raises(RuntimeError, match="CUDA"):
            list(pipe.stream(iter([_batch(), _batch()]), depth=1))


@cpu_only
def test_ops_raise_on_host_tensors():
    from torchio_b200 import ops

    x = torch.rand((1, 1, 8, 8, 8))
    with pytest.raises((RuntimeError, ValueError, TypeError)):
        ops.intensity_fused(x, gamma=torch.ones(1))
    with pytest.raises((RuntimeError, ValueError, TypeError)):
        ops.crop_patches(x[0], [[0, 0, 0]], (4, 4, 4))
    lab = (x * 4).to(torch.int16)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.onehot(lab, torch.arange(4))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.label_argmax(torch.rand((1, 4, 8, 8, 8)), torch.arange(4), 0.0, torch.int16)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.remap(x, (8, 8, 8), (0, 0, 0))
    with pytest.raises(RuntimeError, match="CUDA"):
        ops.rescale(x, sub=0.5)


def test_package_never_imports_the_oracle():
    code = ("import sys; import torchio_b200, torchio_b200.ops, torchio_b200.patches, "
            "torchio_b200.transforms.neighbours; "
            "bad = [m for m in sys.modules if m == 'oracle' or m.startswith('oracle.')]; "
            "assert not bad, bad")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=ROOT)
    for path in (ROOT / "torchio_b200").rglob("*.py"):
        text = path.read_text()
        assert "import oracle" not in text and "from oracle" not in text, path
