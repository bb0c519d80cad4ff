"""`set_differentiable` on the host side: the switch itself, and host-resident batches that require
grad, refused before anything reaches a device (whole-call and streamed `Compose` paths alike)."""

import warnings

import pytest
import torch

import torchio_b200 as tio
from torchio_b200.data import AffineMatrix


@pytest.fixture
def differentiable():
    previous = tio.set_differentiable(True)
    try:
        yield
    finally:
        tio.set_differentiable(previous)


def _host_batch(b):
    x = torch.rand((b, 1, 16, 16, 16), requires_grad=True)
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [AffineMatrix() for _ in range(b)])})


def test_switch_is_off_by_default_and_returns_the_previous_value():
    assert tio.differentiable_default() is False
    assert tio.set_differentiable(True) is False
    try:
        assert tio.differentiable_default() is True
        assert tio.set_differentiable(True) is True
    finally:
        tio.set_differentiable(False)


@pytest.mark.parametrize("chunk_size", [None, 1])
def test_host_batches_that_require_grad_are_refused(differentiable, chunk_size):
    """B = 4 with chunk_size = 1 would take the streamed path, which stages slice by slice."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipeline = tio.Compose([tio.Affine(degrees=10), tio.ElasticDeformation(max_displacement=2.0)], copy=False)
    pipeline.chunk_size = chunk_size
    with pytest.raises(NotImplementedError, match="CUDA tensors only"):
        pipeline(_host_batch(4))
    with pytest.raises(NotImplementedError, match="CUDA tensors only"):
        tio.Affine(degrees=10, copy=False)(_host_batch(4))
