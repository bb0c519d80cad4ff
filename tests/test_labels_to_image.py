"""LabelsToImage: params and RNG order against the reference's fixtures (CPU), and the one-pass
kernel against the reference's op sequence run on the same CUDA tensors from the same CUDA
generator state (GPU): bit-identical images, identical generator offsets afterwards."""

from __future__ import annotations

import hashlib
import json
import warnings

import numpy as np
import pytest
import torch

from labels_to_image_cases import (L2I_CASES, affines, label_map, load_fixture, reference_image,
                                   transform_kwargs)

CASE_NAMES = [c["name"] for c in L2I_CASES]
CASES = {c["name"]: c for c in L2I_CASES}


def _batch(case, labels=None, device=None, pin=False):
    import torchio_b200 as tio

    data = label_map(case) if labels is None else labels
    if device is not None:
        data = data.to(device)
    if pin:
        data = data.pin_memory()
    return tio.SubjectsBatch({"seg": tio.ImagesBatch(data, [tio.AffineMatrix(a) for a in affines(case)],
                                                      image_class=tio.LabelMap)})


def _transform(case):
    import torchio_b200 as tio

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return tio.LabelsToImage(**transform_kwargs(case))


def _sample(case, batch):
    """Gate draw + make_params from the case's CPU seed, as Transform._forward_batch draws them."""
    transform = _transform(case)
    torch.manual_seed(case["seed"])
    assert torch.rand(1).item() < transform.p
    return transform, transform.make_params(batch)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


# ---- CPU ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", CASE_NAMES)
def test_host_params_match_the_reference(name):
    case = CASES[name]
    history, _ = load_fixture(name)
    _, params = _sample(case, _batch(case))
    assert json.dumps([{"name": "LabelsToImage", "params": params}]) == json.dumps(history)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_compose_plan_samples_the_reference_params(name):
    import torchio_b200 as tio

    case = CASES[name]
    history, _ = load_fixture(name)
    pipe = tio.Compose([_transform(case)])
    torch.manual_seed(case["seed"])
    ((_, applied),) = pipe._plan(_batch(case))
    assert json.dumps([{"name": "LabelsToImage", "params": applied[0][1]}]) == json.dumps(history)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_oracle_on_cpu_reproduces_the_reference_image(name):
    """The torch-op port consumes the generator as the reference does: after the same params
    draws, it regenerates the fixture bit for bit."""
    case = CASES[name]
    _, expected = load_fixture(name)
    _, params = _sample(case, _batch(case))
    got = reference_image(label_map(case), params["means"], params["stds"])
    assert torch.equal(_bits(got), _bits(expected))


def test_randn_layout_matches_aten():
    from torchio_b200 import tables

    # H100 SXM: 132 SMs x 2048 threads -> 1056 blocks; 2^29 values take 497 grid-stride rounds
    assert tables.randn_cuda_layout(2**29, 132, 2048) == (1056, 1988)
    assert tables.randn_cuda_layout(2**29, 114, 2048) == (912, ((2**29 - 1) // (4 * 256 * 912) + 1) * 4)
    assert tables.randn_cuda_layout(1000, 132, 2048) == (4, 4)      # grid = ceil(N / 256)
    assert tables.randn_cuda_layout(256, 132, 2048) == (1, 4)
    assert tables.randn_cuda_layout(4 * 256 * 1056, 132, 2048) == (1056, 4)
    assert tables.randn_cuda_layout(4 * 256 * 1056 + 1, 132, 2048) == (1056, 8)
    with pytest.raises(NotImplementedError, match="2\\*\\*29"):
        tables.randn_cuda_layout(2**29 + 1, 132, 2048)


def test_synthesis_tables_follow_the_reference_draw_order():
    from torchio_b200 import tables

    # shared: the dict's order; a label with mean == std == 0 draws nothing
    values, draw, mean, std = tables.label_synthesis_tables({"3": 0.5, "0": 0.0, "1": 0.2},
                                                            {"3": 0.1, "0": 0.0, "1": 0.0}, 2)
    assert values.tolist() == [0, 1, 3] and draw.tolist() == [-1, 1, 0]
    assert mean.shape == std.shape == (2, 3) and mean[1, 2] == np.float32(0.5)
    # per element: sorted union, absent = 0, skipped only when zero in every element
    values, draw, mean, _ = tables.label_synthesis_tables([{0: 0.0, 2: 1.0}, {0: 0.0, 2: 0.0, 5: 1.0}],
                                                          [{0: 0.0, 2: 1.0}, {0: 0.0, 2: 0.0, 5: 1.0}], 2)
    assert values.tolist() == [0, 2, 5] and draw.tolist() == [-1, 0, 1] and mean[0, 2] == 0.0


def test_refusals_before_any_launch():
    import torchio_b200 as tio
    from torchio_b200 import ops

    big = torch.empty((5, 1, 512, 512, 512), dtype=torch.int16, device="meta")  # 5 * 2^27 > 2^29
    with pytest.raises(NotImplementedError, match="2\\*\\*29"):
        ops.labels_to_image(big, [0, 1], [0.1, 0.2], [0.01, 0.02])
    with pytest.raises(TypeError, match="dtype"):
        ops.labels_to_image(torch.zeros((1, 1, 2, 2, 2), dtype=torch.float64), [0], [0.1], [0.01])
    case = CASES["labels_to_image_b1_default"]
    with pytest.raises(KeyError, match="'missing' not found"):
        tio.LabelsToImage("missing").make_params(_batch(case))
    scalar_only = tio.SubjectsBatch({"t1": tio.ImagesBatch(torch.zeros(1, 1, 2, 2, 2), [tio.AffineMatrix(np.eye(4))])})
    with pytest.raises(KeyError, match="No LabelMap"):
        tio.LabelsToImage().make_params(scalar_only)


def test_does_not_stream_in_slices():
    import torchio_b200 as tio

    assert not tio.LabelsToImage().supports_chunks(_batch(CASES["labels_to_image_shared"]))


# ---- GPU ----------------------------------------------------------------------------------------


def _device_run(labels, params, cuda_seed):
    """(ours, reference op sequence, offsets after each) from the same CUDA generator state."""
    from torchio_b200 import ops, tables

    gen = torch.cuda.default_generators[labels.device.index]
    torch.cuda.manual_seed(cuda_seed)
    values, draw, mean, std = tables.label_synthesis_tables(params["means"], params["stds"], labels.shape[0])
    ours = ops.labels_to_image(labels, values, mean, std, draw)
    ours_offset = gen.get_offset()
    torch.cuda.manual_seed(cuda_seed)
    ref = reference_image(labels, params["means"], params["stds"])
    return ours, ref, ours_offset, gen.get_offset()


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_device_image_is_bit_identical_to_the_reference_on_cuda(name):
    case = CASES[name]
    batch = _batch(case, device="cuda")
    _, params = _sample(case, batch)
    ours, ref, off_ours, off_ref = _device_run(batch.images["seg"].data, params, 1000 + case["seed"])
    assert off_ours == off_ref
    assert torch.equal(_bits(ours), _bits(ref))


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [1, 3])
@pytest.mark.parametrize("dtype", [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64, torch.float32])
def test_every_label_dtype_is_bit_identical(dtype, batch_size):
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(7)
    labels = torch.randint(0, 9, (batch_size, 1, 19, 23, 17), generator=g).to(dtype)
    if dtype in (torch.int8, torch.int16, torch.int32, torch.int64, torch.float32):
        labels[:, :, :4] -= 5  # negative labels
    transform = tio.LabelsToImage(ignore_background=True)
    batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(labels.cuda(), [tio.AffineMatrix(np.eye(4))] * batch_size,
                                                       image_class=tio.LabelMap)})
    torch.manual_seed(3)
    params = transform.make_params(batch)
    ours, ref, off_ours, off_ref = _device_run(batch.images["seg"].data, params, 77)
    assert off_ours == off_ref
    assert torch.equal(_bits(ours), _bits(ref))


@pytest.mark.gpu
def test_several_grid_stride_rounds_and_a_ragged_tail():
    """N = 2 * 101 * 103 * 107 spans three rounds of 4S = 4 * 256 * 1056 (H100 SXM) and is not a
    multiple of it; 40 labels, some undrawn."""
    import torchio_b200 as tio

    labels = torch.randint(0, 40, (2, 1, 101, 103, 107), generator=torch.Generator().manual_seed(5))
    labels = labels.to(torch.int16).cuda()
    means = {label: 0.0 if label % 7 == 0 else 0.02 * label for label in range(40)}
    stds = {label: 0.0 if label % 7 == 0 else 0.01 + 0.001 * label for label in range(40)}
    ours, ref, off_ours, off_ref = _device_run(labels, {"means": means, "stds": stds}, 2024)
    assert off_ours == off_ref
    assert torch.equal(_bits(ours), _bits(ref))
    assert tio.LabelsToImage().supports_per_instance_params


@pytest.mark.gpu
def test_full_size_int16_batch_every_voxel():
    """32 x 1 x 256^3 int16, 32 labels, per-element params: N = 2^29, the largest single ATen draw."""
    import torchio_b200 as tio

    labels = torch.empty((32, 1, 256, 256, 256), dtype=torch.int16, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(11)
    labels.copy_(torch.randint(0, 32, labels.shape, generator=g, device="cuda", dtype=torch.int16))
    transform = tio.LabelsToImage()
    batch = tio.SubjectsBatch({"seg": tio.ImagesBatch(labels, [tio.AffineMatrix(np.eye(4))] * 32,
                                                       image_class=tio.LabelMap)})
    torch.manual_seed(12)
    params = transform.make_params(batch)
    ours, ref, off_ours, off_ref = _device_run(labels, params, 13)
    assert off_ours == off_ref
    equal = torch.equal(_bits(ours), _bits(ref))
    digest = hashlib.sha256(ours.cpu().numpy().tobytes()).hexdigest()
    print(f"labels_to_image 32x256^3 int16: sha256 {digest}, bit-identical={equal}")
    assert equal


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASE_NAMES)
def test_device_image_against_the_cpu_fixture(name):
    """Other generator, so other normals: same params, +0 exactly where the reference is 0, and per
    label and element a sample mean and std within 5 standard errors of the params."""
    case = CASES[name]
    history, expected = load_fixture(name)
    batch = _batch(case, device="cuda")
    transform, params = _sample(case, batch)
    assert json.dumps(params) == json.dumps(history[0]["params"])
    torch.cuda.manual_seed(case["seed"])
    out = transform.apply_transform(batch, params).images["image_from_labels"].data.cpu()
    assert out.shape == expected.shape and out.dtype == torch.float32
    zero = expected == 0
    assert torch.equal(out == 0, zero)
    assert not torch.signbit(out[zero]).any()
    labels = label_map(case)[:, 0:1]
    for b in range(case["batch"]):
        means = params["means"][b] if isinstance(params["means"], list) else params["means"]
        stds = params["stds"][b] if isinstance(params["stds"], list) else params["stds"]
        for label, mean in means.items():
            values = out[b][labels[b] == label].double()
            if values.numel() < 2 or (mean == 0.0 and stds[label] == 0.0):
                continue
            std = stds[label]
            if std == 0.0:
                assert torch.all(values == float(np.float32(mean)))
                continue
            n = values.numel()
            assert abs(float(values.mean()) - mean) <= 5 * std / n**0.5, (b, label)
            assert abs(float(values.std()) - std) <= 5 * std / (2 * (n - 1)) ** 0.5, (b, label)


def _chain_batch(device="cuda", pin=False):
    import torchio_b200 as tio

    g = torch.Generator().manual_seed(21)
    labels = torch.randint(0, 6, (2, 1, 32, 28, 24), generator=g).to(torch.int16)
    t1 = torch.rand((2, 1, 32, 28, 24), generator=g)
    if device is not None:
        labels, t1 = labels.to(device), t1.to(device)
    if pin:
        labels, t1 = labels.pin_memory(), t1.pin_memory()
    affine = [tio.AffineMatrix(np.diag([1.0, 1.0, 1.2, 1.0])) for _ in range(2)]
    return tio.SubjectsBatch({"t1": tio.ImagesBatch(t1, affine, image_class=tio.ScalarImage),
                              "seg": tio.ImagesBatch(labels, [a.clone() for a in affine], image_class=tio.LabelMap)})


def _chain():
    import torchio_b200 as tio

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return [tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.LabelsToImage("seg"), tio.BiasField(),
                tio.Blur(std=(0, 1)), tio.Noise(), tio.Gamma()]


def _history(batch):
    return json.dumps([{"name": t.name, "params": t.params} for t in batch.applied_transforms])


@pytest.mark.gpu
def test_compose_equals_the_transforms_one_by_one():
    import torchio_b200 as tio

    torch.manual_seed(31)
    torch.cuda.manual_seed(32)
    batch = _chain_batch()
    for transform in _chain():
        batch = transform(batch)
    results = {}
    for fuse in (False, True):
        pipe = tio.Compose(_chain())
        pipe.fuse = fuse
        torch.manual_seed(31)
        torch.cuda.manual_seed(32)
        results[fuse] = pipe(_chain_batch())
    assert [t.name for t in batch.applied_transforms] == ["Affine", "LabelsToImage", "BiasField", "Blur",
                                                          "Noise", "Gamma"]
    assert set(batch.applied_transforms[1].params) == {"means", "stds", "_batch_size", "_batched_keys"}
    for name in ("t1", "seg", "image_from_labels"):
        # unfused: the same kernels in the same order, bit for bit
        assert torch.equal(results[False].images[name].data, batch.images[name].data), name
        # fused intensity chain: equal up to the fused kernel's fp32 reassociation (test_gpu_properties)
        want = batch.images[name].data.float()
        rng = float(want.max() - want.min()) or 1.0
        assert float((results[True].images[name].data.float() - want).abs().max()) <= 3e-6 * rng, name
    assert _history(results[False]) == _history(batch) == _history(results[True])


@pytest.mark.gpu
@pytest.mark.parametrize("pin", [False, True])
def test_host_batch_returns_the_new_image_on_the_host(pin):
    import torchio_b200 as tio

    outs = []
    for device in ("cuda", None):
        torch.manual_seed(41)
        torch.cuda.manual_seed(42)
        outs.append(tio.LabelsToImage("seg")(_chain_batch(device=device, pin=pin and device is None)))
    on_device, on_host = outs
    image = on_host.images["image_from_labels"].data
    assert image.device.type == "cpu" and image.is_pinned() == pin
    assert on_host.images["seg"].data.device.type == "cpu"
    assert torch.equal(_bits(image), _bits(on_device.images["image_from_labels"].data.cpu()))
    assert _history(on_host) == _history(on_device)
