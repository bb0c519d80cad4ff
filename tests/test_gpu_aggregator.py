"""PatchAggregator on the GPU: every fixture bit for bit, random batches of every dtype and mode bit
for bit against the reference's op sequence on the same CUDA tensors, a 256^3 volume, the
GridSampler -> SubjectsLoader -> model -> PatchAggregator recipe, host callers, no host sync,
non-default streams, launch counts against a profiler trace, and ports of the reference's tests."""

from __future__ import annotations

import json
import subprocess
import sys
import zlib
from pathlib import Path

import pytest
import torch

import aggregator_cases as ac
import torchio_b200 as tio
from oracle.aggregator import OpSequence
from torchio_b200 import ops
from torchio_b200.patches import PatchLocation

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
DEV = "cuda"
CASES = ac.CASES
OK = [n for n in CASES if "error" not in ac.load_fixture(n) and not CASES[n]["deviation"]]


def _buffer(aggregator, key):
    return aggregator._outputs[key]


@pytest.mark.parametrize("name", OK)
def test_fixture_on_the_device(name):
    case = CASES[name]
    got = ac.drive(case, tio.PatchAggregator, PatchLocation, device=DEV, buffers=_buffer)
    ac.check_against_fixture(case, got)


@pytest.mark.parametrize("name", ["aggregator_grid_crop_o234", "aggregator_grid_hann_odd", "aggregator_dtypes_average"])
def test_host_caller_gets_host_tensors(name):
    """Host batches: buffers on the execution device, host outputs equal to the reference's; crop
    returns a copy of its buffer."""
    case = CASES[name]
    got = ac.drive(case, tio.PatchAggregator, PatchLocation, device="cpu", buffers=_buffer)
    for key in [k for k in got if k.startswith("alias_")]:
        assert got[key] is False
        got.pop(key)
    ac.check_against_fixture(case, got)


# ---- random batches against the op sequence on the same CUDA tensors ------------------------------

SHAPE, PATCH, OVERLAP = (13, 11, 17), (5, 4, 6), (2, 1, 3)
PROPERTY = [(dtype, mode) for mode in ("crop", "average", "hann") for dtype in ac.ALL_DTYPES
            if dtype not in ac.ERROR_DTYPES[mode]]


def _random_locations(n: int, g: torch.Generator) -> list[PatchLocation]:
    return [PatchLocation(index=tuple(int(torch.randint(0, SHAPE[a] - PATCH[a] + 1, (1,), generator=g))
                                      for a in range(3)), size=PATCH) for _ in range(n)]


def _equal_bits(a: torch.Tensor, b: torch.Tensor) -> bool:
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype == torch.bool:
        return torch.equal(a, b)
    view = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[a.element_size()]
    return torch.equal(a.contiguous().view(view), b.contiguous().view(view))


@pytest.mark.parametrize("n", [1, 7, 300])
@pytest.mark.parametrize("channels", [1, 3, 64])
@pytest.mark.parametrize("dtype,mode", PROPERTY, ids=[f"{ac.SHORT[d]}-{m}" for d, m in PROPERTY])
def test_random_batches_match_the_op_sequence(dtype, mode, channels, n):
    g = torch.Generator().manual_seed(zlib.crc32(f"{dtype}-{mode}-{channels}-{n}".encode()))
    mine = tio.PatchAggregator(SHAPE, overlap_mode=mode, patch_overlap=OVERLAP)
    theirs = OpSequence(SHAPE, overlap_mode=mode, patch_overlap=OVERLAP)
    for t in range(3):  # several batches into the same buffers
        patches = ac.random_patches(n, channels, PATCH, dtype, int(torch.randint(0, 2 ** 31, (1,), generator=g)), DEV)
        locs = _random_locations(n, g)
        mine.add_batch(patches, locs)
        theirs.add_batch(patches, locs)
        assert _equal_bits(mine.get_output(), theirs.get_output()), f"batch {t}"


@pytest.mark.parametrize("mode", ["crop", "average", "hann"])
def test_256_cubed_with_96_cubed_patches(mode):
    g = torch.Generator().manual_seed(5)
    volume = torch.rand((1, 256, 256, 256), generator=g).to(DEV)
    locs = [PatchLocation(index=i, size=s) for i, s in ac.grid_locations((256,) * 3, (96,) * 3, (16,) * 3)]
    mine = tio.PatchAggregator((256,) * 3, overlap_mode=mode, patch_overlap=16)
    theirs = OpSequence((256,) * 3, overlap_mode=mode, patch_overlap=16)
    for start in range(0, len(locs), 8):
        batch = locs[start:start + 8]
        patches = ops.crop_patches(volume, [loc.index for loc in batch], (96, 96, 96))
        mine.add_batch(patches, batch)
        theirs.add_batch(patches, batch)
    out = mine.get_output()
    assert _equal_bits(out, theirs.get_output())
    if mode == "crop":
        assert torch.equal(out, volume)


@pytest.mark.parametrize("mode", ["crop", "average", "hann"])
def test_grid_sampler_loader_model_aggregator(mode):
    """The reference's dense-inference recipe on a device subject; crop gives the padded input back."""
    volume = torch.rand((2, 37, 30, 41), generator=torch.Generator().manual_seed(3)).to(DEV)
    subject = tio.Subject(t1=tio.ScalarImage(volume))
    sampler = tio.GridSampler(subject, patch_size=(16, 12, 20), patch_overlap=(4, 4, 6), padding_mode="reflect")
    padded = sampler.subject.t1.data
    aggregator = tio.PatchAggregator(spatial_shape=sampler.subject.spatial_shape, overlap_mode=mode,
                                     patch_overlap=(4, 4, 6))
    theirs = OpSequence(sampler.subject.spatial_shape, overlap_mode=mode, patch_overlap=(4, 4, 6))
    for batch in tio.SubjectsLoader(sampler, batch_size=5):
        output = batch.t1.data * 1  # an identity model
        locations = [batch.metadata["patch_location"][i] for i in range(batch.batch_size)]
        aggregator.add_batch(output, locations)
        theirs.add_batch(output, locations)
    result = aggregator.get_output()
    assert result.is_cuda and _equal_bits(result, theirs.get_output())
    if mode == "crop":
        assert torch.equal(result, padded)


def test_no_host_sync_in_add_batch_or_get_output():
    patches = torch.rand((4, 3, 6, 5, 7), device=DEV)
    locs = [PatchLocation(index=(i, i, i), size=(6, 5, 7)) for i in range(4)]
    aggregators = [tio.PatchAggregator((12, 11, 13), overlap_mode=m, patch_overlap=2) for m in ("crop", "average", "hann")]
    for a in aggregators:  # first use: buffers, staging ring
        a.add_batch(patches, locs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for a in aggregators:
            a.add_batch({"__default__": patches}, locs)
            a.get_output()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_non_default_stream():
    patches = torch.rand((6, 2, 5, 4, 6), device=DEV)
    locs = [PatchLocation(index=(i, 6 - i, i), size=(5, 4, 6)) for i in range(6)]
    expected = OpSequence((11, 10, 12), overlap_mode="hann")
    expected.add_batch(patches, locs)
    want = expected.get_output()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        a = tio.PatchAggregator((11, 10, 12), overlap_mode="hann")
        a.add_batch(patches, locs)
        got = a.get_output()
    stream.synchronize()
    assert _equal_bits(got, want)


def test_dtype_change_and_grad_are_refused():
    loc = [PatchLocation(index=(0, 0, 0), size=(4, 4, 4))]
    a = tio.PatchAggregator((6, 6, 6), overlap_mode="average")
    a.add_batch(torch.rand((1, 1, 4, 4, 4), device=DEV), loc)
    with pytest.raises(NotImplementedError, match="cast it before add_batch"):
        a.add_batch(torch.rand((1, 1, 4, 4, 4), device=DEV, dtype=torch.float64), loc)
    with pytest.raises(NotImplementedError, match="detach"):
        a.add_batch(torch.rand((1, 1, 4, 4, 4), device=DEV, requires_grad=True), loc)


# ---- launch counts: ops.launches() against the tio:: kernels of a profiler trace -------------------

def _launch_cases():
    """add_batch: per key, the table upload (`tio_upload`, the library's copy kernel) and one
    `tio_aggregate_patches`; get_output: one `tio_aggregate_finish`, none for crop."""
    loc = [PatchLocation(index=(i, 0, i), size=(4, 5, 6)) for i in range(3)]
    patches = torch.rand((3, 2, 4, 5, 6), device=DEV)
    out = {}
    for mode in ("crop", "average", "hann"):
        a = tio.PatchAggregator((9, 7, 10), overlap_mode=mode)
        out[f"add_one_key_{mode}"] = (lambda a=a: a.add_batch(patches, loc), 2)
        b = tio.PatchAggregator((9, 7, 10), overlap_mode=mode)
        b.add_batch({"x": patches, "y": patches[:, :1]}, loc)
        out[f"add_two_keys_{mode}"] = (lambda b=b: b.add_batch({"x": patches, "y": patches[:, :1]}, loc), 4)
        out[f"get_output_{mode}"] = (lambda b=b: b.get_output("x"), 0 if mode == "crop" else 1)
    return out


def count_every_case(out_path: str) -> None:
    """{case: [expected, ops.launches() delta, tio:: kernels in a CUDA trace]} as JSON."""
    out = Path(out_path)
    trace = out.with_suffix(".trace.json")
    results = {}
    for name, (call, expected) in _launch_cases().items():
        torch.cuda.synchronize()
        before = ops.launches()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        counted = ops.launches() - before
        prof.export_chrome_trace(str(trace))
        events = json.loads(trace.read_text())["traceEvents"]
        traced = sum(1 for e in events if e.get("cat") == "kernel" and "tio::" in e.get("name", ""))
        results[name] = [expected, counted, traced]
    out.write_text(json.dumps(results))


@pytest.fixture(scope="module")
def counts(tmp_path_factory):
    """Traced in a process of its own, as tests/test_launch_count.py does."""
    out = tmp_path_factory.mktemp("aggregator_launches") / "counts.json"
    code = (f"import sys; sys.path[:0] = {[str(ROOT), str(ROOT / 'tests')]!r}; "
            f"import test_gpu_aggregator; test_gpu_aggregator.count_every_case({str(out)!r})")
    subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], check=True)
    return json.loads(out.read_text())


@pytest.mark.parametrize("name", [f"{what}_{mode}" for mode in ("crop", "average", "hann")
                                  for what in ("add_one_key", "add_two_keys", "get_output")])
def test_launch_count_equals_the_kernels_in_a_trace(name, counts):
    expected, counted, traced = counts[name]
    assert counted == expected == traced


# ---- ports of the reference's aggregator tests (tests/test_patches.py) -----------------------------

def _subject(shape):
    return tio.Subject(t1=tio.ScalarImage(torch.rand((1, *shape), generator=torch.Generator().manual_seed(0)).to(DEV)))


def _aggregate_grid(subject, patch_size, sampler_overlap, **kw):
    sampler = tio.GridSampler(subject, patch_size=patch_size, patch_overlap=sampler_overlap)
    aggregator = tio.PatchAggregator(spatial_shape=(20, 20, 20), **kw)
    for i in range(len(sampler)):
        patch = sampler[i]
        aggregator.add_batch(patch.t1.data.unsqueeze(0), [patch.patch_location])
    return aggregator.get_output()


def test_crop_reconstructs_identity():
    subject = _subject((20, 20, 20))
    output = _aggregate_grid(subject, 10, 0, overlap_mode="crop")
    torch.testing.assert_close(output, subject.t1.data)


@pytest.mark.parametrize("mode", ["crop", "average", "hann"])
def test_overlap_modes_give_the_volume_shape(mode):
    kw = dict(overlap_mode=mode, patch_overlap=4) if mode == "crop" else dict(overlap_mode=mode)
    output = _aggregate_grid(_subject((20, 20, 20)), 12, 4, **kw)
    assert output.shape == (1, 20, 20, 20)


def test_downsampled_output():
    aggregator = tio.PatchAggregator(spatial_shape=(20, 20, 20), overlap_mode="average", output_shape=(10, 10, 10))
    aggregator.add_batch(torch.rand(1, 1, 10, 10, 10, device=DEV), [PatchLocation(index=(0, 0, 0), size=(20, 20, 20))])
    assert aggregator.get_output().shape == (1, 10, 10, 10)


def test_dict_output():
    aggregator = tio.PatchAggregator(spatial_shape=(10, 10, 10), overlap_mode="average")
    loc = PatchLocation(index=(0, 0, 0), size=(10, 10, 10))
    aggregator.add_batch({"seg": torch.rand(1, 2, 10, 10, 10, device=DEV),
                          "emb": torch.rand(1, 64, 10, 10, 10, device=DEV)}, [loc])
    assert aggregator.get_output("seg").shape == (2, 10, 10, 10)
    assert aggregator.get_output("emb").shape == (64, 10, 10, 10)
