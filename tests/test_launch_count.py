"""`ops.launches()` is the library's own count of kernel launches (`tio_launch_count`): a call of each
ops entry point must move it by the number of the library's kernels in a profiler trace of the
same call."""

import json
import shutil
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from torchio_b200 import _native, ops, tables

ROOT = Path(__file__).resolve().parent.parent
DEV = "cuda"
ONE = (1.0, 1.0, 1.0)


def test_every_kernel_of_the_library_is_in_namespace_tio():
    """The GPU test below finds the library's kernels in a trace by "tio::" in their names."""
    cuobjdump = shutil.which("cuobjdump")
    if cuobjdump is None:
        pytest.skip("cuobjdump is not on PATH")
    out = subprocess.run([cuobjdump, "-res-usage", str(_native.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout
    kernels = [line.split()[1] for line in out.splitlines() if line.strip().startswith("Function ")]
    assert len(kernels) > 100
    assert [k for k in kernels if not k.startswith("_ZN3tio")] == []


# ---- one representative call per entry point and route: set-up outside the trace, the call inside ----

def _image(shape, seed=0):
    return (torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 100).to(DEV)


def _labels(shape, dtype, seed=0):
    return (_image(shape, seed) / 30).to(dtype)  # labels 0..3


def _blur(sigmas, b):
    t = tables.blur_tables([sigmas] * b, b)
    return dict(taps=t.taps.to(DEV), radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask)


def _bias(b):
    return dict(coarse=(torch.rand((b, 1, 3, 2, 4), generator=torch.Generator().manual_seed(3)) * 0.4).to(DEV))


def _noise(b):
    return dict(mean=torch.zeros(b, device=DEV), std=torch.ones(b, device=DEV), noise_mode=1)


CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


def _resample(shape, dtype, mode, **kw):
    x = _labels(shape, dtype) if dtype != torch.float32 else _image(shape)
    mat = torch.tensor([[1, 0, 0, 0.3, 0, 1, 0, -0.2, 0, 0, 1, 0.1]] * shape[0], device=DEV)
    fill = torch.tensor([1.0], device=DEV) if mode == ops.LABEL_PV else None
    return lambda: ops.resample(x, mat, None, None, ONE, ONE, affine_first=True, mode=mode, fill=fill, **kw)


@case
def upload():
    return lambda: ops.upload(torch.device(DEV), np.arange(100, dtype=np.float32), np.ones(3, np.uint8))


@case
def resample_general_k181():
    """Rows of 181 fp32 are not a multiple of 16 bytes: the tile path declines, one general kernel."""
    return _resample((1, 1, 6, 5, 181), torch.float32, ops.LINEAR)


@case
def resample_tiled():
    return _resample((2, 1, 16, 12, 32), torch.float32, ops.LINEAR)


@case
def resample_tiled_exact_coords():
    return _resample((2, 1, 16, 12, 32), torch.float32, ops.LINEAR, exact_coords=True)


@case
def resample_tiled_int16_nearest():
    return _resample((2, 1, 16, 12, 32), torch.int16, ops.NEAREST)


@case
def resample_label_pv():
    return _resample((2, 1, 16, 12, 32), torch.uint8, ops.LABEL_PV)


@case
def resample_general_by_box_hint():
    return _resample((2, 1, 16, 12, 32), torch.float32, ops.LINEAR, box_hint=-1)


@case
def onehot():
    x = _labels((2, 1, 5, 6, 7), torch.int16)
    return lambda: ops.onehot(x, torch.arange(4, device=DEV))


@case
def label_argmax():
    x = _image((2, 4, 5, 6, 7))
    return lambda: ops.label_argmax(x, torch.arange(4, device=DEV), 0.0, torch.int16)


@case
def min_sample0():
    x = _image((2, 3, 5, 6, 7))
    return lambda: ops.min_sample0(x)


@case
def crop_patches():
    x = _image((2, 8, 8, 8))
    return lambda: ops.crop_patches(x, [[0, 0, 0], [1, 2, 3]], (4, 4, 4))


@case
def remap():
    x = _image((2, 1, 8, 8, 8))
    return lambda: ops.remap(x, (9, 6, 10), (1, -1, 2), mode="reflect")


@case
def permute():
    x = _image((2, 1, 8, 9, 10))
    return lambda: ops.permute(x, (2, 0, 1), 5)


@case
def permute_identity_with_flips():
    x = _image((2, 1, 8, 9, 10))
    return lambda: ops.permute(x, (0, 1, 2), 2)


@case
def blur_jk():
    x, t = _image((2, 1, 8, 6, 20)), _blur([0, 1.5, 1], 2)
    return lambda: ops.blur(x, t["taps"], t["radius"], t["big_r"], t["axes_mask"], None)


@case
def blur_wide():
    x, t = _image((1, 1, 8, 6, 20)), _blur([8.0, 0, 7.0], 1)
    return lambda: ops.blur(x, t["taps"], t["radius"], t["big_r"], t["axes_mask"], None)


@case
def moments():
    x = _image((5, 6, 7))
    return lambda: ops.moments(x)


@case
def quantile_neighbours():
    x = _image((5, 6, 7))
    return lambda: ops.quantile_neighbours(x, [0.01, 0.99])


QS = np.linspace(0.01, 0.99, 15)  # two rounds of the radix select


@case
def quantiles_batched():
    x = _image((3, 1, 5, 6, 7))
    return lambda: ops.quantiles_batched(x, QS)


@case
def histogram_tables():
    vals, w, _, nan = ops.quantiles_batched(_image((3, 1, 5, 6, 7)), QS)
    return lambda: ops.histogram_tables(vals, w, nan, torch.linspace(0, 100, len(QS)))


@case
def histogram_map():
    x = _image((3, 1, 5, 6, 7))
    vals, w, _, nan = ops.quantiles_batched(x, QS)
    t = ops.histogram_tables(vals, w, nan, torch.linspace(0, 100, len(QS)))
    return lambda: ops.histogram_map(x, t, len(QS))


@case
def rescale():
    x = _image((2, 1, 5, 6, 8))
    return lambda: ops.rescale(x, lo=10.0, hi=90.0, sub=[0.5, 1.0], div=2.0)


@case
def rescale_without_tables():
    x = _image((2, 1, 5, 6, 8))
    return lambda: ops.rescale(x, lo=10.0, hi=90.0)


# the routes of intensity_fused
def _intensity(shape, *parts, **kw):
    x = _image(shape)
    for part in parts:
        kw.update(part(shape[0]))
    return lambda: ops.intensity_fused(x, **kw)


@case
def intensity_pass1_only():
    return _intensity((2, 1, 8, 6, 20), _bias)


@case
def intensity_jk_only():
    return _intensity((2, 1, 8, 6, 20), lambda b: _blur([0, 1.5, 1], b))


@case
def intensity_two_passes():
    return _intensity((2, 1, 8, 6, 20), _bias, lambda b: _blur([1, 1.5, 1], b))


@case
def intensity_wide_table():
    return _intensity((1, 1, 8, 6, 20), _bias, lambda b: _blur([8.0, 6.0, 7.0], b))


@case
def intensity_replay_in_pass1():
    """z_replay through pass1_normals_kernel, then the J/K pass."""
    return _intensity((2, 1, 8, 6, 20), _bias, lambda b: _blur([1, 1.5, 1], b), _noise, z_replay=(7, 32))


@case
def intensity_replay_stand_alone():
    """K % 4 != 0: the stand-alone replay, then both passes."""
    return _intensity((2, 1, 8, 4, 18), _bias, lambda b: _blur([1, 1.5, 1], b), _noise, z_replay=(7, 32))


@case
def intensity_pass1_with_normals():
    x, kw = _image((2, 1, 8, 6, 20)), {**_bias(2), **_blur([1, 1.5, 1], 2)}
    return lambda: ops.intensity_pass1_with_normals(x, 5, 64, **kw)


@case
def randn_mt19937():
    return lambda: ops.randn_mt19937(3, 64, 4096, DEV)


@case
def randn_mt19937_past_the_first_16_segments():
    """The coarse jump runs too."""
    return lambda: ops.randn_mt19937(3, 40 << 20, 4096, DEV)


@case
def labels_to_image():
    x = _labels((2, 1, 5, 6, 7), torch.int16)
    return lambda: ops.labels_to_image(x, [0, 1, 2, 3], [0.1, 0.2, 0.3, 0.4], [0.01, 0.02, 0.03, 0.04])


@case
def label_lut():
    x = _labels((2, 1, 5, 6, 7), torch.int16)
    keys, values = tables.label_lut([(1, 5), (2, 0)], torch.int16, DEV)
    return lambda: ops.label_lut(x, keys, values, identity=True)


@case
def label_contour():
    x = _labels((2, 1, 5, 6, 7), torch.uint8)
    return lambda: ops.label_contour(x)


@case
def label_range():
    x = _labels((2, 1, 5, 6, 7), torch.int32)
    return lambda: ops.label_range(x)


@case
def onehot_classes():
    x = _labels((2, 1, 5, 6, 7), torch.int64)
    return lambda: ops.onehot_classes(x, 4)


@case
def channel_argmax():
    x = _image((2, 3, 5, 6, 8))
    return lambda: ops.channel_argmax(x)


@case
def interpolate():
    x, (idx, lam) = _image((2, 1, 5, 6, 7)), tables.resize_tables((5, 6, 7), (3, 9, 4), True)
    return lambda: ops.interpolate(x, (3, 9, 4), idx, lam)


@case
def axis_resample():
    x, t = _image((2, 1, 5, 6, 7)), tables.anisotropy_instance_tables((5, 6, 7), [1, 2], [2.0, 3.0], True)
    return lambda: ops.axis_resample(x, *t, linear=True)


@case
def clamp():
    x = _image((2, 1, 5, 6, 7))
    return lambda: ops.clamp(x, torch.tensor([10.0]), torch.tensor([90.0]))


@case
def mask_by_labels():
    x, m = _image((2, 1, 5, 6, 7)), _labels((1, 5, 6, 7), torch.int16, seed=2)
    keys, _ = tables.label_lut([(1, 0), (2, 0)], torch.int16, DEV)
    return lambda: ops.mask(x, m, keys, torch.tensor([0.0]))


@case
def mask_nonzero():
    x, m = _image((2, 1, 5, 6, 7)), _image((1, 5, 6, 7), seed=2) > 50
    return lambda: ops.mask(x, m, None, torch.tensor([0.0]))


@case
def swap_patches():
    x = _image((2, 1, 8, 8, 8))
    swaps = np.array([[[0, 0, 0, 4, 4, 4, ops.SWAP_EXCHANGE, 0], [0, 0, 0, 1, 1, 1, ops.SWAP_STAGED, 0]]])
    return lambda: ops.swap_patches(x, swaps, (3, 3, 3))


def _keep_largest(dtype, labels):
    x = _labels((2, 1, 6, 7, 8), dtype, seed=4)
    return lambda: ops.keep_largest(x, labels, 0, True)


@case
def keep_largest_of_labels():
    return _keep_largest(torch.int16, [1, 2])


@case
def keep_largest_by_value():
    return _keep_largest(torch.uint8, None)


@case
def keep_largest_by_search():
    return _keep_largest(torch.int32, None)


def _spike_inputs():
    x = _image((2, 1, 6, 8, 10)) - 50  # negative voxels: the peak comes from the spectrum
    intensity = np.array([0.5, 1.0], np.float32)
    (intensity_d,) = ops.upload(x.device, intensity)
    return x, intensity, intensity_d


@case
def spike():
    x, intensity, _ = _spike_inputs()
    spikes = np.zeros((2, 2, 4), np.int32)
    spikes[:, 0] = [1, 2, 3, 1]
    return lambda: ops.spike(x, spikes, intensity)


@case
def spike_stats():
    x, _, intensity_d = _spike_inputs()
    return lambda: ops.spike_stats(x, intensity_d)


@case
def spectrum_peak_in_chunks():
    """A workspace of one row: one chunk per row, three launches each."""
    x, _, intensity_d = _spike_inputs()
    _, flags = ops.spike_stats(x, intensity_d)
    row_bytes = 6 * 8 * (10 // 2 + 1) * 8
    return lambda: ops.spectrum_peak(x, intensity_d, flags, workspace_bytes=row_bytes)


@case
def ghosting_on_two_axes():
    x = _image((2, 1, 6, 8, 10))
    table = np.full((2, 10), 0.5, np.float32)
    return lambda: ops.ghosting(x, table, np.array([0, 2]), np.array([True, True]))


def count_every_case(out_path: str) -> None:
    """{case: [ops.launches() delta, the library's kernels in a CUDA trace]} of every case, as JSON."""
    out = Path(out_path)
    trace = out.with_suffix(".trace.json")
    results = {}
    for name, setup in CASES.items():
        call = setup()
        torch.cuda.synchronize()
        before = ops.launches()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        counted = ops.launches() - before
        prof.export_chrome_trace(str(trace))
        events = json.loads(trace.read_text())["traceEvents"]
        traced = sum(1 for e in events if e.get("cat") == "kernel" and "tio::" in e.get("name", ""))
        results[name] = [counted, traced]
    out.write_text(json.dumps(results))


@pytest.fixture(scope="module")
def counts(tmp_path_factory):
    """The cases are traced in a process of their own: late in a long session that had traced
    before, the profiler returned traces without kernel records."""
    out = tmp_path_factory.mktemp("launch_count") / "counts.json"
    code = (f"import sys; sys.path[:0] = {[str(ROOT), str(ROOT / 'tests')]!r}; "
            f"import test_launch_count; test_launch_count.count_every_case({str(out)!r})")
    subprocess.run([sys.executable, *(["-s"] if sys.flags.no_user_site else []), "-c", code], check=True)
    return json.loads(out.read_text())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_launch_count_equals_the_kernels_in_a_trace(name, counts):
    counted, traced = counts[name]
    assert traced > 0
    assert counted == traced
