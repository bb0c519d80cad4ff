"""Every ops launch goes to the caller's current stream on the tensor's device, whichever device is
current.  Each case of test_launch_count's registry (one call per ops entry point and route) runs on a
stream of its own and, with two GPUs, on the second device while the first is current; both must
compute what the plain run computes, bit for bit."""

import re
import struct

import numpy as np
import pytest
import torch

from test_launch_count import CASES
from torchio_b200 import _native

pytestmark = pytest.mark.gpu

SEED = 1234  # labels_to_image advances the CUDA generator: every run starts from the same state

# the entry points whose last argument is the stream; the others run on the host
_HEADER = re.sub(r"/\*.*?\*/", "", _native.HEADER_PATH.read_text(), flags=re.S)
STREAM_TAKING = set(re.findall(r"\b(tio_\w+)\s*\([^)]*\bvoid\*\s*stream\s*\)", _HEADER))


def _bits(value):
    """``value`` with every tensor, array and float reduced to its bytes on the host."""
    if isinstance(value, torch.Tensor):
        value = value.detach().cpu()
        return str(value.dtype), tuple(value.shape), value.reshape(-1).contiguous().view(torch.uint8).numpy().tobytes()
    if isinstance(value, np.ndarray):
        return str(value.dtype), value.shape, value.tobytes()
    if isinstance(value, float):
        return struct.pack("d", value)
    if isinstance(value, (list, tuple)):
        return [_bits(v) for v in value]
    if isinstance(value, dict):
        return {k: _bits(v) for k, v in value.items()}
    return value


def _inputs(call):
    return [_bits(cell.cell_contents) for cell in call.__closure__ or ()]


def _setup(name):
    """A fresh case, and its inputs' bytes: the in-place entry points change their inputs."""
    torch.cuda.manual_seed_all(SEED)
    call = CASES[name]()
    torch.cuda.synchronize()
    return call, _inputs(call)


def _outputs(name, call, inputs_before, result):
    """What a case computed: its result and the inputs it changed (spike, ghosting, mask, swap_patches,
    keep_largest and histogram_map work in place).  An unchanged input is left out: it may hold bytes
    no kernel wrote, such as the last entry of each row of a histogram table (3 (m - 1) slots for
    3 (m - 1) - 1 values), which is left out of histogram_tables' result too."""
    if name == "histogram_tables":
        result = result[:, :-1]
    changed = [after for after, before in zip(_inputs(call), inputs_before, strict=True) if after != before]
    return _bits(result), changed


def _plain_run(name):
    call, inputs = _setup(name)
    result = call()
    torch.cuda.synchronize()
    return _outputs(name, call, inputs, result)


def test_the_header_names_the_stream_taking_entry_points():
    assert {"tio_upload", "tio_resample", "tio_motion", "tio_aggregate_finish"} <= STREAM_TAKING
    assert not {"tio_mt19937_build_table", "tio_resample_workspace_bytes", "tio_launch_count"} & STREAM_TAKING


@pytest.mark.parametrize("name", list(CASES))
def test_every_launch_goes_to_the_callers_current_stream(name, monkeypatch):
    want = _plain_run(name)
    call, inputs = _setup(name)
    calls, real_call = [], _native.call

    def spy(fn, *args):
        calls.append((fn, args))
        return real_call(fn, *args)

    monkeypatch.setattr(_native, "call", spy)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        result = call()
    stream.synchronize()
    launched = [(fn, args[-1]) for fn, args in calls if fn in STREAM_TAKING]
    assert launched
    assert [fn for fn, handle in launched if handle != stream.cuda_stream] == []
    assert _outputs(name, call, inputs, result) == want


@pytest.mark.parametrize("name", list(CASES))
def test_every_case_runs_on_a_device_that_is_not_current(name):
    """Set up on cuda:1, called with cuda:0 current.  A case whose call itself names "cuda" (upload,
    randn_mt19937) follows the current device, so the results are compared on the host."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs: runs each case on cuda:1 while cuda:0 is current")
    with torch.cuda.device(1):
        want = _plain_run(name)
        call, inputs = _setup(name)
    with torch.cuda.device(0):
        result = call()
    for device in (0, 1):
        torch.cuda.synchronize(device)
    assert _outputs(name, call, inputs, result) == want
