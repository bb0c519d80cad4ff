"""The boundary is executable: the product binds every function from include/tio_b200.h itself, the
stub printed in INTEGRATION.md (what a TorchIO maintainer would paste) must agree with the header
argument for argument, and the stub — run verbatim — must reproduce `ops.resample` on a golden case."""

import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

from torchio_b200 import _native

ROOT = Path(__file__).resolve().parent.parent


def header_prototypes():
    """name -> list of ctypes argument types, as the product parses them from include/tio_b200.h."""
    return {name: argtypes for name, (_, argtypes) in _native.prototypes().items()}


def integration_blocks():
    text = (ROOT / "INTEGRATION.md").read_text()
    section = text[text.index("## B."):]
    return re.findall(r"```python\n(.*?)```", section, flags=re.S)


class _Recorder:
    """Stands in for the CDLL while the INTEGRATION.md argtypes lines are executed."""

    def __init__(self):
        object.__setattr__(self, "fns", {})

    def __getattr__(self, name):
        return self.fns.setdefault(name, type("F", (), {})())


def test_every_declared_function_is_bound_with_the_header_types():
    protos = _native.prototypes()
    text = re.sub(r"/\*.*?\*/", "", (ROOT / "include" / "tio_b200.h").read_text(), flags=re.S)
    assert sorted(protos) == sorted(re.findall(r"\b(tio_\w+)\s*\(", text))
    lib = _native.lib()
    for name, (restype, argtypes) in protos.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, name
    P, I32, I64, U64, SZ, F32 = (ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_size_t,
                                 ctypes.c_float)
    assert protos["tio_rescale"] == (I32, [P, P, I32, I64, F32, F32, P, P, P, P, P, I32, P])
    assert protos["tio_label_argmax"] == (I32, [P, I32, I32, I64, P, F32, P, I32, P])
    assert protos["tio_randn_mt19937"] == (I32, [U64, U64, U64, P, P, P, SZ, P])
    assert protos["tio_quantiles"] == (I32, [P, P, I64, P, I32, P, P, P, P, SZ, P])
    assert protos["tio_quantiles_workspace_bytes"] == (SZ, [])
    assert protos["tio_launch_count"] == (U64, [])
    assert protos["tio_last_error"] == (ctypes.c_char_p, [])


@pytest.mark.parametrize("declaration,message", [
    ("double tio_extra(void);", "does not map"),
    ("int tio_extra(unsigned n, void* stream);", "does not map"),
    ("int tio_extra(void (*done)(int), void* stream);", "prototypes could be parsed"),
], ids=["return-type", "argument-type", "skipped-declaration"])
def test_a_header_the_binding_cannot_read_whole_is_refused(tmp_path, monkeypatch, declaration, message):
    header = tmp_path / "tio_b200.h"
    text = _native.HEADER_PATH.read_text()
    header.write_text(text.replace("#ifdef __cplusplus\n}", f"{declaration}\n#ifdef __cplusplus\n}}"))
    monkeypatch.setattr(_native, "HEADER_PATH", header)
    _native.prototypes.cache_clear()
    try:
        with pytest.raises(RuntimeError, match=message):
            _native.prototypes()
    finally:
        _native.prototypes.cache_clear()


def test_integration_md_argtypes_match_the_header():
    protos = header_prototypes()
    first, second = integration_blocks()[:2]
    rec = _Recorder()
    env = {"ctypes": ctypes, "_lib": rec, "P": ctypes.c_void_p, "I32": ctypes.c_int, "I64": ctypes.c_int64,
           "U64": ctypes.c_uint64, "SZ": ctypes.c_size_t}
    # the argtypes assignments of the stub (they may wrap over two lines) + the table below it
    src = "\n".join(l for l in first.splitlines() if re.match(r"(_lib\.\w+\.(argtypes|restype)\s*=|\s+ctypes\.c_size_t, P\])", l))
    exec(src, env)
    exec(second, env)
    seen = {name: fn.argtypes for name, fn in rec.fns.items() if hasattr(fn, "argtypes")}
    assert len(seen) >= 12
    for name, argtypes in seen.items():
        assert list(argtypes) == protos[name], name
    assert rec.fns["tio_resample_workspace_bytes"].restype is ctypes.c_size_t


@pytest.mark.gpu
def test_integration_md_stub_runs_and_reproduces_ops_resample():
    """Execute the §B stub verbatim (only the library path is pointed at the in-tree build) and
    call it the way the patched reference would."""
    from golden_cases import CASES_BY_NAME
    from oracle import c_port
    from torchio_b200 import ops
    from util import load_golden

    stub = integration_blocks()[0].replace('ctypes.CDLL("libtio_b200.so")', f'ctypes.CDLL("{_native.LIB_PATH}")')
    env: dict = {}
    exec(stub, env)
    name = "config1_affine_deg10_64"
    _, images, history, expected, _ = load_golden(name)
    params = history[0]["params"]
    data = images["t1"]["data"].cuda()
    mat, cp, flags, _ = c_port.spatial_tables(params, data.shape[0], tuple(data.shape[2:]), images["t1"]["affines"][0])
    mat = mat.cuda()
    fill = ops.min_sample0(data)
    got = env["resample_f32"](data, mat, None, None, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), True, True, fill)
    want = ops.resample(data, mat, None, None, (1.0, 1.0, 1.0), (1.0, 1.0, 1.0), affine_first=True,
                        mode=ops.LINEAR, fill=fill)
    assert torch.equal(got, want)
    ref = expected["t1"]
    rng = float(ref.max() - ref.min())
    assert float((got.cpu() - ref).abs().max()) <= 1e-4 * rng
    assert CASES_BY_NAME[name]["batch"] == data.shape[0]
