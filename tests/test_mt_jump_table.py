"""The MT19937 jump-ahead table (host only, no GPU): its header matches what ops
expects, a cached table of another layout is rebuilt, and its polynomials move a
state as far as torch's CPU generator (numpy's MT19937 is the same generator)."""

import ctypes

import numpy as np
import pytest
import torch

from torchio_b200 import _native, ops


@pytest.fixture(scope="module")
def table():
    nbytes = _native.lib().tio_mt19937_table_bytes()
    blob = torch.zeros(nbytes, dtype=torch.uint8)
    _native.call("tio_mt19937_build_table", blob.data_ptr(), nbytes)
    return blob.numpy()


def _header(blob):
    return tuple(int(v) for v in blob[:24].view(np.uint32))


def _seed_window(seed):
    """W_0 of torch's CPU generator: the 624 words of init_genrand(seed)."""
    w = [seed & 0xFFFFFFFF]
    for j in range(1, 624):
        w.append((1812433253 * (w[-1] ^ (w[-1] >> 30)) + j) & 0xFFFFFFFF)
    return np.array(w, dtype=np.uint32)


def _untemper(y):
    y = y ^ (y >> 18)
    y = y ^ ((y << 15) & 0xEFC60000)
    t = y
    for _ in range(4):
        t = y ^ ((t << 7) & 0x9D2C5680)
    t2 = t
    for _ in range(2):
        t2 = t ^ (t2 >> 11)
    return t2


def test_table_header_matches_ops(table):
    assert _header(table) == ops.MT_TABLE_HEADER


def test_cached_table_of_another_layout_is_rebuilt(table, tmp_path, monkeypatch):
    stale = table.copy()
    stale[4:8] = np.array([ops.MT_TABLE_HEADER[1] - 1], dtype=np.uint32).view(np.uint8)  # other log2(L)
    path = tmp_path / "mt19937_jump.bin"
    stale.tofile(path)
    monkeypatch.setattr(ops, "_MT_TABLE_FILE", path)
    monkeypatch.setattr(ops, "_mt_host_table", None)
    got = ops.mt19937_host_table().numpy()
    assert np.array_equal(got, table)
    assert np.array_equal(np.fromfile(path, dtype=np.uint8), table)


@pytest.mark.parametrize("level", ["fine", "coarse"])
def test_jump_polynomial_matches_cpu_generator(table, level):
    """Slot 0 of each level (x^L and x^(S2*L)) applied to W_0 gives W_J, whose tempered
    words are stream words J-624 .. J-1 of the generator.  The state is 19937 bits: of
    the window's first word only the top bit belongs to it (and is ever read)."""
    log2_l, s2 = ops.MT_TABLE_HEADER[1], ops.MT_TABLE_HEADER[2]
    slot, jump = (0, 1 << log2_l) if level == "fine" else (s2 - 1, s2 << log2_l)
    seed = 20240917
    w0 = _seed_window(seed)
    out = np.zeros(624, dtype=np.uint32)
    lib = _native.lib()
    rc = lib.tio_mt19937_apply_poly_host(ctypes.c_void_p(table.ctypes.data), ctypes.c_int(slot),
                                         ctypes.c_void_p(w0.ctypes.data), ctypes.c_void_p(out.ctypes.data))
    assert rc == 0
    bg = np.random.MT19937()
    bg.state = {"bit_generator": "MT19937", "state": {"key": w0, "pos": 624}}
    done = 0
    while done < jump - 624:  # skip in chunks; keep the last 624 words
        k = min(1 << 22, jump - 624 - done)
        bg.random_raw(k)
        done += k
    want = _untemper(bg.random_raw(624).astype(np.uint32))
    assert np.array_equal(out[1:], want[1:])
    assert out[0] >> 31 == want[0] >> 31


def test_device_table_of_cuda_without_an_index_is_the_current_devices(monkeypatch):
    """`randn_mt19937(..., "cuda")` runs on the current device, so it must read that device's table,
    whichever device the table was first copied to."""
    monkeypatch.setattr(ops, "_mt_device_tables", {0: "table on cuda:0", 1: "table on cuda:1"})
    for current in (0, 1):
        monkeypatch.setattr(torch.cuda, "current_device", lambda current=current: current)
        assert ops._mt_table(torch.device("cuda")) == f"table on cuda:{current}"
        assert ops._mt_table(torch.device("cuda", 1 - current)) == f"table on cuda:{1 - current}"
