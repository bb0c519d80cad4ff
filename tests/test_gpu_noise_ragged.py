"""Exact `Noise` on the device for draws of any size at any stream position.

`torch.randn(n, generator=g)` on a CPU mt19937 generator (ATen normal_fill) takes n uniforms from
the stream in 16-groups counted from where the draw starts, and, when n % 16 != 0, 16 more words
that give its last 16 outputs anew.  The device replay (`ops.randn_mt19937`,
`tio_randn_mt19937_window`) must follow that for every start word and size >= 16, and for every
window [lo, hi) of a draw, which is what a slice of a streamed batch uses.  `Noise` then stays on
the host only for draws below 16 values or beyond the jump table's reach (2^31 words)."""

import ctypes
import json
import types
import warnings

import numpy as np
import pytest
import torch

import torchio_b200 as tio
from torchio_b200 import _native, ops
from torchio_b200.transforms import intensity
from torchio_b200.transforms.base import ChunkInfo, chunk_scope

DEV = "cuda"
SEGMENT = 1 << 21  # words per segment of the replay (csrc/mt19937_layout.h)
COARSE = 16 * SEGMENT  # words per coarse jump


def _close(got, want, share=True):
    """The device's uniforms are torch's bit for bit; log/sin/cos differ by <= 4e-6, and most values
    are bit-equal (``share``: checked where there are enough values for the share to mean it)."""
    diff = (got - want).abs()
    assert float(diff.max()) <= 4e-6, (float(diff.max()), int((diff > 4e-6).sum()))
    if share:
        assert float((got == want).float().mean()) > 0.5


def _chain(seed, sizes, skip=0):
    """(offset, n, torch.randn(n)) for consecutive draws of one CPU generator, after `skip` values
    drawn at once."""
    g = torch.Generator().manual_seed(seed)
    offset = 0
    if skip:
        torch.randn(skip, generator=g)
        offset = ops.mt_draw_words(skip)
    draws = []
    for n in sizes:
        draws.append((offset, n, torch.randn(n, generator=g)))
        offset += ops.mt_draw_words(n)
    return draws


# ragged sizes 17..31 first, so that the draws start at every residue modulo 16; then draws that
# cross 624-word blocks, an aligned size at an unaligned start, draws that cross 2^21-word segments
# (7 109 137 = 181 x 217 x 181 crosses three) and the odd 193 x 229 x 193 grid
CHAIN = [*range(17, 32), 1000, 33, 64, 7_109_137, 2**21 + 5, 40, 8_530_021]


@pytest.mark.gpu
def test_replay_follows_a_chain_of_ragged_draws():
    draws = _chain(11, CHAIN)
    assert {offset % 16 for offset, _, _ in draws} == set(range(16))
    assert any(offset // SEGMENT != (offset + n + 16) // SEGMENT for offset, n, _ in draws)
    got = [ops.randn_mt19937(11, offset, n, DEV).cpu() for offset, n, _ in draws]
    for g, (_, n, want) in zip(got, draws, strict=True):
        _close(g, want, share=n >= 1000)
    _close(torch.cat(got[:15]), torch.cat([want for _, _, want in draws[:15]]))


@pytest.mark.gpu
@pytest.mark.parametrize("skip,n", [(COARSE - 37, 1000), (COARSE - 1000, 990), (3 * SEGMENT - 96, 91)],
                         ids=["coarse_jump", "tail_past_the_jump", "tail_across_a_segment"])
def test_replay_across_a_coarse_jump_and_a_segment(skip, n):
    """Groups that straddle the first coarse jump (2^25 words: the draw starts at 2^25 - 21); a
    last group that straddles it and a tail that starts past it (start 2^25 - 984, tail at
    2^25 + 6); a tail that straddles a segment boundary (start 3 * 2^21 - 96, tail at - 5)."""
    [(offset, _, want)] = _chain(5, [n], skip=skip)
    _close(ops.randn_mt19937(5, offset, n, DEV).cpu(), want)


def _windows(n):
    """Ragged windows, the tail alone, windows cutting it and the main groups it overwrites."""
    kept = n - 16 if n % 16 else n
    out = [(0, n), (3, n - 2), (1, 2), (n - 1, n), (n - 16, n), (kept - 5, kept + 3), (n // 2 - 7, n // 2 + 9)]
    return [(lo, hi) for lo, hi in out if 0 <= lo < hi <= n]


@pytest.mark.gpu
@pytest.mark.parametrize("index", [0, 1, 14, 15, 16, 17, 18, 19])
def test_windows_of_a_draw(index):
    """Every window is the same outputs of the whole draw, bit for bit."""
    offset, n, want = _chain(23, CHAIN[: index + 1])[index]
    whole = ops.randn_mt19937(23, offset, n, DEV)
    _close(whole.cpu(), want, share=n >= 1000)
    windows = _windows(n)
    if n > SEGMENT:  # windows that cross a segment boundary and start in the next segment's groups
        edge = (offset // SEGMENT + 1) * SEGMENT - offset
        windows += [(edge - 21, edge + 30), (edge + 3, edge + 5)]
    for lo, hi in windows:
        assert torch.equal(ops.randn_mt19937(23, offset, n, DEV, lo=lo, hi=hi), whole[lo:hi]), (lo, hi)


def _scalar_batch(images, b):
    return tio.SubjectsBatch({k: tio.ImagesBatch(v, [tio.AffineMatrix() for _ in range(b)])
                              for k, v in images.items()})


def _no_host_draws(monkeypatch):
    """torch.randn raises for draws of 16 values or more."""
    real = torch.randn

    def guarded(*args, **kwargs):
        out = real(*args, **kwargs)
        if out.numel() >= 16:
            raise AssertionError(f"host torch.randn of {out.numel()} values")
        return out

    monkeypatch.setattr(torch, "randn", guarded)


@pytest.mark.gpu
@pytest.mark.parametrize("shape,names,rician,p", [
    ((1, 1, 181, 217, 181), ("t1",), False, 1.0),
    ((3, 2, 21, 18, 23), ("t1", "t2"), True, 0.6),
], ids=["mni_1mm", "two_images_rician_gated"])
def test_noise_matches_the_reference_without_host_draws(shape, names, rician, p, monkeypatch):
    from oracle import torch_port

    g = torch.Generator().manual_seed(4)
    imgs = {k: torch.rand(shape, generator=g) for k in names}
    batch = _scalar_batch({k: v.clone().to(DEV) for k, v in imgs.items()}, shape[0])
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        t = tio.Noise(mean=(-0.1, 0.1), std=(0.05, 0.25), rician=rician, p=p)
    torch.manual_seed(2)
    with monkeypatch.context() as m:
        _no_host_draws(m)
        out = t(batch)
    params = out.applied_transforms[0].params
    if p < 1:
        assert sorted(set(params["_keep"])) == [False, True]
    ref = {k: {"kind": "scalar", "data": v.clone(), "affines": [np.eye(4)] * shape[0]} for k, v in imgs.items()}
    torch_port.noise(ref, json.loads(json.dumps(params)))
    for k in names:
        assert float((out.images[k].data.cpu() - ref[k]["data"]).abs().max()) <= 4e-6


def _pipeline(chunk):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        pipeline = tio.Compose([tio.Blur(std=(0.5, 1.5)), tio.Noise(std=(0.05, 0.25)), tio.Gamma(log_gamma=(-0.3, 0.3)),
                                tio.Noise(std=(0.05, 0.25), rician=True)], copy=False)
    pipeline.chunk_size = chunk
    return pipeline


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 3])
def test_ragged_host_batch_streams_and_equals_the_one_shot_rows(chunk, monkeypatch):
    """Rows of 21 x 18 x 23 (8694 % 16 == 6): every slice starts inside a 16-group of the draw."""
    b, shape = 5, (5, 1, 21, 18, 23)
    g = torch.Generator().manual_seed(8)
    imgs = {k: torch.rand(shape, generator=g) + 0.1 for k in ("t1", "t2")}

    def run(size):
        batch = _scalar_batch({k: v.clone() for k, v in imgs.items()}, b)
        pipeline = _pipeline(size)
        streamed = pipeline._chunk_size(batch)
        torch.manual_seed(3)
        return pipeline(batch), streamed

    one_shot, streamed = run(0)
    assert streamed == 0
    with monkeypatch.context() as m:
        _no_host_draws(m)
        out, streamed = run(chunk)
    assert streamed == chunk
    for k in imgs:
        assert not out.images[k].data.is_cuda
        assert torch.equal(out.images[k].data, one_shot.images[k].data)
        for a, o in zip(out.images[k].affines, one_shot.images[k].affines, strict=True):
            assert a == o
    f = lambda h: json.dumps([{"name": t.name, "params": t.params} for t in h], sort_keys=True)
    assert f(out.applied_transforms) == f(one_shot.applied_transforms)


@pytest.mark.gpu
def test_aligned_draws_keep_their_entry_point_and_bits(monkeypatch):
    """Aligned draws and aligned windows still run `tio_randn_mt19937` with its launches; a
    ragged window of an aligned draw equals the same outputs of the whole draw bit for bit, and an
    aligned slice of a streamed draw still makes its normals under the first pass."""
    seed, offset, n = 9, 3 * SEGMENT - 4096, 8192
    calls = []
    real = _native.call
    monkeypatch.setattr(_native, "call", lambda name, *a: (calls.append(name), real(name, *a))[1])
    before = ops.launches()
    whole = ops.randn_mt19937(seed, offset, n, DEV)
    torch.cuda.synchronize()
    assert calls == ["tio_randn_mt19937"] and ops.launches() - before == 3  # seed, fine jump, normals
    assert torch.equal(ops.randn_mt19937(seed, offset, n, DEV, lo=1024, hi=4096), whole[1024:4096])
    calls.clear()
    assert torch.equal(ops.randn_mt19937(seed, offset, n, DEV, lo=1000, hi=4100), whole[1000:4100])
    assert calls == ["tio_randn_mt19937_window"]

    from test_pass1_normals import RADII, _inputs

    x, kw = _inputs(2, 1, (8, 6, 32), RADII, True, seed=3)
    kw.update(mean=torch.zeros(2, device=DEV), std=torch.ones(2, device=DEV), noise_mode=1)
    calls.clear()
    got = ops.intensity_fused(x, **kw, z_replay=(seed, 64, 3 * x.numel(), x.numel()))
    assert calls == ["tio_intensity_pass1_with_normals", "tio_intensity_fused"]
    assert torch.equal(got, ops.intensity_fused(x, **kw, z_replay=(seed, 64 + x.numel())))
    # a ragged slice of the same draw: the stand-alone window, then both passes
    calls.clear()
    got = ops.intensity_fused(x, **kw, z_replay=(seed, 64, 3 * x.numel() + 5, 7))
    assert calls == ["tio_randn_mt19937_window", "tio_intensity_fused"]
    z = ops.randn_mt19937(seed, 64, 3 * x.numel() + 5, DEV, lo=7, hi=7 + x.numel()).view(x.shape)
    assert torch.equal(got, ops.intensity_fused(x, **kw, z=z))


# ---- no GPU needed ----------------------------------------------------------------------------


def test_draw_words_and_aligned_windows():
    assert [ops.mt_draw_words(n) for n in (16, 17, 31, 32, 7_109_137)] == [16, 33, 47, 32, 7_109_153]
    assert ops._mt_aligned_draw(32, 4096, 1024, 2048) == 1056
    for args in [(33, 4096, 0, 4096), (32, 4095, 0, 16), (32, 4096, 8, 4096), (32, 4096, 0, 4090)]:
        assert ops._mt_aligned_draw(*args) is None


def test_randn_refuses_windows_and_positions_out_of_reach():
    """The checks come before anything touches a device."""
    for kwargs in [dict(n=15), dict(lo=5, hi=5), dict(lo=0, hi=101), dict(lo=-1), dict(offset=-16)]:
        args = dict(offset=0, n=100) | kwargs
        with pytest.raises(ValueError, match="0 <= lo < hi <= n"):
            ops.randn_mt19937(1, args.pop("offset"), args.pop("n"), DEV, **args)
    ops_max = ops.MT_MAX_WORDS
    with pytest.raises(ValueError, match="beyond 2\\*\\*31"):
        ops.randn_mt19937(1, ops_max - 100, 99, DEV)  # the tail's 16 words count: 99 + 16 > 100
    with pytest.raises(ValueError, match="beyond 2\\*\\*31"):
        ops.randn_mt19937(1, ops_max - 96, 112, DEV)


def test_window_entry_point_checks_before_launching():
    buf = ctypes.create_string_buffer(4096 + 16)
    p = (ctypes.addressof(buf) + 15) & ~15

    def call(offset, n, lo, hi, z=p):
        _native.call("tio_randn_mt19937_window", 1, offset, n, lo, hi, z, p, p, 64, None)

    with pytest.raises(RuntimeError, match="null pointer"):
        call(0, 32, 0, 32, z=None)
    for n, lo, hi in [(15, 0, 15), (32, 4, 4), (32, 0, 33)]:
        with pytest.raises(RuntimeError, match="lo < hi <= n"):
            call(0, n, lo, hi)
    with pytest.raises(RuntimeError, match="beyond stream word 2\\^31"):
        call(ops.MT_MAX_WORDS - 40, 30, 0, 30)  # 30 + 16 words
    with pytest.raises(RuntimeError, match="workspace too small"):
        call(0, 33, 0, 33)
    with pytest.raises(RuntimeError, match="multiples of 16"):
        _native.call("tio_randn_mt19937", 1, 8, 32, p, p, p, 1 << 20, None)


def test_window_workspace_counts_the_tail_segment():
    lib = _native.lib()
    states = lambda q_hi: (q_hi + 64) * 624 * 4  # start states of segments q < q_hi, + one per coarse jump
    assert lib.tio_randn_mt19937_window_workspace_bytes(SEGMENT - 32, 32) == states(1)
    assert lib.tio_randn_mt19937_window_workspace_bytes(SEGMENT - 20, 20) == states(2)  # tail at 2^21
    assert lib.tio_randn_mt19937_window_workspace_bytes(SEGMENT - 37, 20) == states(1)
    for offset, n in [(0, 16), (SEGMENT - 16, 32), (5 * SEGMENT, 4096)]:
        assert lib.tio_randn_mt19937_window_workspace_bytes(offset, n) <= lib.tio_randn_mt19937_workspace_bytes(offset, n)


def _stage(params, monkeypatch):
    """Noise's stage with device draws recorded instead of made: ((seed, offset, n, lo, hi), ...)."""
    made = []

    def fake(seed, offset, n, device, out=None, *, lo=0, hi=None):
        made.append((seed, offset, n, lo, hi))
        return torch.zeros(hi - lo)

    monkeypatch.setattr(ops, "randn_mt19937", fake)
    monkeypatch.setattr(intensity, "_noise_mode", lambda: "exact")
    return intensity._noise_stage_factory(params), made


def _image(shape):
    return types.SimpleNamespace(data=types.SimpleNamespace(shape=shape, device=torch.device(DEV)))


def test_slices_are_windows_of_the_whole_batch_draw(monkeypatch):
    """Rows [b0, b1) of each draw are outputs [per*b0, per*b1) of the draw over all B rows; the
    second image and the second Rician draw start where the ragged draws before them ended."""
    params = {"mean": 0.0, "std": 0.1, "seed": 77, "rician": True}
    per, total = 21 * 18 * 23, 5
    stage, made = _stage(params, monkeypatch)
    stage(_image((5, 1, 21, 18, 23)), 0)
    stage(_image((5, 1, 21, 18, 23)), 1)
    whole = list(made)
    words = ops.mt_draw_words(per * total)
    assert [m[1] for m in whole] == [0, words, 2 * words, 3 * words]
    assert all(m[2:] == (per * total, 0, per * total) for m in whole)
    for b0, b1 in [(0, 1), (1, 4), (4, 5)]:
        stage, made = _stage(params, monkeypatch)
        with chunk_scope(ChunkInfo(b0, b1, total, {})):
            stage(_image((b1 - b0, 1, 21, 18, 23)), 0)
            stage(_image((b1 - b0, 1, 21, 18, 23)), 1)
        assert made == [(77, m[1], per * total, per * b0, per * b1) for m in whole]


def test_one_draw_is_left_to_the_fused_call(monkeypatch):
    params = {"mean": 0.0, "std": 0.1, "seed": 5, "rician": False}
    stage, made = _stage(params, monkeypatch)
    first = stage(_image((3, 1, 5, 7, 3)), 0)  # 315 values: 331 words
    with chunk_scope(ChunkInfo(1, 2, 3, {})):
        stage2, _ = _stage(params, monkeypatch)
        sliced = stage2(_image((1, 1, 5, 7, 3)), 0)
    assert made == [] and first["z_replay"] == (5, 0, 315, 0) and sliced["z_replay"] == (5, 0, 315, 105)


def test_small_and_out_of_reach_draws_stay_on_the_host(monkeypatch):
    """A draw of < 16 values takes torch's scalar path: it and every later draw are host draws.
    A draw past the reach is a host draw after the generator skips the device draws' words."""
    params = {"mean": 0.0, "std": 0.1, "seed": 5, "rician": False}
    stage, made = _stage(params, monkeypatch)
    small = stage(_image((1, 1, 3, 2, 2)), 0)
    later = stage(_image((1, 1, 20, 20, 20)), 1)
    assert made == [] and "z_host" in small and "z_host" in later
    g = torch.Generator().manual_seed(5)
    torch.randn(12, generator=g)
    assert torch.equal(later["z_host"], torch.randn((1, 1, 20, 20, 20), generator=g))

    monkeypatch.setattr(ops, "MT_MAX_WORDS", 200)
    stage, made = _stage(params, monkeypatch)
    near = stage(_image((1, 1, 5, 7, 3)), 0)  # 105 values, 121 words
    far = stage(_image((1, 1, 5, 7, 3)), 1)   # would end at 242 > 200
    assert near["z_replay"] == (5, 0, 105, 0) and "z_host" in far
    g = torch.Generator().manual_seed(5)
    torch.randn(105, generator=g)
    assert torch.equal(far["z_host"], torch.randn((1, 1, 5, 7, 3), generator=g))


def test_ragged_batches_support_chunks():
    def batch(shape, k=2):
        g = torch.Generator().manual_seed(1)
        return _scalar_batch({f"i{i}": torch.rand(shape, generator=g) for i in range(k)}, shape[0])

    assert tio.Noise().supports_chunks(batch((4, 1, 21, 18, 23)))
    assert tio.Noise(rician=True).supports_chunks(batch((3, 2, 5, 7, 3)))
    assert not tio.Noise().supports_chunks(batch((3, 1, 1, 2, 2)))  # 12 values: torch's scalar path
    big = types.SimpleNamespace(data=torch.empty(1).expand(2, 1, 1024, 1024, 520))  # 2^30 + 2^24 values
    noise = tio.Noise(rician=True)
    noise._get_images = lambda _: {"t1": big}
    assert not noise.supports_chunks(None)  # two draws: beyond 2^31 words
