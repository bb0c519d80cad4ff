"""`tio_intensity_pass1_with_normals`: the first intensity pass and the exact-noise normals from one
persistent kernel.  Both outputs must be what the two stand-alone entry points write, bit for bit
(`tio_intensity_fused` restricted to bias + the I axis, and `tio_randn_mt19937`), and the fused
chain that takes this route must return what it returns with the normals supplied."""

import numpy as np
import pytest
import torch

from torchio_b200 import ops, tables

DEV = "cuda"
SEGMENT = 1 << 21  # words per segment of the replay (csrc/mt19937_layout.h)


def _sigma(radius: int) -> float:
    """A sigma whose taps have radius max(ceil(3 sigma), 1) == radius (0 = no blur)."""
    return 0.0 if radius == 0 else (radius - 0.5) / 3.0


def _inputs(b, c, shape, radii, bias, seed):
    """x, the blur tables of per-element radii (I, J, K) and a coarse bias grid with one identity
    row, all on the device, as keyword arguments of the ops calls."""
    rng = np.random.default_rng(seed)
    x = torch.as_tensor(rng.normal(0, 50, (b, c, *shape)).astype(np.float32)).to(DEV)
    t = tables.blur_tables([[_sigma(r) for r in radii[(e + b) % len(radii)]] for e in range(b)], b)
    kw = dict(taps=t.taps.to(DEV), radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask)
    if bias:
        ident = np.zeros(b, dtype=np.uint8)
        ident[-1] = b > 1
        kw["coarse"] = torch.as_tensor(rng.normal(0, 0.4, (b, c, 3, 2, 4)).astype(np.float32)).to(DEV)
        kw["bias_identity"] = torch.as_tensor(ident).to(DEV)
    return x, kw


# element 0 has no I-axis blur (pure streaming), element 1 the widest table radius, element 2 one between
RADII = [(0, 2, 1), (6, 0, 3), (3, 1, 0)]
CASES = [
    # b, c, (I, J, K): J % 4 != 0 and K < 256 leave ragged tiles; numel % 16 == 0
    (1, 1, (8, 6, 20)),
    (3, 1, (8, 6, 20)),
    (3, 2, (4, 5, 272)),   # two k-blocks, the second one ragged
    (1, 1, (30, 9, 64)),   # more than two unrolled groups of 13 planes
]


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("offset", [0, SEGMENT - 512], ids=["offset0", "across-segments"])
@pytest.mark.parametrize("case", CASES, ids=[f"b{c[0]}c{c[1]}-{'x'.join(map(str, c[2]))}" for c in CASES])
def test_both_outputs_equal_the_stand_alone_calls(case, offset, bias):
    b, c, shape = case
    x, kw = _inputs(b, c, shape, RADII, bias, seed=b + shape[2])
    seed = 1234567 + b
    first, z = ops.intensity_pass1_with_normals(x, seed, offset, **kw)
    want_first = ops.intensity_fused(x, **{**kw, "axes_mask": kw["axes_mask"] & 1})
    want_z = ops.randn_mt19937(seed, offset, x.numel(), DEV).view(x.shape)
    assert torch.equal(z, want_z)
    assert torch.equal(first, want_first)


@pytest.mark.gpu
def test_a_cta_that_runs_a_second_segment_and_many_tiles():
    """More segments than an H100 has SMs: every CTA takes a second segment after a barrier over
    its normal-stage threads, and fetches tiles from the counter many times."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    b, shape = 5, (384, 384, 384)
    assert b * int(np.prod(shape)) > (sms + 1) * SEGMENT
    x = torch.rand((b, 1, *shape), device=DEV)
    t = tables.blur_tables([[_sigma(r) for r in RADII[e % 3]] for e in range(b)], b)
    kw = dict(taps=t.taps.to(DEV), radius=t.radius.to(DEV), big_r=t.big_r, axes_mask=t.axes_mask,
              coarse=torch.randn((b, 1, 4, 4, 4), device=DEV) * 0.3)
    first, z = ops.intensity_pass1_with_normals(x, 99, 4096, **kw)
    assert torch.equal(z, ops.randn_mt19937(99, 4096, x.numel(), DEV).view(x.shape))
    del z
    assert torch.equal(first, ops.intensity_fused(x, **{**kw, "axes_mask": kw["axes_mask"] & 1}))


def _entry_points(monkeypatch, fn):
    """fn() and the library entry points it called, in order."""
    from torchio_b200 import _native

    called, real = [], _native.call

    def spy(name, *args):
        called.append(name)
        return real(name, *args)

    monkeypatch.setattr(_native, "call", spy)
    out = fn()
    monkeypatch.setattr(_native, "call", real)
    return out, called


@pytest.mark.gpu
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_fused_chain_takes_the_route_and_keeps_its_bits(bias, monkeypatch):
    """bias -> blur -> noise -> gamma with the draw handed over as (seed, offset): the combined
    entry point is called, and the result equals the chain run on supplied normals; element 1 is gated out
    of the noise (keep = 0)."""
    b, c, shape = 3, 1, (8, 6, 20)
    x, kw = _inputs(b, c, shape, RADII, bias, seed=5)
    kw.update(mean=torch.tensor([0.1, 0.0, -0.2], device=DEV), std=torch.tensor([0.5, 0.0, 2.0], device=DEV),
              keep=torch.tensor([1, 0, 1], dtype=torch.uint8, device=DEV), noise_mode=1,
              gamma=torch.tensor([0.8, 1.0, 1.3], device=DEV))
    seed, offset = 42, 3 * 16
    got, called = _entry_points(monkeypatch, lambda: ops.intensity_fused(x, **kw, z_replay=(seed, offset)))
    assert called == ["tio_intensity_pass1_with_normals", "tio_intensity_fused"]
    z = ops.randn_mt19937(seed, offset, x.numel(), DEV).view(x.shape)
    assert torch.equal(got, ops.intensity_fused(x, **kw, z=z))


@pytest.mark.gpu
def test_chains_the_kernel_does_not_cover_use_the_two_calls(monkeypatch):
    """Rows that are not a multiple of 16 bytes (K % 4 != 0) and chains without a first pass make
    their normals with the stand-alone replay; the result is the supplied-normals one."""
    for shape, radii in [((8, 4, 18), RADII), ((8, 6, 20), [(0, 2, 1)])]:
        x, kw = _inputs(2, 1, shape, radii, False, seed=7)
        kw.update(mean=torch.zeros(2, device=DEV), std=torch.ones(2, device=DEV), noise_mode=1)
        got, called = _entry_points(monkeypatch, lambda: ops.intensity_fused(x, **kw, z_replay=(7, 32)))
        assert called == ["tio_randn_mt19937", "tio_intensity_fused"]
        z = ops.randn_mt19937(7, 32, x.numel(), DEV).view(x.shape)
        assert torch.equal(got, ops.intensity_fused(x, **kw, z=z))


def test_refuses_what_it_does_not_cover_before_launching():
    """No GPU needed: the checks come first."""
    import ctypes

    from torchio_b200 import _native

    buf = ctypes.create_string_buffer(4096 + 16)
    p = (ctypes.addressof(buf) + 15) & ~15

    def call(k, r, dst):
        _native.call("tio_intensity_pass1_with_normals", p, dst, 1, 1, 2, 2, k, None, 0, 0, 0, None, 0,
                     p, p, r, 1, 0, 0, 16, p + 2048, p, p, 1 << 20, None)

    with pytest.raises(RuntimeError, match="alias"):
        call(16, 2, p)
    with pytest.raises(RuntimeError, match="R <= 6"):
        call(16, 7, p + 1024)
    with pytest.raises(RuntimeError, match="K % 4"):
        call(18, 2, p + 1024)
