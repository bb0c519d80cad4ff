"""GPU parity at the ops / C-ABI level against the C oracle on seeded random
parameters, including the edge cases the reference's tests exercise: 2-D
inputs, odd shapes, large rotations, coordinates far out of bounds,
pass-through rows, multi-channel data, every label dtype."""

import ctypes
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _orc():
    from oracle import c_port

    return c_port


def _random_matrix(rng, shape, big=False):
    ang = rng.uniform(-0.6, 0.6, 3) if big else rng.uniform(-0.2, 0.2, 3)
    cx, sx, cy, sy, cz, sz = np.cos(ang[0]), np.sin(ang[0]), np.cos(ang[1]), np.sin(ang[1]), np.cos(ang[2]), np.sin(ang[2])
    rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    rs = rz @ ry @ rx @ np.diag(rng.uniform(0.8, 1.25, 3))
    c = (np.asarray(shape) - 1) / 2
    m = np.eye(4)
    m[:3, :3] = rs
    m[:3, 3] = c - rs @ c + rng.uniform(-4, 4, 3) * (5 if big else 1)
    return m.astype(np.float32)[:3].reshape(12)


def _run_both(data, mat, cp, flags, sp_in, sp_out, affine_first, mode, fill, box_hint=-1, exact_coords=True):
    from torchio_b200 import ops

    c_port = _orc()
    b, c = data.shape[:2]
    shape = data.shape[2:]
    dev = torch.device("cuda")
    mat_t = torch.as_tensor(mat)
    cp_t = None if cp is None else torch.as_tensor(cp)
    fl_t = None if flags is None else torch.as_tensor(flags)
    fill_t = None if fill is None else torch.as_tensor(fill, dtype=torch.float32)
    got = ops.resample(
        data.to(dev), mat_t.to(dev), None if cp_t is None else cp_t.to(dev),
        None if fl_t is None else fl_t.to(dev), sp_in, sp_out, affine_first=affine_first,
        mode=mode, fill=None if fill_t is None else fill_t.to(dev), box_hint=box_hint,
        exact_coords=exact_coords,
    ).cpu()
    want = torch.empty_like(data)
    ni, nj, nk = (0, 0, 0) if cp is None else cp.shape[1:4]
    spi = torch.as_tensor(np.asarray(sp_in, dtype=np.float32))
    spo = torch.as_tensor(np.asarray(sp_out, dtype=np.float32))
    p = c_port._p
    rc = c_port.lib().orc_resample(
        p(data), p(want), c_port._DTYPES[data.dtype], b, c, *shape, *shape, p(mat_t), p(cp_t),
        p(fl_t), ni, nj, nk, p(spi), p(spo), int(affine_first), mode, p(fill_t),
    )
    assert rc == 0
    return got, want


SHAPES = [(33, 29, 70), (16, 16, 1), (7, 5, 3), (64, 48, 40), (40, 36, 64), (18, 50, 4)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("elastic", [False, True])
def test_resample_bit_exact_vs_c_oracle(shape, mode, elastic):
    rng = np.random.default_rng(hash((shape, mode, elastic)) % 2**32)
    b, c = 3, 2
    g = torch.Generator().manual_seed(5)
    data = torch.rand((b, c, *shape), generator=g) - 0.25
    mat = np.stack([_random_matrix(rng, shape, big=(i == 1)) for i in range(b)])
    flags = np.zeros(b, dtype=np.uint8)
    cp = None
    if elastic:
        cp = rng.uniform(-3, 3, (b, 5, 6, 7, 3)).astype(np.float32)
        flags[:] = 2
        flags[2] = 0  # one element without a grid
    for affine_first in ((True, False) if elastic else (True,)):
        for fill in (None, np.array([-1.0, 0.5], dtype=np.float32)):
            got, want = _run_both(data, mat, cp, flags, (0.8, 1.1, 2.0), (0.8, 1.1, 2.0),
                                  affine_first, mode, fill)
            assert torch.equal(got, want), int((got != want).sum())
            if mode == 1:
                # TMA tile paths: exact = same coordinates, FMA tap blending; fast = one-fma
                # coordinates where no tap leaves the volume.  Same fill decisions either way.
                for hint, exact in ((0, True), (20, True), (22, True), (28, True), (32, True),
                                    (0, False), (20, False), (22, False), (24, False), (28, False), (32, False)):
                    fast, _ = _run_both(data, mat, cp, flags, (0.8, 1.1, 2.0), (0.8, 1.1, 2.0),
                                        affine_first, mode, fill, box_hint=hint, exact_coords=exact)
                    assert float((fast - want).abs().max()) <= (1e-6 if exact else 1e-4), (hint, exact)
                    if fill is not None:
                        for ch in range(c):
                            filled_fast = fast[:, ch] == float(fill[ch])
                            filled_want = want[:, ch] == float(fill[ch])
                            assert torch.equal(filled_fast, filled_want)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64])
def test_label_dtypes_nearest_exact(dtype):
    rng = np.random.default_rng(3)
    shape = (20, 18, 37)
    lo, hi = (0, 200) if dtype == torch.uint8 else (-100, 100)
    data = torch.randint(lo, hi, (2, 1, *shape), dtype=torch.int64).to(dtype)
    mat = np.stack([_random_matrix(rng, shape) for _ in range(2)])
    for fill in (None, np.array([7.0], dtype=np.float32)):
        got, want = _run_both(data, mat, None, None, (1, 1, 1), (1, 1, 1), True, 0, fill)
        assert torch.equal(got, want)


def test_passthrough_rows_are_bit_copies_and_far_oob_is_fill():
    rng = np.random.default_rng(9)
    shape = (12, 10, 33)
    data = torch.rand((3, 1, *shape))
    mat = np.stack([_random_matrix(rng, shape) for _ in range(3)])
    mat[2, 3] = 1e6  # everything out of bounds
    flags = np.array([1, 0, 0], dtype=np.uint8)
    fill = np.array([0.25], dtype=np.float32)
    got, want = _run_both(data, mat, None, flags, (1, 1, 1), (1, 1, 1), True, 1, fill)
    assert torch.equal(got, want)
    assert torch.equal(got[0], data[0])
    assert bool((got[2] == 0.25).all())


def test_min_sample0():
    from torchio_b200 import ops

    for shape in ((2, 3, 16, 16, 16), (1, 2, 5, 7, 3)):
        x = torch.rand(shape) - 0.7
        got = ops.min_sample0(x.cuda()).cpu()
        assert torch.equal(got, x[0].reshape(shape[1], -1).min(dim=1).values)


def test_intensity_kernels_vs_c_oracle():
    """Each intensity stage on its own: a tio_intensity_fused call with only that stage set."""
    from torchio_b200 import ops

    c_port = _orc()
    p = c_port._p
    lib = c_port.lib()
    g = torch.Generator().manual_seed(11)
    for shape in ((3, 2, 24, 20, 16), (2, 1, 9, 7, 5)):
        b, c = shape[:2]
        x = torch.rand(shape, generator=g) - 0.3
        n = x[0].numel()
        # bias
        coarse = torch.randn((b, c, 4, 5, 6), generator=g) * 0.5
        ident = torch.tensor([0, 1, 0][:b], dtype=torch.uint8)
        for divide in (0, 1):
            want = torch.empty_like(x)
            lib.orc_bias_field(p(x), p(want), b, c, *shape[2:], p(coarse), 4, 5, 6, p(ident), divide)
            got = ops.intensity_fused(x.cuda(), coarse=coarse.cuda(), bias_identity=ident.cuda(),
                                      bias_divide=bool(divide)).cpu()
            assert (got - want).abs().max() <= 2e-6 * float(want.abs().max())
            assert torch.equal(got[1], x[1])
        # blur
        from torchio_b200 import tables

        sig = np.array([[0.7, 0.0, 1.9], [0.0, 0.0, 0.0], [1.2, 0.6, 0.4]][:b])
        t = tables.blur_tables(sig, b)
        want = torch.empty_like(x)
        lib.orc_blur(p(x), p(want), None, b, c, *shape[2:], p(t.taps), p(t.radius), t.big_r,
                     p(t.identity))
        got = ops.blur(x.cuda(), t.taps.cuda(), t.radius.cuda(), t.big_r, t.axes_mask,
                       t.identity.cuda()).cpu()
        assert (got - want).abs().max() <= 2e-6
        assert torch.equal(got[1], x[1])
        # noise (gaussian + rician + keep)
        z, z2 = torch.randn(shape, generator=g), torch.randn(shape, generator=g)
        mean = torch.tensor([0.1, -0.2, 0.0][:b]); std = torch.tensor([0.2, 0.1, 0.3][:b])
        keep = torch.tensor([1, 0, 1][:b], dtype=torch.uint8)
        for zz in (None, z2):
            want = torch.empty_like(x)
            lib.orc_noise(p(x), p(want), b, ctypes.c_int64(n), p(mean), p(std), p(keep), p(z), p(zz))
            got = ops.intensity_fused(x.cuda(), mean=mean.cuda(), std=std.cuda(), keep=keep.cuda(),
                                      z=z.cuda(), z2=None if zz is None else zz.cuda(), noise_mode=1,
                                      rician=zz is not None).cpu()
            assert (got - want).abs().max() <= 1e-6
            assert torch.equal(got[1], x[1])
        # gamma
        gam = torch.tensor([0.8, 1.0, 1.3][:b])
        want = torch.empty_like(x)
        lib.orc_gamma(p(x), p(want), b, ctypes.c_int64(n), p(gam))
        got = ops.intensity_fused(x.cuda(), gamma=gam.cuda()).cpu()
        assert (got - want).abs().max() <= 2e-6
        assert torch.equal(got[1], x[1])


def test_philox_noise_statistics():
    """The Philox stream Noise uses under TIO_B200_NOISE=philox (noise_mode 2)."""
    from torchio_b200 import ops

    x = torch.zeros((2, 1, 64, 64, 64), device="cuda")
    mean = torch.tensor([0.5, -1.0], device="cuda")
    std = torch.tensor([2.0, 0.5], device="cuda")

    def philox(seed):
        return ops.intensity_fused(x, mean=mean, std=std, noise_mode=2, philox_seed=seed).cpu()

    y = philox(1234)
    for b in range(2):
        assert abs(float(y[b].mean()) - float(mean[b])) < 0.02 * float(std[b]) + 1e-3
        assert abs(float(y[b].std()) - float(std[b])) < 0.01 * float(std[b])
    y2 = philox(1234)
    assert torch.equal(y, y2)
    y3 = philox(1235)
    assert not torch.equal(y, y3)
    kurt = float(((y[0] - y[0].mean()) ** 4).mean() / y[0].var() ** 2)
    assert abs(kurt - 3.0) < 0.05


@pytest.mark.parametrize("shape", [(2, 1, 40, 36, 64), (3, 2, 19, 33, 70), (2, 1, 9, 7, 5),
                                   (1, 1, 24, 20, 1), (2, 1, 70, 40, 132)])
@pytest.mark.parametrize("sigma_max", [1.9, 4.5])
def test_fused_chain_equals_sequential_kernels(shape, sigma_max):
    """tio_intensity_fused == bias -> blur -> noise -> gamma one after another
    (C oracle), for vector and scalar paths, radii up to 14, ragged tiles."""
    from torchio_b200 import ops, tables

    c_port = _orc()
    p = c_port._p
    lib = c_port.lib()
    b, c = shape[:2]
    g = torch.Generator().manual_seed(17)
    rng = np.random.default_rng(17)
    x = torch.rand(shape, generator=g) - 0.2
    n = x[0].numel()
    coarse = torch.randn((b, c, 4, 5, 6), generator=g) * 0.4
    bias_ident = torch.zeros(b, dtype=torch.uint8)
    sig = rng.uniform(0.0, sigma_max, (b, 3))
    sig[:, 2] = np.where(shape[4] == 1, 0.0, sig[:, 2])
    if b > 1:
        sig[1] = 0.0  # one identity row
        bias_ident[1] = 1
    t = tables.blur_tables(sig, b)
    z = torch.randn(shape, generator=g)
    mean = torch.tensor(rng.uniform(-0.1, 0.1, b), dtype=torch.float32)
    std = torch.tensor(rng.uniform(0.0, 0.3, b), dtype=torch.float32)
    keep = torch.ones(b, dtype=torch.uint8)
    gam = torch.tensor(np.exp(rng.uniform(-0.3, 0.3, b)), dtype=torch.float32)
    if b > 1:
        keep[1] = 0
        gam[1] = 1.0
    # oracle chain
    s1, s2, s3, s4 = (torch.empty_like(x) for _ in range(4))
    lib.orc_bias_field(p(x), p(s1), b, c, *shape[2:], p(coarse), 4, 5, 6, p(bias_ident), 0)
    lib.orc_blur(p(s1), p(s2), None, b, c, *shape[2:], p(t.taps), p(t.radius), t.big_r, p(t.identity))
    lib.orc_noise(p(s2), p(s3), b, ctypes.c_int64(n), p(mean), p(std), p(keep), p(z), None)
    lib.orc_gamma(p(s3), p(s4), b, ctypes.c_int64(n), p(gam))
    dev = "cuda"
    got = ops.intensity_fused(
        x.to(dev), coarse=coarse.to(dev), bias_identity=bias_ident.to(dev),
        taps=t.taps.to(dev), radius=t.radius.to(dev), big_r=t.big_r, axes_mask=t.axes_mask,
        mean=mean.to(dev), std=std.to(dev), keep=keep.to(dev), z=z.to(dev), noise_mode=1,
        gamma=gam.to(dev),
    ).cpu()
    rngv = float(s4.max() - s4.min())
    assert float((got - s4).abs().max()) <= 3e-6 * rngv
    if b > 1:
        assert torch.equal(got[1], x[1])  # fully gated row: bit-exact copy
    # blur alone through the same kernels
    got_b = ops.blur(x.to(dev), t.taps.to(dev), t.radius.to(dev), t.big_r, t.axes_mask,
                     t.identity.to(dev)).cpu()
    want_b = torch.empty_like(x)
    lib.orc_blur(p(x), p(want_b), None, b, c, *shape[2:], p(t.taps), p(t.radius), t.big_r, p(t.identity))
    assert float((got_b - want_b).abs().max()) <= 2e-6


def test_fused_compose_equals_unfused_compose():
    import warnings

    import torchio_b200 as tio

    subjects = []
    for b in range(3):
        gsub = torch.Generator().manual_seed(50 + b)
        subjects.append(tio.Subject(t1=tio.ScalarImage(torch.rand((1, 40, 36, 32), generator=gsub)),
                                    seg=tio.LabelMap(torch.zeros((1, 40, 36, 32), dtype=torch.int16))))
    outs = []
    for fuse in (True, False):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pipe = tio.Compose([tio.BiasField(), tio.Blur(std=(0, 2)), tio.Noise(std=(0, 0.25)),
                                tio.Gamma(log_gamma=(-0.3, 0.3))])
        pipe.fuse = fuse
        torch.manual_seed(5)
        out = pipe(tio.SubjectsBatch.from_subjects(subjects).to("cuda"))
        assert [t.name for t in out.applied_transforms] == ["BiasField", "Blur", "Noise", "Gamma"]
        outs.append(out)
    a, b = outs[0].images["t1"].data, outs[1].images["t1"].data
    assert float((a - b).abs().max()) <= 3e-6 * float(b.max() - b.min())
    assert json_equal(outs[0].applied_transforms, outs[1].applied_transforms)


def json_equal(h1, h2):
    import json

    f = lambda h: json.dumps([{"name": t.name, "params": t.params} for t in h], sort_keys=True)
    return f(h1) == f(h2)


@pytest.mark.parametrize("seed,offset,n", [(0, 0, 16), (1234, 0, 4096), (7, 0, 3 * 2**20 + 1600),
                                           (2**31 - 1, 16 * 12345, 2**20), (99, 40 * 2**20, 2**21 + 32)])
def test_device_mt19937_randn_matches_torch_cpu_stream(seed, offset, n):
    """K4a: the device replay equals torch.randn(generator=CPU(seed)) element for
    element (to ~1 ulp of libm), at any 16-aligned stream position, across
    segment (2^20) and coarse (2^25) jump boundaries."""
    from torchio_b200 import ops

    g = torch.Generator().manual_seed(seed)
    if offset:
        torch.randn(offset, generator=g)
    want = torch.randn(n, generator=g)
    got = ops.randn_mt19937(seed, offset, n, "cuda").cpu()
    diff = (got - want).abs()
    # same uniforms bit for bit; log/sin/cos differ (CUDA libm vs the host's): <= 4e-6 abs
    assert float(diff.max()) <= 4e-6, (float(diff.max()), int((diff > 4e-6).sum()))
    assert float((got == want).float().mean()) > 0.5


def test_noise_exact_mode_uses_device_stream_and_matches_reference():
    """Noise in exact mode == the oracle (host torch.randn) for aligned and ragged
    shapes, two images sharing one stream, and the second Rician draw."""
    import copy
    import warnings

    import torchio_b200 as tio
    from oracle import torch_port

    for shape, rician in (((2, 1, 16, 16, 16), False), ((3, 1, 8, 16, 10), True), ((2, 1, 5, 7, 3), False)):
        g = torch.Generator().manual_seed(3)
        imgs = {"t1": torch.rand(shape, generator=g), "t2": torch.rand(shape, generator=g)}
        batch = tio.SubjectsBatch({k: tio.ImagesBatch(v.clone().cuda(), [tio.AffineMatrix() for _ in range(shape[0])])
                                   for k, v in imgs.items()})
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            t = tio.Noise(mean=(-0.1, 0.1), std=(0.05, 0.25), rician=rician)
        torch.manual_seed(11)
        out = t(batch)
        params = out.applied_transforms[0].params
        ref = {k: {"kind": "scalar", "data": v.clone(), "affines": [np.eye(4)] * shape[0]} for k, v in imgs.items()}
        torch_port.noise(ref, json.loads(json.dumps(params)))
        for k in imgs:
            assert float((out.images[k].data.cpu() - ref[k]["data"]).abs().max()) <= 4e-6


def test_streamed_host_batch_equals_one_shot_rows(coords):
    """Compose streams a host-resident batch through the device in slices of the batch
    axis (copy in / kernels / copy out overlapped); every row, affine and the history
    must equal the one-shot path (tile-vs-general resample paths differ <= 1e-6)."""
    import json
    import warnings

    import torchio_b200 as tio

    def make():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            return tio.Compose([
                tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10), p=0.8), tio.ElasticDeformation(),
                tio.BiasField(), tio.Blur(std=(0, 2), p=0.7), tio.Noise(std=(0, 0.25)),
                tio.Gamma(log_gamma=(-0.3, 0.3))], copy=False)

    g = torch.Generator().manual_seed(5)
    x = torch.rand((5, 1, 32, 40, 48), generator=g) + 0.1
    lab = (torch.rand((5, 1, 32, 40, 48), generator=g) * 4).to(torch.int16)

    def batch():
        return tio.SubjectsBatch({
            "t1": tio.ImagesBatch(x.clone(), [tio.AffineMatrix() for _ in range(5)]),
            "seg": tio.ImagesBatch(lab.clone(), [tio.AffineMatrix() for _ in range(5)],
                                   image_class=tio.LabelMap)})

    outs = []
    for chunk in (0, 2):
        pipe = make()
        pipe.chunk_size = chunk
        torch.manual_seed(77)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            outs.append(pipe(batch()))
    one, streamed = outs
    assert streamed.images["t1"].data.device.type == "cpu"
    rng = float(one.images["t1"].data.max() - one.images["t1"].data.min())
    # (fast coordinates are box relative, and the box edge follows the slice's matrices)
    tol = 3e-6 if coords == "exact" else 3e-5
    assert float((one.images["t1"].data - streamed.images["t1"].data).abs().max()) <= tol * rng
    assert torch.equal(one.images["seg"].data, streamed.images["seg"].data)
    for a, b in zip(one.images["t1"].affines, streamed.images["t1"].affines):
        assert a == b
    h1 = [(t.name, json.dumps(t.params, sort_keys=True)) for t in one.applied_transforms]
    h2 = [(t.name, json.dumps(t.params, sort_keys=True)) for t in streamed.applied_transforms]
    assert h1 == h2


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.int32])
@pytest.mark.parametrize("elastic", [False, True])
def test_nearest_tile_path_is_bit_exact_with_general_path(dtype, elastic):
    """Label maps (nearest) through the TMA tile kernel == the general gather kernel,
    with and without a fill value, for every tiled label dtype."""
    from torchio_b200 import ops

    rng = np.random.default_rng(31)
    g = torch.Generator().manual_seed(9)
    lab = (torch.rand((3, 2, 40, 48, 64), generator=g) * 100).to(dtype).cuda()
    mats = []
    for b in range(3):
        ang = rng.uniform(-0.2, 0.2, 3)
        cx, sx, cy, sy, cz, sz = np.cos(ang[0]), np.sin(ang[0]), np.cos(ang[1]), np.sin(ang[1]), np.cos(ang[2]), np.sin(ang[2])
        r = (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
             @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])) * rng.uniform(0.9, 1.1)
        c = (np.array(lab.shape[2:]) - 1) / 2
        m = np.eye(4); m[:3, :3] = r; m[:3, 3] = c - r @ c + rng.uniform(-2, 2, 3)
        mats.append(m.astype(np.float32)[:3].reshape(12))
    mat = torch.tensor(np.stack(mats)).cuda()
    cp = flags = None
    if elastic:
        cp = torch.tensor(rng.uniform(-4, 4, (3, 7, 7, 7, 3)).astype(np.float32)).cuda()
        flags = torch.tensor([2, 2, 0], dtype=torch.uint8).cuda()
    one = (1.0, 1.0, 1.0)
    for fill in (None, torch.tensor([7.0, 3.0]).cuda()):
        kw = dict(affine_first=True, mode=ops.NEAREST, fill=fill)
        tiled = ops.resample(lab, mat, cp, flags, one, one, **kw)
        general = ops.resample(lab, mat, cp, flags, one, one, box_hint=-1, **kw)
        assert torch.equal(tiled, general)
        assert tiled.dtype == dtype


def test_stream_yields_what_the_plain_calls_return():
    """`for out in pipeline.stream(batches)` keeps a batch in flight (copy-in of batch n+1 under
    the copy-out of batch n); every yielded batch, its history and the RNG consumption must
    equal calling the pipeline batch by batch."""
    import json
    import warnings

    import torchio_b200 as tio

    def make():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            pipe = tio.Compose([
                tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10), p=0.8), tio.ElasticDeformation(),
                tio.BiasField(), tio.Blur(std=(0, 2)), tio.Noise(std=(0, 0.25)),
                tio.Gamma(log_gamma=(-0.3, 0.3))], copy=False)
        pipe.chunk_size = 2
        return pipe

    def batches():
        for t in range(4):
            g = torch.Generator().manual_seed(50 + t)
            x = (torch.rand((5, 1, 24, 28, 32), generator=g) + 0.1).pin_memory()
            lab = (torch.rand((5, 1, 24, 28, 32), generator=g) * 4).to(torch.int16).pin_memory()
            yield tio.SubjectsBatch({
                "t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(5)]),
                "seg": tio.ImagesBatch(lab, [tio.AffineMatrix() for _ in range(5)], image_class=tio.LabelMap)})

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        torch.manual_seed(91)
        pipe = make()
        plain = [pipe(b) for b in batches()]
        after_plain = torch.rand(1).item()
        for depth in (0, 1, 3):
            torch.manual_seed(91)
            streamed = list(make().stream(batches(), depth=depth))
            assert torch.rand(1).item() == after_plain
            assert len(streamed) == len(plain)
            for a, b in zip(plain, streamed):
                assert b.images["t1"].data.device.type == "cpu"
                assert torch.equal(a.images["t1"].data, b.images["t1"].data)
                assert torch.equal(a.images["seg"].data, b.images["seg"].data)
                ha = [(t.name, json.dumps(t.params, sort_keys=True)) for t in a.applied_transforms]
                hb = [(t.name, json.dumps(t.params, sort_keys=True)) for t in b.applied_transforms]
                assert ha == hb
    ticket = make().submit(next(batches()))
    out = ticket.result()
    assert ticket.done() and out.images["t1"].data.device.type == "cpu"


def test_remap_vector_path_equals_c_oracle():
    """tio_remap's 128-bit path (rows that are multiples of 16 bytes): aligned / unaligned crops,
    every padding mode, flips along every axis (a K flip reverses the unit in registers), all
    element sizes — bit for bit against the C oracle."""
    from torchio_b200 import ops

    c_port = _orc()
    rng = np.random.default_rng(12)
    g = torch.Generator().manual_seed(12)
    for trial in range(48):
        dtype = [torch.float32, torch.int16, torch.uint8, torch.int64][trial % 4]
        shape = (int(rng.integers(5, 9)), int(rng.integers(5, 9)), 16 * int(rng.integers(1, 4)))
        x = (torch.rand((2, 2, *shape), generator=g) * 90).to(dtype)
        mode = ["constant", "replicate", "reflect", "circular"][(trial // 4) % 4]
        # K padding in multiples that keep the output row a multiple of 16 elements or not
        pad = [int(rng.integers(0, 4)) for _ in range(4)] + [int(rng.integers(0, 5)) * (4 if trial % 3 else 1),
                                                             int(rng.integers(0, 5)) * (4 if trial % 3 else 1)]
        pad[5] += (-(shape[2] + pad[4] + pad[5])) % 16  # output K a multiple of 16: vector path for every dtype
        if mode in ("reflect", "circular"):
            pad = [min(p, s - 1) for p, s in zip(pad, (shape[0], shape[0], shape[1], shape[1], shape[2], shape[2]))]
            pad[5] -= (shape[2] + pad[4] + pad[5]) % 16 if (shape[2] + pad[4] + pad[5]) % 16 <= pad[5] else 0
        out_shape = tuple(shape[a] + pad[2 * a] + pad[2 * a + 1] for a in range(3))
        offsets = (pad[0], pad[2], pad[4])
        bits = [int(rng.integers(0, 8)) for _ in range(2)]
        want = c_port.remap(x, out_shape, offsets, mode=mode, fill=7, flip_bits=bits)
        got = ops.remap(x.cuda(), out_shape, offsets, mode=mode, fill=7,
                        flip=torch.tensor(bits, dtype=torch.uint8, device="cuda")).cpu()
        assert torch.equal(got, want), (trial, dtype, mode, pad, bits)
        # crop back (negative offsets), aligned and unaligned starts along K
        back_shape = (shape[0], shape[1], 16)
        for k_off in (0, 3, 4):
            if pad[4] + k_off + 16 > out_shape[2]:
                continue
            offs = (-pad[0], -pad[2], -(pad[4] + k_off))
            want_b = c_port.remap(want, back_shape, offs, flip_bits=bits)
            got_b = ops.remap(want.cuda(), back_shape, offs,
                              flip=torch.tensor(bits, dtype=torch.uint8, device="cuda")).cpu()
            assert torch.equal(got_b, want_b), (trial, dtype, k_off, bits)


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.int32])
@pytest.mark.parametrize("elastic", [False, True])
def test_label_pv_tile_path_is_bit_exact_with_general_path_and_oracle(dtype, elastic):
    """label_interpolation="label" (TIO_LABEL_PV) through the TMA tile kernel == the general gather
    kernel == the oracle's one-hot / grid_sample / argmax restatement, on blocky label maps
    (boundaries everywhere), with big translations so that border tiles skip out-of-volume corners,
    and with an exactly axis-aligned half-voxel shift (argmax ties on every boundary voxel)."""
    from oracle import torch_port
    from torchio_b200 import ops

    rng = np.random.default_rng(77)
    shape = (48, 48, 64)
    i, j, k = (torch.arange(n) for n in shape)
    lab = (((i[:, None, None] // 5) * 3 + (j[None, :, None] // 7) * 5 + (k[None, None, :] // 6)) % 6)
    lab = torch.stack([lab, (lab * 7 + 1) % 5, lab.flip(0)]).to(dtype)[:, None].contiguous()  # (3,1,...)
    mats = []
    for b in range(3):
        ang = rng.uniform(-0.2, 0.2, 3)
        cx, sx, cy, sy, cz, sz = np.cos(ang[0]), np.sin(ang[0]), np.cos(ang[1]), np.sin(ang[1]), np.cos(ang[2]), np.sin(ang[2])
        r = (np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]]) @ np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
             @ np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])) * rng.uniform(0.9, 1.1)
        c = (np.array(shape) - 1) / 2
        m = np.eye(4); m[:3, :3] = r; m[:3, 3] = c - r @ c + rng.uniform(-6, 6, 3)
        mats.append(m)
    mats[2] = np.eye(4); mats[2][:3, 3] = (0.5, -0.5, 1.5)  # exact ties
    mat = torch.tensor(np.stack([m.astype(np.float32)[:3].reshape(12) for m in mats])).cuda()
    cp = flags = None
    if elastic:
        cp = torch.tensor(rng.uniform(-4, 4, (3, 7, 7, 7, 3)).astype(np.float32)).cuda()
        flags = torch.tensor([2, 2, 0], dtype=torch.uint8).cuda()
    one = (1.0, 1.0, 1.0)
    pad = torch.tensor([9.0]).cuda()
    kw = dict(affine_first=True, mode=ops.LABEL_PV, fill=pad)
    tiled = ops.resample(lab.cuda(), mat, cp, flags, one, one, **kw)
    general = ops.resample(lab.cuda(), mat, cp, flags, one, one, box_hint=-1, **kw)
    assert tiled.dtype == dtype
    assert torch.equal(tiled, general), int((tiled != general).sum())
    # the oracle's restatement element by element (its sampling grid from the same tables)
    for b in range(3):
        if elastic and b < 2:
            continue  # the displacement part of the grid is covered by the golden fixtures
        a_in = np.eye(4)
        grid = torch_port.map_homogeneous(torch_port.voxel_coordinates(shape), torch.tensor(mats[b], dtype=torch.float64).float())
        want = torch_port.label_partial_volume(lab[b:b + 1], grid, shape, a_in, a_in, False, "linear", 9.0)
        assert torch.equal(general[b:b + 1].cpu(), want), (b, int((general[b:b + 1].cpu() != want).sum()))
