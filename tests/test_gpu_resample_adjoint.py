"""K1ᵀ (`tio_resample_backward`) voxel by voxel against the float64 adjoint of the C oracle.

Each case calls the entry point with a workspace the test owns, so it reads back every tile's
record from the bounds pre-pass, and then checks:

(a) paths: the tile codes the case is built to reach (0 global-atomic fallback, 1 staged box,
    2 nothing sent, 3 pass-through copy) and the box edge the launch uses (24 or 32);
(b) every voxel within `adjoint_bound` of the oracle's grad64: gamma_m * abs64 for m terms, any
    order of fp32 additions, and no term for a coordinate that differs from the oracle's chain;
(c) exact voxels: NaN and Inf where the oracle has them, +0.0 (as bits) where no output voxel
    sends anything, and pass-through elements as bit copies of g.

Each case prints its code counts and its largest |gpu - grad64| / bound.
"""

import ctypes
import math
import time
import warnings
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import c_port
from test_resample_adjoint_oracle import adjoint_bound, check_adjoint
from torchio_b200 import _native, ops
from torchio_b200.transforms import spatial

pytestmark = pytest.mark.gpu

XT = 16


# ---- geometry ------------------------------------------------------------------------------------

def _rot(degrees):
    """3x3 rotation about the I, J, K axes in turn."""
    a, b, c = np.radians(degrees)
    rx = np.array([[1, 0, 0], [0, math.cos(a), -math.sin(a)], [0, math.sin(a), math.cos(a)]])
    ry = np.array([[math.cos(b), 0, math.sin(b)], [0, 1, 0], [-math.sin(b), 0, math.cos(b)]])
    rz = np.array([[math.cos(c), -math.sin(c), 0], [math.sin(c), math.cos(c), 0], [0, 0, 1]])
    return rz @ ry @ rx


def _mat(shape, *, zoom=(1, 1, 1), degrees=(0, 0, 0), shift=(0, 0, 0), out_shape=None):
    """Output-to-input voxel matrix (12 fp32): q = R diag(1 / zoom) (p - c_out) + c_in + shift,
    about the volumes' centres; zoom < 1 zooms out (an output tile reads a wider pre-image)."""
    out_shape = shape if out_shape is None else out_shape
    a = _rot(degrees) @ np.diag(1.0 / np.asarray(zoom, dtype=np.float64))
    c_in = (np.asarray(shape, dtype=np.float64) - 1) / 2
    c_out = (np.asarray(out_shape, dtype=np.float64) - 1) / 2
    m = np.zeros((3, 4))
    m[:, :3] = a
    m[:, 3] = c_in - a @ c_out + np.asarray(shift, dtype=np.float64)
    return m.astype(np.float32).reshape(12)


def _shift(v):
    """The identity plus a translation, exactly: q = p + v."""
    m = np.zeros((3, 4), np.float32)
    m[:, :3] = np.eye(3)
    m[:, 3] = v
    return m.reshape(12)


@dataclass
class Case:
    shape: tuple
    mats: list                    # (12,) fp32 per element; None = pass-through
    must: set                     # tile codes the case is built to reach
    allowed: set                  # every code the records may hold
    box: int = 24
    c: int = 1
    mode: int = ops.LINEAR
    fill: bool = False
    out_shape: tuple = None
    cps: list = None              # (ni, nj, nk, 3) per element or None
    affine_first: bool = True
    spacing_in: tuple = (1.0, 1.0, 1.0)
    spacing_out: tuple = (1.0, 1.0, 1.0)
    box_hint: int = None          # None: the product's `_box_hint`
    needs_32: bool = False        # some tiles fit the 32 box and not the 24 one
    poke: dict = field(default_factory=dict)  # (b, c, oi, oj, ok) -> value written into g

    def tables(self):
        b = len(self.mats)
        mat = np.stack([np.eye(4, dtype=np.float32)[:3].reshape(12) if m is None else m for m in self.mats])
        flags = np.array([1 if m is None else 0 for m in self.mats], np.uint8)
        cp = None
        if self.cps is not None:
            grid = next(g for g in self.cps if g is not None).shape
            cp = np.zeros((b, *grid), np.float32)
            for e, g in enumerate(self.cps):
                if g is not None:
                    cp[e] = g
                    flags[e] |= 2
        return mat, cp, flags


def _cp(rng, grid=(7, 6, 8), amplitude=4.0):
    g = rng.uniform(-amplitude, amplitude, (*grid, 3)).astype(np.float32)
    g[:2] = g[-2:] = 0  # as the reference zeroes the border control points
    return g


def _cases():
    rng = np.random.default_rng(7)
    S = (40, 36, 64)
    small = lambda sh, s=0: _mat(sh, degrees=(8, -5, 6), shift=(1.3, -0.7, 0.4 + s))  # noqa: E731
    cases = {
        # box and flush: K % 4 == 0 takes red.global.add.v4.f32, others the scalar tail, K = 1 is 2-D
        "flush_vector_k64": Case(S, [small(S), small(S, 1)], {1}, {1}),
        "flush_tail_k63": Case((40, 36, 63), [small((40, 36, 63)), small((40, 36, 63), 1)], {1}, {1}),
        "flush_tail_k61_fill": Case((33, 30, 61), [small((33, 30, 61))], {1}, {1, 2}, fill=True),
        "flat_k1": Case((34, 29, 1), [_mat((34, 29, 1), degrees=(0, 0, 20), shift=(2, -1, 0)),
                                      _mat((34, 29, 1), degrees=(0, 0, -35), zoom=(0.9, 1.1, 1))], {1}, {1}),
        "box32_zoom_out": Case((48, 48, 48), [_mat((48, 48, 48), zoom=(0.6, 0.62, 0.6), degrees=(3, 0, 0)),
                                              _mat((48, 48, 48), zoom=(0.65, 0.6, 0.61))],
                               {1}, {0, 1, 2}, box=32, fill=True, needs_32=True),
        # tile codes
        "code0_scale_035": Case((40, 37, 44), [_mat((40, 37, 44), zoom=(0.35, 0.35, 0.35))], {0}, {0, 2},
                                box=32),
        "code0_far_translation": Case((40, 36, 44), [_shift((2e6, 0, 0)), _shift((0, 0, -5e9)),
                                                     _shift((3.0e6, -3.0e6, 1e6))], {0}, {0}, box=24),
        "code2_outside": Case((40, 36, 44), [small((40, 36, 44)), _shift((0, 0, 400))], {1, 2}, {1, 2},
                              fill=True),
        "code3_passthrough": Case((40, 36, 44), [small((40, 36, 44)), None, small((40, 36, 44), 2)],
                                  {1, 3}, {1, 3}, c=2),
        "codes_0_1_2_one_element": Case((50, 44, 40), [_mat((50, 44, 40), degrees=(0, 0, 45),
                                                            zoom=(0.9, 0.9, 1), shift=(30, -4, 0))],
                                        {0, 1, 2}, {0, 1, 2}, box_hint=24, fill=True),
        # geometry (a displacement can carry a whole tile out of the volume: code 2)
        "elastic_and_affine_affine_first": Case(
            (41, 38, 36), [small((41, 38, 36)), small((41, 38, 36), 1), None],
            {1}, {0, 1, 2, 3}, box=32, cps=[_cp(rng), None, None], spacing_in=(1.0, 1.2, 0.9)),
        "elastic_and_affine_affine_last": Case(
            (41, 38, 36), [small((41, 38, 36)), _shift((0, 0, 0)), small((41, 38, 36), 2)],
            {1}, {0, 1, 2}, box=32, cps=[_cp(rng), _cp(rng), None], affine_first=False,
            spacing_out=(1.1, 0.9, 1.0),
            fill=True),
        "target_larger_and_smaller": Case(
            (30, 33, 25), [_mat((30, 33, 25), zoom=(45 / 30, 20 / 33, 37 / 25), degrees=(5, 0, 0),
                                out_shape=(45, 20, 37)),
                           _mat((30, 33, 25), zoom=(45 / 30, 20 / 33, 37 / 25), out_shape=(45, 20, 37))],
            {1}, {0, 1}, out_shape=(45, 20, 37), cps=[_cp(rng, (5, 6, 5)), None],
            spacing_out=(0.7, 1.6, 0.7), box=32, needs_32=True),
        # modes and fills
        "nearest": Case(S, [small(S), small(S, 3)], {1}, {1}, mode=ops.NEAREST),
        "nearest_fill": Case((33, 30, 61), [small((33, 30, 61)), _mat((33, 30, 61), degrees=(0, 30, 0))],
                             {1}, {1, 2}, mode=ops.NEAREST, fill=True),
        # corners within half a voxel outside two faces: the rounded tap is inside, the linear
        # mask (0.7 * 0.7 = 0.49) says filled
        "nearest_fill_corners": Case((33, 20, 24), [_shift((-0.3, -0.3, 0)), _shift((0.3, 0.3, -0.3))],
                                     {1}, {1}, mode=ops.NEAREST, fill=True),
        # faces exactly half a voxel outside (32 and 16 = n - 1 are powers of two, so u = -0.5 and
        # n - 0.5 exactly): the linear mask is exactly 0.5, so those voxels are filled
        "linear_fill_half_voxel_face": Case((33, 20, 17), [_shift((-0.5, 0, 0)), _shift((0, 0, 0.5))],
                                            {1}, {1}, fill=True),
        "nearest_fill_half_voxel_face": Case((33, 20, 17), [_shift((-0.5, 0, 0)), _shift((0, 0, 0.5))],
                                             {1}, {1}, mode=ops.NEAREST, fill=True),
        # zero-weight taps: integer coordinates put weight 0 on the + 1 corners (in bounds inside,
        # out of bounds on the last plane)
        "identity_and_integer_shifts": Case((36, 21, 28), [_shift((0, 0, 0)), _shift((1, -2, 3)),
                                                           _shift((0, 0, -1))], {1}, {1}),
        # floor(-1e-6) = -1: the first plane's weight is 1 - 1e-6 on the lower corner's neighbour
        "shifts_1e-6": Case((36, 21, 28), [_shift((-1e-6, 1e-6, -1e-6)), _shift((1e-6, -1e-6, 1e-6))],
                            {1}, {1}, fill=True),
        # batch and channels: the box is zeroed again for every channel
        "channels_3": Case((40, 36, 44), [small((40, 36, 44)), small((40, 36, 44), 1)], {1}, {1}, c=3,
                           fill=True),
        "batch_32_gated": Case((24, 20, 28), [None if e % 3 == 1 else
                                              _mat((24, 20, 28), degrees=rng.uniform(-12, 12, 3),
                                                   zoom=rng.uniform(0.9, 1.1, 3), shift=rng.uniform(-2, 2, 3))
                                              for e in range(32)], {1, 3}, {1, 3}),
        # non-finite cotangents: on a filled voxel (plane 0 of element 0: mask 0.4), an interior
        # voxel, and voxels whose zero-weight taps are in bounds (element 1's integer shift)
        "nonfinite_g": Case((33, 20, 24), [_shift((-0.6, 0, 0)), _shift((1, 0, 0))], {1}, {1}, fill=True,
                            poke={(0, 0, 0, 5, 5): math.nan, (0, 0, 10, 5, 5): math.inf,
                                  (1, 0, 10, 5, 5): math.nan, (1, 0, 12, 7, 7): -math.inf,
                                  (0, 0, 0, 9, 9): -math.inf}),
    }
    return cases


CASES = _cases()


# ---- the call ----------------------------------------------------------------------------------

def _backward(g, case, box_hint):
    """grad_in and the (B, tiles, 4) records of one tio_resample_backward call."""
    b, c, oi, oj, ok = g.shape
    mat, cp, flags = case.tables()
    dev = g.device
    mat_d = torch.as_tensor(mat).to(dev)
    cp_d = None if cp is None else torch.as_tensor(cp).to(dev)
    flags_d = torch.as_tensor(flags).to(dev)
    fill_d = torch.linspace(-1, 2, c, device=dev) if case.fill else None
    grad_in = torch.full((b, c, *case.shape), float("nan"), device=dev)  # the call must zero it
    ws_bytes = _native.lib().tio_resample_workspace_bytes(b, oi, oj, ok)
    ws = torch.zeros(ws_bytes, dtype=torch.uint8, device=dev)
    sp_in = (ctypes.c_float * 3)(*case.spacing_in)
    sp_out = (ctypes.c_float * 3)(*case.spacing_out)
    ni, nj, nk = (0, 0, 0) if cp is None else cp.shape[1:4]
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    _native.call("tio_resample_backward", g.data_ptr(), grad_in.data_ptr(), b, c, *case.shape, oi, oj, ok,
                 mat_d.data_ptr(), ptr(cp_d), flags_d.data_ptr(), ni, nj, nk, ctypes.addressof(sp_in),
                 ctypes.addressof(sp_out), int(case.affine_first), int(case.mode), ptr(fill_d), int(box_hint),
                 ws.data_ptr(), ws_bytes, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    tiles = b * -(-oi // XT) * -(-oj // XT) * -(-ok // XT)
    records = ws[: tiles * 16].view(torch.int32).view(b, -1, 4).cpu()
    return grad_in, records


def _oracle(g, case, threads=1):
    """grad64, abs64, count of the case for the cotangent g (host), per element on ``threads``."""
    mat, cp, flags = case.tables()
    fill = np.linspace(-1, 2, g.shape[1]).astype(np.float32) if case.fill else None

    def one(e):
        return c_port.resample_adjoint(g[e:e + 1], case.shape, mat[e:e + 1], None if cp is None else cp[e:e + 1],
                                       flags[e:e + 1], case.spacing_in, case.spacing_out,
                                       affine_first=case.affine_first, mode=case.mode, fill=fill)

    with ThreadPoolExecutor(threads) as pool:  # ctypes releases the GIL
        parts = list(pool.map(one, range(g.shape[0])))
    return tuple(torch.cat([p[i] for p in parts]) for i in range(3))


def _launch_box(case):
    mat, cp, _ = case.tables()
    hint = case.box_hint
    if hint is None:
        hint = spatial._box_hint(SimpleNamespace(mat=mat, cp=cp), case.spacing_in, case.spacing_out,
                                 case.out_shape or case.shape)
    return hint, (32 if hint > 24 else 24)


def _cotangent(case, seed=1):
    b, c = len(case.mats), case.c
    g = torch.randn((b, c, *(case.out_shape or case.shape)), generator=torch.Generator().manual_seed(seed))
    for idx, v in case.poke.items():
        g[idx] = v
    return g


def _check_exact(got, g, grad64, count, case):
    """(c): +0.0 bits where nothing arrives, pass-through elements bit for bit."""
    got = got.cpu()
    nothing = count == 0
    assert torch.equal(got[nothing].view(torch.int32), torch.zeros_like(got[nothing]).view(torch.int32))
    for e, m in enumerate(case.mats):
        if m is None:
            assert torch.equal(got[e].view(torch.int32), g[e].view(torch.int32))


def _codes(records):
    codes = (records[..., 3] & 255).reshape(-1)
    return {int(v): int((codes == v).sum()) for v in codes.unique()}


@pytest.mark.parametrize("name", list(CASES))
def test_adjoint_case(name):
    case = CASES[name]
    hint, box = _launch_box(case)
    assert box == case.box, f"{name}: the launch uses the {box} box, the case is built for {case.box}"
    g = _cotangent(case)
    got, records = _backward(g.cuda(), case, hint)
    codes = _codes(records)
    assert case.must <= set(codes) <= case.allowed, (name, codes)
    if case.needs_32:  # tiles staged in the 32 box that the 24 one would not hold
        _, rec24 = _backward(g.cuda(), case, 24)
        assert (rec24[..., 3] & 255).eq(0).sum() > records[..., 3].bitwise_and(255).eq(0).sum(), name
    grad64, abs64, count = _oracle(g, case)
    ratio = check_adjoint(got, grad64, abs64, count)
    _check_exact(got, g, grad64, count, case)
    k = case.shape[2]
    flush = "2-D" if k == 1 else ("vector" if k % 4 == 0 else "scalar tail")
    print(f"[K1T {name}] box {box} (hint {hint}), flush {flush}, tile codes {codes}, "
          f"max |gpu - grad64| / bound = {ratio:.3f}, NaN voxels {int(torch.isnan(grad64).sum())}")


def test_cases_cover_every_path():
    """Across the cases: all four codes, both boxes, all three flush paths, both modes."""
    codes = set().union(*(c.must for c in CASES.values()))
    boxes = {c.box for c in CASES.values()}
    flushes = {("2d" if c.shape[2] == 1 else c.shape[2] % 4 == 0) for c in CASES.values()}
    assert codes == {0, 1, 2, 3} and boxes == {24, 32} and flushes == {"2d", True, False}
    assert {c.mode for c in CASES.values()} == {ops.NEAREST, ops.LINEAR}


# ---- full size, nondeterminism, the public path, refusal ---------------------------------------

def _bench_geometry(b, size):
    """The bench's Affine + ElasticDeformation steps on a (b, 1, size^3) batch: one Case each."""
    import torchio_b200 as tio

    x = torch.rand((b, 1, size, size, size), generator=torch.Generator().manual_seed(2)).cuda()
    torch.manual_seed(12)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = tio.Compose([tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)), tio.ElasticDeformation()],
                          copy=False)(tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(b)])}))
    cases = []
    for step in out.applied_transforms:
        mat, cp, flags, _ = c_port.spatial_tables(step.params, b, (size,) * 3, np.eye(4))
        cps = None if cp is None else [cp[e].numpy() if flags[e] & 2 else None for e in range(b)]
        mats = [mat[e].numpy() for e in range(b)]
        pad = step.params["default_pad_value"]
        has_fill = not (isinstance(pad, (int, float)) and float(pad) == 0.0)
        cases.append((step.name, Case((size,) * 3, mats, {1}, {0, 1, 2}, cps=cps, fill=has_fill,
                                      affine_first=bool(step.params["affine_first"]))))
    return cases


def test_full_size_bench_geometry():
    """8 x 1 x 256^3, the bench's two spatial steps, every voxel against the oracle."""
    for name, case in _bench_geometry(8, 256):
        hint, box = _launch_box(case)
        g = _cotangent(case, seed=3)
        got, records = _backward(g.cuda(), case, hint)
        codes = _codes(records)
        assert case.must <= set(codes) <= case.allowed, codes
        mat, cp, flags = case.tables()
        t0 = time.perf_counter()

        def one(e):  # per element, so that a few GB of host memory suffice
            return c_port.resample_adjoint(g[e:e + 1], case.shape, mat[e:e + 1],
                                           None if cp is None else cp[e:e + 1], flags[e:e + 1], case.spacing_in,
                                           case.spacing_out, affine_first=case.affine_first, mode=case.mode,
                                           fill=np.zeros(1, np.float32) if case.fill else None)

        ratio, got_h = 0.0, got.cpu()
        with ThreadPoolExecutor(8) as pool:  # ctypes releases the GIL
            for e, (grad64, abs64, count) in enumerate(pool.map(one, range(len(case.mats)))):
                ratio = max(ratio, check_adjoint(got_h[e:e + 1], grad64, abs64, count))
                assert torch.equal(got_h[e:e + 1][count == 0].view(torch.int32),
                                   torch.zeros(int((count == 0).sum()), dtype=torch.int32))
        t_oracle = time.perf_counter() - t0
        total = sum(codes.values())
        shares = ", ".join(f"code {k}: {100 * v / total:.1f} %" for k, v in sorted(codes.items()))
        print(f"[K1T 256^3 {name}] box {box}, tiles {shares}; max |gpu - grad64| / bound = {ratio:.3f};"
              f" oracle {t_oracle:.1f} s on 8 threads")


def test_two_runs_differ_only_within_the_bound():
    """Atomics make the order of the additions, and so the last bits, differ between runs."""
    case = Case((96, 96, 96), [_mat((96, 96, 96), zoom=(2.5, 2.5, 2.5), degrees=(7, 3, -4)),
                               _mat((96, 96, 96), zoom=(2.2, 2.6, 2.4))], {1}, {1}, fill=True)
    g = _cotangent(case, seed=4)
    first, _ = _backward(g.cuda(), case, _launch_box(case)[0])
    second, _ = _backward(g.cuda(), case, _launch_box(case)[0])
    grad64, abs64, count = _oracle(g, case, threads=2)
    r1 = check_adjoint(first, grad64, abs64, count)
    r2 = check_adjoint(second, grad64, abs64, count)
    a, b = first.cpu().double(), second.cpu().double()
    differ = a != b
    both = torch.as_tensor(2 * adjoint_bound(abs64.numpy(), count.numpy()))
    assert ((a - b).abs()[differ] <= both[differ]).all()
    print(f"[K1T twice] {int(differ.sum())} of {differ.numel()} voxels differ between runs "
          f"(max m {int(count.max())}); ratios {r1:.3f}, {r2:.3f}")


def _resample_nodes(y):
    """The K1 graph nodes behind y, input side first."""
    nodes, todo, seen = [], [y.grad_fn], set()
    while todo:
        fn = todo.pop()
        if fn is None or fn in seen:
            continue
        seen.add(fn)
        if type(fn).__name__.startswith("_ResampleBackward"):
            nodes.append(fn)
        todo.extend(f for f, _ in fn.next_functions)
    return nodes[::-1]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_public_path_gradient(dtype, coords):
    """Compose([Affine, ElasticDeformation]) with set_differentiable(True): each K1ᵀ node of the
    graph against the oracle on the cotangent it received, and the input's grad after its cast."""
    import torchio_b200 as tio

    b, shape = 3, (96, 80, 64)
    x = (torch.rand((b, 1, *shape), generator=torch.Generator().manual_seed(6)) * 2).to(dtype).cuda()
    x.requires_grad_()
    previous = tio.set_differentiable(True)
    try:
        torch.manual_seed(13)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = tio.Compose([tio.Affine(scales=(0.9, 1.1), degrees=(-10, 10)),
                               tio.ElasticDeformation(max_displacement=4.0)], copy=False)(
                tio.SubjectsBatch({"t1": tio.ImagesBatch(x, [tio.AffineMatrix() for _ in range(b)])}))
        y = out.images["t1"].data
        nodes = _resample_nodes(y)
        assert len(nodes) == 2
        seen = {}
        for i, node in enumerate(nodes):
            node.register_hook(lambda gi, go, i=i: seen.__setitem__(i, (go[0].detach().clone(),
                                                                         gi[0].detach().clone())))
        cot = torch.randn(y.shape, generator=torch.Generator().manual_seed(7)).to(dtype).cuda()
        y.backward(cot)
    finally:
        tio.set_differentiable(previous)
    history = out.applied_transforms
    assert [t.name for t in history] == ["Affine", "ElasticDeformation"]
    round_to = {torch.float16: (2.0**-11, 2.0**-25), torch.bfloat16: (2.0**-8, 2.0**-134)}.get(dtype)
    for i, step in enumerate(history):
        mat, cp, flags, _ = c_port.spatial_tables(step.params, b, shape, np.eye(4))
        pad = step.params["default_pad_value"]
        has_fill = not (isinstance(pad, (int, float)) and float(pad) == 0.0)
        fill = np.zeros(1, np.float32) if has_fill else None
        grad_out, grad_in = seen[i]
        assert grad_out.dtype == torch.float32
        grad64, abs64, count = c_port.resample_adjoint(
            grad_out.cpu(), shape, mat, cp, flags, (1, 1, 1), (1, 1, 1),
            affine_first=bool(step.params["affine_first"]), mode=ops.LINEAR, fill=fill)
        ratio = check_adjoint(grad_in, grad64, abs64, count)
        if i == 0:  # the input's grad: node 0's fp32 result, cast once more to the input's dtype
            assert x.grad.dtype == dtype
            check_adjoint(x.grad, grad64, abs64, count, round_to=round_to)
        print(f"[K1T public {dtype} {coords}] {step.name}: max |gpu - grad64| / bound = {ratio:.3f}")


def test_grid_too_large_is_refused_before_any_launch():
    b = 65536
    g = torch.zeros((b, 1, 1, 1, 1), device="cuda")
    mat = torch.as_tensor(np.tile(np.eye(4, dtype=np.float32)[:3].reshape(12), (b, 1))).cuda()
    before = ops.launches()
    with pytest.raises(RuntimeError, match="grid too large"):
        ops.resample_backward(g, (1, 1, 1), mat, None, None, (1, 1, 1), (1, 1, 1), affine_first=True,
                              mode=ops.LINEAR, fill=None)
    torch.cuda.synchronize()
    assert ops.launches() == before
