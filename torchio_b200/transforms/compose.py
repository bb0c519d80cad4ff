"""Compose (host-side mirror of transforms/compose.py:38-98, TorchIO 2.0.0a2).

Semantics kept: deep-copy once at the top, children run with ``copy=False``
in order, each child draws its gate + params from the global CPU RNG exactly
where the reference does.  Difference by design: a CPU-resident batch is
staged to the GPU once for the whole pipeline (not once per child).
"""

from __future__ import annotations

import copy as _copy
import threading as _threading
from collections.abc import Mapping, Sequence
from typing import Any

import torch as _torch

from ..data import ImagesBatch, SubjectsBatch
from ..params import slice_params
from .base import (ChunkInfo, Transform, _Staging, _finish, chunk_scope, execution_device, refuse_host_grad,
                   wrap_input)
from . import intensity as _int
from .. import ops as _ops


_stream_local = _threading.local()


class Pending:
    """Ticket of `Compose.submit`: the transformed batch once the device has delivered it."""

    def __init__(self, batch, unwrap, event) -> None:
        self._batch, self._unwrap, self._event = batch, unwrap, event

    def done(self) -> bool:
        return self._event is None or self._event.query()

    def result(self):
        if self._event is not None:
            self._event.synchronize()
            self._event = None
        return _finish(self._batch, self._unwrap)


class Compose(Transform):
    def __init__(self, transforms: Sequence[Transform] | Mapping[str, Transform] | None = None,
                 *, copy: bool = True, **kwargs: Any) -> None:
        super().__init__(copy=copy, **kwargs)
        if transforms is None:
            self.transforms: list[Transform] = []
        elif isinstance(transforms, Mapping):
            self.transforms = list(transforms.values())
        else:
            self.transforms = list(transforms)

    def forward(self, data: Any) -> Any:
        return self._submit(data, graph=True).result()

    def submit(self, data: Any) -> "Pending":
        """Issue the whole pipeline for ``data`` and return without waiting for the device.

        For a host-resident batch that is streamed through the device in slices, every copy
        and kernel is queued and the call returns while they run; `Pending.result()` waits
        for the last copy-out and hands back what `forward` returns.  Anything else is
        executed as `forward` does and the ticket is already complete.  Submitting batch
        n+1 before collecting batch n lets its copy-in overlap the copy-out of batch n
        (PCIe is full duplex) — `stream` does exactly that.

        Until `result()` returns, the device is still reading the host tensors of ``data``: a
        loader that refills one staging buffer in place must not touch it before then (fresh
        tensors per batch, as `SubjectsLoader` / `DataLoader` produce, are fine)."""
        return self._submit(data, graph=False)

    def _submit(self, data: Any, graph: bool) -> "Pending":
        """`submit`; ``graph``: a batch that requires grad may record a graph (`forward` only: a
        ticket cannot hand back a graph node)."""
        if self.copy:
            data = _copy.deepcopy(data)
        batch, unwrap = wrap_input(data)
        if not graph and _ops.differentiable_default() and any(
                ib.data.requires_grad for ib in batch.images.values()):
            raise NotImplementedError("Compose.submit / Compose.stream: inputs that require grad are not"
                                      " supported; call the Compose itself")
        refuse_host_grad(batch)  # before the streamed path, which does not stage through _Staging
        chunk = self._chunk_size(batch)
        if chunk:
            batch, done = self._forward_streamed(batch, chunk)
            return Pending(batch, unwrap, done)
        with _Staging(batch):
            batch = self._forward_batch(batch)
        return Pending(batch, unwrap, None)

    def stream(self, batches, depth: int = 1):
        """Loader-style application: ``for out in pipeline.stream(loader)`` yields
        ``pipeline(batch)`` for every batch of ``loader``, in order, with up to ``depth``
        later batches already issued to the device while the caller consumes the current one.
        Results and RNG consumption equal calling the pipeline batch by batch.  ``batches`` must
        yield tensors it does not overwrite while they are in flight (see `submit`)."""
        if depth < 0:
            raise ValueError(f"depth must be >= 0, got {depth}")
        window: list[Pending] = []
        for data in batches:
            window.append(self.submit(data))
            if len(window) > depth:
                yield window.pop(0).result()
        while window:
            yield window.pop(0).result()

    #: Elements per slice when a host-resident batch is streamed through the device
    #: (None = choose from the batch's size; 0 = never stream).
    chunk_size: int | None = None
    #: auto mode: slices of about this many bytes, and only batches of >= 2 slices
    chunk_bytes = 256 << 20

    def _chunk_size(self, batch: SubjectsBatch) -> int:
        """Slice length for streamed execution, or 0 for the one-shot path.  Streaming
        applies to host-resident batches whose pipeline is made of transforms that
        are row-wise separable given their recorded params (`supports_chunks`)."""
        if self.chunk_size == 0 or not self.transforms:
            return 0
        b = batch.batch_size
        if b < 2 or any(ib.data.is_cuda for ib in batch.images.values()):
            return 0
        if not _torch.cuda.is_available():
            return 0
        if not all(t.supports_chunks(batch) for t in self.transforms):
            return 0
        if self.chunk_size is not None:
            return min(int(self.chunk_size), b) if self.chunk_size < b else 0
        per_sample = sum(ib.data[0].numel() * ib.data.element_size() for ib in batch.images.values())
        chunk = max(1, self.chunk_bytes // max(per_sample, 1))
        return int(chunk) if chunk * 2 <= b else 0

    def _plan(self, batch: SubjectsBatch):
        """Gate draws and `make_params` of every child on the whole batch, in
        pipeline order — the RNG sequence of sequential application, since no
        child's sampling reads voxel data.  Entries: (children, [(child, params)])."""
        plan = []
        index = 0
        while index < len(self.transforms):
            group = self._fusable_run(index) if self.fuse else []
            if len(group) < 2:
                group = [self.transforms[index]]
            applied = _sample_group(group, batch)
            for transform, params in applied:
                checks = getattr(transform, "plan_checks", None)
                if checks is not None:
                    checks(batch, params)
            plan.append((group, applied))
            index += len(group)
        return plan

    def _forward_streamed(self, batch: SubjectsBatch, chunk: int) -> SubjectsBatch:
        """Host batch -> device -> host in slices of the batch axis on three streams,
        so the copy in of slice n+1, the kernels of slice n and the copy out of
        slice n-1 overlap (PCIe is full duplex).  Params are sampled for the whole
        batch first; results equal the one-shot path row for row."""
        plan = self._plan(batch)
        device = execution_device()
        streams = self._streams(device)
        h2d, compute, d2h = streams
        total = batch.batch_size
        cache: dict = {}
        for step, (_, applied) in enumerate(plan):
            for transform, params in applied:
                transform.prepare_stream(batch, params, cache, step)
        names = list(batch.images)
        outputs: dict[str, Any] = {}
        affines: dict[str, list] = {name: [] for name in names}
        caller = _torch.cuda.current_stream(device)
        for s in streams:
            s.wait_stream(caller)
        for b0 in range(0, total, chunk):
            b1 = min(b0 + chunk, total)
            staged = {}
            with _torch.cuda.stream(h2d):
                for name in names:
                    ib = batch.images[name]
                    staged[name] = ib.data[b0:b1].to(device, non_blocking=True)
                arrived = h2d.record_event()
            compute.wait_event(arrived)
            with _torch.cuda.stream(compute):
                sub = SubjectsBatch({
                    name: ImagesBatch(staged[name], list(batch.images[name].affines[b0:b1]),
                                      image_class=batch.images[name]._image_class)
                    for name in names})
                for tensor in staged.values():
                    tensor.record_stream(compute)
                for step, (group, applied) in enumerate(plan):
                    with chunk_scope(ChunkInfo(b0, b1, total, cache, step)):
                        sliced = [(t, slice_params(p, b0, b1)) for t, p in applied]
                        _apply_group(sliced, sub)
                done = compute.record_event()
            d2h.wait_event(done)
            with _torch.cuda.stream(d2h):
                for name in names:
                    result = sub.images[name].data.contiguous()
                    result.record_stream(d2h)
                    if name not in outputs:
                        source = batch.images[name].data
                        outputs[name] = _torch.empty((total, *result.shape[1:]), dtype=result.dtype,
                                                     pin_memory=source.is_pinned())
                    outputs[name][b0:b1].copy_(result, non_blocking=True)
                    affines[name].extend(sub.images[name].affines)
            del staged, sub
        done = d2h.record_event()
        caller.wait_stream(compute)
        for name in names:
            ib = batch.images[name]
            ib.data = outputs[name]
            ib.affines[:] = affines[name]
        for _, applied in plan:
            for transform, params in applied:
                transform._record(batch, params)
        return batch, done

    def _streams(self, device):
        """(copy-in, kernels, copy-out) streams of the calling thread for ``device``.  Kept per
        thread and outside the module's ``__dict__``: a `Queue` calls one Compose from several
        worker threads (each gets its own triple, so their subjects overlap instead of
        serialising on shared streams), and the Compose stays picklable / deep-copyable."""
        cache = getattr(_stream_local, "streams", None)
        if cache is None:
            cache = _stream_local.streams = {}
        key = (device.type, device.index)
        triple = cache.get(key)
        if triple is None:
            # the kernel stream also carries the small table uploads of every slice: high
            # priority, or the copy engine serves them only after the queued bulk copies
            triple = cache[key] = (_torch.cuda.Stream(device=device),
                                   _torch.cuda.Stream(device=device, priority=-1),
                                   _torch.cuda.Stream(device=device))
        return triple

    def _forward_batch(self, batch):
        # Children never copy (compose.py:88-92).  Unlike the reference we do
        # not mutate child.copy: Queue calls one Compose from several threads.
        index = 0
        while index < len(self.transforms):
            group = self._fusable_run(index) if self.fuse else []
            if len(group) >= 2:
                batch = _run_fused(group, batch)
                index += len(group)
            else:
                batch = self.transforms[index]._forward_batch(batch)
                index += 1
        return batch

    #: Fuse runs of consecutive intensity transforms into one kernel pair.
    fuse = True

    def _fusable_run(self, start: int) -> list[Transform]:
        """Longest run from ``start`` of BiasField < Blur < Noise < Gamma (each at
        most once, in that order, same include/exclude): exactly the chains whose
        per-voxel arithmetic the fused kernel reproduces."""
        order = {_int.BiasField: 0, _int.Blur: 1, _int.Noise: 2, _int.Gamma: 3}
        run: list[Transform] = []
        last = -1
        for transform in self.transforms[start:]:
            rank = order.get(type(transform))
            if rank is None or rank <= last:
                break
            if run and (transform.include != run[0].include or transform.exclude != run[0].exclude):
                break
            run.append(transform)
            last = rank
        return run

    def __len__(self) -> int:
        return len(self.transforms)

    def __getitem__(self, index: int) -> Transform:
        return self.transforms[index]

    def to_hydra(self) -> dict[str, Any]:
        cfg = super().to_hydra()
        cfg["transforms"] = [t.to_hydra() for t in self.transforms]
        return cfg


def _sample_group(group: list[Transform], batch):
    """Gate draw then `make_params` for each transform of the group, in order:
    the draws `Transform._forward_batch` makes.  Returns the non-gated (t, params)."""
    applied = []
    for transform in group:
        if not transform._per_instance_p_active(batch) and _torch.rand(1).item() >= transform.p:
            continue
        applied.append((transform, transform.make_params(batch)))
    return applied


def _apply_group(applied, batch) -> None:
    """Apply sampled transforms: a run of >= 2 intensity transforms goes through one
    fused launch pair per image, anything else through its own `apply_transform`."""
    if len(applied) >= 2 and all(type(t) in _FUSABLE for t, _ in applied):
        builders = []
        for transform, params in applied:
            if isinstance(transform, _int.BiasField):
                builders.append(lambda ib, index, p=params: _int._bias_stage(
                    ib.data.shape, ib.affines, p["std"], p["seed"], p["scale"], divide=False))
            elif isinstance(transform, _int.Blur):
                builders.append(lambda ib, index, p=params: _int._blur_stage(ib, p, index))
            elif isinstance(transform, _int.Noise):
                builders.append(_int._noise_stage_factory(params))
            else:
                builders.append(lambda ib, index, p=params: {
                    "gamma": _int.tables.gamma_values(p["log_gamma"], ib.data.shape[0])})
        _int.run_stages(applied[0][0]._get_images(batch), builders)
        return
    for transform, params in applied:
        transform.apply_transform(batch, params)


_FUSABLE = (_int.BiasField, _int.Blur, _int.Noise, _int.Gamma)


def _run_fused(group: list[Transform], batch):
    """Sample every transform of the run exactly as sequential application would
    (gate draw, then make_params, in order — none of them reads voxel data),
    then apply all non-gated stages with one fused launch pair per image."""
    applied = _sample_group(group, batch)
    for transform, _ in applied:
        transform._check_differentiable(batch)
    if applied:
        _apply_group(applied, batch)
        for transform, params in applied:
            transform._record(batch, params)
    return batch
