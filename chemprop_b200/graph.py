"""Whole-step CUDA graph (SURVEY.md section 8f-2): the training step of the path -- device layout build, forward, loss, backward,
optionally the optimizer -- captured ONCE for a batch signature and replayed with one `cudaGraphLaunch` per step.

Why it is possible: the step is sync-free (layout meta words come from the host, `engine.HOST_META`), every kernel of
libdmpnn_sm90.so launches on the caller's current stream with plain pointer arguments, the TMA descriptors are passed by value
(`__grid_constant__`), and the library never allocates.  Why it pays: a 10 k-molecule fwd+bwd is ~60 launches of 5-250 us each;
the host needs ~1 ms of Python + ctypes to issue them, a graph launch needs ~20 us, so the GPU queue never runs dry and the
host is free for the loader.  (The reference reaches the same point only through `torch.compile(mode="reduce-overhead")`.)

A graph is bound to a batch SIGNATURE -- atom / edge / molecule counts and the layout meta words (tile count, flags, max
in-degree, ...): everything that a launch parameter was derived from at capture time.  `CudaGraphStep` keeps one graph per
signature (LRU) and copies each new batch's five tensors into the static input buffers of the matching graph; a batch with a new
signature is captured on first sight (two eager warm-up steps + the capture, ~10 ms).  Fixed-shape loaders (bucketed or padded
batches, or a resident batch as in bench.py) therefore replay one graph for the whole run.

That holds because every host-side argument of every launch is derived from the signature, and everything that depends on
the batch's contents (layout, window table, atom tiles, segment pointers, mol-atom-bond index maps) is rebuilt inside the
graph from the static inputs.  tests/test_graph_signature_host.py checks the first on the CPU for every capturable path
and head, on batches of one signature and different topology (tests/graph_twins.py); tests/test_gpu_graph_replay.py
replays such batches with the optimizer in the graph against the eager steps, bit for bit, and against float64.
"""
from __future__ import annotations

import weakref
from collections import OrderedDict
from typing import Callable

import torch

from .data.collate import BatchMolGraph


def batch_signature(bmg: BatchMolGraph) -> tuple:
    meta = getattr(bmg, "_meta_host", None)
    if meta is None:
        raise ValueError("CudaGraphStep needs a batch with host-computed layout meta words (chemprop_b200's collate / loader / "
                         "packed data set produce them); a batch built from device tensors would need a device read-back")
    return (int(bmg.V.shape[0]), int(bmg.V.shape[1]), int(bmg.E.shape[0]), int(bmg.E.shape[1]), len(bmg), tuple(int(x) for x in meta))


class _Captured:
    __slots__ = ("graph", "bmg", "out", "last", "last_ref", "launches")


def _static_copy(bmg: BatchMolGraph) -> BatchMolGraph:
    static = BatchMolGraph.from_tensors(bmg.V.clone(), bmg.E.clone(), bmg.edge_index.clone(), bmg.rev_edge_index.clone(),
                                        bmg.batch.clone(), len(bmg))
    static._meta_host = list(bmg._meta_host)
    return static


class CudaGraphStep:
    """`step = CudaGraphStep(fn)`; `loss = step(bmg)`.

    `fn(bmg) -> Tensor | tuple[Tensor, ...]` runs one full step on a DEVICE batch and must not synchronise with the host: e.g.

        def fn(bmg):
            opt.zero_grad(set_to_none=False)          # gradients are static buffers of the graph
            loss = criterion(head(agg(mp(bmg), bmg.batch)), targets)
            loss.backward()
            opt.step()                                # torch.optim.*(capturable=True)
            return loss

    The returned tensors are static outputs of the graph: valid until the next call with the same signature.  Parameters'
    `.grad` tensors must exist before the first call (run one eager step, or `p.grad = torch.zeros_like(p)`), so that the
    captured backward accumulates into fixed buffers.

    `step(bmgs)` also takes a list or tuple of batches (one per component of a multicomponent model with unshared
    encoders): `fn` then receives a list of static batches, one per given batch, and the graph's signature is the tuple of
    the batches' signatures."""

    def __init__(self, fn: Callable, max_graphs: int = 8, warmup: int = 2, pool=None):
        self.fn, self.max_graphs, self.warmup = fn, int(max_graphs), int(warmup)
        self._graphs: OrderedDict = OrderedDict()
        self._pool = pool
        self.captures = 0
        self.replays = 0
        self.last_launches = 0

    def _capture(self, bmg) -> _Captured:
        many = isinstance(bmg, (list, tuple))
        dev = (bmg[0] if many else bmg).V.device
        static = [_static_copy(b) for b in bmg] if many else _static_copy(bmg)
        statics = static if many else [static]

        def run():
            for s in statics:
                s._layout = None
            return self.fn(static)

        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                 # warm-up on a side stream, as torch's capture protocol asks
            for _ in range(self.warmup):
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        cap = _Captured()
        cap.graph = torch.cuda.CUDAGraph()
        cap.bmg = static
        cap.last = cap.last_ref = None
        kw = {} if self._pool is None else {"pool": self._pool}
        from . import _lib

        l0 = _lib.load().dmpnn_launch_count()
        with torch.cuda.graph(cap.graph, **kw):
            cap.out = run()
        cap.launches = int(_lib.load().dmpnn_launch_count() - l0)      # libdmpnn kernels one replay launches
        if self._pool is None:
            self._pool = cap.graph.pool()             # later graphs share this one's memory pool
        self.captures += 1
        return cap

    def load(self, cap: _Captured, bmg):
        # The very same (unmodified) batch object as last time -- a resident batch replayed step after step: nothing to copy.
        # "Same" = the object itself (held through a weak reference: an `id()` is reused as soon as a batch is freed, and a
        # fresh batch's tensors are all at version 0), the same storage and no in-place change torch knows of.  Tensors that
        # are rewritten through raw pointers behind torch's back are not seen: pass such a batch as a new object.
        # A list of batches is compared batch by batch.
        many = isinstance(cap.bmg, list)
        bmgs, statics = (list(bmg), cap.bmg) if many else ([bmg], [cap.bmg])
        stamp = tuple(tuple((t.data_ptr(), t._version, tuple(t.shape)) for t in (b.V, b.E, b.edge_index, b.rev_edge_index,
                                                                                   b.batch)) for b in bmgs)
        if (cap.last_ref is not None and len(cap.last_ref) == len(bmgs)
                and all(r() is b for r, b in zip(cap.last_ref, bmgs)) and cap.last == stamp):
            return
        try:
            cap.last_ref, cap.last = [weakref.ref(b) for b in bmgs], stamp
        except TypeError:                                  # a batch type without weak references: copied every time
            cap.last_ref = cap.last = None
        for s, b in zip(statics, bmgs):
            s.V.copy_(b.V, non_blocking=True)
            s.E.copy_(b.E, non_blocking=True)
            s._edge_index.copy_(b.edge_index, non_blocking=True)
            s._rev_edge_index.copy_(b.rev_edge_index, non_blocking=True)
            s._batch.copy_(b.batch, non_blocking=True)

    def __call__(self, bmg):
        many = isinstance(bmg, (list, tuple))
        bmgs = list(bmg) if many else [bmg]
        if not bmgs:
            raise ValueError("CudaGraphStep needs at least one batch")
        if not all(b.V.is_cuda for b in bmgs):
            raise ValueError("CudaGraphStep takes a device batch (BatchMolGraph.cuda_copy / a resident data set)")
        sig = tuple(batch_signature(b) for b in bmgs) if many else batch_signature(bmg)
        cap = self._graphs.get(sig)
        if cap is None:
            cap = self._capture(bmgs if many else bmg)
            self._graphs[sig] = cap
            while len(self._graphs) > self.max_graphs:
                self._graphs.popitem(last=False)
        else:
            self._graphs.move_to_end(sig)
        self.load(cap, bmgs if many else bmg)
        cap.graph.replay()
        self.replays += 1
        self.last_launches = cap.launches
        return cap.out
