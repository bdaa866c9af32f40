"""`BatchMolGraph` / `collate_batch` with the public surface of chemprop/data/collate.py:13-97.

Public view (unchanged): ``V`` f32 (V x d_v), ``E`` f32 (E x d_e), ``edge_index`` int64 (2 x E),
``rev_edge_index`` int64 (E), ``batch`` int64 (V), ``len(bmg)`` = number of molecules,
in-place ``.to(device)`` returning None.

What differs from the reference: concatenation is done by one C call
(`dmpnn_collate_host`, replacing the per-molecule Python loop at collate.py:48-62), host tensors
can be pinned, and the engine's device layout (dst-sorted CSR + tile table, built by
`dmpnn_layout_build`) is cached on the object after first use so the depth loop, the readout and
the backward pass all share it.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, NamedTuple, Sequence

import numpy as np
import torch
from torch import Tensor

from .. import _lib
from .molgraph import MolGraph


_EXT = None          # the CPython collate extension (chemprop_b200/csrc/collate_ext.c); False = unavailable


def _collate_ext():
    """Loads lib/_collate_ext*.so once.  Host-side convenience only: without it the ctypes path below is used."""
    global _EXT
    if _EXT is None:
        _EXT = False
        try:
            import importlib.util

            from ..build import collate_ext_path

            path = collate_ext_path()
            if path.exists():
                spec = importlib.util.spec_from_file_location("chemprop_b200._collate_ext", path)
                mod = importlib.util.module_from_spec(spec)
                spec.loader.exec_module(mod)
                _EXT = mod
        except Exception:  # noqa: BLE001
            _EXT = False
    return _EXT or None


def host_meta(edge_index: Tensor, rev_edge_index: Tensor, batch: Tensor, n_mols: int) -> list | None:
    """The layout meta words (flags, max in-degree, tile count, largest tile) of a batch whose int64 index tensors are
    in host memory -- `dmpnn_batch_meta_host`, one C pass.  None when the tensors are not plain host int64."""
    ts = (edge_index, rev_edge_index, batch)
    if any(t.is_cuda or t.dtype != torch.int64 for t in ts):
        return None
    edge_index, rev_edge_index, batch = (t.contiguous() for t in ts)
    if edge_index.dim() != 2 or edge_index.shape[0] != 2 or rev_edge_index.shape[0] != edge_index.shape[1]:
        return None
    V, E = int(batch.shape[0]), int(edge_index.shape[1])
    if max(V, E, n_mols) >= 2 ** 31:
        return None
    meta = np.zeros(_lib.META_WORDS, dtype=np.int32)
    lib = _lib.load()
    rc = lib.dmpnn_batch_meta_host(edge_index.data_ptr() if E else None, rev_edge_index.data_ptr() if E else None,
                                   batch.data_ptr() if V else None, V, E, int(n_mols), meta.ctypes.data)
    _lib.check(rc, "dmpnn_batch_meta_host")
    return meta.tolist()


def tile_packing_order(n_atoms, n_edges) -> np.ndarray:
    """A permutation of the molecules of a batch under which the engine's tiles come out nearly full
    (`dmpnn_tile_pack_order`: best-fit decreasing on the edge counts).  The order of molecules inside a batch is the
    loader's choice (the reference reshuffles it every epoch); use it as `mgs = [mgs[i] for i in order]` -- and order the
    targets the same way -- before building the BatchMolGraph.  Purely a performance matter."""
    na = np.ascontiguousarray(n_atoms, dtype=np.int64)
    ne = np.ascontiguousarray(n_edges, dtype=np.int64)
    if na.shape != ne.shape or na.ndim != 1:
        raise ValueError("n_atoms / n_edges must be one-dimensional and of equal length")
    order = np.empty(na.shape[0], dtype=np.int64)
    lib = _lib.load()
    _lib.check(lib.dmpnn_tile_pack_order(na.shape[0], na.ctypes.data, ne.ctypes.data, order.ctypes.data),
               "dmpnn_tile_pack_order")
    return order


def tile_packing_order_of(mgs: Sequence[MolGraph]) -> np.ndarray:
    return tile_packing_order([mg.V.shape[0] for mg in mgs], [mg.edge_index.shape[1] for mg in mgs])


class BatchMolGraph:
    # the three index tensors sit behind properties: replacing one drops the cached device layout and host meta
    # (`__weakref__`: chemprop_b200.graph.CudaGraphStep remembers the last batch it loaded without keeping it alive)
    __slots__ = ("V", "E", "_edge_index", "_rev_edge_index", "_batch", "_size", "_layout", "_xfer", "_meta_host", "__weakref__")

    def _index_property(name):  # noqa: N805
        def get(self):
            return getattr(self, name)

        def set_(self, value):
            setattr(self, name, value)
            self._layout = None
            self._meta_host = None

        return property(get, set_)

    edge_index = _index_property("_edge_index")
    rev_edge_index = _index_property("_rev_edge_index")
    batch = _index_property("_batch")
    del _index_property

    def __init__(self, mgs: Sequence[MolGraph], pin_memory: bool = False, transfer_dtype: torch.dtype | None = None,
                 use_extension: bool = True):
        """``transfer_dtype=torch.bfloat16`` (opt-in, for the bf16 tier) additionally keeps a compact host staging
        copy -- features in bf16, indices in int32 -- that `.to(cuda)` / `.cuda_copy()` ship over PCIe instead of
        the f32 / int64 tensors (half the bytes); the public device tensors are widened back to f32 / int64 on
        the GPU.  The bf16 tier rounds V and E to bf16 when it assembles its GEMM operands anyway, so its results
        are bit-identical; the fp32 tier would see bf16-rounded features, hence opt-in."""
        self._size = len(mgs)
        self._layout = None
        self._xfer = None
        self._meta_host = None
        if transfer_dtype is not None and transfer_dtype != torch.bfloat16:
            raise ValueError("transfer_dtype must be torch.bfloat16 or None")
        kw = dict(pin_memory=True) if pin_memory else {}
        ext = _collate_ext() if use_extension else None
        if ext is not None:
            self._init_ext(ext, mgs, kw, transfer_dtype is not None)
        else:
            self._init_ctypes(mgs, kw, transfer_dtype is not None)
        # flags / tile count of this batch, computed here in the loader so that the training step needs no device read-back
        self._meta_host = host_meta(self._edge_index, self._rev_edge_index, self._batch, self._size)

    def _alloc(self, Vt: int, Et: int, d_v: int, d_e: int, kw: dict, compact: bool):
        self.V = torch.empty((Vt, d_v), dtype=torch.float32, **kw)
        self.E = torch.empty((Et, d_e), dtype=torch.float32, **kw)
        self.edge_index = torch.empty((2, Et), dtype=torch.int64, **kw)
        self.rev_edge_index = torch.empty((Et,), dtype=torch.int64, **kw)
        self.batch = torch.empty((Vt,), dtype=torch.int64, **kw)
        if not compact:
            return None
        if max(Vt, Et) >= 2 ** 31:
            raise ValueError("batch too large for int32 transfer indices")
        return (torch.empty((Vt, d_v), dtype=torch.bfloat16, **kw), torch.empty((Et, d_e), dtype=torch.bfloat16, **kw),
                torch.empty((2, Et), dtype=torch.int32, **kw), torch.empty((Et,), dtype=torch.int32, **kw),
                torch.empty((Vt,), dtype=torch.int32, **kw))

    def _init_ext(self, ext, mgs, kw: dict, compact: bool):
        """One C call per phase: the extension walks the MolGraph list through the CPython / NumPy C API."""
        mgs = mgs if isinstance(mgs, (list, tuple)) else list(mgs)
        n_atoms, n_edges, d_v, d_e = ext.sizes(mgs)
        Vt, Et = int(n_atoms.sum()), int(n_edges.sum())
        xf = self._alloc(Vt, Et, d_v, d_e, kw, compact)
        out = (self.V, self.E, self.edge_index, self.rev_edge_index, self.batch) + (xf or ())
        ext.fill(mgs, d_v, d_e, Et, *(t.data_ptr() for t in out))
        self._xfer = xf

    def _init_ctypes(self, mgs, kw: dict, compact: bool):
        n = len(mgs)
        n_atoms = np.fromiter((mg.V.shape[0] for mg in mgs), dtype=np.int64, count=n)
        n_edges = np.fromiter((mg.edge_index.shape[1] for mg in mgs), dtype=np.int64, count=n)
        d_v = int(mgs[0].V.shape[1]) if n else 0
        d_e = int(mgs[0].E.shape[1]) if n else 0
        Vt, Et = int(n_atoms.sum()), int(n_edges.sum())
        # keep converted arrays alive for the duration of the C call
        Vs = [np.ascontiguousarray(mg.V, dtype=np.float32) for mg in mgs]
        Es = [np.ascontiguousarray(mg.E, dtype=np.float32) for mg in mgs]
        EIs = [np.ascontiguousarray(mg.edge_index, dtype=np.int64) for mg in mgs]
        RVs = [np.ascontiguousarray(mg.rev_edge_index, dtype=np.int64) for mg in mgs]
        for mg, e, ne in zip(mgs, Es, n_edges):
            if e.shape[0] != ne:
                raise ValueError(f"MolGraph.E has {e.shape[0]} rows but edge_index has {ne} edges")

        def ptrs(arrs):
            return np.fromiter((a.__array_interface__["data"][0] for a in arrs), dtype=np.uint64, count=n)

        pV, pE, pEI, pRV = ptrs(Vs), ptrs(Es), ptrs(EIs), ptrs(RVs)
        xf = self._alloc(Vt, Et, d_v, d_e, kw, compact)
        lib = _lib.load()
        rc = lib.dmpnn_collate_host(
            n, n_atoms.ctypes.data, n_edges.ctypes.data, pV.ctypes.data, pE.ctypes.data, pEI.ctypes.data,
            pRV.ctypes.data, d_v, d_e, self.V.data_ptr(), self.E.data_ptr(), self.edge_index.data_ptr(),
            self.rev_edge_index.data_ptr(), self.batch.data_ptr(),
        )
        _lib.check(rc, "dmpnn_collate_host")
        if xf is not None:
            rc = lib.dmpnn_collate_host_compact(
                n, n_atoms.ctypes.data, n_edges.ctypes.data, pV.ctypes.data, pE.ctypes.data, pEI.ctypes.data,
                pRV.ctypes.data, d_v, d_e, *(t.data_ptr() for t in xf))
            _lib.check(rc, "dmpnn_collate_host_compact")
        self._xfer = xf

    @classmethod
    def from_tensors(cls, V: Tensor, E: Tensor, edge_index: Tensor, rev_edge_index: Tensor, batch: Tensor,
                     size: int) -> "BatchMolGraph":
        """Wrap already-batched tensors (e.g. the five leaves of a reference BatchMolGraph)."""
        bmg = object.__new__(cls)
        bmg.V, bmg.E, bmg._edge_index, bmg._rev_edge_index, bmg._batch = V, E, edge_index, rev_edge_index, batch
        bmg._size = int(size)
        bmg._layout = None
        bmg._xfer = None
        bmg._meta_host = host_meta(edge_index, rev_edge_index, batch, int(size))   # None for device tensors
        return bmg

    def __len__(self) -> int:
        return self._size

    def _moved(self, dev: torch.device, non_blocking: bool):
        """The five public tensors on `dev` (through the compact staging copy when there is one)."""
        if self._xfer is not None and dev.type == "cuda" and not self.V.is_cuda:
            Vb, Eb, ei, rv, bt = (t.to(dev, non_blocking=non_blocking) for t in self._xfer)
            return Vb.float(), Eb.float(), ei.long(), rv.long(), bt.long()
        return tuple(t.to(dev, non_blocking=non_blocking)
                     for t in (self.V, self.E, self.edge_index, self.rev_edge_index, self.batch))

    def transfer_nbytes(self) -> int:
        """Bytes a host -> device move of this batch copies."""
        ts = self._xfer if self._xfer is not None else (self.V, self.E, self.edge_index, self.rev_edge_index, self.batch)
        return sum(t.numel() * t.element_size() for t in ts)

    def to(self, device, non_blocking: bool = False):
        """In place, returns None (chemprop/data/collate.py:68-73)."""
        dev = torch.device(device)
        meta = self._meta_host                     # the index values do not change with the device
        self.V, self.E, self.edge_index, self.rev_edge_index, self.batch = self._moved(dev, non_blocking)
        self._meta_host = meta
        if dev.type == "cuda":
            self._xfer = None

    def cuda_copy(self, device="cuda", non_blocking: bool = True) -> "BatchMolGraph":
        """A device-resident copy; this (pinned) host batch stays intact, e.g. for reuse by a loader."""
        out = BatchMolGraph.from_tensors(*self._moved(torch.device(device), non_blocking), self._size)
        out._meta_host = self._meta_host
        return out

    def __copy__(self):
        # GraphTransform makes a shallow copy and replaces V / E (chemprop/nn/transforms.py:69-72);
        # the index layout stays valid for the copy.
        new = object.__new__(type(self))
        for s in self.__slots__:
            if s != "__weakref__":
                setattr(new, s, getattr(self, s))
        return new


class Datum(NamedTuple):
    """chemprop/data/datasets.py `Datum` (fields in the same order)."""
    mg: MolGraph
    V_d: np.ndarray | None
    x_d: np.ndarray | None
    y: np.ndarray | None
    weight: float
    lt_mask: np.ndarray | None
    gt_mask: np.ndarray | None


class TrainingBatch(NamedTuple):
    bmg: BatchMolGraph
    V_d: Tensor | None
    X_d: Tensor | None
    Y: Tensor | None
    w: Tensor
    lt_mask: Tensor | None
    gt_mask: Tensor | None


def collate_batch(batch: Iterable[Datum], pack_tiles: bool = False) -> TrainingBatch:
    """Same contract as chemprop/data/collate.py:86-97.  `pack_tiles=True` (training loaders:
    `DataLoader(..., collate_fn=functools.partial(collate_batch, pack_tiles=True))`) reorders the data of the batch --
    molecules, descriptors, targets, weights, masks, all alike -- by `tile_packing_order` so that the engine's tiles come
    out nearly full; leave it off where the caller relies on the order inside a batch (prediction)."""
    batch = list(batch)
    if pack_tiles and len(batch) > 1:
        order = tile_packing_order_of([d[0] for d in batch])
        batch = [batch[i] for i in order]
    mgs, V_ds, *rest = zip(*batch)
    return TrainingBatch(BatchMolGraph(mgs), _cat_V_d(V_ds), *_molecule_tensors(*rest))


def _cat_V_d(V_ds) -> Tensor | None:
    return None if V_ds[0] is None else torch.from_numpy(np.concatenate(V_ds)).float()


def _molecule_tensors(x_ds, ys, weights, lt_masks, gt_masks) -> tuple:
    """X_d, Y, w, lt_mask, gt_mask of a batch (chemprop/data/collate.py:90-96)."""
    return (
        None if x_ds[0] is None else torch.from_numpy(np.array(x_ds)).float(),
        None if ys[0] is None else torch.from_numpy(np.array(ys)).float(),
        torch.tensor(weights, dtype=torch.float).unsqueeze(1),
        None if lt_masks[0] is None else torch.from_numpy(np.array(lt_masks)),
        None if gt_masks[0] is None else torch.from_numpy(np.array(gt_masks)),
    )


class MulticomponentTrainingBatch(NamedTuple):
    """chemprop/data/collate.py:186-193.  `bmgs`: one batch per component, or ONE union batch (see
    `collate_multicomponent`); `V_ds` accordingly a list per component or one tensor in union atom order."""
    bmgs: list[BatchMolGraph] | BatchMolGraph
    V_ds: list[Tensor | None] | Tensor | None
    X_d: Tensor | None
    Y: Tensor | None
    w: Tensor
    lt_mask: Tensor | None
    gt_mask: Tensor | None


def collate_multicomponent(batches: Iterable[Sequence[Datum]], union: bool = False) -> MulticomponentTrainingBatch:
    """chemprop/data/collate.py:196-208: `batches` holds one sequence of N Datums (one per component) per data point.
    `union=False`: one BatchMolGraph per component, as the reference.  `union=True`: ONE BatchMolGraph of all N * b
    molecules in datapoint-major interleaved order -- union molecule m * N + c is component c of data point m -- with its
    host layout meta words (graph-capturable), for a shared encoder (EngineMulticomponentMPNN); its `V_ds` is one tensor
    in union atom order (None when component 0 has none).  X_d, Y, weights and masks come from component 0, as in the
    reference."""
    batches = [list(dp) for dp in batches]
    comps = list(zip(*batches))
    head = _molecule_tensors(*list(zip(*comps[0]))[2:])
    if not union:
        tbs = [collate_batch(batch) for batch in comps]
        return MulticomponentTrainingBatch([tb.bmg for tb in tbs], [tb.V_d for tb in tbs], *head)
    union_data = [d for dp in batches for d in dp]
    V_ds = None if comps[0][0].V_d is None else _cat_V_d([d.V_d for d in union_data])
    return MulticomponentTrainingBatch(BatchMolGraph([d.mg for d in union_data]), V_ds, *head)
