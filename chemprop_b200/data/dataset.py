"""`PackedMolGraphDataset`: every molecule of a (pre-featurised) data set in six flat arrays, on the host or resident
in HBM, and batch assembly as ONE gather (SURVEY.md section 8f-1).

What it replaces: the reference builds a batch with `[dataset[i] for i in ids]` (`MoleculeDataset.__getitem__`,
chemprop/data/datasets.py:222-244) followed by `collate_batch` (chemprop/data/collate.py:86-97), i.e. a Python loop over
molecules plus `np.concatenate` per field (collate.py:48-62; ~15 k molecules/s per worker process), and then copies
the batch to the GPU.  Here the molecules are packed once (`from_molgraphs`):

    V_all  (sum V x d_v, f32)      atom_ptr (n + 1, int64)      edge_index local to the molecule (2 x sum E, int32)
    E_all  (sum E x d_e, f32)      edge_ptr (n + 1, int64)      rev_edge_index local to the molecule (sum E, int32)

and `batch(ids)` returns the same `BatchMolGraph` the collate would have built for those molecules (bit-identical
tensors, tests/test_dataset.py) from contiguous row copies:

  * host data set   -> `dmpnn_dataset_gather_host` (one C pass; optionally also the bf16 / int32 transfer copy);
  * `.to("cuda")`   -> `dmpnn_dataset_gather` (one kernel launch; the step uploads 24 bytes per molecule -- ids and
                       output offsets -- instead of ~5.7 kB per molecule of features and indices).

Either way the batch carries its layout meta words (flags, tile count), computed on the host in O(batch size) from
per-molecule sizes, so the training step issues no host <-> device synchronisation.  Molecules are validated once,
here, instead of per batch.
"""
from __future__ import annotations

from typing import Sequence

import numpy as np
import torch

from .. import _lib
from .collate import BatchMolGraph, tile_packing_order
from .molgraph import MolGraph


class HostBatchBuffer:
    """Reusable (optionally pinned) staging memory for host batches.  A loader keeps two or three of these and passes
    one to `PackedMolGraphDataset.batch(ids, buffer=...)`: the gather then writes into memory that is already mapped
    (fresh allocations make the gather page-fault bound: ~2 GB/s instead of memcpy speed) and, when pinned, ready for
    an asynchronous host -> device copy.  The returned BatchMolGraph's tensors are views of this buffer: it is valid
    until the buffer is handed to the next `batch` call."""

    def __init__(self, d_v: int, d_e: int, atoms: int = 0, edges: int = 0, pin_memory: bool = False, compact: bool = False):
        self.d_v, self.d_e, self.pin_memory, self.compact = int(d_v), int(d_e), bool(pin_memory), bool(compact)
        self.cap_atoms = self.cap_edges = -1
        self._reserve(int(atoms), int(edges))

    def _reserve(self, atoms: int, edges: int):
        if atoms <= self.cap_atoms and edges <= self.cap_edges:
            return
        self.cap_atoms = max(atoms, int(self.cap_atoms * 1.25))
        self.cap_edges = max(edges, int(self.cap_edges * 1.25))
        kw = dict(pin_memory=True) if self.pin_memory else {}
        A, Eg = max(self.cap_atoms, 1), max(self.cap_edges, 1)
        self.V = torch.empty((A, self.d_v), dtype=torch.float32, **kw)
        self.E = torch.empty((Eg, self.d_e), dtype=torch.float32, **kw)
        self.ei = torch.empty((2 * Eg,), dtype=torch.int64, **kw)
        self.rev = torch.empty((Eg,), dtype=torch.int64, **kw)
        self.bt = torch.empty((A,), dtype=torch.int64, **kw)
        if self.compact:
            self.Vb = torch.empty((A, self.d_v), dtype=torch.bfloat16, **kw)
            self.Eb = torch.empty((Eg, self.d_e), dtype=torch.bfloat16, **kw)
            self.ei32 = torch.empty((2 * Eg,), dtype=torch.int32, **kw)
            self.rev32 = torch.empty((Eg,), dtype=torch.int32, **kw)
            self.bt32 = torch.empty((A,), dtype=torch.int32, **kw)

    def views(self, Vt: int, Et: int):
        self._reserve(Vt, Et)
        pub = (self.V[:Vt], self.E[:Et], self.ei[:2 * Et].view(2, Et), self.rev[:Et], self.bt[:Vt])
        xf = ((self.Vb[:Vt], self.Eb[:Et], self.ei32[:2 * Et].view(2, Et), self.rev32[:Et], self.bt32[:Vt])
              if self.compact else None)
        return pub, xf


class PackedMolGraphDataset:
    def __init__(self, V_all, E_all, ei_local, rev_local, atom_ptr, edge_ptr, mol_max_indeg):
        self.V_all, self.E_all, self.ei_local, self.rev_local = V_all, E_all, ei_local, rev_local
        self.atom_ptr, self.edge_ptr = atom_ptr, edge_ptr              # int64 torch tensors on the data set's device
        self._atom_ptr_h = atom_ptr.cpu().numpy() if atom_ptr.is_cuda else atom_ptr.numpy()   # host copies: offsets of a
        self._edge_ptr_h = edge_ptr.cpu().numpy() if edge_ptr.is_cuda else edge_ptr.numpy()   # batch are computed on the host
        self._max_indeg_h = np.ascontiguousarray(mol_max_indeg, dtype=np.int32)

    # ------------------------------------------------------------------------------------------------
    @classmethod
    def from_molgraphs(cls, mgs: Sequence[MolGraph], pin_memory: bool = False) -> "PackedMolGraphDataset":
        """Pack a list of MolGraphs (one collate of the whole data set, then global -> molecule-local indices)."""
        whole = BatchMolGraph(mgs, pin_memory=pin_memory)
        n = len(whole)
        meta = whole._meta_host
        if meta is None or meta[_lib.META_FLAGS] != 7:
            from ..engine import check_flags

            check_flags(0 if meta is None else meta[_lib.META_FLAGS])
        ei, rev, bt = whole.edge_index.numpy(), whole.rev_edge_index.numpy(), whole.batch.numpy()
        V, E = int(bt.shape[0]), int(ei.shape[1])
        atom_ptr = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(bt, minlength=n), out=atom_ptr[1:])
        mol_of_edge = bt[ei[0]] if E else np.zeros(0, np.int64)
        edge_ptr = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(np.bincount(mol_of_edge, minlength=n), out=edge_ptr[1:])
        if E and np.any(np.diff(mol_of_edge) < 0):
            raise ValueError("edges of a molecule must be contiguous")   # cannot happen for a collate of MolGraphs
        if (np.diff(atom_ptr) >= 2 ** 31).any() or (np.diff(edge_ptr) >= 2 ** 31).any():
            raise ValueError("molecule too large for int32 local indices")
        ei_local = (ei - atom_ptr[mol_of_edge][None, :]).astype(np.int32)
        rev_local = (rev - edge_ptr[mol_of_edge]).astype(np.int32)
        deg = np.bincount(ei[1], minlength=V) if E else np.zeros(V, np.int64)
        mol_max_indeg = np.zeros(n, dtype=np.int32)
        nz = np.flatnonzero(np.diff(atom_ptr) > 0)
        if V:
            mol_max_indeg[nz] = np.maximum.reduceat(deg, atom_ptr[nz]).astype(np.int32)
        kw = dict(pin_memory=True) if pin_memory else {}

        def t(a, dtype):
            out = torch.empty(a.shape, dtype=dtype, **kw)
            out.copy_(torch.from_numpy(np.ascontiguousarray(a)))
            return out

        return cls(whole.V, whole.E, t(ei_local, torch.int32), t(rev_local, torch.int32), t(atom_ptr, torch.int64),
                   t(edge_ptr, torch.int64), mol_max_indeg)

    # ------------------------------------------------------------------------------------------------
    def __len__(self) -> int:
        return int(self._atom_ptr_h.shape[0]) - 1

    @property
    def device(self) -> torch.device:
        return self.V_all.device

    @property
    def d_v(self) -> int:
        return int(self.V_all.shape[1])

    @property
    def d_e(self) -> int:
        return int(self.E_all.shape[1])

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in (self.V_all, self.E_all, self.ei_local, self.rev_local,
                                                          self.atom_ptr, self.edge_ptr))

    def n_atoms(self, ids=None) -> np.ndarray:
        d = np.diff(self._atom_ptr_h)
        return d if ids is None else d[np.asarray(ids, dtype=np.int64)]

    def n_edges(self, ids=None) -> np.ndarray:
        d = np.diff(self._edge_ptr_h)
        return d if ids is None else d[np.asarray(ids, dtype=np.int64)]

    def host_buffer(self, pin_memory: bool = False, compact: bool = False) -> HostBatchBuffer:
        """Staging memory for `batch(ids, buffer=...)` of this data set."""
        return HostBatchBuffer(self.d_v, self.d_e, pin_memory=pin_memory, compact=compact)

    def to(self, device, non_blocking: bool = False) -> "PackedMolGraphDataset":
        """A copy of the data set on `device` (the six arrays; a few GB per million molecules)."""
        dev = torch.device(device)
        mv = lambda x: x.to(dev, non_blocking=non_blocking)  # noqa: E731
        return PackedMolGraphDataset(mv(self.V_all), mv(self.E_all), mv(self.ei_local), mv(self.rev_local),
                                     mv(self.atom_ptr), mv(self.edge_ptr), self._max_indeg_h)

    def replicate(self, k: int) -> "PackedMolGraphDataset":
        """The data set repeated `k` times (molecule i + j * len(self) is a copy of molecule i): a cheap way to a large
        synthetic data set (bench.py's 1 M-molecule configuration) from a generator that makes ~7 k molecules/s."""
        k = int(k)
        if k < 1:
            raise ValueError("k >= 1")
        if k == 1:
            return self
        return PackedMolGraphDataset.concatenate([self] * k)

    @classmethod
    def concatenate(cls, datasets: Sequence["PackedMolGraphDataset"]) -> "PackedMolGraphDataset":
        """One data set holding the molecules of `datasets` one after the other (molecule i of datasets[j] is molecule
        i + sum_{j' < j} len(datasets[j'])); the feature widths and the device must agree."""
        if not datasets:
            raise ValueError("nothing to concatenate")
        d0 = datasets[0]
        if any((d.d_v, d.d_e, d.device) != (d0.d_v, d0.d_e, d0.device) for d in datasets):
            raise ValueError("data sets of different feature widths or devices cannot be concatenated")

        def cat_ptr(ptrs):
            out, base = [], 0
            for p in ptrs:
                out.append(torch.from_numpy(p[:-1] + base))
                base += int(p[-1])
            return torch.cat(out + [torch.tensor([base], dtype=torch.int64)]).to(d0.device)

        return cls(torch.cat([d.V_all for d in datasets]), torch.cat([d.E_all for d in datasets]),
                   torch.cat([d.ei_local for d in datasets], 1), torch.cat([d.rev_local for d in datasets]),
                   cat_ptr([d._atom_ptr_h for d in datasets]), cat_ptr([d._edge_ptr_h for d in datasets]),
                   np.concatenate([d._max_indeg_h for d in datasets]))

    def molgraph(self, i: int) -> MolGraph:
        """Molecule `i` as a MolGraph (host data sets; for inspection and tests)."""
        a0, a1, e0, e1 = (int(x) for x in (*self._atom_ptr_h[i:i + 2], *self._edge_ptr_h[i:i + 2]))
        return MolGraph(self.V_all[a0:a1].cpu().numpy(), self.E_all[e0:e1].cpu().numpy(),
                        self.ei_local[:, e0:e1].cpu().numpy().astype(np.int64),
                        self.rev_local[e0:e1].cpu().numpy().astype(np.int64))

    # ------------------------------------------------------------------------------------------------
    def _plan(self, ids):
        """ids (int64), output offsets and the batch's layout meta words -- all on the host, O(len(ids))."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        if ids.ndim != 1:
            raise ValueError("ids must be one-dimensional")
        n = int(ids.shape[0])
        plan = np.empty(3 * n + 2, dtype=np.int64)        # [ids | out_atom_ptr (n + 1) | out_edge_ptr (n + 1)]
        plan[:n] = ids
        meta = np.zeros(_lib.META_WORDS, dtype=np.int32)
        lib = _lib.load()
        rc = lib.dmpnn_dataset_batch_meta_host(
            n, plan.ctypes.data, len(self), self._atom_ptr_h.ctypes.data, self._edge_ptr_h.ctypes.data,
            self._max_indeg_h.ctypes.data, plan[n:].ctypes.data, plan[2 * n + 1:].ctypes.data, meta.ctypes.data)
        _lib.check(rc, "dmpnn_dataset_batch_meta_host")
        return plan, n, int(plan[2 * n]), int(plan[3 * n + 1]), meta.tolist()

    def packed_order(self, ids) -> np.ndarray:
        """`ids` reordered so that the batch's tiles come out nearly full (see `tile_packing_order`)."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        na = self._atom_ptr_h[ids + 1] - self._atom_ptr_h[ids]
        ne = self._edge_ptr_h[ids + 1] - self._edge_ptr_h[ids]
        return ids[tile_packing_order(na, ne)]

    def plan(self, ids):
        """The host half of `batch(ids)`: ids, output offsets and the layout meta words (O(len(ids)), pure host work, safe to
        run on a loader thread ahead of time); hand the result to `batch(ids, plan=...)`."""
        return self._plan(ids)

    def batch(self, ids, pin_memory: bool = False, transfer_dtype: torch.dtype | None = None,
              buffer: HostBatchBuffer | None = None, n_threads: int = 0, plan=None) -> BatchMolGraph:
        """The BatchMolGraph of molecules `ids` (in that order; repeats allowed), on this data set's device.
        Host data sets: `buffer` = reusable staging memory to gather into (see HostBatchBuffer); its `compact` flag
        then decides whether the bf16 / int32 transfer copy is produced; `n_threads` host threads share the copy (0 =
        automatic: one per 2048 molecules, at most 8).  `plan`: the result of `plan(ids)` computed earlier."""
        plan, n, Vt, Et, meta = self._plan(ids) if plan is None else plan
        lib = _lib.load()
        if self.device.type == "cuda":
            if transfer_dtype is not None:
                raise ValueError("transfer_dtype applies to host data sets (a resident data set transfers nothing)")
            dev = self.device
            stage = torch.empty(plan.shape[0], dtype=torch.int64, pin_memory=True)
            stage.numpy()[:] = plan
            dplan = stage.to(dev, non_blocking=True)          # 24 bytes per molecule: all a step uploads
            f32, i64 = dict(dtype=torch.float32, device=dev), dict(dtype=torch.int64, device=dev)
            V, E = torch.empty((Vt, self.d_v), **f32), torch.empty((Et, self.d_e), **f32)
            ei, rev, bt = torch.empty((2, Et), **i64), torch.empty((Et,), **i64), torch.empty((Vt,), **i64)
            if n > 0:
                with torch.cuda.device(dev):
                    rc = lib.dmpnn_dataset_gather(
                        dplan.data_ptr(), dplan[n:].data_ptr(), dplan[2 * n + 1:].data_ptr(), n,
                        self.atom_ptr.data_ptr(), self.edge_ptr.data_ptr(), self.V_all.data_ptr(), self.E_all.data_ptr(),
                        self.ei_local.data_ptr(), self.rev_local.data_ptr(), int(self.ei_local.shape[1]), self.d_v,
                        self.d_e, V.data_ptr(), E.data_ptr(), ei.data_ptr(), rev.data_ptr(), bt.data_ptr(), Et,
                        torch.cuda.current_stream(dev).cuda_stream)
                _lib.check(rc, "dmpnn_dataset_gather")
            bmg = BatchMolGraph.from_tensors(V, E, ei, rev, bt, n)
            bmg._meta_host = meta
            return bmg
        if transfer_dtype is not None and transfer_dtype != torch.bfloat16:
            raise ValueError("transfer_dtype must be torch.bfloat16 or None")
        bmg = object.__new__(BatchMolGraph)
        bmg._size, bmg._layout, bmg._xfer, bmg._meta_host = n, None, None, None
        if buffer is not None:
            if (buffer.d_v, buffer.d_e) != (self.d_v, self.d_e):
                raise ValueError("buffer feature widths do not match the data set")
            pub, xf = buffer.views(Vt, Et)
            bmg.V, bmg.E, bmg._edge_index, bmg._rev_edge_index, bmg._batch = pub
        else:
            kw = dict(pin_memory=True) if pin_memory else {}
            xf = bmg._alloc(Vt, Et, self.d_v, self.d_e, kw, transfer_dtype is not None)
        out = (bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch) + (xf or (None,) * 5)
        rc = lib.dmpnn_dataset_gather_host(
            n, plan.ctypes.data, plan[n:].ctypes.data, plan[2 * n + 1:].ctypes.data, self._atom_ptr_h.ctypes.data,
            self._edge_ptr_h.ctypes.data, self.V_all.data_ptr(), self.E_all.data_ptr(), self.ei_local.data_ptr(),
            self.rev_local.data_ptr(), int(self.ei_local.shape[1]), self.d_v, self.d_e,
            *(None if t is None else t.data_ptr() for t in out), int(n_threads))
        _lib.check(rc, "dmpnn_dataset_gather_host")
        bmg._xfer = xf
        bmg._meta_host = meta
        return bmg


class MulticomponentPackedDataset:
    """N aligned `PackedMolGraphDataset`s (component c of data point m is molecule m of `datasets[c]`) behind the interface
    `PackedBatchLoader` draws from, so that the loader's samplers, sharding, `drop_last` rule, `arrays` / `extras`,
    prefetching and host / HBM-resident modes apply unchanged; ids are DATA POINT ids.

      * `union=True` (shared encoder; the components must agree in d_v / d_e): the components are stacked once, component c
        of data point m being packed molecule c * n + m, and `batch(ids)` is ONE union BatchMolGraph in datapoint-major
        interleaved order (union molecule k * N + c is component c of ids[k]) -- one `dmpnn_dataset_gather` (or its host
        twin) over the expanded ids [m_0, n + m_0, ..., m_1, n + m_1, ...], its layout meta words planned on the host.  Only
        the stacked copy is kept (the given data sets are not referenced), so the features are held once.
      * `union=False`: `batch(ids)` is the list of the N components' batches of the same ids.

    `packed_order(ids)` orders data points by their summed sizes (`tile_packing_order`); each data point's molecules then
    stay together, in component order."""

    def __init__(self, datasets: Sequence[PackedMolGraphDataset], union: bool = False):
        datasets = list(datasets)
        if not datasets:
            raise ValueError("no components")
        n = len(datasets[0])
        if any(len(d) != n for d in datasets):
            raise ValueError("the components' data sets must have one molecule per data point each (equal lengths)")
        if len({d.device for d in datasets}) != 1:
            raise ValueError("the components' data sets must live on one device")
        self.union, self._n, self._N = bool(union), n, len(datasets)
        # per data point, the atoms and edges of all its components (host arrays: the tile-packing order)
        self._atoms = sum(d.n_atoms() for d in datasets)
        self._edges = sum(d.n_edges() for d in datasets)
        self.components = None if self.union else datasets
        self.stacked = PackedMolGraphDataset.concatenate(datasets) if self.union else None

    def __len__(self) -> int:
        return self._n

    @property
    def n_components(self) -> int:
        return self._N

    @property
    def device(self) -> torch.device:
        return self.stacked.device if self.union else self.components[0].device

    def to(self, device, non_blocking: bool = False) -> "MulticomponentPackedDataset":
        out = object.__new__(MulticomponentPackedDataset)
        out.__dict__.update(self.__dict__)
        if self.union:
            out.stacked = self.stacked.to(device, non_blocking)
        else:
            out.components = [d.to(device, non_blocking) for d in self.components]
        return out

    def union_ids(self, ids) -> np.ndarray:
        """The packed molecule ids of the union batch of data points `ids`: [m_0, n + m_0, ..., m_1, n + m_1, ...]."""
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        return (ids[:, None] + self._n * np.arange(self._N, dtype=np.int64)[None, :]).reshape(-1)

    def packed_order(self, ids) -> np.ndarray:
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        return ids[tile_packing_order(self._atoms[ids], self._edges[ids])]

    def plan(self, ids):
        if self.union:
            return self.stacked.plan(self.union_ids(ids))
        return [d.plan(ids) for d in self.components]

    def host_buffer(self, pin_memory: bool = False, compact: bool = False):
        if self.union:
            return self.stacked.host_buffer(pin_memory, compact)
        return [d.host_buffer(pin_memory, compact) for d in self.components]

    def batch(self, ids, pin_memory: bool = False, transfer_dtype: torch.dtype | None = None, buffer=None,
              n_threads: int = 0, plan=None):
        """The union BatchMolGraph of data points `ids` (union=True), or the list of the components' BatchMolGraphs."""
        kw = dict(pin_memory=pin_memory, transfer_dtype=transfer_dtype, n_threads=n_threads)
        if self.union:
            return self.stacked.batch(self.union_ids(ids), buffer=buffer, plan=plan, **kw)
        buffers = [None] * self._N if buffer is None else buffer
        plans = [None] * self._N if plan is None else plan
        return [d.batch(ids, buffer=b, plan=p, **kw) for d, b, p in zip(self.components, buffers, plans)]
