"""`PackedBatchLoader`: the loader side of the path for pre-featurised data -- what `build_dataloader`
(chemprop/data/dataloader.py:24-96: `DataLoader(dataset, batch_size, sampler=SeededSampler | RandomSampler, collate_fn=
collate_batch, drop_last=...)`) and Lightning's `DistributedSampler` (chemprop/cli/train.py:1930-1939) do in the reference,
on top of a `PackedMolGraphDataset`:

  * index order: `SeededSampler` semantics when `shuffle and seed is not None` (chemprop/data/samplers.py:8-27: one
    `default_rng(seed)`, `rg.shuffle(idxs)` in place at the start of every epoch -- the same permutations as the reference,
    tests/test_loader.py), `torch.randperm` when unseeded, `arange` when not shuffling;
  * `drop_last=None` drops a trailing batch of size 1 (dataloader.py:77-86: batch norm cannot take it);
  * data parallel: rank r of `world` takes every world-th index of the (padded) epoch order, like `DistributedSampler`;
  * batch assembly: host data set -> a producer thread gathers batch i+1 (`dmpnn_dataset_gather_host`, multi-threaded)
    into a ring of reusable (pinned) `HostBatchBuffer`s while the consumer trains on batch i; with `device="cuda"` the
    host -> device copy is issued asynchronously on a side stream and the consumer's stream waits on its event; a data
    set that is already resident in HBM is gathered directly on the device (one launch, no thread, no copy).

  * `pack_tiles=True` (default): inside each batch the molecules are ordered by `dmpnn_tile_pack_order` so that the
    engine's 128-row tiles come out ~0.94 full instead of ~0.81 (the fused depth step costs the same per tile whatever its
    fill); batch membership is the sampler's, `LoadedBatch.ids` / `extras` follow the order used.

A `MulticomponentPackedDataset` is drawn from the same way, by data point: each batch is one union BatchMolGraph of its
data points' components in interleaved order (`union=True`) or the list of the components' batches of the same ids.

Per-molecule side arrays (`Y`, `weights`, `X_d`, ... -- anything indexed by molecule) given as `arrays={name: ndarray}`
come back gathered for the batch in `batch.extras[name]`.
"""
from __future__ import annotations

import queue
import threading
from typing import Iterator, NamedTuple

import numpy as np
import torch

from .collate import BatchMolGraph
from .dataset import MulticomponentPackedDataset, PackedMolGraphDataset


class LoadedBatch(NamedTuple):
    bmg: BatchMolGraph       # a list of one batch per component for MulticomponentPackedDataset(union=False)
    ids: np.ndarray          # molecule (data point) ids of the batch, in batch order
    extras: dict             # name -> tensor gathered from `arrays`


def epoch_shard(order: np.ndarray, rank: int, world: int) -> np.ndarray:
    """DistributedSampler's split: pad the epoch order to a multiple of `world` by repeating its head, then stride."""
    if world <= 1:
        return order
    n = order.shape[0]
    total = -(-n // world) * world
    if total > n:
        reps = -(-(total - n) // max(n, 1))
        order = np.concatenate([order] + [order] * reps)[:total] if n else order
    return order[rank:total:world]


def _cuda_copy(host, device):
    """A host batch -- or a list of them (MulticomponentPackedDataset(union=False)) -- copied to `device` asynchronously."""
    if isinstance(host, list):
        return [h.cuda_copy(device, non_blocking=True) for h in host]
    return host.cuda_copy(device, non_blocking=True)


class PackedBatchLoader:
    def __init__(self, dataset: PackedMolGraphDataset | MulticomponentPackedDataset, batch_size: int = 64, shuffle: bool = True,
                 seed: int | None = None, drop_last: bool | None = None, rank: int = 0, world: int = 1,
                 device: str | torch.device | None = None, prefetch: int = 3, transfer_dtype: torch.dtype | None = None,
                 arrays: dict | None = None, n_threads: int = 0, pack_tiles: bool = True):
        if batch_size <= 0 or world <= 0 or not 0 <= rank < world or prefetch < 2:
            raise ValueError("bad batch_size / rank / world / prefetch (prefetch >= 2)")
        self.dataset, self.batch_size, self.shuffle = dataset, int(batch_size), bool(shuffle)
        self.rank, self.world, self.prefetch, self.n_threads = int(rank), int(world), int(prefetch), int(n_threads)
        self.device = None if device is None else torch.device(device)
        self.transfer_dtype = transfer_dtype
        self.pack_tiles = bool(pack_tiles)
        self.arrays = {k: np.asarray(v) for k, v in (arrays or {}).items()}
        n = len(dataset)
        for k, v in self.arrays.items():
            if v.shape[0] != n:
                raise ValueError(f"arrays[{k!r}] has {v.shape[0]} rows for {n} molecules")
        self._idxs = np.arange(n)                                   # samplers.py:16
        self._rg = np.random.default_rng(seed) if (shuffle and seed is not None) else None   # samplers.py:17
        per_rank = -(-n // self.world) if self.world > 1 else n
        if drop_last is None:                                       # dataloader.py:77-86
            drop_last = per_rank % self.batch_size == 1
        self.drop_last = bool(drop_last)
        self._per_rank = per_rank

    def __len__(self) -> int:
        full, rem = divmod(self._per_rank, self.batch_size)
        return full + (1 if rem and not self.drop_last else 0)

    # ------------------------------------------------------------------------------------------------
    def epoch_order(self) -> np.ndarray:
        """This epoch's molecule order for THIS rank (advances the sampler state, like iterating the reference's)."""
        if not self.shuffle:
            order = self._idxs
        elif self._rg is not None:
            self._rg.shuffle(self._idxs)                            # samplers.py:21 (in place, cumulative over epochs)
            order = self._idxs.copy()
        else:
            order = torch.randperm(len(self.dataset)).numpy()
        return epoch_shard(order, self.rank, self.world)

    def batches_of(self, order: np.ndarray, pack: bool | None = None) -> list[np.ndarray]:
        out = [order[i:i + self.batch_size] for i in range(0, order.shape[0], self.batch_size)]
        if out and self.drop_last and out[-1].shape[0] < self.batch_size:
            out.pop()
        if self.pack_tiles if pack is None else pack:   # same molecules per batch, ordered for full tiles; `LoadedBatch.ids` reports the order
            out = [self.dataset.packed_order(ids) for ids in out]
        return out

    def _extras(self, ids: np.ndarray) -> dict:
        out = {}
        for k, v in self.arrays.items():
            t = torch.from_numpy(np.ascontiguousarray(v[ids]))
            if self.device is not None and self.device.type == "cuda":
                t = t.pin_memory().to(self.device, non_blocking=True)
            out[k] = t
        return out

    def _resident_batches(self, epochs: int | None) -> Iterator[LoadedBatch]:
        """Resident data set: the batch is gathered on the device (one launch), but its HOST half -- the tile-packing order of
        the molecules (~1.6 ms per 10 k molecules) and the plan (ids, output offsets, meta words) -- runs on a producer
        thread `prefetch` batches ahead (across epoch boundaries when `epochs` is None or > 1), so that the training loop's
        thread only uploads the plan and launches."""
        ds = self.dataset
        q: queue.Queue = queue.Queue(maxsize=self.prefetch)
        stop = threading.Event()

        def put(item):
            # the queue is bounded: never block for good on a consumer that has gone away (early `break`, exception)
            while not stop.is_set():
                try:
                    q.put(item, timeout=0.1)
                    return
                except queue.Full:
                    pass

        def produce_plans():
            try:
                e = 0
                while (epochs is None or e < epochs) and not stop.is_set():
                    for ids in self.batches_of(self.epoch_order(), pack=False):
                        if stop.is_set():
                            return
                        ids = ds.packed_order(ids) if self.pack_tiles else ids
                        put((ids, ds.plan(ids)))
                    e += 1
                put(None)
            except BaseException as ex:  # noqa: BLE001 -- handed to the consumer
                put(ex)

        th = threading.Thread(target=produce_plans, daemon=True, name="packed-batch-planner")
        th.start()
        try:
            while True:
                item = q.get()
                if item is None:
                    break
                if isinstance(item, BaseException):
                    raise item
                ids, plan = item
                yield LoadedBatch(ds.batch(ids, plan=plan), ids, self._extras(ids))
        finally:
            stop.set()
            th.join(timeout=5)

    def stream(self) -> Iterator[LoadedBatch]:
        """Batches for ever, epoch after epoch (the sampler reshuffles at every epoch boundary), without draining the
        prefetch pipeline between epochs.  `for batch in loader` is one epoch."""
        if self.dataset.device.type == "cuda":
            yield from self._resident_batches(epochs=None)
        else:
            while True:
                yield from iter(self)

    def __iter__(self) -> Iterator[LoadedBatch]:
        ds = self.dataset
        if ds.device.type == "cuda":
            yield from self._resident_batches(epochs=1)
            return
        chunks = self.batches_of(self.epoch_order())
        to_cuda = self.device is not None and self.device.type == "cuda"
        compact = self.transfer_dtype is not None
        ring = [ds.host_buffer(pin_memory=to_cuda, compact=compact) for _ in range(self.prefetch)]
        free_evt = [None] * self.prefetch                           # H2D-complete event of the last use of each buffer
        free: queue.Queue = queue.Queue()                           # staging buffers the producer may write
        for k in range(self.prefetch):
            free.put(k)
        q: queue.Queue = queue.Queue()                              # gathered batches (bounded by the buffers)
        stop = threading.Event()

        def produce():
            try:
                for ids in chunks:
                    k = free.get()
                    if k < 0 or stop.is_set():
                        return
                    if free_evt[k] is not None:
                        free_evt[k].synchronize()                   # its previous H2D copy has left the buffer
                    q.put((k, ids, ds.batch(ids, buffer=ring[k], n_threads=self.n_threads)))
                q.put(None)
            except BaseException as e:  # noqa: BLE001 -- handed to the consumer
                q.put(e)

        th = threading.Thread(target=produce, daemon=True, name="packed-batch-loader")
        th.start()
        copy_stream = torch.cuda.Stream(device=self.device) if to_cuda else None
        try:
            while True:
                item = q.get()
                if item is None:
                    break
                if isinstance(item, BaseException):
                    raise item
                k, ids, host = item
                if to_cuda:
                    with torch.cuda.stream(copy_stream):
                        bmg = _cuda_copy(host, self.device)
                        ev = torch.cuda.Event()
                        ev.record(copy_stream)
                    free_evt[k] = ev
                    free.put(k)                                     # reusable once `ev` has completed (the producer waits)
                    cur = torch.cuda.current_stream(self.device)
                    cur.wait_event(ev)
                    for b in (bmg if isinstance(bmg, list) else [bmg]):
                        for t in (b.V, b.E, b.edge_index, b.rev_edge_index, b.batch):
                            t.record_stream(cur)
                    yield LoadedBatch(bmg, ids, self._extras(ids))
                else:
                    yield LoadedBatch(host, ids, self._extras(ids))  # views of ring[k]: valid until the next batch is drawn
                    free.put(k)
        finally:
            stop.set()
            free.put(-1)                                            # unblock a producer waiting for a buffer
            th.join(timeout=5)
