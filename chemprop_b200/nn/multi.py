"""Multicomponent models on the engine: `EngineMulticomponentMessagePassing` (chemprop/nn/message_passing/multi.py) and
`EngineMulticomponentMPNN` (chemprop/models/multi.py), for data points made of N molecules (solute + solvent, reactant +
catalyst, ...).

Two inputs are accepted wherever the reference takes `bmgs`, a list of N batches:

  * the list itself -- component c's block encodes batch c (the reference's behaviour; the only input for unshared blocks);
  * one UNION batch (shared encoder only): the N components of b data points in datapoint-major interleaved order, union
    molecule m * N + c being component c of data point m (`collate_multicomponent(..., union=True)`, or a
    `MulticomponentPackedDataset(..., union=True)`).  The block then runs once over all components: one depth-step chain
    per step instead of N, and one weight-gradient GEMM per weight over every component's rows.  Because the order is
    datapoint-major, the union's per-molecule aggregation (N * b x d, row-major) IS the reference fingerprint
    `torch.cat([agg(H_0), ..., agg(H_{N-1})], 1)` (b x N * d) viewed with another shape: no copy, and it holds for every
    Aggregation (all of them reduce over the segments of `batch`).
"""
from __future__ import annotations

import logging
from typing import Sequence

import torch
from torch import Tensor, nn

from .. import engine
from .agg import Aggregation, AttentiveAggregation
from .head import EngineMPNN

logger = logging.getLogger(__name__)


def _is_list_input(bmgs) -> bool:
    return isinstance(bmgs, (list, tuple))


class EngineMulticomponentMessagePassing(nn.Module):
    """chemprop/nn/message_passing/multi.py:13-84: same constructor, validation, `hparams`, `__len__`, `output_dim` and
    module tree (`shared=True` keeps `nn.ModuleList([blocks[0]] * n_components)`, so the state dict carries the reference's
    duplicated `blocks.<c>.*` keys).  `forward(bmgs, V_ds)` takes a list of N batches (returns the list of each
    component's H_v) or, with `shared=True`, one union batch in interleaved order (returns the union's H_v; `V_ds` is then
    one tensor in union atom order)."""

    def __init__(self, blocks: Sequence[nn.Module], n_components: int | None = None, shared: bool = False):
        super().__init__()
        self.hparams = {
            "cls": self.__class__,
            "blocks": [block.hparams for block in blocks],
            "n_components": n_components,
            "shared": shared,
        }
        if len(blocks) == 0:
            raise ValueError("arg 'blocks' was empty!")
        if shared and len(blocks) > 1:
            logger.warning("More than 1 block was supplied but 'shared' was True! Using only the 0th block...")
        if shared and n_components is None:
            raise ValueError("'shared' is True, so arg 'n_components' is required!")
        self.n_components = n_components
        self.shared = shared
        self.blocks = nn.ModuleList([blocks[0]] * self.n_components if shared else blocks)

    def __len__(self) -> int:
        return len(self.blocks)

    @property
    def output_dim(self) -> int:
        return sum(block.output_dim for block in self.blocks)

    def forward(self, bmgs, V_ds=None):
        if _is_list_input(bmgs):
            if len(bmgs) != len(self.blocks):
                raise ValueError(f"{len(bmgs)} batches for {len(self.blocks)} components")
            if V_ds is None:
                return [block(bmg) for block, bmg in zip(self.blocks, bmgs)]
            return [block(bmg, V_d) for block, bmg, V_d in zip(self.blocks, bmgs, V_ds)]
        if not self.shared:
            raise ValueError("a union batch (one BatchMolGraph for all components) needs a shared encoder (shared=True); "
                             "unshared blocks take a list of one batch per component")
        if V_ds is not None and not isinstance(V_ds, Tensor):
            raise ValueError("with a union batch, V_ds is one tensor in union atom order")
        return self.blocks[0](bmgs, V_ds)


class EngineMulticomponentMPNN(EngineMPNN):
    """`chemprop.models.MulticomponentMPNN` (models/multi.py:16-66) on the engine: EngineMPNN's head, criterion and
    `training_loss`, with the multicomponent fingerprint.  `forward` / `fingerprint` / `training_loss` take the
    multicomponent batch where EngineMPNN takes `bmg`: a list of N batches, or one union batch with a shared encoder.

    Fingerprint: union input -> `agg(H_union, union.batch)` viewed as b x N * d; list input with Mean / Sum / Norm
    aggregation -> each component's aggregation writes its own column block of one b x sum(d_c) buffer
    (SegmentAggColumnsFunction); any other aggregation -> per component and `torch.cat`, as the reference.  Then batch
    norm, then the scaled X_d.  A reference MulticomponentMPNN state dict without its `metrics.*` entries loads with
    strict=True."""

    def __init__(self, message_passing: EngineMulticomponentMessagePassing, agg: Aggregation | None = None,
                 predictor: nn.Module | None = None, batch_norm: bool = False, X_d_transform: nn.Module | None = None):
        super().__init__(message_passing, agg, predictor, batch_norm, X_d_transform)

    def fingerprint(self, bmgs, V_ds=None, X_d: Tensor | None = None) -> Tensor:
        H = self._union_fingerprint(bmgs, V_ds) if not _is_list_input(bmgs) else self._list_fingerprint(bmgs, V_ds)
        H = self.bn(H)
        return H if X_d is None else torch.cat((H, self.X_d_transform(X_d)), dim=1)

    def _union_fingerprint(self, bmg, V_d) -> Tensor:
        N = len(self.message_passing)
        if len(bmg) % N:
            raise ValueError(f"a union batch of {len(bmg)} molecules is not a whole number of {N}-component data points")
        H = self.agg(self.message_passing(bmg, V_d), bmg.batch)
        return H.view(len(bmg) // N, N * H.shape[1])

    def _list_fingerprint(self, bmgs, V_ds) -> Tensor:
        H_vs = self.message_passing(bmgs, V_ds)
        if not isinstance(self.agg, Aggregation) or isinstance(self.agg, AttentiveAggregation):
            return torch.cat([self.agg(H_v, bmg.batch) for H_v, bmg in zip(H_vs, bmgs)], 1)
        segs = [engine.segments_of(bmg.batch, len(bmg)) for bmg in bmgs]
        if len({s[2] for s in segs}) != 1:
            raise ValueError("the components' batches hold different numbers of molecules")
        return engine.SegmentAggColumnsFunction.apply(segs, self.agg._mode, float(self.agg._scale), *H_vs)
