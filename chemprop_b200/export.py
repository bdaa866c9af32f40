"""`torch.export` support for inference (reference: tests/integration/test_export.py:15-46, which exports an MPNN with
dynamic atom / edge counts and runs it on a batch without edges).

The engine's forward is a sequence of C-ABI calls on raw pointers, which a tracer cannot see through.  For export the
whole message-passing forward and the aggregation are therefore presented as two `torch.library` custom ops with fake
(shape-only) implementations -- `dmpnn::mp_forward` and `dmpnn::segment_agg`; the modules switch to them when
`torch.compiler.is_exporting()` reports an export trace.  The ops build the device layout themselves from the
graph's index tensors (the number of molecules and of output rows is data dependent: an unbacked size in the fake
implementation), run the monolithic forward without autograd and return fresh tensors.  Scope: inference on the
monolithic tiers (ReLU / LeakyReLU / Tanh / ELU); the composed tier is built of autograd functions and is not exported.

`register_batch_mol_graph_pytree()` registers `chemprop_b200.data.BatchMolGraph` as a pytree node, the way the
reference's test fixture does for its own class (tests/conftest.py:21-53), so that a BatchMolGraph can be an export input.
"""
from __future__ import annotations

import torch
from torch import Tensor

from . import engine
from ._lib import SCALE_NONE  # noqa: F401  (re-exported for callers building op arguments)

KIND_BOND, KIND_ATOM = 0, 1


def is_tracing() -> bool:
    """True inside torch.export.export (not under torch.compile: the custom ops carry no autograd formula, and a
    compiled TRAINING step must keep the autograd functions)."""
    return bool(getattr(torch.compiler, "is_exporting", lambda: False)())


@torch.library.custom_op("dmpnn::mp_forward", mutates_args=())
def mp_forward(V: Tensor, E: Tensor, edge_index: Tensor, rev_edge_index: Tensor, batch: Tensor, W_i: Tensor,
               b_i: Tensor | None, W_h: Tensor, b_h: Tensor | None, W_o: Tensor, b_o: Tensor | None, kind: int,
               depth: int, act: int, act_param: float, undirected: bool, bf16: bool, fused: bool) -> Tensor:
    """{Bond, Atom}MessagePassing.forward up to tau(W_o(.)) (base.py:196-212, :180-182), inference only."""
    engine._require_cuda(V, E, W_i, W_h, W_o)
    n_mols = int(batch[-1].item()) + 1 if batch.numel() else 0        # every molecule has >= 1 atom and `batch` is sorted
    lay = engine.build_layout(edge_index, rev_edge_index, batch, n_mols)
    lay.validate()
    cfg = engine.MPConfig(depth=int(depth), act=int(act), act_param=float(act_param), undirected=bool(undirected),
                          hidden_dtype=torch.bfloat16 if bf16 else torch.float32, fused=bool(fused))
    f = lambda t: None if t is None else t.detach().contiguous().float()  # noqa: E731
    Vf, Ef = V.contiguous().float(), E.contiguous().float()
    # the atom forward here is atom_forward_tc or atom_forward, never the fused atom step: that step rounds to bf16 at other
    # points, so moving exported atom models onto it would change their results
    p = engine.plan("bond" if kind == KIND_BOND else "export_atom", cfg, lay, W_i.shape[0], Vf.shape[1], Ef.shape[1])
    with torch.no_grad():
        Hv, _ = p.forward(lay, Vf, Ef, f(W_i), f(b_i), f(W_h), f(b_h), f(W_o), f(b_o), cfg, p)
    return Hv.clone(memory_format=torch.contiguous_format)


@mp_forward.register_fake
def _mp_forward_fake(V, E, edge_index, rev_edge_index, batch, W_i, b_i, W_h, b_h, W_o, b_o, kind, depth, act, act_param,
                     undirected, bf16, fused):
    return V.new_empty((V.shape[0], W_o.shape[0]), dtype=torch.bfloat16 if bf16 else torch.float32)


@torch.library.custom_op("dmpnn::segment_agg", mutates_args=())
def segment_agg(H: Tensor, batch: Tensor, scale_mode: int, scale: float) -> Tensor:
    """Mean / Sum / Norm aggregation (chemprop/nn/agg.py:73-78, 90-95, 112-113), inference only."""
    ptr, _, B = engine.segments_of(batch)
    Hc = H if H.stride(1) == 1 else H.contiguous()
    out = torch.empty((B, H.shape[1]), dtype=torch.float32, device=H.device)     # molecule level: always f32 (engine.SegmentAggFunction)
    engine.segment_sum(Hc, ptr, B, H.shape[1], out, scale_mode=int(scale_mode), scale=float(scale), pad_to=H.shape[1])
    return out


@segment_agg.register_fake
def _segment_agg_fake(H, batch, scale_mode, scale):
    n_mols = torch.library.get_ctx().new_dynamic_size()               # batch.max() + 1: data dependent (agg.py:75)
    return H.new_empty((n_mols, H.shape[1]), dtype=torch.float32)


_PYTREE_DONE = False


def register_batch_mol_graph_pytree():
    """Make `chemprop_b200.data.BatchMolGraph` a pytree node (leaves: V, E, edge_index, rev_edge_index, batch; context:
    the number of molecules) -- the counterpart of the reference's tests/conftest.py:21-53."""
    global _PYTREE_DONE
    if _PYTREE_DONE:
        return
    from torch.utils._pytree import GetAttrKey, register_pytree_node

    from .data import BatchMolGraph

    def flatten(bmg):
        return [bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch], len(bmg)

    def unflatten(children, size):
        bmg = object.__new__(BatchMolGraph)
        bmg.V, bmg.E, bmg._edge_index, bmg._rev_edge_index, bmg._batch = children
        bmg._size, bmg._layout, bmg._xfer, bmg._meta_host = size, None, None, None
        return bmg

    def flatten_with_keys(bmg):
        children, context = flatten(bmg)
        keys = [GetAttrKey(k) for k in ("V", "E", "edge_index", "rev_edge_index", "batch")]
        return list(zip(keys, children)), context

    register_pytree_node(BatchMolGraph, flatten, unflatten, flatten_with_keys_fn=flatten_with_keys,
                         serialized_type_name="chemprop_b200.data.BatchMolGraph")
    _PYTREE_DONE = True
