"""`ConstrainerFFN` with the API of chemprop/nn/ffn.py:70-145 (SURVEY.md 8f-4): atom- or bond-level predictions are adjusted
so that they sum to a per-molecule constraint, the adjustment being shared out with a per-molecule softmax of an MLP's
output.

- The MLP is the reference's plain torch stack (same module tree, so state-dict keys `ffn.<i>.<j>.*` match), run on the
  engine's GEMMs as the predictors run theirs (`engine_mlp`: dmpnn_linear_fwd / dmpnn_linear_wgrad with each fused
  activation in the GEMM epilogue).
- The segmented part (ffn.py:120-141: exp, the two per-molecule sums, the softmax weights, the deviation and the scatter into
  the constrained columns) is one launch each way, dmpnn_constrain_fwd / dmpnn_constrain_bwd (ConstrainFunction).  Which
  columns are constrained is decided on the device, so a call never synchronises with the host for it.
- Molecule row offsets: `offsets` when the caller has them (EngineMolAtomBondMPNN passes its layout's), otherwise
  `segments_of(batch)`, which reads a status word back once.
- A constrainer whose MLP has more than one output checks once, after the launch, that the reference accepts the shape
  (n_c equal to the number of constrained columns, or 1) and raises as the reference does when it does not.  That read is
  skipped while the stream is capturing a CUDA graph or torch's sync debug mode is on: the constrained columns are then NaN
  and `status` (the last call's int32 device word) holds the number of constrained columns."""
from __future__ import annotations

from typing import Sequence

import torch
from torch import Tensor, nn

from .. import _lib
from .. import engine as K
from ..engine import SegmentAggFunction, SegmentBcastFunction, segments_of
from .message_passing import DEFAULT_HIDDEN_DIM, get_activation_function


def build_mlp(input_dim: int, output_dim: int, hidden_dim: int | Sequence[int] = 300, n_layers: int = 1,
              dropout: float = 0.0, activation="relu") -> nn.Sequential:
    """Module tree of chemprop/nn/ffn.py `MLP.build` (:38-61): [Linear], then [act, dropout, Linear] per further layer."""
    drop, act = nn.Dropout(dropout), get_activation_function(activation)
    hidden = [hidden_dim] * n_layers if isinstance(hidden_dim, int) else list(hidden_dim)
    dims = [input_dim] + hidden + [output_dim]
    blocks = [nn.Sequential(nn.Linear(dims[0], dims[1]))]
    blocks += [nn.Sequential(act, drop, nn.Linear(d1, d2)) for d1, d2 in zip(dims[1:-1], dims[2:])]
    return nn.Sequential(*blocks)


class ConstrainFunction(torch.autograd.Function):
    """(Kl, preds, ptr, constraints) -> (P', status): ffn.py:120-141 given the MLP output Kl (R x n_c), the predictions
    (R x t), the molecule row offsets ptr (int32, m + 1) and the constraints (m x t).  One dmpnn_constrain_fwd; mirror one
    dmpnn_constrain_bwd (dP and dKl; the constraints are data and get no gradient)."""

    @staticmethod
    def forward(ctx, Kl, preds, ptr, constraints):
        K._require_cuda(Kl, preds, ptr, constraints)
        Klc, P, Cn = Kl.float().contiguous(), preds.float().contiguous(), constraints.float().contiguous()
        if Cn.shape[1] != P.shape[1]:
            raise ValueError(f"constraints have {Cn.shape[1]} columns, the predictions {P.shape[1]}")
        out = torch.empty_like(P)
        status = torch.zeros(1, dtype=torch.int32, device=P.device)
        if P.shape[0] > 0 and P.shape[1] > 0:
            K.constrain_fwd(Klc, P, ptr, Cn, out, status)
        ctx.save_for_backward(Klc, P, ptr, Cn)
        ctx.dtypes = (Kl.dtype, preds.dtype)
        ctx.mark_non_differentiable(status)
        return out.to(preds.dtype), status

    @staticmethod
    def backward(ctx, g, _g_status):
        Klc, P, ptr, Cn = ctx.saved_tensors
        G = g.float().contiguous()
        dP, dKl = torch.empty_like(P), torch.empty_like(Klc)
        if P.shape[0] > 0 and P.shape[1] > 0:
            K.constrain_bwd(G, Klc, P, ptr, Cn, dP, dKl)
        else:
            dP.copy_(G)
            dKl.zero_()
        return dKl.to(ctx.dtypes[0]), dP.to(ctx.dtypes[1]), None, None


def _on_engine(t: Tensor) -> bool:
    """Whether the constrain kernels take this tensor (a module-level test seam, like the engine's op wrappers)."""
    return t.is_cuda


def _may_synchronise() -> bool:
    return not torch.cuda.is_current_stream_capturing() and torch.cuda.get_sync_debug_mode() == 0


class ConstrainerFFN(nn.Module):
    def __init__(self, n_constraints: int = 1, fp_dim: int = DEFAULT_HIDDEN_DIM, hidden_dim: int | Sequence[int] = 300,
                 n_layers: int = 1, dropout: float = 0.0, activation="relu"):
        super().__init__()
        self.hparams = dict(n_constraints=n_constraints, fp_dim=fp_dim, hidden_dim=hidden_dim, n_layers=n_layers,
                            dropout=dropout, activation=activation, cls=self.__class__)
        self.ffn = build_mlp(fp_dim, n_constraints, hidden_dim, n_layers, dropout, activation)
        self.status: Tensor | None = None

    def forward(self, fp: Tensor, preds: Tensor, batch: Tensor, constraints: Tensor, *,
                offsets: Tensor | None = None) -> Tensor:
        """fp: b x h fingerprints; preds: b x t; batch: b (molecule of each atom / bond, sorted); constraints: m x t (NaN in
        row 0 marks an unconstrained column, ffn.py:135).  `offsets`: the molecules' row offsets (int32, m + 1) when the
        caller has them, so `batch` is not read.  Returns the adjusted b x t predictions."""
        if not _on_engine(preds):
            return self._composed_forward(fp, preds, batch, constraints)
        # ffn.py:123 sizes everything by the constraints' row count: molecules without an atom / bond row (a trailing
        # single-heavy-atom SMILES has no bond) are empty segments, not an error
        n_mols = int(constraints.shape[0])
        if offsets is None:
            offsets = segments_of(batch, n_seg=n_mols)[0]
        elif tuple(offsets.shape) != (n_mols + 1,) or offsets.dtype != torch.int32:
            raise ValueError(f"offsets must be int32 with {n_mols + 1} entries (one per constraint row, plus one), got "
                             f"{offsets.dtype} {tuple(offsets.shape)}")
        from .head import EdgePairOperand, engine_mlp     # head imports build_mlp from this module

        # ffn.py:119 on the engine; the model's bond fingerprint goes through its pair-mean wrapper of this MLP
        Kl = self.ffn(fp) if isinstance(fp, EdgePairOperand) else engine_mlp(self.ffn, fp)
        out, self.status = ConstrainFunction.apply(Kl, preds, offsets, constraints)
        n_c = Kl.shape[1]
        if n_c > 1 and _may_synchronise():
            nq = int(self.status.item())
            if nq:
                raise RuntimeError(f"ConstrainerFFN: the MLP has {n_c} outputs and the constraints {nq} set columns; "
                                   "the reference broadcasts only equal counts or a single output (ffn.py:138-140)")
        return out

    def _composed_forward(self, fp: Tensor, preds: Tensor, batch: Tensor, constraints: Tensor) -> Tensor:
        """The reference's op sequence on the engine's segment ops, for tensors the constrain kernels cannot take.  A CPU
        tensor is refused by those ops as well (DmpnnError); this path serves torch stand-ins of the engine's wrappers."""
        n_mols = int(constraints.shape[0])
        ptr, seg, _ = segments_of(batch, n_seg=n_mols)
        rows = preds.shape[0]
        has = ~torch.isnan(constraints)[0]                                                           # ffn.py:135
        if rows == 0 or not bool(has.any()):             # nothing to adjust (the segment kernels need >= 1 column)
            return preds + torch.zeros_like(preds)
        expk = self.ffn(fp).exp()                                                                  # ffn.py:119-120
        Z = SegmentAggFunction.apply(expk.float(), ptr, seg, n_mols, _lib.SCALE_NONE, 1.0)           # ffn.py:124-126
        w = expk / SegmentBcastFunction.apply(Z, ptr, seg, rows)                                     # ffn.py:127-128
        per_mol = SegmentAggFunction.apply(preds.float(), ptr, seg, n_mols, _lib.SCALE_NONE, 1.0)    # ffn.py:130-133
        deviation = (constraints[:, has] - per_mol[:, has]).contiguous()                             # ffn.py:136
        corrections = w * SegmentBcastFunction.apply(deviation, ptr, seg, rows)                      # ffn.py:138
        out = torch.zeros_like(preds)
        out[:, has] = corrections.to(preds.dtype)                                                    # ffn.py:139-140
        return preds + out
