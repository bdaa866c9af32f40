"""`MABBondMessagePassing` / `MABAtomMessagePassing` (SURVEY.md 8f-3) with the module API of
chemprop/nn/message_passing/mol_atom_bond.py: the same depth loop as Bond / AtomMessagePassing, followed by a vertex
read-out (`W_vo`, optional `W_vd` on extra atom descriptors) and an edge read-out (`W_eo` on `[E || H]` per directed
edge, optional `W_ed` on extra bond descriptors); `forward(bmg, V_d=None, E_d=None) -> (H_v | None, H_e | None)`.
Per-edge outputs are handed back in the caller's edge order.  CUDA only, like the rest.

`precision` selects the tier, as for Bond / AtomMessagePassing:
  * "fp32" (default): the composed tier (chemprop_b200/composed.py) -- one libdmpnn kernel per reference op, `tau` /
    `dropout` applied by torch in between, f32 hidden states; matches the reference within 1e-5.
  * "bf16": engine.MABMPFunction -- bf16 hidden states, the fused depth step of the bf16 tier, the W_vo read-out and the
    per-edge W_eo head as tensor-core GEMMs with bias, tau and an f32 store in their epilogues; within 1e-2.  It applies
    when the activation is fused (ReLU, LeakyReLU, Tanh, ELU), `undirected=False`, no active dropout (except on a
    forward-only call of MABBondMessagePassing: keep bits in the fused depth step, dmpnn_scale_mask after W_vo / W_eo), and the GEMM
    sizes fit the tensor-core kernels (d_h <= engine.MAX_TC_HIDDEN and a multiple of 4, every inner dimension -- d_e + d_h
    for W_eo included -- <= engine.MAX_TC_K).  Anything else runs on the composed tier, with a one-time RuntimeWarning
    naming the reason.
    No host synchronisation on the path: a training step captures into CudaGraphStep.
Both tiers return f32 `H_v` / `H_e`: every consumer (atom / bond predictors, W_vd / W_ed, MolAtomBondMPNN) holds f32
parameters.
"""
from __future__ import annotations

import torch
from torch import Tensor, nn

from .. import composed
from ..engine import MABMPFunction, MPConfig, _warn_once, get_layout, plan
from ..exceptions import InvalidShapeError
from .message_passing import (DEFAULT_ATOM_FDIM, DEFAULT_BOND_FDIM, DEFAULT_HIDDEN_DIM, activation_name,
                              engine_activation, get_activation_function, is_fused_activation)


class _MABMessagePassingBase(nn.Module):
    _kind = None

    def __init__(self, d_v: int = DEFAULT_ATOM_FDIM, d_e: int = DEFAULT_BOND_FDIM, d_h: int = DEFAULT_HIDDEN_DIM,
                 bias: bool = False, depth: int = 3, dropout: float = 0.0, activation="relu", undirected: bool = False,
                 d_vd: int | None = None, d_ed: int | None = None, V_d_transform: nn.Module | None = None,
                 E_d_transform: nn.Module | None = None, graph_transform: nn.Module | None = None,
                 return_vertex_embeddings: bool = True, return_edge_embeddings: bool = True, precision: str = "fp32"):
        super().__init__()
        if precision not in ("fp32", "bf16"):
            raise ValueError("precision must be 'fp32' or 'bf16'")
        # same keys as the reference's save_hyperparameters() result (mol_atom_bond.py `__init__`), plus `precision`
        self.hparams = dict(d_v=d_v, d_e=d_e, d_h=d_h, bias=bias, depth=depth, dropout=dropout, activation=activation,
                            undirected=undirected, d_vd=d_vd, d_ed=d_ed, return_vertex_embeddings=return_vertex_embeddings,
                            return_edge_embeddings=return_edge_embeddings, V_d_transform=V_d_transform,
                            E_d_transform=E_d_transform, graph_transform=graph_transform, precision=precision,
                            cls=self.__class__)
        self.return_vertex_embeddings = return_vertex_embeddings
        self.return_edge_embeddings = return_edge_embeddings
        self.W_i, self.W_h, self.W_vo, self.W_vd, self.W_eo, self.W_ed = self.setup(d_v, d_e, d_h, d_vd, d_ed, bias)
        self.depth = depth
        self.undirected = undirected
        self.dropout = nn.Dropout(dropout)
        self.tau = get_activation_function(activation)
        self.V_d_transform = V_d_transform if V_d_transform is not None else nn.Identity()
        self.E_d_transform = E_d_transform if E_d_transform is not None else nn.Identity()
        self.graph_transform = graph_transform if graph_transform is not None else nn.Identity()
        self.precision = precision

    def setup(self, d_v, d_e, d_h, d_vd, d_ed, bias):
        raise NotImplementedError

    def _readouts(self, d_v, d_e, d_h, d_vd, d_ed):
        W_vo = nn.Linear(d_v + d_h, d_h) if self.return_vertex_embeddings else None
        W_eo = nn.Linear(d_e + d_h, d_h) if self.return_edge_embeddings else None
        W_vd = nn.Linear(d_h + d_vd, d_h + d_vd) if d_vd else None
        W_ed = nn.Linear(d_h + d_ed, d_h + d_ed) if d_ed else None
        return W_vo, W_vd, W_eo, W_ed

    @property
    def output_dims(self) -> tuple[int | None, int | None]:
        v = None if not self.return_vertex_embeddings else (self.W_vd or self.W_vo).out_features
        e = None if not self.return_edge_embeddings else (self.W_ed or self.W_eo).out_features
        return v, e

    def composed_reason(self) -> str | None:
        """Why this module, as configured now, runs on the composed tier with precision='bf16' (None: it does not)."""
        if not is_fused_activation(self.tau):
            return f"activation {activation_name(self.tau)}"
        if self.undirected:
            return "undirected=True"
        if self.dropout_active() and not self._forward_only_dropout():
            return "training-mode dropout" if self._kind == "bond" or not self.forward_only() else "dropout on atom states"
        return plan("mab_" + self._kind, self._config(), None, self.W_h.out_features, self.hparams["d_v"],
                    self.hparams["d_e"]).reason

    def dropout_active(self) -> bool:
        """nn.Dropout's own test (mol_atom_bond.py `update` / `*_finalize`): its training flag and p > 0, read now."""
        return bool(self.dropout.training and self.dropout.p > 0)

    def forward_only(self) -> bool:
        """No backward can follow this call: autograd is off, or no parameter asks for a gradient."""
        return not torch.is_grad_enabled() or not any(p.requires_grad for p in self.parameters())

    def _forward_only_dropout(self) -> bool:
        """Active dropout on the bf16 tier: forward-only bond calls (the atom kind's restatement on atoms needs every
        out-edge of an atom to carry the same state, which per-edge masks break)."""
        return self._kind == "bond" and 0.0 < self.dropout.p < 1.0 and self.forward_only()

    def uses_composed_tier(self) -> bool:
        return self.precision != "bf16" or self.composed_reason() is not None

    def _config(self) -> MPConfig:
        act, ap = engine_activation(self.tau)
        return MPConfig(depth=int(self.depth), act=act, act_param=ap, undirected=False, hidden_dtype=torch.bfloat16)

    def _descriptors(self, H: Tensor, X_d: Tensor | None, transform, W_d, W_o, name: str) -> Tensor:
        """Second half of vertex_finalize / edge_finalize: W_d on [H || X_d], dropout, no activation."""
        if X_d is None:
            return H
        X_d = transform(X_d)
        try:
            H = self.dropout(W_d(torch.cat((H.to(W_d.weight.dtype), X_d), dim=1)))
        except (RuntimeError, AttributeError):
            raise InvalidShapeError(name, X_d.shape, [len(H), (W_d.in_features - W_o.out_features) if W_d is not None else 0])
        return H

    def forward(self, bmg, V_d: Tensor | None = None, E_d: Tensor | None = None):
        bmg = self.graph_transform(bmg)
        lay = get_layout(bmg)
        why = self.composed_reason() if self.precision == "bf16" else None
        if self.precision == "bf16" and why is None:
            W_vo, W_eo = self.W_vo, self.W_eo
            cfg = self._config()
            if self.dropout_active():
                cfg.dropout_p, cfg.forward_only = float(self.dropout.p), True
                cfg.mask_fn = getattr(self, "_mask_fn", None)      # test hook: where the keep masks come from
            H_v, H_e = MABMPFunction.apply(
                bmg.V, bmg.E, self.W_i.weight, self.W_i.bias, self.W_h.weight, self.W_h.bias,
                None if W_vo is None else W_vo.weight, None if W_vo is None else W_vo.bias,
                None if W_eo is None else W_eo.weight, None if W_eo is None else W_eo.bias, lay, cfg, self._kind)
            H_v = H_v if W_vo is not None else None
            H_e = H_e if W_eo is not None else None
        else:
            if why is not None:
                # no silent cliff: the composed tier keeps f32 hidden states and launches one kernel per reference op
                _warn_once(f"mab_composed_bf16:{why}",
                           f"chemprop_b200: precision='bf16' requested, but this configuration ({why}) runs on the composed "
                           "tier: f32 hidden states, one kernel per reference op, no fused depth step (expect several times "
                           "the step time of the fused bf16 tier)")
            H_v, H_e = composed.mab_forward(self, bmg, lay, self._kind)
        if H_v is not None:
            H_v = self._descriptors(H_v, V_d, self.V_d_transform, self.W_vd, self.W_vo, "V_d")
        if H_e is not None:
            H_e = self._descriptors(H_e, E_d, self.E_d_transform, self.W_ed, self.W_eo, "E_d")
        return H_v, H_e


class MABBondMessagePassing(_MABMessagePassingBase):
    _kind = "bond"

    def setup(self, d_v=DEFAULT_ATOM_FDIM, d_e=DEFAULT_BOND_FDIM, d_h=DEFAULT_HIDDEN_DIM, d_vd=None, d_ed=None, bias=False):
        W_i = nn.Linear(d_v + d_e, d_h, bias)
        W_h = nn.Linear(d_h, d_h, bias)
        W_vo, W_vd, W_eo, W_ed = self._readouts(d_v, d_e, d_h, d_vd, d_ed)
        return W_i, W_h, W_vo, W_vd, W_eo, W_ed


class MABAtomMessagePassing(_MABMessagePassingBase):
    _kind = "atom"

    def setup(self, d_v=DEFAULT_ATOM_FDIM, d_e=DEFAULT_BOND_FDIM, d_h=DEFAULT_HIDDEN_DIM, d_vd=None, d_ed=None, bias=False):
        W_i = nn.Linear(d_v, d_h, bias)
        W_h = nn.Linear(d_e + d_h, d_h, bias)
        W_vo, W_vd, W_eo, W_ed = self._readouts(d_v, d_e, d_h, d_vd, d_ed)
        return W_i, W_h, W_vo, W_vd, W_eo, W_ed
