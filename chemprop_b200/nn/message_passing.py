"""`BondMessagePassing` / `AtomMessagePassing` with the module API of
chemprop/nn/message_passing/base.py:16-289 (same constructor arguments, `hparams`, parameter names
W_i / W_h / W_o / W_d, `output_dim`, `forward(bmg, V_d=None)`), executed by the sm_90a engine.

Differences a user can see: the module must live on a CUDA device (there is no CPU fallback), and a
`precision` keyword selects the hidden-state storage type: "fp32" (default; matches the reference
within 1e-5) or "bf16" (bf16 hidden states + tensor-core depth step; within 1e-2).

Two execution tiers sit behind `forward`: the monolithic autograd functions of engine.py (tau fused into the
kernels: ReLU / LeakyReLU / Tanh / ELU) and the composed tier of composed.py (the reference's op sequence, one libdmpnn
kernel per op, `self.tau` / `self.dropout` applied by torch in between) for everything else: PReLU, SELU or user
activation modules, LeakyReLU / ELU with a negative parameter, AtomMessagePassing(undirected=True), and active dropout
that the monolithic tier cannot take.

Dropout is active when `self.dropout` is in training mode with p > 0 -- the flag of the nn.Dropout module, as in the
reference (base.py:139, :182), so that chemprop's DropoutEstimator, which trains only the nn.Dropout modules of an eval-mode
model, samples the encoder too.  `p` is read at call time.  Active dropout runs on the monolithic tier
  * on a forward-only call (`torch.is_grad_enabled()` false, or no parameter requiring grad) of BondMessagePassing: keep
    bits in the fused bf16 depth step for every fused activation, dmpnn_scale_mask on every other bond path;
  * in a training step of BondMessagePassing on the fused bf16 / ReLU path (engine.Plan.dropout_ok).
AtomMessagePassing's monolithic tiers restate the reference on atoms, which needs every out-edge of an atom to carry the
same state; the reference drops each edge's copy independently, so active dropout runs it on the composed tier.
"""
from __future__ import annotations

import math

import torch
from torch import Tensor, nn

from .. import _lib, composed
from ..engine import AtomMPFunction, BondMPFunction, MPConfig, _warn_once, get_layout, plan
from ..exceptions import InvalidShapeError

try:                                   # custom-op registration for torch.export (inference); optional
    from .. import export as _export
except Exception:  # noqa: BLE001 -- an old torch without torch.library.custom_op: export support is simply absent
    _export = None

DEFAULT_ATOM_FDIM, DEFAULT_BOND_FDIM, DEFAULT_HIDDEN_DIM = 72, 14, 300  # chemprop/conf.py

_ACT_NAMES = {"relu": nn.ReLU, "leakyrelu": lambda: nn.LeakyReLU(0.1), "prelu": nn.PReLU, "tanh": nn.Tanh,
              "elu": nn.ELU}
_FUSED_ACTS = (nn.ReLU, nn.LeakyReLU, nn.Tanh, nn.ELU, nn.Identity)


def get_activation_function(activation) -> nn.Module:
    """chemprop/nn/utils.py:19-55 (string / enum-like / module -> module)."""
    if isinstance(activation, nn.Module):
        return activation
    name = getattr(activation, "name", activation)
    key = str(name).lower()
    if key == "selu":
        return nn.SELU()
    if key not in _ACT_NAMES:
        raise KeyError(f"Unsupported activation: {activation!r}; one of {sorted(_ACT_NAMES)}")
    return _ACT_NAMES[key]()


def engine_activation(tau: nn.Module) -> tuple[int, float]:
    """Map a torch activation module to the engine's fused activation code."""
    if not is_fused_activation(tau):
        raise NotImplementedError(
            f"activation {activation_name(tau)} is not fused into the sm_90a kernels "
            "(fused: ReLU, Tanh, Identity, LeakyReLU / ELU with a parameter >= 0; anything else runs on the composed tier)"
        )
    code = {nn.ReLU: _lib.ACT_RELU, nn.LeakyReLU: _lib.ACT_LEAKYRELU, nn.Tanh: _lib.ACT_TANH, nn.ELU: _lib.ACT_ELU,
            nn.Identity: _lib.ACT_NONE}[type(tau)]
    p = _act_param(tau)
    return code, 0.0 if p is None else p


def _act_param(tau: nn.Module) -> float | None:
    if type(tau) is nn.LeakyReLU:
        return float(tau.negative_slope)
    if type(tau) is nn.ELU:
        return float(tau.alpha)
    return None


def is_fused_activation(tau: nn.Module) -> bool:
    """Exact stock classes only: a user subclass may override forward, so it goes to the composed tier.  LeakyReLU and ELU
    only with a finite parameter >= 0: the kernels' backward passes take tau' from the stored output (act_grad_from_out in
    csrc/common.cuh: y > 0 ? 1 : slope, y > 0 ? 1 : y + alpha), which is tau'(z) only while tau keeps the sign of z."""
    if type(tau) not in _FUSED_ACTS:
        return False
    p = _act_param(tau)
    return p is None or (math.isfinite(p) and p >= 0.0)


def activation_name(tau: nn.Module) -> str:
    """How the composed-tier warnings name an activation: the class, or the module with its parameter when only the
    parameter keeps it off the fused path."""
    return repr(tau) if type(tau) in _FUSED_ACTS else type(tau).__name__


class _MessagePassingBase(nn.Module):
    _function = None
    _composed_forward = None

    def __init__(self, d_v: int = DEFAULT_ATOM_FDIM, d_e: int = DEFAULT_BOND_FDIM, d_h: int = DEFAULT_HIDDEN_DIM,
                 bias: bool = False, depth: int = 3, dropout: float = 0.0, activation="relu",
                 undirected: bool = False, d_vd: int | None = None, V_d_transform: nn.Module | None = None,
                 graph_transform: nn.Module | None = None, precision: str = "fp32",
                 output_dtype: torch.dtype | None = None):
        super().__init__()
        if precision not in ("fp32", "bf16"):
            raise ValueError("precision must be 'fp32' or 'bf16'")
        if output_dtype not in (None, torch.float32, torch.bfloat16):
            raise ValueError("output_dtype must be None, torch.float32 or torch.bfloat16")
        # same keys as the reference's save_hyperparameters() result (base.py:70-80)
        self.hparams = dict(d_v=d_v, d_e=d_e, d_h=d_h, bias=bias, depth=depth, dropout=dropout,
                            activation=activation, undirected=undirected, d_vd=d_vd,
                            V_d_transform=V_d_transform, graph_transform=graph_transform,
                            precision=precision, output_dtype=output_dtype, cls=self.__class__)
        self.W_i, self.W_h, self.W_o, self.W_d = self.setup(d_v, d_e, d_h, d_vd, bias)
        self.depth = depth
        self.undirected = undirected
        self.dropout = nn.Dropout(dropout)
        self.tau = get_activation_function(activation)
        self.V_d_transform = V_d_transform if V_d_transform is not None else nn.Identity()
        self.graph_transform = graph_transform if graph_transform is not None else nn.Identity()
        self.precision = precision
        # dtype of the atom-level output H_v.  None = the tier's storage type (bf16 for precision="bf16": what the engine's
        # Aggregation consumes without a pass over V x h; the aggregation itself always returns f32).  Heads that read H_v
        # directly with f32 parameters (atom-level predictors of the mol-atom-bond models) want torch.float32.
        self.output_dtype = output_dtype
        self.fused = True

    @property
    def output_dim(self) -> int:
        return self.W_d.out_features if self.W_d is not None else self.W_o.out_features

    def setup(self, d_v, d_e, d_h, d_vd, bias):
        raise NotImplementedError

    def _config(self) -> MPConfig:
        act, ap = engine_activation(self.tau)
        return MPConfig(depth=int(self.depth), act=act, act_param=ap, undirected=bool(self.undirected),
                        hidden_dtype=torch.bfloat16 if self.precision == "bf16" else torch.float32,
                        fused=bool(self.fused))

    def _dropout_on_fused_path(self, lay) -> bool:
        """Training-mode dropout that can stay on the fused bf16 path for this batch (BondMessagePassing only)."""
        return False

    def dropout_active(self) -> bool:
        """nn.Dropout's own test (base.py:139): its training flag and p > 0, read now (DropoutEstimator rewrites p)."""
        return bool(self.dropout.training and self.dropout.p > 0)

    def forward_only(self) -> bool:
        """No backward can follow this call: autograd is off, or no parameter asks for a gradient."""
        return not torch.is_grad_enabled() or not any(p.requires_grad for p in self.parameters())

    def _forward_only_dropout(self) -> bool:
        """Active dropout that runs on the monolithic tier because no mirror needs its masks (BondMessagePassing only)."""
        return False

    def uses_composed_tier(self, lay=None) -> bool:
        """True when this call cannot run on the monolithic functions (see the module docstring).  Active dropout stays
        monolithic on a forward-only bond call, and in training on the fused bf16 / ReLU path, which depends on the batch's
        layout `lay`."""
        if not is_fused_activation(self.tau):
            return True
        if self.dropout_active():
            if self._forward_only_dropout():
                return False
            return not (lay is not None and self._dropout_on_fused_path(lay))
        return False

    _kind = 0

    def _traced_forward(self, bmg) -> Tensor:
        """Under torch.export: the whole forward as ONE custom op (chemprop_b200/export.py), inference only."""
        if self.uses_composed_tier():
            raise NotImplementedError("torch.export covers the monolithic tiers (ReLU / LeakyReLU / Tanh / ELU, no "
                                      "training-mode dropout, AtomMessagePassing directed)")
        cfg = self._config()
        return torch.ops.dmpnn.mp_forward(
            bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch, self.W_i.weight, self.W_i.bias, self.W_h.weight,
            self.W_h.bias, self.W_o.weight, self.W_o.bias, type(self)._kind, cfg.depth, cfg.act, cfg.act_param,
            cfg.undirected, self.precision == "bf16", bool(self.fused))

    def forward(self, bmg, V_d: Tensor | None = None) -> Tensor:
        bmg = self.graph_transform(bmg)
        if _export is not None and _export.is_tracing():
            return self.finalize_descriptors(self._traced_forward(bmg), V_d)
        lay = get_layout(bmg)
        out_dtype = self.output_dtype or (torch.bfloat16 if self.precision == "bf16" else torch.float32)
        if self.uses_composed_tier(lay):
            if self.precision == "bf16":
                # no silent cliff: this tier keeps f32 hidden states; its W_h GEMMs run as 3xTF32 on the tensor cores (a sixth
                # of the bf16 rate), W_i / W_o on the f32 FMA pipes, and every reference op is a launch of its own
                why = (f"activation {activation_name(self.tau)}" if not is_fused_activation(self.tau) else
                       "undirected AtomMessagePassing" if (self.undirected and type(self)._kind == 1) else
                       "dropout in AtomMessagePassing" if type(self)._kind == 1 else
                       "training-mode dropout outside the fused ReLU path")
                _warn_once("composed_bf16", f"chemprop_b200: precision='bf16' requested, but this configuration ({why}) runs on "
                           "the composed tier: f32 hidden states, one kernel per reference op, no fused depth step "
                           "(expect several times the step time of the fused bf16 tier)")
            H = type(self)._composed_forward(self, bmg, lay)          # computed in f32 on this tier
        else:
            cfg = self._config()
            if self.dropout_active():
                cfg.dropout_p = float(self.dropout.p)
                cfg.forward_only = self._forward_only_dropout()
                cfg.mask_fn = getattr(self, "_mask_fn", None)      # test hook: where the keep masks come from
            H = type(self)._function.apply(
                bmg.V, bmg.E, self.W_i.weight, self.W_i.bias, self.W_h.weight, self.W_h.bias,
                self.W_o.weight, self.W_o.bias, lay, cfg,
            )
        if H.dtype != out_dtype:
            H = H.to(out_dtype)
        return self.finalize_descriptors(H, V_d)

    def finalize_descriptors(self, H: Tensor, V_d: Tensor | None) -> Tensor:
        """Second half of `finalize` (base.py:184-194): optional W_d on [H || V_d]; no activation."""
        if V_d is None:
            return H
        V_d = self.V_d_transform(V_d)
        try:
            H = self.W_d(torch.cat((H.to(self.W_d.weight.dtype), V_d), dim=1))
            H = self.dropout(H)
        except RuntimeError:
            raise InvalidShapeError("V_d", V_d.shape, [len(H), self.W_d.in_features - self.W_o.out_features])
        return H


class BondMessagePassing(_MessagePassingBase):
    """Directed-bond message passing (chemprop/nn/message_passing/base.py:215-251)."""
    _function = BondMPFunction
    _composed_forward = staticmethod(composed.bond_forward)

    def _forward_only_dropout(self) -> bool:
        return 0.0 < self.dropout.p < 1.0 and self.forward_only()

    def _dropout_on_fused_path(self, lay) -> bool:
        if not (self.precision == "bf16" and 0.0 < self.dropout.p < 1.0 and is_fused_activation(self.tau)):
            return False
        h = self.W_h.out_features
        d_v = self.W_o.in_features - h
        cfg = self._config()
        cfg.dropout_p = float(self.dropout.p)
        return plan("bond", cfg, lay, h, d_v, self.W_i.in_features - d_v).dropout_ok

    def setup(self, d_v=DEFAULT_ATOM_FDIM, d_e=DEFAULT_BOND_FDIM, d_h=DEFAULT_HIDDEN_DIM, d_vd=None, bias=False):
        W_i = nn.Linear(d_v + d_e, d_h, bias)
        W_h = nn.Linear(d_h, d_h, bias)
        W_o = nn.Linear(d_v + d_h, d_h)
        W_d = nn.Linear(d_h + d_vd, d_h + d_vd) if d_vd else None
        return W_i, W_h, W_o, W_d


class AtomMessagePassing(_MessagePassingBase):
    """Atom message passing (chemprop/nn/message_passing/base.py:254-289)."""
    _function = AtomMPFunction
    _composed_forward = staticmethod(composed.atom_forward)
    _kind = 1

    def setup(self, d_v=DEFAULT_ATOM_FDIM, d_e=DEFAULT_BOND_FDIM, d_h=DEFAULT_HIDDEN_DIM, d_vd=None, bias=False):
        W_i = nn.Linear(d_v, d_h, bias)
        W_h = nn.Linear(d_e + d_h, d_h, bias)
        W_o = nn.Linear(d_v + d_h, d_h)
        W_d = nn.Linear(d_h + d_vd, d_h + d_vd) if d_vd else None
        return W_i, W_h, W_o, W_d

    def uses_composed_tier(self, lay=None) -> bool:
        # undirected averaging (base.py:202-203) breaks the atom-granular restatement the monolithic tier relies on
        return bool(self.undirected) or super().uses_composed_tier(lay)
