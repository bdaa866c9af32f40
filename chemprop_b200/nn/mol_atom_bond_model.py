"""`EngineMolAtomBondMPNN`: chemprop's `MolAtomBondMPNN` (chemprop/models/mol_atom_bond.py) without Lightning, on the
engine -- what follows the MAB message passing: three batch norms (molecule, atom and edge fingerprints), the bond
fingerprint `[H_e || H_e[rev]]`, molecule-, atom- and bond-level predictors, the bond predictor's average over each
reverse-edge pair, atom and bond constraints, and the sum of the per-level criteria.

- The bond fingerprint is an EdgePairOperand: the bond predictor's first layer gathers `H_e[rev]` inside its GEMM
  (PairLinearFunction), so the E x 2h concatenation is never stored, and its mirror sends the gradient back into H_e.
- The pair mean `(P[2i] + P[2i+1]) / 2` is dmpnn_edge_pair_mean (NaN rows where edge 2i+1 is not the reverse of edge 2i),
  applied by the model to the bond predictor's output and, through `_EdgePairMeanMLP`, to the bond constrainer's MLP
  output, as the reference's wrappers do.
- Atom- and bond-level criteria: each engine criterion's `row_loss`, which runs the row-parallel kernel the criterion
  names (dmpnn_regression_loss_rows for MSE, MAE, RMSE and their bounded variants, dmpnn_bce_loss_rows,
  dmpnn_ce_loss_rows), or its own kernel where it names none.  The molecule level, and any criterion that is not an engine
  criterion, is called as a module, as EngineMPNN does.
- No host synchronisation: a training step, with or without atom and bond constraints, captures into CudaGraphStep.  The
  constrainers get the molecules' atom and bond offsets from the layout and decide on the device which constraint columns
  are set (ConstrainerFFN, dmpnn_constrain_fwd / _bwd); the constraints are inputs of the graph like the targets.

Module tree and state-dict keys are the reference's (`bns.*`, `{mol,atom,bond}_predictor.*`, `{atom,bond}_constrainer.*`):
a reference `MolAtomBondMPNN` state dict without its `metricss.*` entries loads with `strict=True`."""
from __future__ import annotations

import torch
from torch import Tensor, nn

from .. import engine as K
from .head import EdgePairOperand, _Criterion, _predict, EngineBatchNorm1d, engine_mlp

_LEVELS = ("mol", "atom", "bond")


class EdgePairMeanFunction(torch.autograd.Function):
    """P (E x ...) -> (P[2i] + P[2i+1]) / 2 (E/2 x ...) in one launch (dmpnn_edge_pair_mean; mirror
    dmpnn_edge_pair_mean_bwd).  An odd E is refused."""

    @staticmethod
    def forward(ctx, P, rev):
        K._require_cuda(P, rev)
        E = P.shape[0]
        if E % 2:
            raise ValueError(f"the reverse-edge pair mean needs an even number of directed edges, got {E}")
        X = P.float().reshape(E, -1).contiguous()
        out = torch.empty((E // 2, X.shape[1]), dtype=torch.float32, device=P.device)
        if E > 0 and X.shape[1] > 0:
            K.edge_pair_mean(X, rev, out)
        ctx.cfg = (tuple(P.shape), P.dtype)
        return out.view(E // 2, *P.shape[1:])

    @staticmethod
    def backward(ctx, g):
        shape, dt = ctx.cfg
        E = shape[0]
        G = g.float().reshape(E // 2, -1).contiguous()
        dP = torch.empty((E, G.shape[1]), dtype=torch.float32, device=g.device)
        if E > 0 and G.shape[1] > 0:
            K.edge_pair_mean_bwd(G, dP)
        return dP.view(shape).to(dt), None


class _EdgePairMeanMLP(nn.Sequential):
    """The bond constrainer's MLP (`ConstrainerFFN.ffn`, same children and state-dict keys) followed by the reverse-edge
    pair mean, as the reference wraps `bond_constrainer.ffn.forward`.  It takes the model's EdgePairOperand: the first
    Linear gathers H_e[rev] in its GEMM (PairLinearFunction), and every layer runs on the engine as ConstrainerFFN runs it."""

    def forward(self, x):
        if not isinstance(x, EdgePairOperand):
            raise TypeError("the bond constrainer of EngineMolAtomBondMPNN takes the model's bond-level fingerprint "
                            "(an EdgePairOperand)")
        return EdgePairMeanFunction.apply(engine_mlp(self, x), x.rev)


class EngineMolAtomBondMPNN(nn.Module):
    """chemprop's `MolAtomBondMPNN` (models/mol_atom_bond.py) reduced to its path, on the engine: MAB message passing ->
    (aggregation) -> three batch norms -> molecule-, atom- and bond-level predictors (any Engine*FFN) -> constraints ->
    the sum of the per-level criteria.

    - `fingerprint(bmg, V_d, E_d, X_d) -> (H_g, H_v, H_e)`, H_e an EdgePairOperand standing for `[H_e || H_e[rev]]`.
    - `forward(bmg, V_d, E_d, X_d, constraints=None)`: the list of the three predictions (None for an absent level), the
      bond level averaged over each reverse-edge pair, with the constrainers applied as the reference does (to
      `preds[..., 0]` for multi-target predictors).
    - `training_loss(bmg, targetss, weightss, V_d, E_d, X_d, lt_masks=None, gt_masks=None, constraints=None)`:
      `MolAtomBondMPNN.training_step` without logging.  NaN targets are masked.  The step, constraints included, never
      synchronises with the host while a graph is being captured, and captures into CudaGraphStep.  Eagerly, a
      constrainer with more than one MLP output reads one status word to raise on shapes the reference rejects.

    A bond constrainer gets its MLP wrapped in `_EdgePairMeanMLP` (same children, same state-dict keys), which averages the
    MLP output over each reverse-edge pair as the reference's wrapper does; that constrainer then takes this model's bond
    fingerprint only.  The molecule index of each bond is derived on the device, `batch[edge_index[0, ::2]]`."""

    def __init__(self, message_passing: nn.Module, agg: nn.Module | None = None, mol_predictor: nn.Module | None = None,
                 atom_predictor: nn.Module | None = None, bond_predictor: nn.Module | None = None,
                 atom_constrainer: nn.Module | None = None, bond_constrainer: nn.Module | None = None,
                 batch_norm: bool = False, X_d_transform: nn.Module | None = None):
        if all(p is None for p in (mol_predictor, atom_predictor, bond_predictor)):
            raise ValueError("At least one of mol_predictor, atom_predictor, or bond_predictor must be provided.")
        if mol_predictor is not None and agg is None:
            raise ValueError("If mol_predictor is provided, agg must also be provided.")
        super().__init__()
        self.message_passing = message_passing
        self.agg = agg
        self.mol_predictor = mol_predictor
        self.atom_predictor = atom_predictor
        self.atom_constrainer = atom_constrainer
        self.bond_predictor = bond_predictor
        if bond_constrainer is not None and not isinstance(bond_constrainer.ffn, _EdgePairMeanMLP):
            bond_constrainer.ffn = _EdgePairMeanMLP(*bond_constrainer.ffn)
        self.bond_constrainer = bond_constrainer
        fp_dims = [message_passing.output_dims[0]] * 2 + [message_passing.output_dims[1]]
        self.bns = nn.ModuleList([EngineBatchNorm1d(d) if batch_norm and p is not None else nn.Identity()
                                  for d, p in zip(fp_dims, self.predictors)])
        self.X_d_transform = X_d_transform if X_d_transform is not None else nn.Identity()

    @property
    def predictors(self) -> tuple:
        return self.mol_predictor, self.atom_predictor, self.bond_predictor

    @property
    def criterions(self) -> tuple:
        return tuple(None if p is None else p.criterion for p in self.predictors)

    @property
    def n_taskss(self) -> tuple:
        return tuple(None if p is None else p.n_tasks for p in self.predictors)

    def fingerprint(self, bmg, V_d: Tensor | None = None, E_d: Tensor | None = None, X_d: Tensor | None = None):
        H_v, H_e = self.message_passing(bmg, V_d, E_d)
        H_g = self.agg(H_v, bmg.batch) if self.agg is not None else None
        H_g = self.bns[0](H_g) if H_g is not None else None
        H_v = self.bns[1](H_v) if H_v is not None else None
        H_e = self.bns[2](H_e) if H_e is not None else None
        if H_g is not None and X_d is not None:
            H_g = torch.cat((H_g, self.X_d_transform(X_d)), dim=1)
        if H_e is not None:
            H_e = EdgePairOperand(H_e, bmg.rev_edge_index.to(torch.int32))
        return H_g, H_v, H_e

    def _predictions(self, fps, train: bool) -> list:
        predss = []
        for level, (fp, predictor) in enumerate(zip(fps, self.predictors)):
            if predictor is None:
                predss.append(None)
                continue
            preds = predictor.train_step(fp) if train else predictor(fp)
            if level == 2:
                preds = EdgePairMeanFunction.apply(preds, fp.rev)
            predss.append(preds)
        return predss

    def _constrain(self, bmg, fps, predss, constraints) -> list:
        out = list(predss)
        lay = K.get_layout(bmg)
        for level, constrainer in ((1, self.atom_constrainer), (2, self.bond_constrainer)):
            c = constraints[level - 1]
            if constrainer is None or out[level] is None or c is None:
                continue
            batch = bmg.batch if level == 1 else bmg.batch[bmg.edge_index[0, ::2]]
            # the molecules' atom offsets, and their bond offsets: each molecule's directed edges are contiguous and
            # paired (2i, 2i + 1), which the pair mean already requires, so its bonds are its edges halved
            offsets = lay.mol_atom_ptr if level == 1 else lay.mol_row_ptr // 2
            preds = out[level]
            if preds.dim() > 2:
                preds = preds.clone()
                preds[..., 0] = constrainer(fps[level], preds[..., 0], batch, c, offsets=offsets)
            else:
                preds = constrainer(fps[level], preds, batch, c, offsets=offsets)
            out[level] = preds
        return out

    def forward(self, bmg, V_d: Tensor | None = None, E_d: Tensor | None = None, X_d: Tensor | None = None,
                constraints=None) -> list:
        fps = self.fingerprint(bmg, V_d, E_d, X_d)
        predss = self._predictions(fps, train=False)
        return predss if constraints is None else self._constrain(bmg, fps, predss, constraints)

    def predict(self, batches, *, active_dropout: bool = False) -> list:
        """chemprop's `predict_step` over `batches` (tuples `(bmg, V_d, E_d, X_d, ..., constraints)`, as the reference's
        MolAtomBondTrainingBatch), each level concatenated along its rows (models/mol_atom_bond.py:435-440 followed by
        the estimators' `torch.concat(preds, 0)`): `[mol, atom, bond]`, None for an absent level.  Eval mode under
        torch.inference_mode(); `active_dropout` trains every nn.Dropout module (DropoutEstimator).  Every module's
        training flag is restored, even on error; no host synchronisation."""
        return _predict(self, batches, lambda b: self(b[0], b[1], b[2], b[3], b[-1]), active_dropout,
                        lambda outs: [None if level[0] is None else torch.cat(level, 0) for level in zip(*outs)])

    def training_loss(self, bmg, targetss, weightss, V_d: Tensor | None = None, E_d: Tensor | None = None,
                      X_d: Tensor | None = None, lt_masks=None, gt_masks=None, constraints=None) -> Tensor:
        fps = self.fingerprint(bmg, V_d, E_d, X_d)
        predss = self._predictions(fps, train=True)
        if constraints is not None:
            predss = self._constrain(bmg, fps, predss, constraints)
        total = None
        for level, (predictor, preds) in enumerate(zip(self.predictors, predss)):
            if predictor is None:
                continue
            crit = predictor.criterion
            weights = None if weightss is None else weightss[level]
            lt = None if lt_masks is None else lt_masks[level]
            gt = None if gt_masks is None else gt_masks[level]
            masks = () if lt is None and gt is None else (lt, gt)
            if level > 0 and isinstance(crit, _Criterion):
                l = crit.row_loss(preds, targetss[level], weights, *masks)
            else:
                l = crit(preds, targetss[level], None, weights, *masks)
            total = l if total is None else total + l
        return total
