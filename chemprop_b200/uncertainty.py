"""chemprop's uncertainty estimators (chemprop/uncertainty/estimator.py) on the engine's models.

`EngineUncertaintyEstimatorRegistry` holds them under the reference's names.  Each estimator is called as
`estimator(batches, models)`: the reference's `estimator(dataloader, models, trainer)` without the trainer, the predictions
coming from each model's `predict(batches)` (chemprop's `trainer.predict` followed by `torch.concat(preds, 0)`).  `models`
are EngineMPNN / EngineMulticomponentMPNN objects, or EngineMolAtomBondMPNN objects, for which every estimator returns
`(mol, atom, bond)` predictions and uncertainties with None for an absent level, as the reference does.  Shapes, dtypes, the
leading model dimension and the population (`correction=0`) variances are the reference's.

`dropout` (Monte Carlo dropout) trains only the nn.Dropout modules of an eval-mode model, as the reference does.  The
encoder honours that flag; on a forward-only call BondMessagePassing keeps its fused depth step and tensor-core GEMMs with
dropout active (DESIGN.md 4.10).  Calibrators and evaluators take tensors only: chemprop's own classes run on these outputs.
"""
from __future__ import annotations

import torch
from torch import Tensor, nn

from .nn.mol_atom_bond_model import EngineMolAtomBondMPNN


class _Registry(dict):
    """name -> estimator class, with the reference ClassRegistry's `register` decorator."""

    def register(self, name: str):
        def deco(cls):
            self[name] = cls
            return cls

        return deco


EngineUncertaintyEstimatorRegistry = _Registry()


def _is_mab(models) -> bool:
    return isinstance(models[0], EngineMolAtomBondMPNN)


def _levels(batches, models) -> tuple:
    """Per level (one for EngineMPNN, mol / atom / bond for EngineMolAtomBondMPNN) the list of every model's predictions
    (empty where a level is absent)."""
    if not _is_mab(models):
        return ([m.predict(batches) for m in models],)
    out = ([], [], [])
    for m in models:
        for level, preds in zip(out, m.predict(batches)):
            if preds is not None:
                level.append(preds)
    return out


def _result(models, per_level: list) -> tuple:
    """(preds, uncs) of the reference: the single level's pair for EngineMPNN, the pair of per-level lists otherwise."""
    if not _is_mab(models):
        return per_level[0]
    return [p for p, _ in per_level], [u for _, u in per_level]


class UncertaintyEstimator:
    """Base class: `__call__(batches, models) -> (preds, uncs)`."""

    def __call__(self, batches, models):
        raise NotImplementedError


@EngineUncertaintyEstimatorRegistry.register("none")
class NoUncertaintyEstimator(UncertaintyEstimator):
    """estimator.py:66-114: the stacked predictions, no uncertainty."""

    def __call__(self, batches, models):
        preds = [torch.stack(lv) if lv else None for lv in _levels(batches, models)]
        return (preds[0], None) if not _is_mab(models) else (preds, (None, None, None))


class _SplitEstimator(UncertaintyEstimator):
    """The estimators that stack the models' predictions and split the last dimension (`_split`)."""
    _float = False

    def __call__(self, batches, models):
        per_level = []
        for lv in _levels(batches, models):
            if not lv:
                per_level.append((None, None))
                continue
            stacked = torch.stack(lv)
            per_level.append(self._split(stacked.float() if self._float else stacked))
        return _result(models, per_level)

    def _split(self, stacked: Tensor) -> tuple:
        raise NotImplementedError


@EngineUncertaintyEstimatorRegistry.register("mve")
class MVEEstimator(_SplitEstimator):
    """estimator.py:117-180: (mean, variance) of mean-variance estimation heads."""

    def _split(self, stacked):
        mean, var = stacked.unbind(dim=-1)
        return mean, var


@EngineUncertaintyEstimatorRegistry.register("ensemble")
class EnsembleEstimator(_SplitEstimator):
    """estimator.py:183-249: the stacked predictions and their variance over the models (1 x ...)."""
    _float = True

    def __call__(self, batches, models):
        if len(models) <= 1:
            raise ValueError("Ensemble method for uncertainty is only available when multiple models are provided.")
        return super().__call__(batches, models)

    def _split(self, stacked):
        return stacked, torch.var(stacked, dim=0, correction=0).unsqueeze(0)


@EngineUncertaintyEstimatorRegistry.register("classification")
class ClassEstimator(_SplitEstimator):
    """estimator.py:252-299: the predicted probabilities serve as both prediction and uncertainty."""

    def _split(self, stacked):
        return stacked, stacked


class _EvidentialEstimator(_SplitEstimator):
    def _split(self, stacked):
        mean, v, alpha, beta = stacked.unbind(-1)
        return mean, self._unc(v, alpha, beta)


@EngineUncertaintyEstimatorRegistry.register("evidential-total")
class EvidentialTotalEstimator(_EvidentialEstimator):
    """estimator.py:302-365: (1 + 1 / v) beta / (alpha - 1)."""

    @staticmethod
    def _unc(v, alpha, beta):
        return (1 + 1 / v) * (beta / (alpha - 1))


@EngineUncertaintyEstimatorRegistry.register("evidential-epistemic")
class EvidentialEpistemicEstimator(_EvidentialEstimator):
    """estimator.py:368-426: (1 / v) beta / (alpha - 1)."""

    @staticmethod
    def _unc(v, alpha, beta):
        return (1 / v) * (beta / (alpha - 1))


@EngineUncertaintyEstimatorRegistry.register("evidential-aleatoric")
class EvidentialAleatoricEstimator(_EvidentialEstimator):
    """estimator.py:429-487: beta / (alpha - 1)."""

    @staticmethod
    def _unc(v, alpha, beta):
        return beta / (alpha - 1)


@EngineUncertaintyEstimatorRegistry.register("classification-dirichlet")
class ClassificationDirichletEstimator(_SplitEstimator):
    """estimator.py:648-719: (probability, uncertainty K / S) of the binary Dirichlet head."""

    def _split(self, stacked):
        y, u = stacked.unbind(dim=-1)
        return y, u


@EngineUncertaintyEstimatorRegistry.register("quantile-regression")
class QuantileRegressionEstimator(_SplitEstimator):
    """estimator.py:823-877: (mean, half the predicted interval)."""
    _float = True

    def _split(self, stacked):
        mean, interval = stacked.unbind(-1)
        return mean, interval / 2


@EngineUncertaintyEstimatorRegistry.register("multiclass-dirichlet")
class MulticlassDirichletEstimator(UncertaintyEstimator):
    """estimator.py:722-820: each predictor's forward is replaced for the call by alpha = train_step(Z) ->
    [alpha / S || C / S] (S = sum of alpha), and the outputs split into the class probabilities and the uncertainty.  Of
    an EngineMolAtomBondMPNN every present predictor is replaced."""

    def __call__(self, batches, models):
        outs = ([], [], [])
        for model in models:
            predictors = list(model.predictors) if _is_mab(models) else [model.predictor]
            patched = [p for p in predictors if p is not None]
            try:
                for p in patched:
                    p.forward = _dirichlet_forward(p)
                levels = model.predict(batches)
                levels = levels if _is_mab(models) else [levels]
            finally:
                for p in patched:
                    del p.forward                      # the instance attribute shadowed the class's forward
            for out, output in zip(outs, levels):
                if output is not None:
                    out.append(output)
        per_level = [(torch.stack([o[..., :-1] for o in out], 0), torch.stack([o[..., -1] for o in out], 0))
                     if out else (None, None) for out in outs]
        if not _is_mab(models):
            return per_level[0]
        return tuple(p for p, _ in per_level), tuple(u for _, u in per_level)


def _dirichlet_forward(predictor: nn.Module):
    def forward(Z):
        alpha = predictor.train_step(Z)
        u = alpha.shape[2] / alpha.sum(-1, keepdim=True)
        return torch.concat([alpha / alpha.sum(-1, keepdim=True), u], -1)

    return forward


@EngineUncertaintyEstimatorRegistry.register("dropout")
class DropoutEstimator(UncertaintyEstimator):
    """estimator.py:490-636: Monte Carlo dropout.  For each model: `p` of every nn.Dropout module replaced by `dropout`
    when given (truthy), `ensemble_size` passes of `predict` with the nn.Dropout modules trained and the rest in eval mode,
    then the mean and the population variance over the passes; `p` and every training flag are restored, even on error.
    The masks come from torch's generator, so `torch.manual_seed` makes a run repeatable."""

    def __init__(self, ensemble_size: int, dropout: float | None = None):
        self.ensemble_size = ensemble_size
        self.dropout = dropout

    def _samples(self, batches, model) -> list:
        drops = [m for m in model.modules() if isinstance(m, nn.Dropout)]
        ps = [m.p for m in drops]
        try:
            if self.dropout:
                for m in drops:
                    m.p = self.dropout
            return [model.predict(batches, active_dropout=True) for _ in range(self.ensemble_size)]
        finally:
            for m, p in zip(drops, ps):
                m.p = p

    def __call__(self, batches, models):
        mab = _is_mab(models)
        meanss, varss = ([], [], []), ([], [], [])
        for model in models:
            samples = self._samples(batches, model)
            levels = zip(*samples) if mab else [samples]
            for level, passes in enumerate(levels):
                if passes[0] is None:
                    continue
                stacked = torch.stack(list(passes), dim=0).float()
                meanss[level].append(torch.mean(stacked, dim=0))
                varss[level].append(torch.var(stacked, dim=0, correction=0))
        if not mab:
            return torch.stack(meanss[0]), torch.stack(varss[0])
        return (tuple(torch.stack(m) if m else None for m in meanss), tuple(torch.stack(v) if v else None for v in varss))


__all__ = ["EngineUncertaintyEstimatorRegistry", "UncertaintyEstimator", "NoUncertaintyEstimator", "MVEEstimator",
           "EnsembleEstimator", "ClassEstimator", "EvidentialTotalEstimator", "EvidentialEpistemicEstimator",
           "EvidentialAleatoricEstimator", "DropoutEstimator", "ClassificationDirichletEstimator",
           "MulticlassDirichletEstimator", "QuantileRegressionEstimator"]
