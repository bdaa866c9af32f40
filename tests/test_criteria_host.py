"""CPU tier: the criteria's shared host path (chemprop_b200/nn/head.py: CriterionLossFunction, `_Criterion.row_loss`)
through the torch emulations of their kernel wrappers: the weights every kernel receives, and which kernel each criterion
runs at atom and bond level."""
from __future__ import annotations

import pytest
import torch

from tests.test_mab_model_host import patch_mab_model
from tests.test_spectral_host import _check_weights
from tests.util import golden_bmg, load_golden

LOSS_WRAPPERS = ("mse_loss", "bce_loss", "ce_loss", "regression_loss", "mve_loss", "evidential_loss", "quantile_loss",
                 "dirichlet_loss", "sid_loss", "wasserstein_loss", "regression_loss_rows", "bce_loss_rows", "ce_loss_rows")


def _mse_bce_ce(b, T, C=3):
    """(criterion, preds, targets) of chemprop's MSE, BCE and cross-entropy on b molecules and T tasks."""
    import chemprop_b200.nn as N

    torch.manual_seed(b + T)
    return (("mse", N.EngineRegressionFFN(n_tasks=T, input_dim=4).criterion, torch.randn(b, T), torch.randn(b, T)),
            ("bce", N.EngineBinaryClassificationFFN(n_tasks=T, input_dim=4).criterion, torch.randn(b, T),
             torch.randint(0, 2, (b, T)).float()),
            ("ce", N.EngineMulticlassClassificationFFN(n_classes=C, n_tasks=T, input_dim=4).criterion, torch.randn(b, T, C),
             torch.randint(0, C, (b, T)).float()))


@pytest.mark.parametrize("rows", [False, True])
def test_mse_bce_and_ce_broadcast_one_task_weight_and_refuse_other_sizes(rows, monkeypatch):
    """A 1-entry task weight reaches the kernel as T entries, as the reference broadcasts it; weights that are not one per
    molecule (row), and task weights of any other size, are refused on the host before a kernel could read past them."""
    from chemprop_b200 import engine

    patch_mab_model(monkeypatch)
    for name in ("mse_loss", "bce_loss", "ce_loss", "regression_loss_rows", "bce_loss_rows", "ce_loss_rows"):
        def checked(P, Y, w, tw, *rest, _fn=getattr(engine, name)):
            _check_weights(Y, w, tw)                    # the kernels read exactly b weights and T task weights
            return _fn(P, Y, w, tw, *rest)

        monkeypatch.setattr(engine, name, checked)
    b, T = 6, 3
    w = torch.rand(b) + 0.5
    for kind, crit, preds, Y in _mse_bce_ce(b, T):
        Y[1, 2] = float("nan")
        loss = crit.row_loss if rows else (lambda P, Y, w: crit(P, Y, None, w))  # noqa: E731
        crit.task_weights = torch.full((1, 1), 2.0)
        one = loss(preds, Y, w)
        crit.task_weights = torch.full((1, T), 2.0)
        assert torch.equal(one, loss(preds, Y, w)), kind
        with pytest.raises(ValueError, match="weights must have"):
            loss(preds, Y, torch.ones(b + 1))
        crit.task_weights = torch.ones(1, T - 1)
        with pytest.raises(ValueError, match="weights must have"):
            loss(preds, Y, None)


def test_uncertainty_and_spectral_criteria_keep_their_own_kernel_at_atom_and_bond_level(monkeypatch):
    """An MVE criterion on atoms and a SID criterion on bonds have no row-parallel kernel: each level runs its criterion's
    own single-block kernel, once, on every row of the level."""
    import chemprop_b200.nn as N
    from chemprop_b200 import engine

    patch_mab_model(monkeypatch)
    census = []
    for name in LOSS_WRAPPERS:
        def recorded(P, *a, _fn=getattr(engine, name), _name=name):
            census.append((_name, int(P.shape[0])))
            return _fn(P, *a)

        monkeypatch.setattr(engine, name, recorded)
    g = load_golden("fixture_mab_model_reg")
    bmg = golden_bmg(g, "cpu")
    V, E = int(bmg.V.shape[0]), int(bmg.E.shape[0])
    torch.manual_seed(0)
    model = N.EngineMolAtomBondMPNN(N.MABBondMessagePassing(d_h=16), atom_predictor=N.EngineMveFFN(n_tasks=2, input_dim=16),
                                    bond_predictor=N.EngineSpectralFFN(n_tasks=5, input_dim=32)).train()
    Ye = torch.rand(E // 2, 5) + 0.1
    loss = model.training_loss(bmg, [None, torch.randn(V, 2), Ye / Ye.sum(1, keepdim=True)], None)
    loss.backward()
    assert torch.isfinite(loss)
    assert sorted(census) == sorted([("mve_loss", V), ("sid_loss", E // 2)]), census
