"""TEST INFRASTRUCTURE ONLY.  Generates the spectral-predictor and regression-loss fixtures under tests/golden/ by running
the UNMODIFIED reference (chemprop v2.3.1, imported through oracle/ref_shim.py); the outputs are committed, the reference
does not travel with the tests.

    python -m tools.make_golden_spectral

Each fixture is the reference's own training step (chemprop/models/model.py:148-161),
`MPNN(BondMessagePassing(d_h = 40), MeanAggregation(), <predictor>(n_layers = 2), batch_norm = True).training_step(batch)`
on 14 seeded molecules with per-molecule weights and non-uniform task weights:

1. fixture_mpnn_spectral_sid: SpectralFFN with 40 bins, softplus and SID(threshold = 0.025), which clamps about half of
   the predictions (each near 1 / 40).  The targets are positive synthetic spectra normalised per row, with NaN bins, one of
   them the first bin of a row.
2. fixture_mpnn_spectral_wasserstein: the same with spectral_activation="exp" and criterion=Wasserstein(tw, 0.025).  The
   MLP outputs stay within a few units, so exp(exp(x)) is finite.
3. fixture_mpnn_{mae,rmse,bounded_mse,bounded_mae,bounded_rmse}: RegressionFFN with 3 tasks, NaN targets and the named
   criterion.  The bounded ones get lt_mask / gt_mask with set entries on both sides of their bound and on masked targets.

Recorded: the initial state dict, targets, weights and masks, the training-mode predictions before the step, the loss,
every gradient, the batch-norm running statistics after the step, the eval-mode predictions and the reference
predictor's hparams keys.  Weights and outputs only."""
from __future__ import annotations

import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import import_reference  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
N_MOLS, N_BINS, T_REG, THRESHOLD = 14, 40, 3, 0.025
KINDS = {"spectral_sid": 191, "spectral_wasserstein": 193, "mae": 197, "rmse": 199, "bounded_mse": 211,
         "bounded_mae": 223, "bounded_rmse": 227}


def _graph_arrays(bmg, n_mols: int) -> dict:
    return {"V": bmg.V.numpy(), "E": bmg.E.numpy(), "edge_index": bmg.edge_index.numpy(),
            "rev_edge_index": bmg.rev_edge_index.numpy(), "batch": bmg.batch.numpy(), "n_mols": np.int64(n_mols)}


def _spectra(rng) -> np.ndarray:
    """Positive spectra: a baseline plus three Gaussian bands per row, normalised to sum 1; NaN bins afterwards."""
    x = np.arange(N_BINS, dtype=np.float64)
    Y = np.full((N_MOLS, N_BINS), 0.05)
    for _ in range(3):
        c, s, a = rng.uniform(0, N_BINS, (N_MOLS, 1)), rng.uniform(1.5, 6, (N_MOLS, 1)), rng.uniform(0.2, 1.0, (N_MOLS, 1))
        Y += a * np.exp(-0.5 * ((x - c) / s) ** 2)
    Y /= Y.sum(1, keepdims=True)
    Y = Y.astype(np.float32)
    Y[rng.random(Y.shape) < 0.08] = np.nan
    Y[4, 0] = np.nan                                       # a masked first bin
    return Y


def training_case(kind: str, seed: int) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MPNN
    from chemprop.nn import metrics as M

    from chemprop_b200.data.synthetic import make_molecules

    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    mgs = make_molecules(N_MOLS, seed=seed, mean_atoms=9, std_atoms=3, min_atoms=1)
    bmg = RefBMG([RefMG(*m) for m in mgs])
    mp = ref_nn.BondMessagePassing(d_h=40, depth=3)
    lt = gt = None
    if kind.startswith("spectral"):
        tw = torch.linspace(0.5, 2.0, N_BINS)
        kw = dict(n_tasks=N_BINS, input_dim=40, hidden_dim=24, n_layers=2)
        if kind == "spectral_sid":
            predictor = ref_nn.SpectralFFN(**kw, task_weights=tw, threshold=THRESHOLD)
        else:
            predictor = ref_nn.SpectralFFN(**kw, criterion=M.Wasserstein(tw, threshold=THRESHOLD),
                                           spectral_activation="exp")
        Y = _spectra(rng)
    else:
        tw = torch.tensor([1.0, 0.5, 2.0])
        crit = {"mae": M.MAE, "rmse": M.RMSE, "bounded_mse": M.BoundedMSE, "bounded_mae": M.BoundedMAE,
                "bounded_rmse": M.BoundedRMSE}[kind](tw)
        predictor = ref_nn.RegressionFFN(n_tasks=T_REG, input_dim=40, hidden_dim=24, n_layers=2, criterion=crit)
        Y = rng.normal(0.0, 1.0, size=(N_MOLS, T_REG)).astype(np.float32)
        Y[2, 0] = Y[11, 1] = Y[7, 2] = np.nan
        if kind.startswith("bounded"):
            sel = rng.random(Y.shape)
            lt, gt = sel < 0.35, sel > 0.65
            lt[2, 0] = gt[11, 1] = True                    # set on masked targets
    model = MPNN(mp, ref_nn.MeanAggregation(), predictor, batch_norm=True)
    model.log = lambda *a, **k: None                     # Lightning's logger is not part of the path
    with torch.no_grad():                                # non-trivial affine / running statistics
        model.bn.weight.uniform_(0.5, 1.5)
        model.bn.bias.normal_(0, 0.2)
        model.bn.running_mean.normal_(0, 0.1)
        model.bn.running_var.uniform_(0.5, 2.0)
    state0 = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    w = rng.uniform(0.5, 2.0, size=(N_MOLS,)).astype(np.float32)
    with torch.no_grad():                                # the training-mode predictions the criterion sees
        probe = copy.deepcopy(model).train()
        preds_train = probe.predictor.train_step(probe.fingerprint(bmg)).numpy()
    model.train()
    lt_t = None if lt is None else torch.from_numpy(lt)
    gt_t = None if gt is None else torch.from_numpy(gt)
    batch = (bmg, None, None, torch.from_numpy(Y), torch.from_numpy(w), lt_t, gt_t)
    loss = model.training_step(batch, 0)
    loss.backward()
    with torch.no_grad():
        model.eval()
        preds_eval = model(bmg)
    d = _graph_arrays(bmg, N_MOLS)
    d.update({"Y": Y, "w": w, "loss": loss.detach().numpy(), "preds_train": preds_train, "preds_eval": preds_eval.numpy(),
              "hp_keys": np.array(sorted(predictor.hparams.keys()))})
    if lt is not None:
        d.update({"lt_mask": lt, "gt_mask": gt})
    for k, v in state0.items():
        if not k.startswith("metrics."):
            d["param." + k] = v
    for k, v in model.state_dict().items():
        if k.startswith("bn.running") or k == "bn.num_batches_tracked":
            d["after." + k] = v.detach().numpy()
    for k, p in model.named_parameters():
        if p.grad is not None:
            d["grad." + k] = p.grad.numpy()
    return d


def main():
    torch.set_num_threads(1)  # deterministic summation order
    for kind, seed in KINDS.items():
        d = training_case(kind, seed)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mpnn_{kind}.npz"), **d)
        print(f"fixture_mpnn_{kind}: loss={float(d['loss']):.6f} preds_eval{tuple(d['preds_eval'].shape)}")


if __name__ == "__main__":
    main()
