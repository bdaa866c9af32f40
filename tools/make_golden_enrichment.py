"""TEST INFRASTRUCTURE ONLY.  Generates the count-data regression fixtures under tests/golden/ by running the UNMODIFIED
reference (chemprop v2.3.1, imported through oracle/ref_shim.py); the outputs are committed, the reference does not travel
with the tests.

    python -m tools.make_golden_enrichment

Each fixture is the reference's own training step (chemprop/models/model.py:148-161),
`MPNN(BondMessagePassing(d_h = 40), MeanAggregation(), RegressionFFN(n_layers = 2, ...), batch_norm = True)
.training_step(batch)` on 14 seeded molecules with per-molecule weights:

1. fixture_mpnn_enrichment_{sqrt,score,wald}: the recipe of examples/training_NLogProbEnrichment.ipynb,
   `RegressionFFN(criterion=NLogProbEnrichment(tw, n1, n2, method, zscale, zinterval), output_transform=Softplus())`, on
   Poisson counts (k1, k2) with zeros and one NaN count; n1 and n2 are the column totals.  sqrt runs at zinterval 1.5, so
   that terms sit at the clamp; score at zscale 1.7; wald with the defaults.  score and wald keep every row's counts
   (after nan_to_num) off (0, 0), where their z is NaN and the reference raises.
2. fixture_mpnn_enrichment_score_raises: the score batch with one row of zero counts, on which the reference's
   training step raises "Got nan loss ..."; recorded are the inputs and the message.
3. fixture_mpnn_quantile_point: RegressionFFN with 3 tasks, NaN targets and PointQuantileLoss(tw, alpha = 0.3).

Recorded (1, 3): the initial state dict, targets, weights, the training-mode predictions before the step, the loss, every
gradient, the batch-norm running statistics after the step, the eval-mode predictions and the reference predictor's
hparams keys; and the same step re-run in float64 from the same state (`f64.loss`, `f64.grad.*`, `f64.after.bn.*`,
`f64.preds_train`): the reference's own f32-vs-f64 gap sets the bar the engine is held to.  Weights and outputs only."""
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
N_MOLS, T_REG, ALPHA = 14, 3, 0.3
ENRICH = {"sqrt": dict(seed=229, zscale=1.0, zinterval=1.5),
          "score": dict(seed=233, zscale=1.7, zinterval=5.0),
          "wald": dict(seed=239, zscale=1.0, zinterval=5.0)}
QUANTILE_SEED = 241


def _graph_arrays(bmg, n_mols: int) -> dict:
    return {"V": bmg.V.numpy(), "E": bmg.E.numpy(), "edge_index": bmg.edge_index.numpy(),
            "rev_edge_index": bmg.rev_edge_index.numpy(), "batch": bmg.batch.numpy(), "n_mols": np.int64(n_mols)}


def _counts(rng, method: str, zero_row: bool) -> np.ndarray:
    """Poisson (k1, k2) with zeros in both columns and one NaN count; for score / wald no row is (0, 0) after nan_to_num
    unless `zero_row` asks for one."""
    Y = np.stack([rng.poisson(3.0, N_MOLS), rng.poisson(2.0, N_MOLS)], 1).astype(np.float32)
    Y[1, 0] = Y[6, 1] = 0.0
    Y[9, 1] = np.nan
    Y[3] = (40.0, 1.0)                                     # a strongly enriched molecule: |z| large
    if method != "sqrt":
        k = np.nan_to_num(Y)
        Y[(k == 0).all(1), 0] = 1.0
    if zero_row:
        Y[5] = (0.0, 0.0)
    return Y


def _model(predictor, seed: int):
    import chemprop.nn as ref_nn
    from chemprop.models import MPNN

    torch.manual_seed(seed)
    model = MPNN(ref_nn.BondMessagePassing(d_h=40, depth=3), ref_nn.MeanAggregation(), predictor, batch_norm=True)
    model.log = lambda *a, **k: None                     # Lightning's logger is not part of the path
    with torch.no_grad():                                # non-trivial affine / running statistics
        model.bn.weight.uniform_(0.5, 1.5)
        model.bn.bias.normal_(0, 0.2)
        model.bn.running_mean.normal_(0, 0.1)
        model.bn.running_var.uniform_(0.5, 2.0)
    return model


def _step(model, bmg, Y, w):
    """training_step + backward; returns (loss, grads, bn statistics after, training-mode predictions before)."""
    with torch.no_grad():
        probe = copy.deepcopy(model).train()
        preds_train = probe.predictor.train_step(probe.fingerprint(bmg))
    model.train()
    loss = model.training_step((bmg, None, None, Y, w, None, None), 0)
    loss.backward()
    grads = {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}
    after = {k: v.detach().clone() for k, v in model.state_dict().items()
             if k.startswith("bn.running") or k == "bn.num_batches_tracked"}
    return loss.detach(), grads, after, preds_train


def _bmg64(bmg):
    b = copy.copy(bmg)
    b.V, b.E = bmg.V.double(), bmg.E.double()
    return b


def training_case(kind: str) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.nn import metrics as M

    from chemprop_b200.data.synthetic import make_molecules

    method = kind.split("_")[1] if kind.startswith("enrichment") else None
    seed = ENRICH[method]["seed"] if method else QUANTILE_SEED
    raises = kind.endswith("_raises")
    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    mgs = make_molecules(N_MOLS, seed=seed, mean_atoms=9, std_atoms=3, min_atoms=1)
    bmg = RefBMG([RefMG(*m) for m in mgs])
    extra = {}
    if method:
        cfg = ENRICH[method]
        Y = _counts(rng, method, raises)
        n1, n2 = int(np.nansum(Y[:, 0])), int(np.nansum(Y[:, 1]))
        tw = torch.tensor([1.0, 0.5])
        crit = M.NLogProbEnrichment(tw, n1=n1, n2=n2, method=method, zscale=cfg["zscale"], zinterval=cfg["zinterval"])
        predictor = ref_nn.RegressionFFN(n_tasks=1, input_dim=40, hidden_dim=24, n_layers=2, criterion=crit,
                                         output_transform=torch.nn.Softplus())
        extra = {"n1": np.int64(n1), "n2": np.int64(n2), "method": np.array(method), "zscale": np.float64(cfg["zscale"]),
                 "zinterval": np.float64(cfg["zinterval"])}
    else:
        tw = torch.tensor([1.0, 0.5, 2.0])
        crit = M.PointQuantileLoss(tw, alpha=ALPHA)
        predictor = ref_nn.RegressionFFN(n_tasks=T_REG, input_dim=40, hidden_dim=24, n_layers=2, criterion=crit)
        Y = rng.normal(0.0, 1.0, size=(N_MOLS, T_REG)).astype(np.float32)
        Y[2, 0] = Y[11, 1] = Y[7, 2] = np.nan
        extra = {"alpha": np.float64(ALPHA)}
    model = _model(predictor, seed)
    state0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
    w = rng.uniform(0.5, 2.0, size=(N_MOLS,)).astype(np.float32)
    d = _graph_arrays(bmg, N_MOLS)
    d.update({"Y": Y, "w": w, "hp_keys": np.array(sorted(predictor.hparams.keys())), **extra})
    for k, v in state0.items():
        if not k.startswith("metrics."):
            d["param." + k] = v.numpy()
    if raises:
        try:
            _step(model, bmg, torch.from_numpy(Y), torch.from_numpy(w))
        except ValueError as e:
            d["error"] = np.array(str(e))
            return d
        raise AssertionError("the reference did not raise")
    loss, grads, after, preds_train = _step(model, bmg, torch.from_numpy(Y), torch.from_numpy(w))
    with torch.no_grad():
        model.eval()
        preds_eval = model(bmg)
    d.update({"loss": loss.numpy(), "preds_train": preds_train.numpy(), "preds_eval": preds_eval.numpy()})
    d.update({"after." + k: v.numpy() for k, v in after.items()})
    d.update({"grad." + k: v.numpy() for k, v in grads.items()})
    # the same step in float64 from the same state
    m64 = _model(copy.deepcopy(predictor), seed)
    m64.load_state_dict(state0)
    m64.double()
    # torchmetrics' Metric.double() also turns the states' defaults to float64; the stand-in keeps them apart
    c64 = m64.predictor.criterion
    c64.__dict__["_state_defaults"] = {n: v.double() if v.is_floating_point() else v
                                       for n, v in c64.__dict__.get("_state_defaults", {}).items()}
    loss64, grads64, after64, preds64 = _step(m64, _bmg64(bmg), torch.from_numpy(Y).double(), torch.from_numpy(w).double())
    d.update({"f64.loss": loss64.numpy(), "f64.preds_train": preds64.numpy()})
    d.update({"f64.after." + k: v.numpy() for k, v in after64.items()})
    d.update({"f64.grad." + k: v.numpy() for k, v in grads64.items()})
    return d


KINDS = ("enrichment_sqrt", "enrichment_score", "enrichment_wald", "enrichment_score_raises", "quantile_point")


def main():
    torch.set_num_threads(1)  # deterministic summation order
    for kind in KINDS:
        d = training_case(kind)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mpnn_{kind}.npz"), **d)
        if "error" in d:
            print(f"fixture_mpnn_{kind}: raises {d['error']}")
        else:
            print(f"fixture_mpnn_{kind}: loss={float(d['loss']):.6f} f64={float(d['f64.loss']):.6f} "
                  f"preds_eval{tuple(d['preds_eval'].shape)}")


if __name__ == "__main__":
    main()
