"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/fixture_mpnn_binary.npz and fixture_mpnn_multiclass.npz by running the
UNMODIFIED reference (chemprop v2.3.1, imported through oracle/ref_shim.py) on seeded batches; the outputs are committed, the
reference does not travel with the tests.

    python -m tools.make_golden_classification

Each case is the reference's own training step (chemprop/models/model.py:148-161): `MPNN(BondMessagePassing(d_h = 40),
MeanAggregation(), <predictor>(n_layers = 2), batch_norm = True).training_step(batch)` on 14 seeded molecules with NaN targets,
per-molecule weights and non-uniform task weights -- BinaryClassificationFFN on 3 tasks with one soft label,
MulticlassClassificationFFN on 2 tasks of 4 classes.  Recorded: the initial state dict, targets, weights, the loss, every
gradient, the batch-norm running statistics after the step and the eval-mode predictions."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import import_reference  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def classification_case(kind: str, seed: int) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MPNN

    from chemprop_b200.data.synthetic import make_molecules

    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    mgs = make_molecules(14, seed=seed, mean_atoms=9, std_atoms=3, min_atoms=1)
    bmg = RefBMG([RefMG(*m) for m in mgs])
    mp = ref_nn.BondMessagePassing(d_h=40, depth=3)
    if kind == "binary":
        T = 3
        tw = torch.tensor([1.0, 0.5, 2.0])
        predictor = ref_nn.BinaryClassificationFFN(n_tasks=T, input_dim=40, hidden_dim=24, n_layers=2, task_weights=tw)
        Y = rng.integers(0, 2, size=(14, T)).astype(np.float32)
        Y[5, 2] = 0.3                                    # a soft label
        Y[2, 0] = Y[11, 1] = Y[7, 2] = np.nan
    else:
        T, C = 2, 4
        tw = torch.tensor([0.75, 1.5])
        predictor = ref_nn.MulticlassClassificationFFN(n_classes=C, n_tasks=T, input_dim=40, hidden_dim=24, n_layers=2,
                                                       task_weights=tw)
        Y = rng.integers(0, C, size=(14, T)).astype(np.float32)
        Y[4, 1] = np.nan
        Y[10, 0] = np.nan
    model = MPNN(mp, ref_nn.MeanAggregation(), predictor, batch_norm=True)
    model.log = lambda *a, **k: None                     # Lightning's logger is not part of the path
    with torch.no_grad():                                # non-trivial affine / running statistics
        model.bn.weight.uniform_(0.5, 1.5)
        model.bn.bias.normal_(0, 0.2)
        model.bn.running_mean.normal_(0, 0.1)
        model.bn.running_var.uniform_(0.5, 2.0)
    state0 = {k: v.detach().clone().numpy() for k, v in model.state_dict().items()}
    w = rng.uniform(0.5, 2.0, size=(14,)).astype(np.float32)
    model.train()
    batch = (bmg, None, None, torch.from_numpy(Y), torch.from_numpy(w), None, None)
    loss = model.training_step(batch, 0)
    loss.backward()
    with torch.no_grad():
        model.eval()
        preds_eval = model(bmg)
    d = {"V": bmg.V.numpy(), "E": bmg.E.numpy(), "edge_index": bmg.edge_index.numpy(),
         "rev_edge_index": bmg.rev_edge_index.numpy(), "batch": bmg.batch.numpy(), "n_mols": np.int64(14), "Y": Y, "w": w,
         "loss": loss.detach().numpy(), "preds_eval": preds_eval.numpy()}
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
    for kind, seed in (("binary", 131), ("multiclass", 137)):
        d = classification_case(kind, seed)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mpnn_{kind}.npz"), **d)
        print(f"fixture_mpnn_{kind}: loss={float(d['loss']):.6f} preds_eval{tuple(d['preds_eval'].shape)} "
              f"params={sorted(k for k in d if k.startswith('param.'))}")


if __name__ == "__main__":
    main()
