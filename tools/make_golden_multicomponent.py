"""TEST INFRASTRUCTURE ONLY.  Generates the multicomponent model fixtures tests/golden/fixture_mc_<case>.npz by running the
UNMODIFIED reference (chemprop v2.3.1, imported through oracle/ref_shim.py); the outputs are committed, the reference does
not travel with the tests.

    python -m tools.make_golden_multicomponent

Each fixture is the reference's own `MulticomponentMPNN.training_step` (models/model.py:179-193 with models/multi.py's
fingerprint) on seeded synthetic molecules, two components:
  - shared_reg: one shared BondMessagePassing (d_h = 32), MeanAggregation, regression (MSE) with NaN targets and weights;
  - unshared_bn_xd: BondMessagePassing (d_h = 32, ReLU) + AtomMessagePassing (d_h = 24, ELU, bias), SumAggregation,
    batch_norm=True, molecule descriptors X_d through a ScaleTransform, regression (MSE);
  - shared_bin_edgeless: shared BondMessagePassing (d_h = 32, tanh, bias), NormAggregation, binary classification, and a
    second component of single-atom, edge-less molecules.
Recorded: every component's batch, the initial state dict (minus `metrics.*`), targets, weights, X_d, the train-mode
fingerprint, the train-mode predictions, the loss, every gradient, the batch-norm running statistics after the step and
the eval-mode predictions."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import import_reference  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
N_DP, D_XD, T = 12, 3, 2
CASES = {"shared_reg": 401, "unshared_bn_xd": 409, "shared_bin_edgeless": 419}


def case(name: str, seed: int) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MulticomponentMPNN
    from chemprop.nn.transforms import ScaleTransform

    from chemprop_b200.data.synthetic import make_molecules

    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    solutes = make_molecules(N_DP, seed=seed, mean_atoms=9, std_atoms=3, min_atoms=2)
    if name == "shared_bin_edgeless":
        solvents = make_molecules(N_DP, seed=seed + 1, mean_atoms=1, std_atoms=0, min_atoms=1, max_atoms=1)
    else:
        solvents = make_molecules(N_DP, seed=seed + 1, mean_atoms=4, std_atoms=2, min_atoms=1, max_atoms=8)
    bmgs = [RefBMG([RefMG(*m) for m in mgs]) for mgs in (solutes, solvents)]
    X_d = None
    if name == "shared_reg":
        blocks, shared = [ref_nn.BondMessagePassing(d_h=32)], True
        agg = ref_nn.MeanAggregation()
    elif name == "unshared_bn_xd":
        blocks, shared = [ref_nn.BondMessagePassing(d_h=32), ref_nn.AtomMessagePassing(d_h=24, activation="elu", bias=True)], False
        agg = ref_nn.SumAggregation()
        X_d = rng.normal(1.0, 2.0, size=(N_DP, D_XD)).astype(np.float32)
    else:
        blocks, shared = [ref_nn.BondMessagePassing(d_h=32, activation="tanh", bias=True)], True
        agg = ref_nn.NormAggregation(norm=20.0)
    mcmp = ref_nn.MulticomponentMessagePassing(blocks, n_components=2, shared=shared)
    d_fp = mcmp.output_dim + (D_XD if X_d is not None else 0)
    kw = dict(n_tasks=T, input_dim=d_fp, hidden_dim=24, n_layers=2)
    if name == "shared_bin_edgeless":
        predictor = ref_nn.BinaryClassificationFFN(**kw)
    else:
        predictor = ref_nn.RegressionFFN(**kw, task_weights=torch.tensor([1.0, 0.5]))
    batch_norm = name == "unshared_bn_xd"
    X_d_transform = None
    if X_d is not None:
        X_d_transform = ScaleTransform(X_d.mean(0).tolist(), X_d.std(0).tolist())
    model = MulticomponentMPNN(mcmp, agg, predictor, batch_norm=batch_norm, X_d_transform=X_d_transform)
    model.log = lambda *a, **k: None                     # Lightning's logger is not part of the path
    if batch_norm:
        with torch.no_grad():                            # non-trivial affine / running statistics
            model.bn.weight.uniform_(0.5, 1.5)
            model.bn.bias.normal_(0, 0.2)
            model.bn.running_mean.normal_(0, 0.1)
            model.bn.running_var.uniform_(0.5, 2.0)
    state0 = {k: v.detach().clone().numpy() for k, v in model.state_dict().items() if not k.startswith("metrics.")}
    if name == "shared_bin_edgeless":
        Y = (rng.random((N_DP, T)) < 0.4).astype(np.float32)
    else:
        Y = rng.normal(0.0, 1.0, size=(N_DP, T)).astype(np.float32)
    Y[rng.random(Y.shape) < 0.1] = np.nan
    w = rng.uniform(0.5, 2.0, size=(N_DP, 1)).astype(np.float32)
    t = lambda a: None if a is None else torch.from_numpy(a)  # noqa: E731
    model.train()
    with torch.no_grad():                                # the train-mode fingerprint / predictions on the initial state
        bn_state = {k: v.clone() for k, v in model.bn.state_dict().items()}
        fp = model.fingerprint(bmgs, None, t(X_d)).numpy()
        preds_train = model.predictor.train_step(torch.from_numpy(fp)).numpy()
        model.bn.load_state_dict(bn_state)
    loss = model.training_step((bmgs, [None, None], t(X_d), t(Y), t(w), None, None), 0)
    loss.backward()
    with torch.no_grad():
        model.eval()
        preds_eval = model(bmgs, None, t(X_d)).numpy()
    d = {"loss": loss.detach().numpy(), "batch_norm": np.int64(batch_norm), "shared": np.int64(shared),
         "n_dp": np.int64(N_DP), "Y": Y, "w": w, "fingerprint": fp, "preds_train": preds_train, "preds_eval": preds_eval}
    for c, bmg in enumerate(bmgs):
        d.update({f"V.{c}": bmg.V.numpy(), f"E.{c}": bmg.E.numpy(), f"edge_index.{c}": bmg.edge_index.numpy(),
                  f"rev_edge_index.{c}": bmg.rev_edge_index.numpy(), f"batch.{c}": bmg.batch.numpy()})
    if X_d is not None:
        d["X_d"] = X_d
    for k, v in state0.items():
        d["param." + k] = v
    if batch_norm:
        for k in ("running_mean", "running_var", "num_batches_tracked"):
            d["after.bn." + k] = getattr(model.bn, k).detach().numpy()
    for k, p in model.named_parameters():
        if p.grad is not None:
            d["grad." + k] = p.grad.numpy()
    return d


def main():
    torch.set_num_threads(1)  # deterministic summation order
    for name, seed in CASES.items():
        d = case(name, seed)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mc_{name}.npz"), **d)
        print(f"fixture_mc_{name}: loss={float(d['loss']):.6f} fingerprint {d['fingerprint'].shape}")


if __name__ == "__main__":
    main()
