"""TEST INFRASTRUCTURE ONLY.  Generates the uncertainty-predictor fixtures under tests/golden/ by running the UNMODIFIED
reference (chemprop v2.3.1, imported through oracle/ref_shim.py); the outputs are committed, the reference does not travel
with the tests.

    python -m tools.make_golden_uncertainty

1. fixture_mpnn_{mve,evidential,quantile,binary_dirichlet,multiclass_dirichlet}: the reference's own training step
   (chemprop/models/model.py:148-161), `MPNN(BondMessagePassing(d_h = 40), MeanAggregation(), <predictor>(n_layers = 2),
   batch_norm = True).training_step(batch)` on 14 seeded molecules with 3 tasks, NaN targets, per-molecule weights and
   non-uniform task weights.  The criteria use non-default v_kl / eps / alpha; the regression kinds carry an
   UnscaleTransform with non-trivial mean and scale; the Dirichlet labels include -1 (the last class, as
   `torch.eye(C)[targets.long()]` wraps it).  Recorded: the initial state dict, targets, weights, the loss, every gradient,
   the batch-norm running statistics after the step and the eval-mode predictions.
2. fixture_ckpt_{regression,regression_mve,regression_evidential,regression_quantile,classification_dirichlet,
   multiclass_dirichlet}: the reference's trained checkpoints tests/data/example_model_v2_<kind>_mol.pt -- the hparams
   needed to rebuild each one, its state dict (without `metrics.*`) with every tensor after the encoder in full and the
   encoder's tensors as key and shape only (`shape.message_passing.*`: its 228 k floats would make each fixture 1.2 MB; the
   regression checkpoint's encoder is the `bond_d3_trained` golden's), and, on 24 seeded synthetic molecules of the default
   widths (d_v = 72, d_e = 14), the reference's aggregated encoder output H (before batch norm) and its eval-mode
   predictions `model(bmg)`, which equal `predictor(bn(H))`.  Weights and outputs only."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import REFERENCE_ROOT, import_reference  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
T = 3
TRAIN_KINDS = {"mve": 151, "evidential": 157, "quantile": 163, "binary_dirichlet": 167, "multiclass_dirichlet": 173}
CKPT_KINDS = ("regression", "regression_mve", "regression_evidential", "regression_quantile", "classification_dirichlet",
              "multiclass_dirichlet")
UNSCALE_MEAN, UNSCALE_SCALE = [2.12, -0.7, 0.4], [1.36, 0.5, 3.0]
V_KL, EPS, ALPHA, N_CLASSES = 0.35, 0.05, 0.3, 4


def _graph_arrays(bmg, n_mols: int) -> dict:
    return {"V": bmg.V.numpy(), "E": bmg.E.numpy(), "edge_index": bmg.edge_index.numpy(),
            "rev_edge_index": bmg.rev_edge_index.numpy(), "batch": bmg.batch.numpy(), "n_mols": np.int64(n_mols)}


def training_case(kind: str, seed: int) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MPNN
    from chemprop.nn.metrics import DirichletLoss, EvidentialLoss, QuantileLoss
    from chemprop.nn.transforms import UnscaleTransform

    from chemprop_b200.data.synthetic import make_molecules

    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    mgs = make_molecules(14, seed=seed, mean_atoms=9, std_atoms=3, min_atoms=1)
    bmg = RefBMG([RefMG(*m) for m in mgs])
    mp = ref_nn.BondMessagePassing(d_h=40, depth=3)
    tw = torch.tensor([1.0, 0.5, 2.0])
    kw = dict(n_tasks=T, input_dim=40, hidden_dim=24, n_layers=2)
    unscale = UnscaleTransform(UNSCALE_MEAN, UNSCALE_SCALE)
    if kind == "mve":
        predictor = ref_nn.MveFFN(**kw, task_weights=tw, output_transform=unscale)
    elif kind == "evidential":
        predictor = ref_nn.EvidentialFFN(**kw, criterion=EvidentialLoss(tw, v_kl=V_KL, eps=EPS), output_transform=unscale)
    elif kind == "quantile":
        predictor = ref_nn.QuantileFFN(**kw, criterion=QuantileLoss(tw, alpha=ALPHA), output_transform=unscale)
    elif kind == "binary_dirichlet":
        predictor = ref_nn.BinaryDirichletFFN(**kw, criterion=DirichletLoss(tw, v_kl=V_KL))
    else:
        predictor = ref_nn.MulticlassDirichletFFN(n_classes=N_CLASSES, **kw, criterion=DirichletLoss(tw, v_kl=V_KL))
    if kind.endswith("dirichlet"):
        C = 2 if kind.startswith("binary") else N_CLASSES
        Y = rng.integers(0, C, size=(14, T)).astype(np.float32)
        Y[3, 1] = -1.0                                   # torch.eye(C)[-1]: the last class
    else:
        Y = rng.normal(0.0, 1.0, size=(14, T)).astype(np.float32)
    Y[2, 0] = Y[11, 1] = Y[7, 2] = np.nan
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
    d = _graph_arrays(bmg, 14)
    d.update({"Y": Y, "w": w, "loss": loss.detach().numpy(), "preds_eval": preds_eval.numpy()})
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


def checkpoint_case(kind: str) -> dict:
    import pickle
    import types

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MPNN
    from chemprop.nn.transforms import UnscaleTransform

    from chemprop_b200.data.synthetic import make_molecules

    class _Anything(dict):           # stands in for classes of packages that are not installed (lightning.fabric ...)
        def __init__(self, *a, **k):
            pass

        def __setstate__(self, state):
            pass

    class _Unpickler(pickle.Unpickler):
        def find_class(self, module, name):
            try:
                return super().find_class(module, name)
            except Exception:
                return type(name, (_Anything,), {})

    pm = types.ModuleType("permissive_pickle")
    pm.__dict__.update(pickle.__dict__)
    pm.Unpickler = _Unpickler
    path = os.path.join(REFERENCE_ROOT, "tests", "data", f"example_model_v2_{kind}_mol.pt")
    ck = torch.load(path, map_location="cpu", weights_only=False, pickle_module=pm)
    hp, sd = ck["hyper_parameters"], {k: v for k, v in ck["state_dict"].items() if not k.startswith("metrics.")}
    mp_hp, agg_hp, pr_hp = hp["message_passing"], hp["agg"], hp["predictor"]
    mp = ref_nn.BondMessagePassing(d_v=mp_hp["d_v"], d_e=mp_hp["d_e"], d_h=mp_hp["d_h"], depth=mp_hp["depth"])
    agg = ref_nn.NormAggregation(norm=agg_hp["norm"]) if "norm" in agg_hp else ref_nn.MeanAggregation()
    n_classes = int(pr_hp.get("n_classes", 0))
    kw = dict(n_tasks=pr_hp["n_tasks"], input_dim=pr_hp["input_dim"], hidden_dim=pr_hp["hidden_dim"],
              n_layers=pr_hp["n_layers"])
    if n_classes:
        kw["n_classes"] = n_classes
    if "predictor.output_transform.mean" in sd:
        kw["output_transform"] = UnscaleTransform(sd["predictor.output_transform.mean"][0].tolist(),
                                                  sd["predictor.output_transform.scale"][0].tolist())
    predictor = pr_hp["cls"](**kw)
    model = MPNN(mp, agg, predictor, batch_norm=bool(hp["batch_norm"]))
    res = model.load_state_dict(sd, strict=False)
    # the only keys the checkpoint lacks are torchmetrics states (total_loss, num_samples) and the metrics list
    assert all(k.startswith("metrics.") or k.endswith(("total_loss", "num_samples")) for k in res.missing_keys), res
    assert not res.unexpected_keys, res
    mgs = make_molecules(24, seed=181)
    bmg = RefBMG([RefMG(*m) for m in mgs])
    model.eval()
    with torch.no_grad():
        preds = model(bmg)
        H = model.agg(model.message_passing(bmg), bmg.batch)
        assert torch.equal(model.predictor(model.bn(H)), preds)
    d = _graph_arrays(bmg, 24)
    d["H"] = H.numpy()
    d.update({"preds_eval": preds.numpy(), "hp.n_tasks": np.int64(pr_hp["n_tasks"]), "hp.n_classes": np.int64(n_classes),
              "hp.n_layers": np.int64(pr_hp["n_layers"]), "hp.hidden_dim": np.int64(pr_hp["hidden_dim"]),
              "hp.d_h": np.int64(mp_hp["d_h"]), "hp.depth": np.int64(mp_hp["depth"]),
              "hp.norm": np.float64(agg_hp.get("norm", 0.0)), "hp.batch_norm": np.int64(bool(hp["batch_norm"])),
              "hp.predictor": np.str_(pr_hp["cls"].__name__)})
    for k, v in sd.items():
        if k.startswith("message_passing."):
            d["shape." + k] = np.asarray(v.shape, dtype=np.int64)
        else:
            d["param." + k] = v.detach().numpy()
    return d


def main():
    torch.set_num_threads(1)  # deterministic summation order
    for kind, seed in TRAIN_KINDS.items():
        d = training_case(kind, seed)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mpnn_{kind}.npz"), **d)
        print(f"fixture_mpnn_{kind}: loss={float(d['loss']):.6f} preds_eval{tuple(d['preds_eval'].shape)}")
    for kind in CKPT_KINDS:
        d = checkpoint_case(kind)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_ckpt_{kind}.npz"), **d)
        print(f"fixture_ckpt_{kind}: {d['hp.predictor']} preds_eval{tuple(d['preds_eval'].shape)}")


if __name__ == "__main__":
    main()
