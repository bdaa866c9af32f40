"""TEST INFRASTRUCTURE ONLY.  Generates the mol-atom-bond model fixtures under tests/golden/ by running the UNMODIFIED
reference (chemprop v2.3.1, imported through oracle/ref_shim.py); the outputs are committed, the reference does not
travel with the tests.

    python -m tools.make_golden_mab_model

1. fixture_mab_model_<case>.npz: the reference's own `MolAtomBondMPNN.training_step` (models/mol_atom_bond.py:291-339)
   on seeded synthetic molecules, MABBondMessagePassing(d_h = 32), predictors with n_layers = 2:
   - reg: regression at all three levels, batch_norm=True, NaN targets, per-row weights and molecule descriptors X_d;
   - bin_bounded: no molecule level; binary classification at atom level; BoundedMSE at bond level with lt / gt masks;
   - constrained: regression at all three levels with atom and bond constrainers and their constraints.
   Recorded: the initial state dict (minus `metricss.*`), targets, weights, masks, constraints, the loss, every gradient,
   the batch-norm running statistics after the step and the eval-mode predictions (with the constraints).
2. fixture_mab_ckpt_<name>.npz: the reference's trained checkpoints tests/data/mol_atom_bond/example_models/<name>.pt
   (regression, regression_mve, regression_constrained).  The trained heads hold 0.36 - 0.63 M weights (1.4 - 2.5 MB in
   f32, too large for a test vector), so a fixture holds:
   - the shape of every key of the checkpoint's state dict (encoder and heads) and the hparams that rebuild the model:
     the engine model must load a state dict of exactly these keys and shapes with strict=True;
   - the trained heads cut to their first HIDDEN_KEPT hidden units (rows of each MLP's first layer, columns of its last;
     every other tensor -- biases of the last layers, task weights, the target scalers -- in full), and the eval-mode
     predictions of the reference model with those heads (with constraints where the checkpoint has constrainers);
   - the reference's pre-batch-norm fingerprints (H_v, H_e and the aggregated H_g) of the checkpoint's trained encoder on
     6 synthetic molecules."""
from __future__ import annotations

import os
import pickle
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import REFERENCE_ROOT, import_reference  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
N_MOLS, D_H, D_XD = 10, 32, 3
TRAIN_CASES = {"reg": 301, "bin_bounded": 307, "constrained": 311}
CKPT_CASES = ("regression", "regression_mve", "regression_constrained")
N_CKPT_MOLS, HIDDEN_KEPT = 6, 16


def _graph_arrays(bmg, n_mols: int) -> dict:
    return {"V": bmg.V.numpy(), "E": bmg.E.numpy(), "edge_index": bmg.edge_index.numpy(),
            "rev_edge_index": bmg.rev_edge_index.numpy(), "batch": bmg.batch.numpy(), "n_mols": np.int64(n_mols)}


def _rows(bmg):
    return int(bmg.V.shape[0]), int(bmg.E.shape[0]) // 2


def training_case(case: str, seed: int) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data.collate import BatchMolAtomBondGraph
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MolAtomBondMPNN
    from chemprop.nn import metrics as M
    from chemprop.nn.ffn import ConstrainerFFN
    from chemprop.nn.message_passing import MABBondMessagePassing

    from chemprop_b200.data.synthetic import make_molecules

    rng = np.random.default_rng(seed)
    torch.manual_seed(seed)
    bmg = BatchMolAtomBondGraph([RefMG(*m) for m in make_molecules(N_MOLS, seed=seed, mean_atoms=9, std_atoms=3,
                                                                   min_atoms=2)])
    V, Eh = _rows(bmg)
    mp = MABBondMessagePassing(d_h=D_H, depth=3)
    kw = dict(hidden_dim=24, n_layers=2)
    preds = dict(mol_predictor=None, atom_predictor=None, bond_predictor=None)
    cons = dict()
    X_d = None
    T = (2, 2, 1)
    if case in ("reg", "constrained"):
        d_mol = D_H + (D_XD if case == "reg" else 0)
        preds["mol_predictor"] = ref_nn.RegressionFFN(n_tasks=T[0], input_dim=d_mol, **kw,
                                                      task_weights=torch.tensor([1.0, 0.5]))
        preds["atom_predictor"] = ref_nn.RegressionFFN(n_tasks=T[1], input_dim=D_H, **kw,
                                                       task_weights=torch.tensor([2.0, 0.75]))
        preds["bond_predictor"] = ref_nn.RegressionFFN(n_tasks=T[2], input_dim=2 * D_H, **kw)
        if case == "reg":
            X_d = rng.normal(size=(N_MOLS, D_XD)).astype(np.float32)
        else:
            cons = dict(atom_constrainer=ConstrainerFFN(n_constraints=T[1], fp_dim=D_H, hidden_dim=16),
                        bond_constrainer=ConstrainerFFN(n_constraints=T[2], fp_dim=2 * D_H, hidden_dim=16))
    else:
        preds["atom_predictor"] = ref_nn.BinaryClassificationFFN(n_tasks=T[1], input_dim=D_H, **kw)
        preds["bond_predictor"] = ref_nn.RegressionFFN(n_tasks=T[2], input_dim=2 * D_H, **kw,
                                                       criterion=M.BoundedMSE(torch.ones(T[2])))
    batch_norm = case != "constrained"
    model = MolAtomBondMPNN(mp, ref_nn.SumAggregation() if preds["mol_predictor"] is not None else None,
                            batch_norm=batch_norm, **preds, **cons)
    model.log = lambda *a, **k: None                     # Lightning's logger is not part of the path
    if batch_norm:
        with torch.no_grad():                            # non-trivial affine / running statistics
            for bn in model.bns:
                if isinstance(bn, torch.nn.BatchNorm1d):
                    bn.weight.uniform_(0.5, 1.5)
                    bn.bias.normal_(0, 0.2)
                    bn.running_mean.normal_(0, 0.1)
                    bn.running_var.uniform_(0.5, 2.0)
    state0 = {k: v.detach().clone().numpy() for k, v in model.state_dict().items() if not k.startswith("metricss.")}
    rows = (N_MOLS, V, Eh)
    targetss, weightss, lts, gts = [], [], [None] * 3, [None] * 3
    w_mol = rng.uniform(0.5, 2.0, size=(N_MOLS, 1)).astype(np.float32)
    counts = (np.ones(N_MOLS, np.int64), np.bincount(bmg.batch.numpy(), minlength=N_MOLS),
              np.bincount(bmg.bond_batch.numpy()[::2], minlength=N_MOLS))
    for level, p in enumerate(model.predictors):
        if p is None:
            targetss.append(None)
            weightss.append(None)
            continue
        if isinstance(p, ref_nn.BinaryClassificationFFN):
            Y = (rng.random((rows[level], T[level])) < 0.4).astype(np.float32)
        else:
            Y = rng.normal(0.0, 1.0, size=(rows[level], T[level])).astype(np.float32)
        Y[rng.random(Y.shape) < 0.12] = np.nan
        targetss.append(Y)
        weightss.append(np.repeat(w_mol, counts[level], axis=0))
        if isinstance(p.criterion, M.BoundedMSE):
            sel = rng.random(Y.shape)
            lts[level], gts[level] = sel < 0.35, sel > 0.65
    constraints = None
    if cons:
        constraints = [rng.normal(size=(N_MOLS, T[1])).astype(np.float32),
                       rng.normal(size=(N_MOLS, T[2])).astype(np.float32)]
    t = lambda a: None if a is None else torch.from_numpy(a)  # noqa: E731
    model.train()
    batch = (bmg, None, None, t(X_d), [t(y) for y in targetss], [t(w) for w in weightss], [t(m) for m in lts],
             [t(m) for m in gts], None if constraints is None else [t(c) for c in constraints])
    loss = model.training_step(batch, 0)
    loss.backward()
    with torch.no_grad():
        model.eval()
        preds_eval = model(bmg, None, None, t(X_d), None if constraints is None else [t(c) for c in constraints])
    d = _graph_arrays(bmg, N_MOLS)
    d.update({"loss": loss.detach().numpy(), "batch_norm": np.int64(batch_norm)})
    if X_d is not None:
        d["X_d"] = X_d
    for level, name in enumerate(("mol", "atom", "bond")):
        if targetss[level] is None:
            continue
        d[f"Y.{name}"], d[f"w.{name}"] = targetss[level], weightss[level]
        d[f"preds_eval.{name}"] = preds_eval[level].numpy()
        if lts[level] is not None:
            d[f"lt.{name}"], d[f"gt.{name}"] = lts[level], gts[level]
    if constraints is not None:
        d["constraints.atom"], d["constraints.bond"] = constraints
    for k, v in state0.items():
        d["param." + k] = v
    for k, v in model.state_dict().items():
        if k.startswith("bns.") and ("running" in k or k.endswith("num_batches_tracked")):
            d["after." + k] = v.detach().numpy()
    for k, p in model.named_parameters():
        if p.grad is not None:
            d["grad." + k] = p.grad.numpy()
    return d


def _load_checkpoint(path: str):
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
    return torch.load(path, map_location="cpu", weights_only=False, pickle_module=pm)


def checkpoint_case(name: str) -> dict:
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data.collate import BatchMolAtomBondGraph
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MolAtomBondMPNN
    from chemprop.nn.ffn import ConstrainerFFN
    from chemprop.nn.message_passing import MABBondMessagePassing
    from chemprop.nn.transforms import UnscaleTransform

    from chemprop_b200.data.synthetic import make_molecules

    ck = _load_checkpoint(os.path.join(REFERENCE_ROOT, "tests", "data", "mol_atom_bond", "example_models", f"{name}.pt"))
    hp, sd = ck["hyper_parameters"], {k: v for k, v in ck["state_dict"].items() if not k.startswith("metricss.")}
    mph = hp["message_passing"]
    mp = MABBondMessagePassing(d_v=mph["d_v"], d_e=mph["d_e"], d_h=mph["d_h"], depth=mph["depth"])
    agg = ref_nn.NormAggregation(norm=hp["agg"]["norm"])
    def heads(hidden):
        """The checkpoint's predictors and constrainers, each MLP with `hidden(h)` hidden units (h: the trained width)."""
        mods, rec = {}, {}
        for level in ("mol", "atom", "bond"):
            ph = hp[f"{level}_predictor"]
            assert ph["n_layers"] == 1
            ot = UnscaleTransform(sd[f"{level}_predictor.output_transform.mean"][0].tolist(),
                                  sd[f"{level}_predictor.output_transform.scale"][0].tolist())
            mods[f"{level}_predictor"] = ph["cls"](n_tasks=ph["n_tasks"], input_dim=ph["input_dim"],
                                                  hidden_dim=hidden(ph["hidden_dim"]), n_layers=1, output_transform=ot)
            rec.update({f"hp.{level}.cls": np.str_(ph["cls"].__name__), f"hp.{level}.n_tasks": np.int64(ph["n_tasks"]),
                        f"hp.{level}.input_dim": np.int64(ph["input_dim"]),
                        f"hp.{level}.hidden_dim": np.int64(ph["hidden_dim"]), f"hp.{level}.n_layers": np.int64(1)})
        for level in ("atom", "bond"):
            ch = hp[f"{level}_constrainer"]
            if ch is not None:
                assert ch["n_layers"] == 1
                mods[f"{level}_constrainer"] = ConstrainerFFN(n_constraints=ch["n_constraints"], fp_dim=ch["fp_dim"],
                                                              hidden_dim=hidden(ch["hidden_dim"]), n_layers=1)
                rec.update({f"hp.{level}_constrainer.n_constraints": np.int64(ch["n_constraints"]),
                            f"hp.{level}_constrainer.fp_dim": np.int64(ch["fp_dim"]),
                            f"hp.{level}_constrainer.hidden_dim": np.int64(ch["hidden_dim"]),
                            f"hp.{level}_constrainer.n_layers": np.int64(1)})
        return mods, rec

    def load(model, state):
        res = model.load_state_dict(state, strict=False)
        # the only keys the checkpoint lacks are torchmetrics states (total_loss, num_samples) and the metrics lists
        assert all(k.startswith("metricss.") or k.endswith(("total_loss", "num_samples")) for k in res.missing_keys), res
        assert not res.unexpected_keys, res

    mods, rec = heads(lambda h: h)
    model = MolAtomBondMPNN(mp, agg, batch_norm=bool(hp["batch_norm"]), **mods)
    load(model, sd)
    # the same model with every head MLP cut to its first HIDDEN_KEPT hidden units
    cut = {}
    for k, v in sd.items():
        if k.startswith("message_passing."):
            cut[k] = v
        elif k.endswith(".ffn.0.0.weight") or k.endswith(".ffn.0.0.bias"):
            cut[k] = v[:HIDDEN_KEPT].clone()
        elif k.endswith(".ffn.1.2.weight"):
            cut[k] = v[:, :HIDDEN_KEPT].clone()
        else:
            cut[k] = v
    small = MolAtomBondMPNN(mp, agg, batch_norm=bool(hp["batch_norm"]), **heads(lambda h: HIDDEN_KEPT)[0])
    load(small, cut)
    n = N_CKPT_MOLS
    bmg = BatchMolAtomBondGraph([RefMG(*m) for m in make_molecules(n, seed=331, mean_atoms=9, std_atoms=3, min_atoms=2)])
    rng = np.random.default_rng(331)
    constraints = None
    if "atom_constrainer" in mods:
        constraints = []
        for level in ("atom", "bond"):             # one column per task, NaN where the task is not constrained
            c = rng.normal(size=(n, hp[f"{level}_predictor"]["n_tasks"])).astype(np.float32)
            c[:, hp[f"{level}_constrainer"]["n_constraints"]:] = np.nan
            constraints.append(torch.from_numpy(c))
    small.eval()
    with torch.no_grad():
        preds = small(bmg, constraints=constraints)
        H_v, H_e = small.message_passing(bmg)
        H_g = small.agg(H_v, bmg.batch)
    d = _graph_arrays(bmg, n)
    d.update({"H_v": H_v.numpy(), "H_e": H_e.numpy(), "H_g": H_g.numpy(), "hp.norm": np.float64(hp["agg"]["norm"]),
              "hp.batch_norm": np.int64(bool(hp["batch_norm"])), "hp.d_h": np.int64(mph["d_h"]),
              "hp.hidden_kept": np.int64(HIDDEN_KEPT)}, **rec)
    for level, p in zip(("mol", "atom", "bond"), preds):
        d[f"preds_eval.{level}"] = p.numpy()
    if constraints is not None:
        d["constraints.atom"], d["constraints.bond"] = constraints[0].numpy(), constraints[1].numpy()
    for k, v in sd.items():
        d["shape." + k] = np.asarray(v.shape, dtype=np.int64)
        if not k.startswith("message_passing."):
            d["param." + k] = cut[k].detach().numpy()
    return d


def main():
    torch.set_num_threads(1)  # deterministic summation order
    for case, seed in TRAIN_CASES.items():
        d = training_case(case, seed)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mab_model_{case}.npz"), **d)
        print(f"fixture_mab_model_{case}: loss={float(d['loss']):.6f}")
    for name in CKPT_CASES:
        d = checkpoint_case(name)
        np.savez_compressed(os.path.join(GOLDEN_DIR, f"fixture_mab_ckpt_{name}.npz"), **d)
        print(f"fixture_mab_ckpt_{name}: preds " + " ".join(str(d[f'preds_eval.{lv}'].shape) for lv in ("mol", "atom", "bond")))


if __name__ == "__main__":
    main()
