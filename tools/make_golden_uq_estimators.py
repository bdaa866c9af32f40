"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/fixture_uq_estimators.npz by running the UNMODIFIED reference
estimators (chemprop/uncertainty/estimator.py, chemprop v2.3.1, imported through oracle/ref_shim.py); the output is
committed, the reference does not travel with the tests.

    python -m tools.make_golden_uq_estimators

The estimators are called with fixed model outputs: a trainer stand-in whose `predict(model, dataloader)` returns the
per-batch predictions recorded for that model (and, for `dropout`, for that pass), so the fixture pins what each estimator
does with the predictions -- which outputs it splits, stacks, averages and how, shapes, dtypes, the leading model
dimension and the population variances -- for `MPNN` (MulticomponentMPNN is an MPNN to the estimators) and for
`MolAtomBondMPNN` (mol / atom / bond levels, the atom level absent in one case).  `multiclass-dirichlet` replaces
`predictor.forward`, so its stand-in model calls that forward on the recorded concentrations.

Recorded per case `<estimator>.<family>`: `in.m<i>.b<j>[.l<level>][.k<pass>]` (the per-batch predictions) and
`out.<preds|uncs>[.l<level>]` (the reference's outputs; absent when None)."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fixture_uq_estimators.npz")
N_MODELS, N_PASSES, BATCHES = 3, 4, (5, 3)                 # molecules per batch
LEVEL_ROWS = ((5, 3), (17, 9), (22, 14))                   # rows per batch of the mol / atom / bond levels
T, C = 2, 3

# estimator -> the last dimensions of one model output (after rows)
KINDS = {"none": (T,), "mve": (T, 2), "ensemble": (T,), "classification": (T, C), "evidential-total": (T, 4),
         "evidential-epistemic": (T, 4), "evidential-aleatoric": (T, 4), "dropout": (T,),
         "classification-dirichlet": (T, 2), "multiclass-dirichlet": (T, C), "quantile-regression": (T, 2)}


def _output(rng, kind: str, rows: int) -> np.ndarray:
    shape = (rows, *KINDS[kind])
    x = rng.normal(size=shape).astype(np.float32)
    if kind.startswith("evidential") or kind == "multiclass-dirichlet":
        x = (np.abs(x) + 1.5).astype(np.float32)               # v, alpha > 1, beta > 0 / concentrations > 1
    if kind == "multiclass-dirichlet":
        return x
    if kind == "mve":
        x[..., 1] = np.abs(x[..., 1]) + 0.1
    return x


def main():
    import_reference()
    from chemprop.models import MPNN
    from chemprop.uncertainty.estimator import UncertaintyEstimatorRegistry as Reg

    rng = np.random.default_rng(2024)
    out = {}

    class _Predictor(torch.nn.Module):
        def __init__(self, alpha_per_batch):
            super().__init__()
            self.alpha = alpha_per_batch
            self.calls = 0

        def train_step(self, Z):
            a = self.alpha[self.calls % len(self.alpha)]
            self.calls += 1
            return a

    def stand_in_model(mab: bool):
        if mab:
            m = torch.nn.Module()
        else:
            m = MPNN.__new__(MPNN)
            torch.nn.Module.__init__(m)
        m.predict_step = lambda *a, **k: None                   # DropoutEstimator wraps it; the trainer never calls it
        return m

    class Trainer:
        """`predict(model, dataloader)`: the recorded predictions of `model`, pass after pass."""

        def __init__(self, table):
            self.table, self.calls = table, {}

        def predict(self, model, dataloader, **_):
            k = self.calls.get(id(model), 0)
            self.calls[id(model)] = k + 1
            if hasattr(model, "predictor"):                     # multiclass-dirichlet: through the replaced forward
                return [model.predictor.forward(None) for _ in BATCHES]
            return self.table[id(model)][k]

    for kind in KINDS:
        for family in ("mpnn", "mab"):
            mab = family == "mab"
            n_models = 1 if kind == "dropout" and not mab else (2 if kind == "dropout" else N_MODELS)
            passes = N_PASSES if kind == "dropout" else 1
            levels = (0, 2) if mab else (0,)                    # the MAB case has no atom level
            models, table = [], {}
            case = f"{kind}.{family}"
            for i in range(n_models):
                m = stand_in_model(mab)
                recs = []
                for k in range(passes):
                    per_batch = []
                    for j in range(len(BATCHES)):
                        if mab:
                            item = []
                            for lv in range(3):
                                if lv in levels:
                                    x = _output(rng, kind, LEVEL_ROWS[lv][j])
                                    out[f"{case}.in.m{i}.b{j}.l{lv}" + (f".k{k}" if passes > 1 else "")] = x
                                    item.append(torch.from_numpy(x))
                                else:
                                    item.append(None)
                            per_batch.append(tuple(item))
                        else:
                            x = _output(rng, kind, BATCHES[j])
                            out[f"{case}.in.m{i}.b{j}" + (f".k{k}" if passes > 1 else "")] = x
                            per_batch.append(torch.from_numpy(x))
                    recs.append(per_batch)
                if kind == "multiclass-dirichlet":
                    if mab:
                        continue                                # the reference reads model.predictor: MPNN only
                    m.predictor = _Predictor([r for r in recs[0]])
                table[id(m)] = recs
                models.append(m)
            if not models:
                continue
            est = Reg[kind](ensemble_size=N_PASSES, dropout=0.3) if kind == "dropout" else Reg[kind]()
            preds, uncs = est(None, models, Trainer(table))
            for name, val in (("preds", preds), ("uncs", uncs)):
                vals = val if mab else [val]
                for lv, v in enumerate(vals or [None] * 3):
                    if v is not None:
                        out[f"{case}.out.{name}" + (f".l{lv}" if mab else "")] = v.detach().numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
