"""TEST INFRASTRUCTURE ONLY.  Generates tests/golden/fixture_metrics.npz by running the UNMODIFIED reference's own metric
classes (chemprop v2.3.1, chemprop/nn/metrics.py, imported through oracle/ref_shim.py); the output is committed, the
reference does not travel with the tests.

    python -m tools.make_golden_metrics

Recorded, each over three `update`s then `compute`, with masks, per-row weights and task weights:
  - mse, mae, rmse, bounded-mse, bounded-mae, bounded-rmse (with lt / gt masks);
  - binary-mcc and multiclass-mcc (C = 3), once on probabilities and once on logits (the reference's sigmoid / softmax
    switch);
  - the criterion-as-metric path: for the criteria mse, mae, rmse, bounded-mse, bounded-mae, bounded-rmse, bce and sid,
    the batches, the per-batch values of `forward` (the reference's validation-loss logging), the batch mask counts and
    the epoch value.
The torchmetrics-derived metrics (r2, roc, prc, accuracy, f1) are not here: torchmetrics is not installed, and
tests/test_metrics_host.py pins the restatement of those against sklearn."""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.ref_shim import import_reference  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fixture_metrics.npz")
SIZES = (17, 9, 23)
T = 3


def _reference_metrics():
    import_reference()
    import torchmetrics.utilities.data as tud

    tud.dim_zero_cat = torch.cat
    import chemprop.nn.metrics as M

    M.dim_zero_cat = torch.cat           # bound at the reference module's import
    return M


def _update(r, b, kind, logits=False):
    if kind == "reg":
        P = r.normal(size=(b, T))
        Y = r.normal(size=(b, T))
    elif kind == "bin":
        P = r.normal(size=(b, T)) * 2 if logits else r.random((b, T))
        Y = (r.random((b, T)) < 0.4).astype(float)
    elif kind == "mc":
        x = r.normal(size=(b, T, 3)) * 2
        P = x if logits else np.exp(x) / np.exp(x).sum(-1, keepdims=True)
        Y = r.integers(0, 3, (b, T)).astype(float)
    else:                                 # spectra
        P = r.random((b, T)) + 0.05
        P /= P.sum(1, keepdims=True)
        Y = r.random((b, T)) + 0.05
        Y /= Y.sum(1, keepdims=True)
    return dict(preds=P.astype(np.float32), targets=Y.astype(np.float32), mask=r.random((b, T)) > 0.25,
                weights=(r.random(b) + 0.5).astype(np.float32), lt_mask=r.random((b, T)) < 0.3,
                gt_mask=r.random((b, T)) < 0.3)


def _t(u):
    return {k: torch.from_numpy(v) for k, v in u.items()}


def main():
    M = _reference_metrics()
    r = np.random.default_rng(2026)
    out = {}
    metric_cls = {"mse": M.MSE, "mae": M.MAE, "rmse": M.RMSE, "bounded-mse": M.BoundedMSE, "bounded-mae": M.BoundedMAE,
                  "bounded-rmse": M.BoundedRMSE, "binary-mcc": M.BinaryMCCMetric, "multiclass-mcc": M.MulticlassMCCMetric}
    for name, cls in metric_cls.items():
        tw = (r.random(T) + 0.5).astype(np.float32)
        out[f"{name}.task_weights"] = tw
        out[f"{name}.n"] = np.int64(len(SIZES))
        kind = "mc" if name == "multiclass-mcc" else "bin" if name == "binary-mcc" else "reg"
        for variant in ("prob", "logit") if kind != "reg" else ("plain",):
            m = cls(task_weights=tw)
            for i, b in enumerate(SIZES):
                u = _update(r, b, kind, logits=variant == "logit")
                tu = _t(u)
                if kind == "reg":
                    m.update(tu["preds"], tu["targets"], tu["mask"], tu["weights"].view(-1, 1), tu["lt_mask"], tu["gt_mask"])
                else:
                    m.update(tu["preds"], tu["targets"], tu["mask"], tu["weights"].view(-1, 1))
                    u = {k: u[k] for k in ("preds", "targets", "mask", "weights")}
                if not name.startswith("bounded"):
                    u = {k: v for k, v in u.items() if k not in ("lt_mask", "gt_mask")}
                for k, v in u.items():
                    out[f"{name}.{variant}.{i}.{k}"] = v
            out[f"{name}.{variant}.value"] = np.float64(m.compute())
    out["names"] = np.array(list(metric_cls))

    crit_cls = {"mse": M.MSE, "mae": M.MAE, "rmse": M.RMSE, "bounded-mse": M.BoundedMSE, "bounded-mae": M.BoundedMAE,
                "bounded-rmse": M.BoundedRMSE, "bce": M.BCELoss, "sid": M.SID}
    for name, cls in crit_cls.items():
        tw = (r.random(T) + 0.5).astype(np.float32)
        c = cls(task_weights=tw)
        out[f"crit.{name}.task_weights"] = tw
        vals, counts = [], []
        kind = "bin" if name == "bce" else "spec" if name == "sid" else "reg"
        for i, b in enumerate(SIZES):
            u = _update(r, b, kind, logits=True)
            for k, v in u.items():
                out[f"crit.{name}.{i}.{k}"] = v
            tu = _t(u)
            vals.append(float(c(tu["preds"], tu["targets"], tu["mask"], tu["weights"].view(-1, 1), tu["lt_mask"],
                                tu["gt_mask"])))
            counts.append(int(tu["mask"].sum()))
        out[f"crit.{name}.batch_values"] = np.array(vals, np.float32)
        out[f"crit.{name}.batch_counts"] = np.array(counts, np.int64)
        out[f"crit.{name}.value"] = np.float64(c.compute())
    out["criteria"] = np.array(list(crit_cls))
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays")


if __name__ == "__main__":
    main()
