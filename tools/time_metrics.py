"""Time of the device metrics on the GPU (CUDA events, medians of repeated timed loops), with the card name and power limit
read in the same run:

  * `compute()` of AUROC + AUPRC (dmpnn_rank_curve, one sort each) at 1 M and 10 M (score, label) pairs, scores quantised
    to 256 levels, and sklearn's roc_auc_score + precision_recall_curve / auc on the same pairs on this host's CPU;
  * `update` per batch of 10 000 x 12 for every registry metric;
  * `EngineMPNN.evaluate(stage="val")` on a C2-shaped held-out set: bf16 BondMessagePassing d_h = 300, depth 3, 12-task
    binary head, 10 batches of 10 000 molecules (100 000 molecules), metrics roc, prc, accuracy, f1, binary-mcc.

    python tools/time_metrics.py [--reps 5] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.time_mab import card  # noqa: E402
from tools.time_mab_head import median_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_metrics.py measures on the GPU; no CUDA device found")

    import chemprop_b200.nn as N
    from chemprop_b200.data import BatchMolGraph, TrainingBatch, make_molecules
    from chemprop_b200.nn.metrics import EngineMetricRegistry

    res = {"card": card()}
    g = np.random.default_rng(0)

    # ---- ranking compute at 1 M and 10 M pairs ----
    for n in (1_000_000, 10_000_000):
        s = (np.floor(g.random(n) * 256) / 256).astype(np.float32)
        y = (g.random(n) < 0.3).astype(np.float32)
        P, Y = torch.from_numpy(s).cuda().view(-1, 1), torch.from_numpy(y).cuda().view(-1, 1)
        M = torch.ones_like(Y, dtype=torch.bool)
        roc, prc = EngineMetricRegistry["roc"](), EngineMetricRegistry["prc"]()
        roc.update(P, Y, M)
        prc.update(P, Y, M)

        def both():
            roc.compute()
            prc.compute()

        ms = median_ms(both, 3, args.reps)
        entry = {"engine_roc_prc_compute_ms": ms}
        try:
            from sklearn.metrics import auc, precision_recall_curve, roc_auc_score

            t0 = time.perf_counter()
            roc_auc_score(y, s)
            p_, r_, _ = precision_recall_curve(y, s)
            auc(r_, p_)
            entry["sklearn_cpu_ms"] = (time.perf_counter() - t0) * 1e3
        except ImportError:
            entry["sklearn_cpu_ms"] = "not measured (sklearn not installed)"
        res[f"rank_{n}"] = entry
        print(n, entry, flush=True)

    # ---- update per batch ----
    B, T = 10_000, 12
    P = torch.rand(B, T, device="cuda")
    Y = (torch.rand(B, T, device="cuda") < 0.4).float()
    M = torch.rand(B, T, device="cuda") > 0.1
    w = torch.ones(B, 1, device="cuda")
    Pm = torch.stack([1 - P, P], -1)
    upd = {}
    for name, cls in EngineMetricRegistry.items():
        m = cls()
        args_ = (Pm if name == "multiclass-mcc" else P, Y, M, w)
        upd[name] = median_ms(lambda: m.update(*args_), 20, args.reps)
        if name in ("roc", "prc"):
            m.reset()
    res["update_ms_per_10000x12"] = upd
    print(upd, flush=True)

    # ---- evaluate over a C2-shaped held-out set ----
    torch.manual_seed(0)
    model = N.EngineMPNN(N.BondMessagePassing(d_h=300, depth=3, precision="bf16"),
                         predictor=N.EngineBinaryClassificationFFN(n_tasks=T, input_dim=300)).cuda()
    mgs = make_molecules(100_000, seed=1)
    batches = []
    for lo in range(0, len(mgs), 10_000):
        bmg = BatchMolGraph(mgs[lo:lo + 10_000])
        bmg.to("cuda")
        Yb = (torch.rand(10_000, T, device="cuda") < 0.3).float()
        Yb[torch.rand(10_000, T, device="cuda") < 0.1] = float("nan")
        batches.append(TrainingBatch(bmg, None, None, Yb, torch.ones(10_000, 1, device="cuda"), None, None))
    metrics = [EngineMetricRegistry[k]() for k in ("roc", "prc", "accuracy", "f1", "binary-mcc")]
    model.evaluate(batches, metrics)
    torch.cuda.synchronize()
    times = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        model.evaluate(batches, metrics)          # ends in its one host sync
        times.append((time.perf_counter() - t0) * 1e3)
    res["evaluate_val_100k_mols_ms"] = float(np.median(times))

    def fwd_only():
        model.eval()
        with torch.no_grad():
            for b in batches:
                model(b.bmg)
        model.train()

    res["forward_only_100k_mols_ms"] = median_ms(fwd_only, 1, args.reps)
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_metrics.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
