"""GPU timing of the uncertainty heads (csrc/head.cu).

  1. each kernel alone, CUDA events over many launches, at B = 10 000: dmpnn_pred_transform and dmpnn_pred_transform_bwd
     for MVE / evidential / quantile (T = 12) and Dirichlet (T = 1, C = 10), dmpnn_mve_loss / dmpnn_evidential_loss /
     dmpnn_quantile_loss (T = 12), dmpnn_dirichlet_loss (T = 1, C = 10);
  2. the C2-sized training step (tools/time_head.py: 10 000 ~25-atom molecules, BondMessagePassing h = 300 depth 3 bf16,
     MeanAggregation, batch norm, FFN of width 300) as ONE CUDA graph with each uncertainty head, next to the regression head.

The card name and power limit are read in the same run.  Prints one JSON line; `--out DIR` also writes it to
DIR/time_uq_head.json.  Usage: python tools/time_uq_head.py [--steps K] [--out DIR]"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.time_head import card, per_call_us  # noqa: E402


def time_kernels() -> dict:
    from chemprop_b200 import _lib
    from chemprop_b200 import engine as K

    g = torch.Generator(device="cuda").manual_seed(0)
    B = 10_000
    out = {}
    w = torch.rand(B, device="cuda", generator=g) + 0.5
    loss = torch.empty(1, device="cuda")
    for name, kind, T, u in (("mve", _lib.PRED_MVE, 12, 2), ("evidential", _lib.PRED_EVIDENTIAL, 12, 4),
                             ("quantile", _lib.PRED_QUANTILE, 12, 2), ("dirichlet", _lib.PRED_DIRICHLET, 1, 10)):
        X = torch.randn(B, T * u, device="cuda", generator=g) * 3
        P, dP, dX = torch.empty_like(X), torch.empty_like(X), torch.empty_like(X)
        tw = torch.rand(T, device="cuda", generator=g) + 0.5
        if name == "dirichlet":
            Y = torch.randint(0, u, (B, T), device="cuda", generator=g).float()
        else:
            Y = torch.randn(B, T, device="cuda", generator=g)
        Y[torch.rand(B, T, device="cuda", generator=g) < 0.2] = float("nan")
        K.pred_transform(X, kind, u, None, None, P)
        tag = f"B10000_T{T}" + (f"_C{u}" if name == "dirichlet" else "")
        out[f"pred_transform_{name}_{tag}_us"] = per_call_us(lambda: K.pred_transform(X, kind, u, None, None, P))
        out[f"pred_transform_bwd_{name}_{tag}_us"] = per_call_us(lambda: K.pred_transform_bwd(X, dP, kind, u, None, dX))
        if name == "mve":
            fn = lambda: K.mve_loss(P, Y, w, tw, loss, dP)  # noqa: E731
        elif name == "evidential":
            fn = lambda: K.evidential_loss(P, Y, w, tw, 0.2, 1e-8, loss, dP)  # noqa: E731
        elif name == "quantile":
            fn = lambda: K.quantile_loss(P, Y, w, tw, 0.1, loss, dP)  # noqa: E731
        else:
            fn = lambda: K.dirichlet_loss(P, Y, w, tw, u, 0.2, loss, dP)  # noqa: E731
        out[f"{name}_loss_{tag}_us"] = per_call_us(fn)
    return out


def time_steps(steps: int) -> dict:
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedMolGraphDataset, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    n = 10_000
    ds = PackedMolGraphDataset.from_molgraphs(make_molecules(n, seed=1, mean_atoms=25.0)).to("cuda")
    bmg = ds.batch(ds.packed_order(np.arange(n, dtype=np.int64)))
    rng = np.random.default_rng(0)
    reg = rng.normal(size=(n, 12))
    heads = {
        "regression_T12": (lambda: N.EngineRegressionFFN(n_tasks=12), reg),
        "mve_T12": (lambda: N.EngineMveFFN(n_tasks=12), reg),
        "evidential_T12": (lambda: N.EngineEvidentialFFN(n_tasks=12), reg),
        "quantile_T12": (lambda: N.EngineQuantileFFN(n_tasks=12), reg),
        "binary_dirichlet_T12": (lambda: N.EngineBinaryDirichletFFN(n_tasks=12), rng.integers(0, 2, size=(n, 12))),
        "multiclass_dirichlet_T1_C10": (lambda: N.EngineMulticlassDirichletFFN(n_classes=10),
                                        rng.integers(0, 10, size=(n, 1))),
    }
    out = {}
    for name, (make_head, y) in heads.items():
        torch.manual_seed(0)
        model = N.EngineMPNN(N.BondMessagePassing(precision="bf16"), N.MeanAggregation(), make_head(),
                             batch_norm=True).cuda().train()
        Y = torch.from_numpy(y.astype(np.float32)).cuda()
        for p in model.parameters():
            p.grad = torch.zeros_like(p)

        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            b._layout = None                     # the device layout build is part of every step (as bench.py)
            loss = model.training_loss(b, Y)
            loss.backward()
            return loss

        step = CudaGraphStep(fn)
        for _ in range(5):
            step(bmg)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(3):
            e0.record()
            for _ in range(steps):
                loss = step(bmg)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) / steps)
        assert step.captures == 1 and bool(torch.isfinite(loss))
        out[f"step_graph_{name}_ms"] = float(np.median(ts))
        del step, model
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_uq_head.py measures on the GPU; no CUDA device found")
    res = {"card": card()}
    res.update(time_kernels())
    res.update(time_steps(args.steps))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_uq_head.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
