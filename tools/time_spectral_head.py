"""GPU timing of the spectral head (csrc/head.cu) at b = 10 000, T = 1 801, d_h = 300.

  1. each kernel alone, CUDA events over many launches: dmpnn_spectral_transform and dmpnn_spectral_transform_bwd (softplus),
     dmpnn_sid_loss and dmpnn_wasserstein_loss (with a threshold), each next to its algorithmic bytes (every b x T f32 operand
     read or written once: 72 MB each) and the bandwidth that implies;
  2. the C2-sized training step (tools/time_head.py: 10 000 ~25-atom molecules, BondMessagePassing h = 300 depth 3 bf16,
     MeanAggregation, batch norm, FFN of width 300) as ONE CUDA graph with EngineSpectralFFN (T = 1 801, SID) next to the
     regression head (T = 12).

The card name and power limit are read in the same run.  Prints one JSON line; `--out DIR` also writes it to
DIR/time_spectral_head.json.  Usage: python tools/time_spectral_head.py [--steps K] [--out DIR]"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.time_head import card, per_call_us  # noqa: E402

B, T = 10_000, 1801


def time_kernels() -> dict:
    from chemprop_b200 import _lib
    from chemprop_b200 import engine as K

    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.randn(B, T, device="cuda", generator=g) * 2
    P, dP, dX = torch.empty_like(X), torch.empty_like(X), torch.empty_like(X)
    K.spectral_transform(X, _lib.SPEC_SOFTPLUS, P)
    dP.copy_(torch.randn(B, T, device="cuda", generator=g) * 1e-7)      # the mirror's dOut: a gradient-sized input
    Y = torch.rand(B, T, device="cuda", generator=g) + 0.05
    Y = Y / Y.sum(1, keepdim=True)
    Y[torch.rand(B, T, device="cuda", generator=g) < 0.1] = float("nan")
    w = torch.rand(B, device="cuda", generator=g) + 0.5
    tw = torch.rand(T, device="cuda", generator=g) + 0.5
    loss = torch.empty(1, device="cuda")
    thr = float(P.median())
    mb = B * T * 4 / 1e6
    cases = {   # name -> (call, operands read or written once: X / P / Y / dOut / dP / dX)
        "spectral_transform": (lambda: K.spectral_transform(X, _lib.SPEC_SOFTPLUS, P), 2),
        "spectral_transform_bwd": (lambda: K.spectral_transform_bwd(X, dP, _lib.SPEC_SOFTPLUS, dX), 3),
        "sid_loss": (lambda: K.sid_loss(P, Y, w, tw, thr, loss, dP), 3),
        "wasserstein_loss": (lambda: K.wasserstein_loss(P, Y, w, tw, thr, loss, dP), 3),
    }
    out = {}
    for name, (fn, n_ops) in cases.items():
        us = per_call_us(fn)
        out[f"{name}_B{B}_T{T}_us"] = us
        out[f"{name}_algorithmic_MB"] = n_ops * mb
        out[f"{name}_algorithmic_TBps"] = n_ops * mb / us             # MB / us = TB / s
    return out


def time_steps(steps: int) -> dict:
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedMolGraphDataset, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    n = B
    ds = PackedMolGraphDataset.from_molgraphs(make_molecules(n, seed=1, mean_atoms=25.0)).to("cuda")
    bmg = ds.batch(ds.packed_order(np.arange(n, dtype=np.int64)))
    rng = np.random.default_rng(0)
    spec = rng.uniform(0.05, 1.0, size=(n, T))
    spec = spec / spec.sum(1, keepdims=True)
    spec[rng.random(spec.shape) < 0.1] = np.nan
    heads = {
        "regression_T12": (lambda: N.EngineRegressionFFN(n_tasks=12), rng.normal(size=(n, 12))),
        f"spectral_sid_T{T}": (lambda: N.EngineSpectralFFN(n_tasks=T, threshold=1e-4), spec),
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
        raise SystemExit("time_spectral_head.py measures on the GPU; no CUDA device found")
    res = {"card": card()}
    res.update(time_kernels())
    res.update(time_steps(args.steps))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_spectral_head.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
