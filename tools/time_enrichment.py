"""GPU timing of count-data regression (csrc/head.cu, csrc/row_head.cu).

  1. each kernel alone at b = 10 000, 100 000 and 1 000 000, CUDA events over many launches: dmpnn_enrichment_loss (sqrt
     method, loss and gradient), dmpnn_pred_transform / _bwd kind 7 (Softplus) and dmpnn_pinball_loss_rows (T = 1), each
     next to the reference's torch op sequence for the same result on the same GPU (NLogProbEnrichment's get_zstats, clamp,
     erf and log with its masked reduction and autograd; nn.Softplus forward and backward; PointQuantileLoss's where);
  2. the C2-sized training step (tools/time_head.py: 10 000 ~25-atom molecules, BondMessagePassing h = 300 depth 3 bf16,
     MeanAggregation, batch norm, FFN of width 300) as ONE CUDA graph with the DEL head (Softplus output,
     NLogProbEnrichment on two count columns) next to the MSE head with one task.

The card name and power limit are read in the same run.  Prints one JSON line; `--out DIR` also writes it to
DIR/time_enrichment.json.  Usage: python tools/time_enrichment.py [--steps K] [--out DIR]"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.time_head import card, per_call_us  # noqa: E402

SIZES = (10_000, 100_000, 1_000_000)


def _counts(b: int, g) -> torch.Tensor:
    Y = torch.poisson(torch.full((b, 2), 4.0, device="cuda"), generator=g)
    Y[torch.rand(b, 2, device="cuda", generator=g) < 0.05] = float("nan")
    return Y


def _torch_enrichment(R, Y, w, tw, d):
    """The reference's op sequence (metrics.py:78-123, 656-689) on the device, loss and dLoss/dR."""
    m = Y.isfinite()
    k = Y.nan_to_num(0.0)
    Rl = R.detach().requires_grad_(True)
    Rd = Rl.squeeze() / d
    z = 2 * (torch.sqrt(k[:, 0] + 3 / 8.0) - torch.sqrt((k[:, 1] + 3 / 8.0) * Rd)) / torch.sqrt(1 + Rd)
    z = torch.clamp(z, -5.0, 5.0).abs()
    L = -torch.log(1 - torch.erf(z / math.sqrt(2))).unsqueeze(1)
    loss = (L * w.view(-1, 1) * tw * m).sum() / m.sum()
    (g,) = torch.autograd.grad(loss, Rl)
    return loss, g


def time_kernels() -> dict:
    from chemprop_b200 import _lib
    from chemprop_b200 import engine as K

    out = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for b in SIZES:
        R = torch.rand(b, 1, device="cuda", generator=g) * 2 + 0.05
        Y = _counts(b, g)
        w = torch.rand(b, device="cuda", generator=g) + 0.5
        tw = torch.tensor([1.0, 0.5], device="cuda")
        d = float(torch.nansum(Y[:, 1]) / torch.nansum(Y[:, 0]))
        loss, dR = torch.empty(1, device="cuda"), torch.empty_like(R)
        out[f"enrichment_loss_b{b}_us"] = per_call_us(
            lambda: K.enrichment_loss(R, Y, w, tw, d, _lib.ENRICH_METHODS["sqrt"], 1.0, 5.0, loss, dR))
        out[f"torch_enrichment_b{b}_us"] = per_call_us(lambda: _torch_enrichment(R, Y, w, tw.view(1, 2), d), calls=50)
        X = torch.randn(b, 1, device="cuda", generator=g)
        o, dX = torch.empty_like(X), torch.empty_like(X)
        out[f"softplus_fwd_bwd_b{b}_us"] = per_call_us(
            lambda: (K.pred_transform(X, _lib.PRED_SOFTPLUS, 1, None, None, o),
                     K.pred_transform_bwd(X, R, _lib.PRED_SOFTPLUS, 1, None, dX)))
        sp = torch.nn.Softplus()

        def torch_softplus():
            x = X.detach().requires_grad_(True)
            torch.autograd.grad(sp(x), x, R)

        out[f"torch_softplus_fwd_bwd_b{b}_us"] = per_call_us(torch_softplus, calls=50)
        Yp = torch.randn(b, 1, device="cuda", generator=g)
        out[f"pinball_loss_rows_b{b}_us"] = per_call_us(lambda: K.pinball_loss_rows(X, Yp, w, None, 0.3, loss, dX))

        def torch_pinball():
            x = X.detach().requires_grad_(True)
            diff = Yp - x
            L = torch.where(diff > 0, 0.3 * diff, 0.7 * (-diff)) * w.view(-1, 1)
            torch.autograd.grad(L.sum() / b, x)

        out[f"torch_pinball_b{b}_us"] = per_call_us(torch_pinball, calls=50)
    return out


def time_steps(steps: int) -> dict:
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedMolGraphDataset, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    n = 10_000
    ds = PackedMolGraphDataset.from_molgraphs(make_molecules(n, seed=1, mean_atoms=25.0)).to("cuda")
    bmg = ds.batch(ds.packed_order(np.arange(n, dtype=np.int64)))
    rng = np.random.default_rng(0)
    counts = rng.poisson(4.0, size=(n, 2)).astype(np.float32)
    n1, n2 = int(counts[:, 0].sum()), int(counts[:, 1].sum())
    heads = {
        "mse_T1": (lambda: N.EngineRegressionFFN(n_tasks=1), rng.normal(size=(n, 1))),
        "del_enrichment": (lambda: N.EngineRegressionFFN(criterion=N.EngineNLogProbEnrichment(n1=n1, n2=n2),
                                                         output_transform=torch.nn.Softplus()), counts),
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
        raise SystemExit("time_enrichment.py measures on the GPU; no CUDA device found")
    res = {"card": card()}
    res.update(time_kernels())
    res.update(time_steps(args.steps))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_enrichment.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
