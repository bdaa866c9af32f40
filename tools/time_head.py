"""GPU timing of the classification heads (csrc/head.cu).

  1. the three kernels alone, CUDA events over many launches: dmpnn_bce_loss at B = 10 000, T = 12 (binary), dmpnn_ce_loss at
     B = 10 000, T = 1, C = 10 (multiclass), dmpnn_class_probs for both shapes, dmpnn_mse_loss at B = 10 000, T = 12 beside them;
  2. the C2-sized training step (10 000 ~25-atom molecules, BondMessagePassing h = 300 depth 3 bf16, MeanAggregation, batch
     norm, 1-hidden-layer FFN of width 300) as ONE CUDA graph, with the regression head (12 tasks), the binary head (12 tasks)
     and the multiclass head (1 task, 10 classes).

The card name and power limit are read in the same run.  Prints one JSON line; `--out DIR` also writes it to DIR/time_head.json.
Usage: python tools/time_head.py [--steps K] [--out DIR]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card() -> dict:
    out = {"name": torch.cuda.get_device_name(), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        out["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        out["power_limit_w"] = f"unavailable ({e})"
    return out


def per_call_us(fn, calls: int = 200, windows: int = 5) -> float:
    """Median over `windows` of (event time of `calls` back-to-back launches) / calls."""
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(windows):
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / calls)
    return float(np.median(ts))


def time_kernels() -> dict:
    from chemprop_b200 import engine as K

    g = torch.Generator(device="cuda").manual_seed(0)
    B = 10_000
    out = {}
    P = torch.randn(B, 12, device="cuda", generator=g)
    Y = (torch.rand(B, 12, device="cuda", generator=g) < 0.5).float()
    Y[torch.rand(B, 12, device="cuda", generator=g) < 0.2] = float("nan")
    w, tw = torch.rand(B, device="cuda", generator=g) + 0.5, torch.rand(12, device="cuda", generator=g) + 0.5
    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    out["bce_loss_B10000_T12_us"] = per_call_us(lambda: K.bce_loss(P, Y, w, tw, loss, dP))
    out["mse_loss_B10000_T12_us"] = per_call_us(lambda: K.mse_loss(P, Y, w, tw, loss, dP))
    out["sigmoid_probs_B10000_T12_us"] = per_call_us(lambda: K.class_probs(P, 1, False, dP))
    P10 = torch.randn(B, 10, device="cuda", generator=g)
    Y1 = torch.randint(0, 10, (B, 1), device="cuda", generator=g).float()
    dP10 = torch.empty_like(P10)
    out["ce_loss_B10000_T1_C10_us"] = per_call_us(lambda: K.ce_loss(P10, Y1, w, None, 10, loss, dP10))
    out["softmax_probs_B10000_T1_C10_us"] = per_call_us(lambda: K.class_probs(P10, 10, True, dP10))
    return out


def time_steps(steps: int) -> dict:
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedMolGraphDataset, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    n = 10_000
    ds = PackedMolGraphDataset.from_molgraphs(make_molecules(n, seed=1, mean_atoms=25.0)).to("cuda")
    bmg = ds.batch(ds.packed_order(np.arange(n, dtype=np.int64)))
    rng = np.random.default_rng(0)
    heads = {
        "regression_T12": (lambda: N.EngineRegressionFFN(n_tasks=12), rng.normal(size=(n, 12))),
        "binary_T12": (lambda: N.EngineBinaryClassificationFFN(n_tasks=12), rng.integers(0, 2, size=(n, 12))),
        "multiclass_T1_C10": (lambda: N.EngineMulticlassClassificationFFN(n_classes=10), rng.integers(0, 10, size=(n, 1))),
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
        raise SystemExit("time_head.py measures on the GPU; no CUDA device found")
    res = {"card": card()}
    res.update(time_kernels())
    res.update(time_steps(args.steps))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_head.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
