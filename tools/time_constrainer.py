"""Time of ConstrainerFFN and of a constrained mol-atom-bond training step on the GPU (CUDA events, medians of repeated
timed loops), on a batch of C4's size (10 000 molecules of ~80 atoms), d_h = 300:

  * the constrainer forward + backward at atom level (V rows, fp width h, 2 constraint columns) and bond level (E/2 rows,
    fp width 2h, 1 column): the previous composition (torch MLP on cuBLAS, dmpnn_segment_sum / dmpnn_segment_bcast with
    torch elementwise ops and a host read of the constraint mask) against the engine MLP + dmpnn_constrain_fwd / _bwd;
  * the two kernels alone at both levels;
  * the training step of EngineMolAtomBondMPNN (bf16 MAB encoder, atom and bond regression heads, atom and bond
    constrainers) eagerly and replayed as one CUDA graph.
The card name, power limit and SM clocks are read in the same run.

    python tools/time_constrainer.py [--mols 10000] [--steps 20] [--reps 5] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tools.time_mab import card  # noqa: E402
from tools.time_mab_head import median_ms  # noqa: E402


def clocks() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        sm, mx = (float(x) for x in q.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": sm, "max_sm_clock_mhz": mx}
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        return {"sm_clock_mhz": f"unavailable ({e})"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import chemprop_b200.nn as N
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.graph import CudaGraphStep
    from chemprop_b200.nn.constrainer import ConstrainerFFN, build_mlp

    dev = "cuda"
    torch.manual_seed(0)
    h = 300
    bmg = BatchMolGraph(make_molecules(args.mols, seed=1, mean_atoms=80.0))
    bmg.to(dev)
    V, E, B = int(bmg.V.shape[0]), int(bmg.E.shape[0]), len(bmg)
    res = {"card": card(), "clocks_before": clocks(), "n_mols": B, "atoms": V, "directed_edges": E, "d_h": h}
    t = lambda fn: median_ms(fn, args.steps, args.reps)  # noqa: E731
    lay = engine.get_layout(bmg)

    levels = {"atom": (V, h, 2, bmg.batch, lay.mol_atom_ptr),
              "bond": (E // 2, 2 * h, 1, bmg.batch[bmg.edge_index[0, ::2]], lay.mol_row_ptr // 2)}
    con = {}
    for name, (R, d, n_c, batch, offsets) in levels.items():
        mod = ConstrainerFFN(n_constraints=n_c, fp_dim=d).to(dev)
        torch_ffn = build_mlp(d, n_c, 300, 1).to(dev)            # the previous MLP: nn.Linear on cuBLAS
        torch_ffn.load_state_dict(mod.ffn.state_dict())
        previous = types.SimpleNamespace(ffn=torch_ffn)
        fp = torch.randn(R, d, device=dev, requires_grad=True)
        preds = torch.randn(R, n_c, device=dev, requires_grad=True)
        cons = torch.randn(B, n_c, device=dev)
        G = torch.randn(R, n_c, device=dev)

        def old():
            (ConstrainerFFN._composed_forward(previous, fp, preds, batch, cons) * G).sum().backward()

        def new():
            (mod(fp, preds, batch, cons, offsets=offsets) * G).sum().backward()

        Kl = torch.randn(R, n_c, device=dev) * 0.1
        P = torch.randn(R, n_c, device=dev)
        out, status = torch.empty_like(P), torch.zeros(1, dtype=torch.int32, device=dev)
        dP, dKl = torch.empty_like(P), torch.empty_like(Kl)
        con[name] = {"rows": R, "fp_dim": d, "n_c": n_c,
                     "previous_fwd_bwd_ms": t(old), "engine_fwd_bwd_ms": t(new),
                     "constrain_fwd_ms": t(lambda: engine.constrain_fwd(Kl, P, offsets, cons, out, status)),
                     "constrain_bwd_ms": t(lambda: engine.constrain_bwd(G, Kl, P, offsets, cons, dP, dKl))}
    res["constrainer"] = con

    Yv, Ye = torch.randn(V, 2, device=dev), torch.randn(E // 2, 1, device=dev)
    cons = [torch.randn(B, 2, device=dev), torch.randn(B, 1, device=dev)]
    model = N.EngineMolAtomBondMPNN(N.MABBondMessagePassing(d_h=h, precision="bf16"),
                                    atom_predictor=N.EngineRegressionFFN(n_tasks=2, input_dim=h),
                                    bond_predictor=N.EngineRegressionFFN(n_tasks=1, input_dim=2 * h),
                                    atom_constrainer=ConstrainerFFN(n_constraints=2, fp_dim=h),
                                    bond_constrainer=ConstrainerFFN(n_constraints=1, fp_dim=2 * h)).to(dev).train()
    for p in model.parameters():
        p.grad = torch.zeros_like(p)

    def step(bb=bmg):
        for p in model.parameters():
            p.grad.zero_()
        out = model.training_loss(bb, [None, Yv, Ye], None, constraints=cons)
        out.backward()
        return out

    cg = CudaGraphStep(step)
    res["constrained_step_ms"] = {"eager": t(step), "graph": t(lambda: cg(bmg))}
    res["clocks_after"] = clocks()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_constrainer.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
