"""Training-step time of EngineMulticomponentMPNN on the GPU (CUDA events, medians of repeated timed loops): two components,
10 000 data points -- a C2-like solute (~25 atoms) and a small solvent (1-10 atoms, the single-atom ones edge-less) --
BondMessagePassing d_h = 300, depth 3, regression head, in bf16 and fp32, at batch sizes 10 000, 1 000 and 64:

  * shared encoder, one union batch (one message-passing chain over both components);
  * shared encoder, a list of the two components' batches (one chain per component, as the reference runs it);
  * unshared encoders (one block per component), list of batches;
each eagerly and replayed as one CUDA graph, with the libdmpnn kernels one step launches.  The card name and power limit
are read in the same run.

    python tools/time_multicomponent.py [--dps 10000] [--steps 10] [--reps 5] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tools.time_mab import card  # noqa: E402
from tools.time_mab_head import median_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dps", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_multicomponent.py measures on the GPU; no CUDA device found")

    import chemprop_b200.nn as N
    from chemprop_b200 import _lib
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    dev, h = "cuda", 300
    solutes = make_molecules(args.dps, seed=1, mean_atoms=25.0, std_atoms=5.0)
    solvents = make_molecules(args.dps, seed=2, mean_atoms=4.0, std_atoms=3.0, min_atoms=1, max_atoms=10)
    lib = _lib.load()
    rows = []
    for b in sorted({args.dps, 1000, 64}, reverse=True):
        comps = [solutes[:b], solvents[:b]]
        union = BatchMolGraph([comps[c][m] for m in range(b) for c in range(2)])
        union.to(dev)
        per = [BatchMolGraph(m) for m in comps]
        for x in per:
            x.to(dev)
        Y = torch.randn(b, 1, device=dev)
        for precision in ("bf16", "fp32"):
            torch.manual_seed(0)
            blk = N.BondMessagePassing(d_h=h, precision=precision)
            models = {
                "shared, union batch": (N.EngineMulticomponentMessagePassing([blk], n_components=2, shared=True), union),
                "shared, per-component batches": (N.EngineMulticomponentMessagePassing([blk], n_components=2, shared=True), per),
                "unshared, per-component batches": (N.EngineMulticomponentMessagePassing(
                    [N.BondMessagePassing(d_h=h, precision=precision) for _ in range(2)], n_components=2), per),
            }
            for mode, (mcmp, batch) in models.items():
                model = N.EngineMulticomponentMPNN(mcmp, N.MeanAggregation()).to(dev)
                params = list(model.parameters())
                for p in params:
                    p.grad = torch.zeros_like(p)

                def step(bt, model=model, params=params):
                    for p in params:
                        p.grad.zero_()
                    loss = model.training_loss(bt, Y)
                    loss.backward()
                    return loss

                step(batch)
                torch.cuda.synchronize()
                l0 = lib.dmpnn_launch_count()
                step(batch)
                torch.cuda.synchronize()
                launches = int(lib.dmpnn_launch_count() - l0)
                eager = median_ms(lambda: step(batch), args.steps, args.reps)
                graph = CudaGraphStep(step)
                graphed = median_ms(lambda: graph(batch), args.steps, args.reps)
                rows.append({"batch": b, "precision": precision, "encoder": mode, "launches": launches,
                             "eager_ms": round(eager, 3), "graph_ms": round(graphed, 3)})
                print(json.dumps(rows[-1]), flush=True)
                del graph
    res = {"card": card(), "data_points": args.dps, "d_h": h, "depth": 3,
           "atoms_per_data_point": {"solute": sum(m.V.shape[0] for m in solutes) / args.dps,
                                    "solvent": sum(m.V.shape[0] for m in solvents) / args.dps},
           "edgeless_solvents": sum(m.edge_index.shape[1] == 0 for m in solvents), "rows": rows}
    lines = [f"card: {res['card']['name']}, power limit {res['card']['power_limit_w']} W", "",
             "| batch | precision | encoder | launches / step | eager ms / step | CUDA graph ms / step |", "|---|---|---|---|---|---|"]
    lines += [f"| {r['batch']} | {r['precision']} | {r['encoder']} | {r['launches']} | {r['eager_ms']} | {r['graph_ms']} |"
              for r in rows]
    print("\n".join(lines))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_multicomponent.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "time_multicomponent.md"), "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
