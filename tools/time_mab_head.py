"""Time of the mol-atom-bond model's heads on the GPU (CUDA events, medians of repeated timed loops), on the C2 batch of
bench.py (10 000 ~25-atom molecules: ~249 k atoms, ~502 k directed edges), d_h = 300:

  * each level's head forward + backward from fixed fingerprints (molecule: RegressionFFN on the aggregate; atom:
    RegressionFFN on H_v with dmpnn_regression_loss_rows; bond: RegressionFFN on [H_e || H_e[rev]] through the gathered
    first layer, the pair mean and dmpnn_regression_loss_rows), and the bond head's first layer alone (SIMT, forward and
    backward);
  * each _rows criterion against its single-block twin at 249 k and 502 k rows (T = 1);
  * dmpnn_edge_pair_mean and its mirror;
  * the whole three-level training step (EngineMolAtomBondMPNN, bf16 MAB encoder) eager and as one CUDA graph, against
    MABBondMessagePassing alone with a loss on both outputs.
The card name and power limit are read in the same run.

    python tools/time_mab_head.py [--mols 10000] [--steps 20] [--reps 5] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tools.time_mab import card  # noqa: E402


def median_ms(fn, steps: int, reps: int, warmup: int = 3) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / steps)
    return statistics.median(out)


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
    from chemprop_b200.nn.head import EdgePairOperand, PairLinearFunction
    from chemprop_b200.nn.mol_atom_bond_model import EdgePairMeanFunction

    dev = "cuda"
    torch.manual_seed(0)
    h = 300
    bmg = BatchMolGraph(make_molecules(args.mols, seed=1, mean_atoms=25.0))
    bmg.to(dev)
    V, E, B = int(bmg.V.shape[0]), int(bmg.E.shape[0]), len(bmg)
    res = {"card": card(), "n_mols": B, "atoms": V, "directed_edges": E, "d_h": h}
    t = lambda fn: median_ms(fn, args.steps, args.reps)  # noqa: E731
    rev = bmg.rev_edge_index.to(torch.int32)

    # ---- per-level heads from fixed fingerprints
    Hg = torch.randn(B, h, device=dev, requires_grad=True)
    Hv = torch.randn(V, h, device=dev, requires_grad=True)
    He = torch.randn(E, h, device=dev, requires_grad=True)
    Yg, Yv, Ye = torch.randn(B, 1, device=dev), torch.randn(V, 1, device=dev), torch.randn(E // 2, 1, device=dev)
    mol, atom, bond = (N.EngineRegressionFFN(input_dim=d).to(dev) for d in (h, h, 2 * h))

    def mol_head():
        mol.criterion(mol.train_step(Hg), Yg).backward()

    def atom_head():
        atom.criterion.row_loss(atom.train_step(Hv), Yv).backward()

    def bond_head():
        P = EdgePairMeanFunction.apply(bond.train_step(EdgePairOperand(He, rev)), rev)
        bond.criterion.row_loss(P, Ye).backward()

    res["head_fwd_bwd_ms"] = {"mol": t(mol_head), "atom": t(atom_head), "bond": t(bond_head)}
    W, b = bond.ffn[0][0].weight, bond.ffn[0][0].bias
    fwd = lambda: PairLinearFunction.apply(He, rev, W, b, engine.ACT_RELU, 0.0)  # noqa: E731
    Y1 = fwd()
    G1 = torch.randn_like(Y1)
    res["bond_first_layer_simt_ms"] = {"forward": t(fwd), "backward": t(lambda: torch.autograd.grad(Y1, (He, W, b), G1,
                                                                                                   retain_graph=True))}

    # ---- _rows criteria against their single-block twins
    crit = {}
    for R in (V, E // 2, E):
        P, Y = torch.randn(R, 1, device=dev), torch.randn(R, 1, device=dev)
        Yb = torch.rand(R, 1, device=dev)
        Pc, Yc = torch.randn(R, 10, device=dev), torch.randint(0, 10, (R, 1), device=dev).float()
        loss = torch.empty(1, device=dev)
        dP, dPc = torch.empty_like(P), torch.empty_like(Pc)
        row = {}
        for name, rows_fn, one_fn in (
                ("mse", lambda: engine.regression_loss_rows(P, Y, None, None, None, None, 0, loss, dP),
                 lambda: engine.regression_loss(P, Y, None, None, None, None, 0, loss, dP)),
                ("bce", lambda: engine.bce_loss_rows(P, Yb, None, None, loss, dP),
                 lambda: engine.bce_loss(P, Yb, None, None, loss, dP)),
                ("ce_C10", lambda: engine.ce_loss_rows(Pc, Yc, None, None, 10, loss, dPc),
                 lambda: engine.ce_loss(Pc, Yc, None, None, 10, loss, dPc))):
            row[name] = {"rows_ms": t(rows_fn), "single_block_ms": t(one_fn)}
        crit[str(R)] = row
    res["criteria"] = crit

    # ---- pair mean
    P = torch.randn(E, 1, device=dev)
    out, dP = torch.empty(E // 2, 1, device=dev), torch.empty(E, 1, device=dev)
    res["pair_mean_ms"] = {"forward": t(lambda: engine.edge_pair_mean(P, rev, out)),
                           "backward": t(lambda: engine.edge_pair_mean_bwd(out, dP))}

    # ---- whole step, with and without the three batch norms
    mp = N.MABBondMessagePassing(d_h=h, precision="bf16").to(dev)
    targetss, weightss = [Yg, Yv, Ye], [None, None, None]
    steps = {}
    for bn in (True, False):
        model = N.EngineMolAtomBondMPNN(mp, N.MeanAggregation(), N.EngineRegressionFFN(input_dim=h),
                                        N.EngineRegressionFFN(input_dim=h), N.EngineRegressionFFN(input_dim=2 * h),
                                        batch_norm=bn).to(dev).train()
        for p in model.parameters():
            p.grad = torch.zeros_like(p)

        def step(bb=bmg, model=model):
            for p in model.parameters():
                p.grad.zero_()
            out = model.training_loss(bb, targetss, weightss)
            out.backward()
            return out

        cg = CudaGraphStep(step)
        sfx = "" if bn else "_no_batch_norm"
        steps["three_level_eager" + sfx] = t(step)
        steps["three_level_graph" + sfx] = t(lambda: cg(bmg))
    # the three batch norms alone (forward + backward) on the step's fingerprint shapes
    bns = [N.EngineBatchNorm1d(h).to(dev).train() for _ in range(3)]
    Xs = [torch.randn(r, h, device=dev, requires_grad=True) for r in (B, V, E)]
    steps["batch_norms_fwd_bwd"] = {str(r): t(lambda bn=bn, X=X: bn(X).sum().backward()) for bn, X, r in
                                    zip(bns, Xs, (B, V, E))}

    agg = N.MeanAggregation()
    Gm, Ge = torch.randn(B, h, device=dev) / 16, torch.randn(E, h, device=dev) / 16

    def mp_only():
        for p in mp.parameters():
            p.grad = None
        H_v, H_e = mp(bmg)
        ((agg(H_v, bmg.batch) * Gm).sum() + (H_e * Ge).sum()).backward()

    steps["mab_bond_mp_only"] = t(mp_only)
    res["step_ms"] = steps
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_mab_head.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
