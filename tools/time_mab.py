"""Forward + backward time of the mol-atom-bond message passing on the GPU, precision="bf16" against "fp32" (CUDA events).

Loss: sum(mean_agg(H_v) * G) + sum(H_e * G_e).
  * MABBondMessagePassing(d_h=300, depth=3) on the C2 batch of bench.py (10 000 ~25-atom molecules), with
    BondMessagePassing(precision="bf16") on the same batch as the floor (vertex read-out only, no edge head);
  * MABAtomMessagePassing(d_h=300, depth=3) on C4-shaped condensed-reaction graphs (make_cgr_graphs, d_v=106, d_e=28).
For the bf16 edge head, the kernel times of its forward GEMM and its mirror-mode gradient entry are reported next to their
algorithmic bytes.  The card name and power limit are read in the same run.

    python tools/time_mab.py [--mols 10000] [--cgr 10000] [--steps 10] [--warmup 3] [--out DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

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


def time_step(fn, steps: int, warmup: int) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def mab_step(mp, bmg, Gm, Ge):
    from chemprop_b200.nn import MeanAggregation

    agg = MeanAggregation()
    params = list(mp.parameters())

    def step():
        for p in params:
            p.grad = None
        H_v, H_e = mp(bmg)
        loss = (agg(H_v, bmg.batch).float() * Gm).sum()
        if H_e is not None:
            loss = loss + (H_e.float() * Ge).sum()
        loss.backward()
    return step


def bond_floor_step(mp, bmg, Gm):
    from chemprop_b200.nn import MeanAggregation

    agg = MeanAggregation()
    params = list(mp.parameters())

    def step():
        for p in params:
            p.grad = None
        (agg(mp(bmg), bmg.batch).float() * Gm).sum().backward()
    return step


def edge_head_kernels(kind: str, bmg, d_v: int, d_e: int, h: int, steps: int) -> dict:
    """CUDA-event times of the edge head's two new launches on this batch: H_e = tau(X_e . W_eo^T + b) (f32 store) and the
    mirror-mode entry dZ[inv_perm[e]] = (dY_e . W_eo[:, d_e:] + dM_v[dst(e)]) * tau'(H^{T-1}) (bond) / its V-row counterpart
    (atom), with their algorithmic bytes (every operand read once, every result written once)."""
    from chemprop_b200 import engine

    lay = engine.get_layout(bmg)
    nE, nV = lay.E, lay.V
    hp = engine.pad_hidden(h)
    dev = bmg.V.device
    W = torch.randn(h, d_e + h, device=dev) / (d_e + h) ** 0.5
    b = torch.randn(h, device=dev)
    Xe = torch.randn(nE, (d_e + h + 15) // 16 * 16, device=dev).to(torch.bfloat16)
    He = torch.empty(nE, h, device=dev)
    Wpk, WTpk = engine.pack_weight_tc(W), engine.pack_weight_tc(W[:, d_e:], transpose=True)
    rows = nE if kind == "bond" else nV
    dY = torch.randn(rows, hp, device=dev).to(torch.bfloat16)
    Y = torch.randn(nE if kind == "bond" else nV, hp, device=dev).to(torch.bfloat16)
    res = torch.randn(nV, hp, device=dev).to(torch.bfloat16)
    out = torch.empty(nE if kind == "bond" else nV, hp, device=dev, dtype=torch.bfloat16)
    relu = engine.ACT_RELU
    fwd = lambda: engine.linear_tc_rows(Xe, d_e + h, Wpk, h, He, R=nE, bias=b, act=relu)  # noqa: E731
    if kind == "bond":
        dst_e = engine.mab_tables(lay)[0]
        mir = lambda: engine.linear_tc_rows(dY, h, WTpk, h, out, R=nE, act=relu, Y=Y, out_row=lay.inv_perm, res=res,  # noqa: E731
                                            res_row=dst_e)
        # per edge: the dY_e row read, the H^{T-1} row read, the dZ row written (bf16 each) and two int32 indices; dM_v is
        # gathered by destination atom, read once: nV rows
        mir_bytes = nE * (3 * h * 2 + 8) + nV * h * 2
    else:
        mir = lambda: engine.linear_tc_rows(dY, h, WTpk, h, out, R=nV, act=relu, Y=Y, res=res)  # noqa: E731
        mir_bytes = nV * 4 * h * 2
    fwd_bytes = nE * ((d_e + h) * 2 + h * 4)                       # X_e (bf16) in, H_e (f32) out
    ms_f, ms_m = time_step(fwd, steps, 2), time_step(mir, steps, 2)
    return {"rows_E": nE, "rows_V": nV,
            "fwd_ms": ms_f, "fwd_MB": fwd_bytes / 1e6, "fwd_GBs": fwd_bytes / ms_f / 1e6,
            "mirror_ms": ms_m, "mirror_MB": mir_bytes / 1e6, "mirror_GBs": mir_bytes / ms_m / 1e6}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mols", type=int, default=10_000)
    ap.add_argument("--cgr", type=int, default=10_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None, help="directory for a JSON copy of the result")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("tools/time_mab.py measures on the GPU; no CUDA device found")
    from chemprop_b200.data import BatchMolGraph, make_cgr_graphs, make_molecules
    from chemprop_b200.nn import BondMessagePassing, MABAtomMessagePassing, MABBondMessagePassing

    dev = torch.device("cuda")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup}
    h = 300
    for kind, n, gen, d_v, d_e in (("bond", args.mols, lambda n: make_molecules(n, seed=1, mean_atoms=25.0), 72, 14),
                                   ("atom", args.cgr, lambda n: make_cgr_graphs(n, seed=1), 106, 28)):
        bmg = BatchMolGraph(gen(n))
        bmg.to(dev)
        g = torch.Generator(device=dev).manual_seed(0)
        Gm = torch.randn(n, h, device=dev, generator=g)
        Ge = torch.randn(bmg.E.shape[0], h, device=dev, generator=g) / 16
        cls = MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing
        row = {"n_mols": n, "atoms": int(bmg.V.shape[0]), "directed_edges": int(bmg.E.shape[0])}
        for precision in ("bf16", "fp32"):
            torch.manual_seed(0)
            mp = cls(d_v=d_v, d_e=d_e, d_h=h, depth=3, precision=precision).to(dev)
            ms = time_step(mab_step(mp, bmg, Gm, Ge), args.steps, args.warmup)
            row[f"mab_{precision}_ms"] = ms
            row[f"mab_{precision}_mols_per_s"] = n / ms * 1e3
            del mp
            torch.cuda.empty_cache()
        row["speedup_bf16_over_fp32"] = row["mab_fp32_ms"] / row["mab_bf16_ms"]
        if kind == "bond":
            torch.manual_seed(0)
            mp = BondMessagePassing(d_v=d_v, d_e=d_e, d_h=h, depth=3, precision="bf16").to(dev)
            row["floor_bond_mp_bf16_ms"] = time_step(bond_floor_step(mp, bmg, Gm), args.steps, args.warmup)
            del mp
        row["edge_head_kernels"] = edge_head_kernels(kind, bmg, d_v, d_e, h, max(args.steps, 20))
        res[f"mab_{kind}"] = row
        print(json.dumps({f"mab_{kind}": row}), flush=True)
        del bmg
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "time_mab.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
