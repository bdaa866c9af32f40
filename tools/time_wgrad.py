"""GPU time of the bf16 weight-gradient GEMM (k_wgrad_tc + k_wgrad_reduce) at the four call shapes of a C2 training step.

The batch is the seeded synthetic C2 batch of tools/time_step.py (10 000 ~25-atom molecules, h = 300): E edge rows, V atom
rows, operands of normal random data in the layouts engine.bond_backward_tc hands over (hidden states at the padded leading
dimension).  Per shape: CUDA events around timed windows of at least 200 ms after a warm-up, microseconds per call, the
operand bytes of the shape (every dY and X element read once; the f32 partial sums and dW are not counted), GB/s, and that
rate as a fraction of the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.
DMPNN_EXP selects the kernel's timing experiments in a -DDMPNN_EXPERIMENTS=1 build (csrc/wgrad_tc.cu).

    python tools/time_wgrad.py [--mols 10000] [--hidden 300] [--windows 3] [--window-ms 200]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

DATA_SHEET_GBS = 3350.0          # H100 SXM, HBM3


def card() -> str:
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return f"{name}, power limit / max SM clock: {q.stdout.strip().splitlines()[0]}"
    except Exception as e:  # noqa: BLE001 -- reported, not fatal
        return f"{name}, power limit unavailable ({e})"


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--mols", type=int, default=10000)
    ap.add_argument("--hidden", type=int, default=300)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--window-ms", type=float, default=200.0)
    args = ap.parse_args()

    from chemprop_b200.data import BatchMolGraph, make_molecules

    bmg = BatchMolGraph(make_molecules(args.mols, seed=1))
    h, d_v, d_e = args.hidden, bmg.V.shape[1], bmg.E.shape[1]
    print(f"batch: {args.mols} molecules, {bmg.V.shape[0]} atoms, {bmg.E.shape[0]} directed edges, d_v {d_v}, d_e {d_e}, h {h}")
    if not torch.cuda.is_available():
        sys.exit("time_wgrad.py measures on the GPU and none is present: nothing was timed")

    from chemprop_b200.engine import get_layout, pad_hidden, wgrad_tc, wgrad_tc_multi

    bmg.to("cuda")
    lay = get_layout(bmg)
    E, V, hp = lay.E, bmg.V.shape[0], pad_hidden(h)
    g = torch.Generator(device="cuda").manual_seed(1)

    def operand(rows: int, cols: int, ld: int) -> torch.Tensor:
        t = torch.zeros(rows, ld, dtype=torch.bfloat16, device="cuda")
        t[:, :cols] = torch.randn(rows, cols, device="cuda", generator=g).bfloat16()
        return t

    pad8 = lambda k: (k + 7) // 8 * 8                                  # noqa: E731
    k_o, k_i = d_v + h + 1, d_v + d_e                                  # XO = [V | H_v | 1], X_0 = [V[src] | E]
    shapes = [                                                         # name, R, K, dY terms, X
        ("dW_o (dY, XO)", V, k_o, 1),
        ("dW_h, t = 2 (G, H^1)", E, h, 1),
        ("dW_h, t = 1 (dZ^1, M^1)", E, h, 1),
        ("dW_i (three dZ terms, X_0)", E, k_i, 3),
    ]
    print(f"card: {card()}; DMPNN_EXP={os.environ.get('DMPNN_EXP', '0')}")
    for name, R, K, n_terms in shapes:
        dYs = [operand(R, h, hp) for _ in range(n_terms)]
        X = operand(R, K, hp if K == h else pad8(K))
        dW = torch.empty(h, K, device="cuda")
        call = (lambda: wgrad_tc(dYs[0], X, R, h, K, dW)) if n_terms == 1 else (lambda: wgrad_tc_multi(dYs, X, R, h, K, dW))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def window(n: int) -> float:
            e0.record()
            for _ in range(n):
                call()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n                            # ms per call

        window(10)                                                     # warm-up: module load, workspace allocations
        n = max(10, int(args.window_ms / window(10)) + 1)
        us = sorted(window(n) * 1e3 for _ in range(args.windows))
        byt = R * (n_terms * h + K) * 2
        med = us[len(us) // 2]
        print(f"{name}: R {R}, N {h}, K {K}, {n_terms} term(s): {med:.1f} us per call (median of {args.windows} windows of {n} "
              f"calls, {us[0]:.1f} - {us[-1]:.1f}); operands {byt / 1e9:.3f} GB, {byt / med / 1e3:.0f} GB/s = "
              f"{byt / med / 1e3 / DATA_SHEET_GBS:.2f} of the data sheet's 3 350 GB/s")
        del dYs, X, dW


if __name__ == "__main__":
    main()
