"""GPU: the time of one Monte Carlo dropout sample (a forward-only encoder pass with the nn.Dropout modules trained),
three ways -- forward-only (keep bits in the fused bond step, dmpnn_scale_mask at the read-out), the same call with
gradients enabled (the composed tier, where such a call ran before; with ReLU the training path of Plan.dropout_ok), and a
plain eval forward -- for config 2's batch (10 k ~25-atom molecules, BondMessagePassing h = 300, depth 3, bf16) with ReLU
and with tanh, and config 4's atom batch (10 k ~80-atom condensed reaction graphs, AtomMessagePassing h = 300, depth 3,
bf16; its dropout stays on the composed tier).
CUDA events, median of 5 timed loops of 10 calls after a warm-up; prints the card's name and power limit.

    python tools/time_mc_dropout.py"""
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from chemprop_b200.data import BatchMolGraph, make_cgr_graphs, make_molecules, tile_packing_order_of  # noqa: E402
from chemprop_b200.engine import get_layout  # noqa: E402
from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing  # noqa: E402

CONFIGS = {
    "C2": (lambda: make_molecules(10_000, seed=1), BondMessagePassing, dict(d_h=300, depth=3, precision="bf16")),
    "C2-tanh": (lambda: make_molecules(10_000, seed=1), BondMessagePassing, dict(d_h=300, depth=3, precision="bf16",
                                                                                 activation="tanh")),
    "C4": (lambda: make_cgr_graphs(10_000, seed=1), AtomMessagePassing, dict(d_v=106, d_e=28, d_h=300, depth=3,
                                                                              precision="bf16")),
}


def _time(fn, loops=5, calls=10) -> float:
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(loops):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / calls)
    return statistics.median(ms)


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"gpu": card}))
    import warnings

    warnings.simplefilter("ignore")
    for name, (graphs, cls, kw) in CONFIGS.items():
        mgs = graphs()
        mgs = [mgs[i] for i in tile_packing_order_of(mgs)]
        bmg = BatchMolGraph(mgs)
        bmg.to("cuda")
        torch.manual_seed(0)
        mp = cls(dropout=0.1, **kw).cuda().eval()

        def eval_forward():
            with torch.inference_mode():
                mp(bmg)

        def mc_sample():
            mp.dropout.train()
            with torch.inference_mode():
                mp(bmg)
            mp.dropout.eval()

        def grad_sample():
            mp.dropout.train()
            mp(bmg)                                    # gradients enabled: not forward-only
            mp.dropout.eval()

        mp.dropout.train()
        with torch.inference_mode():
            mono = not mp.uses_composed_tier(get_layout(bmg))
        mono_grad = not mp.uses_composed_tier(get_layout(bmg))
        mp.dropout.eval()
        row = {"config": name, "module": cls.__name__, **kw, "molecules": len(bmg), "directed_edges": int(bmg.E.shape[0]),
               "mc_sample_on_monolithic_tier": mono, "with_grad_on_monolithic_tier": mono_grad,
               "ms_eval_forward": _time(eval_forward), "ms_mc_sample": _time(mc_sample),
               "ms_mc_sample_with_grad": _time(grad_sample)}
        print(json.dumps(row))


if __name__ == "__main__":
    main()
