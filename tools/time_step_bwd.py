"""GPU timing of the fused step's autograd-mirror modes alone (CUDA events): MODE 1 (masked by tau' of the activation),
MODE 3 (tau' of the pre-activation) without addends, as the engine runs it, and MODE 3 with one and two addends, a C ABI
capability.  Molecules in the loader's tile-packing order; prints the card and its power limit."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from chemprop_b200 import _lib
from chemprop_b200.data import BatchMolGraph, make_molecules, tile_packing_order_of
from chemprop_b200.engine import bond_step_bwd_fused, get_layout, pack_weight_bf16, pad_hidden

if not torch.cuda.is_available():
    sys.exit("time_step_bwd.py needs a GPU")
n_mols = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
h = int(sys.argv[2]) if len(sys.argv) > 2 else 300
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                     capture_output=True, text=True).stdout.strip())
mgs = make_molecules(n_mols, seed=1)
mgs = [mgs[i] for i in tile_packing_order_of(mgs)]
bmg = BatchMolGraph(mgs); bmg.to("cuda")
lay = get_layout(bmg); hp = pad_hidden(h)


def rows():
    x = torch.zeros(lay.E, hp, dtype=torch.bfloat16, device="cuda")
    x[:, :h] = torch.randn(lay.E, h, device="cuda").bfloat16()
    return x


dZ, Y, A0, A1 = rows(), rows(), rows(), rows()
out = torch.zeros_like(dZ)
WpkT = pack_weight_bf16((torch.randn(h, h, device="cuda") / h ** 0.5).t().contiguous())
cases = [("MODE 1", False, ()), ("MODE 3", True, ()), ("MODE 3 + 1 addend", True, (A0,)),
         ("MODE 3 + 2 addends", True, (A0, A1))]
for name, pre, add in cases:
    run = lambda: bond_step_bwd_fused(dZ, Y, out, h, WpkT, lay, _lib.ACT_RELU, 0.0, None, pre, add)  # noqa: E731
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(10):
        e0.record(); run(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[len(ts) // 2]
    byt = (3 + len(add)) * lay.E * h * 2   # dZ, Y, addends read once, dOut written once
    print(f"{name}: E={lay.E} h={h}: {ms * 1e3:.1f} us  {byt / ms / 1e6:.0f} GB/s  "
          f"frac={byt / ms / 1e6 / 3350.0:.3f} of the H100 SXM data sheet's HBM bandwidth")
