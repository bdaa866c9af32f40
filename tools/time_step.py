"""GPU timing of the fused depth step alone (CUDA events), optional experiments via DMPNN_EXP.
PACK=1: molecules in the loader's tile-packing order (fuller tiles) instead of generator order."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from chemprop_b200 import _lib
from chemprop_b200.data import BatchMolGraph, make_molecules, tile_packing_order_of
from chemprop_b200.engine import bond_step_fused, get_layout, pack_weight_bf16, pad_hidden

n_mols = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
h = int(sys.argv[2]) if len(sys.argv) > 2 else 300
mgs = make_molecules(n_mols, seed=1)
if os.environ.get("PACK", "0") != "0":
    mgs = [mgs[i] for i in tile_packing_order_of(mgs)]
bmg = BatchMolGraph(mgs); bmg.to("cuda")
lay = get_layout(bmg); hp = pad_hidden(h)
H0 = torch.zeros(lay.E, hp, dtype=torch.bfloat16, device="cuda"); H0[:, :h] = torch.randn(lay.E, h, device="cuda").bfloat16()
Hp = torch.relu(H0).clone(); Hn = torch.zeros_like(H0)
W = torch.randn(h, h, device="cuda") / h ** 0.5; Wpk = pack_weight_bf16(W)
for first in (False, True):
    for _ in range(3): bond_step_fused(H0 if first else Hp, H0, Hn, h, Wpk, None, lay, _lib.ACT_RELU, 0.0, first)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(10):
        e0.record(); bond_step_fused(H0 if first else Hp, H0, Hn, h, Wpk, None, lay, _lib.ACT_RELU, 0.0, first); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ms = sorted(ts)[len(ts) // 2]
    byt = (2 if first else 3) * lay.E * h * 2
    print(f"PACK={os.environ.get('PACK','0')} EXP={os.environ.get('DMPNN_EXP','0')} first={first} E={lay.E} tiles={lay.n_tiles} h={h}: {ms*1e3:.1f} us  {byt/ms/1e6:.0f} GB/s  frac={byt/ms/1e6/3350.0:.3f} of the H100 SXM data sheet's HBM bandwidth")
