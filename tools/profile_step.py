"""In-situ per-kernel durations of the bench step (torch.profiler / CUPTI; warm caches, real overlap)."""
import collections, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile
from chemprop_b200.data import BatchMolGraph, make_molecules
from chemprop_b200.nn import BondMessagePassing, MeanAggregation

n = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
steps = 5
dev = torch.device("cuda")
torch.manual_seed(0)
mp = BondMessagePassing(d_h=300, depth=3, precision="bf16").to(dev)
agg = MeanAggregation()
bmg = BatchMolGraph(make_molecules(n, seed=1, mean_atoms=25.0)); bmg.to(dev)
params = list(mp.parameters())

def step():
    bmg._layout = None
    for p in params: p.grad = None
    loss = agg(mp(bmg), bmg.batch).float().square().mean()
    loss.backward()

for _ in range(3): step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(steps): step()
    torch.cuda.synchronize()
agg_t = collections.OrderedDict()
span0, span1 = None, None
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
        k = ev.name.split("(")[0].replace("void ", "")[:80]
        a = agg_t.setdefault(k, [0, 0.0, []]); a[0] += 1; a[1] += ev.device_time if hasattr(ev, "device_time") else ev.cuda_time
        a[2].append(ev.device_time if hasattr(ev, "device_time") else ev.cuda_time)
        t0 = ev.time_range.start; t1 = ev.time_range.end
        span0 = t0 if span0 is None else min(span0, t0); span1 = t1 if span1 is None else max(span1, t1)
tot = sum(v[1] for v in agg_t.values())
print(f"{steps} steps: kernel-time sum {tot/steps:.0f} us/step; device span {(span1-span0)/steps:.0f} us/step")
for k, (c, v, ds) in sorted(agg_t.items(), key=lambda kv: -kv[1][1]):
    per = c // steps
    each = " [" + " ".join(f"{d:.0f}" for d in ds[-per:]) + "]" if 1 < per <= 6 else ""
    print(f"{100*v/tot:5.1f}%  {v/steps:8.1f} us/step  {c/steps:5.1f}/step  {k}{each}")
