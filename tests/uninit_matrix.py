"""TEST INFRASTRUCTURE ONLY.  The poisoned-allocation differential shared by tests/test_uninit_host.py (CPU, through the
kernel emulations) and tests/test_gpu_uninit.py (H100): the same module configurations run forward + backward once with every
uninitialised floating-point buffer of the library zero-filled and once with it filled with a poison value.  Nothing the
library computes may depend on memory it never wrote, so outputs and gradients must be bit-identical (the engine has no
float atomics, DESIGN.md section 2) and finite.

The fill reaches the library through `PoisonTorch`, a proxy installed as the `torch` global of the allocating modules
(engine, composed, nn.*): `torch.empty` / `torch.empty_like` of a floating-point dtype come back filled.  Integer buffers are
never filled -- an index read before it is written would be an out-of-bounds access, not a wrong number."""
from __future__ import annotations

import torch

# NaN reaches a result through any product (0 * NaN = NaN); 1e30 (finite in bf16 and f32) through the reads a NaN-blind op
# would hide: the packed-bf16 ReLU mask, a max, a comparison
POISONS = {"nan": float("nan"), "huge": 1e30}

# (d_h, padding columns [d_h, pad16(d_h))): 300 -> 4, 296 -> 8, 100 -> 12, 64 -> 0
D_H = (300, 296, 100, 64)
ACTS = ("relu", "leakyrelu", "tanh", "elu")
MODULES = ("bond-bf16", "bond-fp32", "atom-bf16", "atom-fp32", "mabbond-bf16", "mabatom-bf16")


def _grid():
    """Every module with every d_h (24 cases); depth, activation, bias and d_vd rotate so that every module meets every depth
    and activation, and every d_h every depth and activation."""
    out = []
    for m, mod in enumerate(MODULES):
        for j, h in enumerate(D_H):
            out.append(dict(module=mod, d_h=h, depth=1 + (m + 2 * j) % 3, act=ACTS[(m + j) % 4], bias=(m + j) % 2 == 0,
                            d_vd=8 if (not mod.startswith("mab") and (3 * m + j) % 4 == 1) else None))
    return out


CASES = _grid() + [
    # training-mode dropout on the fused bf16 path (keep masks from mask_fn, the same in every run)
    dict(module="bond-bf16", d_h=300, depth=3, act="relu", bias=True, dropout=0.25),
    dict(module="bond-bf16", d_h=100, depth=2, act="relu", bias=False, dropout=0.25),
    # undirected: the reverse-edge average prologue of the fused step (bf16) / the 3xTF32 tier (fp32)
    dict(module="bond-bf16", d_h=296, depth=3, act="tanh", bias=True, undirected=True),
    dict(module="bond-fp32", d_h=100, depth=3, act="relu", bias=False, undirected=True),
    # molecules of more than 128 directed edges: 128-row windows of the fused step (FAR)
    dict(module="bond-bf16", d_h=300, depth=3, act="relu", bias=True, batch="bigmol"),
    dict(module="mabbond-bf16", d_h=300, depth=3, act="elu", bias=False, batch="bigmol"),
    dict(module="atom-bf16", d_h=300, depth=3, act="relu", bias=False, batch="bigmol"),
    # a molecule of more than 128 atoms: the two-launch atom step
    dict(module="atom-bf16", d_h=300, depth=3, act="relu", bias=True, batch="bigatom"),
    dict(module="mabatom-bf16", d_h=296, depth=3, act="leakyrelu", bias=False, batch="bigatom"),
    # one EngineMPNN.training_loss step per aggregation
    dict(module="mpnn-bond-bf16", d_h=300, depth=3, act="relu", bias=False, agg="mean"),
    dict(module="mpnn-atom-bf16", d_h=300, depth=3, act="relu", bias=False, agg="sum", batch_norm=True),
    dict(module="mpnn-bond-fp32", d_h=100, depth=2, act="tanh", bias=True, agg="norm"),
]


def case_id(c: dict) -> str:
    extra = [k for k in ("dropout", "undirected", "batch", "agg") if c.get(k)]
    tags = [f"{k}={c[k]}" if k in ("batch", "agg") else k for k in extra]
    return "-".join([c["module"], f"h{c['d_h']}", f"d{c['depth']}", c["act"], "bias" if c["bias"] else "nobias"]
                    + (["vd"] if c.get("d_vd") else []) + tags)


class PoisonTorch:
    """Stands in for the `torch` module inside the library: floating-point `empty` / `empty_like` results are filled."""

    def __init__(self, fill: float):
        self._fill = fill

    def __getattr__(self, name):
        return getattr(torch, name)

    def _filled(self, t):
        if t.is_floating_point():
            t.fill_(self._fill)
        return t

    def empty(self, *args, **kwargs):
        return self._filled(torch.empty(*args, **kwargs))

    def empty_like(self, *args, **kwargs):
        return self._filled(torch.empty_like(*args, **kwargs))


def install_poison(monkeypatch, fill: float):
    """Route the allocations of engine, composed and nn.* through PoisonTorch(fill) for the rest of the test."""
    import chemprop_b200.composed as composed
    import chemprop_b200.engine as engine
    import chemprop_b200.nn.agg as agg
    import chemprop_b200.nn.constrainer as constrainer
    import chemprop_b200.nn.head as head
    import chemprop_b200.nn.message_passing as message_passing
    import chemprop_b200.nn.mol_atom_bond as mol_atom_bond
    import chemprop_b200.nn.transforms as transforms

    proxy = PoisonTorch(fill)
    for mod in (engine, composed, agg, constrainer, head, message_passing, mol_atom_bond, transforms):
        if hasattr(mod, "torch"):
            monkeypatch.setattr(mod, "torch", proxy)

    def _empty_hidden(rows, hp, dtype, dev):
        return proxy.empty((max(rows, 1), hp), dtype=dtype, device=dev)

    monkeypatch.setattr(engine, "_empty_hidden", _empty_hidden)


def make_batch(c: dict, device: str, n_mols: int, seed: int = 0):
    """A shuffled-edge batch of ~12-atom molecules; `bigmol` adds three molecules of more than 128 directed edges, `bigatom`
    one molecule of more than 128 atoms."""
    from chemprop_b200.data import BatchMolGraph, make_molecules

    mgs = make_molecules(n_mols, seed=seed, mean_atoms=12.0, std_atoms=4.0, min_atoms=1, max_atoms=30, shuffle_edges=True)
    batch = c.get("batch")
    if batch == "bigmol":
        big = make_molecules(3, seed=seed + 1, mean_atoms=85.0, std_atoms=8.0, min_atoms=70, max_atoms=100, shuffle_edges=True)
        for i, m in enumerate(big):
            mgs.insert(min(len(mgs), 1 + i * max(1, len(mgs) // 3)), m)
    elif batch == "bigatom":
        big = make_molecules(1, seed=seed + 1, mean_atoms=135.0, std_atoms=3.0, min_atoms=130, max_atoms=140, shuffle_edges=True)
        mgs.insert(len(mgs) // 2, big[0])
    bmg = BatchMolGraph(mgs)
    bmg.to(device)
    return bmg


def _module(c: dict):
    import chemprop_b200.nn as N

    kind, precision = c["module"].rsplit("-", 1)
    kw = dict(d_h=c["d_h"], depth=c["depth"], activation=c["act"], bias=c["bias"], precision=precision)
    if kind in ("bond", "atom", "mpnn-bond", "mpnn-atom"):
        cls = N.AtomMessagePassing if kind.endswith("atom") else N.BondMessagePassing
        mp = cls(dropout=c.get("dropout", 0.0), undirected=c.get("undirected", False), d_vd=c.get("d_vd"), **kw)
    else:
        cls = N.MABAtomMessagePassing if kind == "mabatom" else N.MABBondMessagePassing
        mp = cls(**kw)
    if not kind.startswith("mpnn"):
        return mp
    agg = {"mean": N.MeanAggregation, "sum": N.SumAggregation, "norm": N.NormAggregation}[c["agg"]]()
    return N.EngineMPNN(mp, agg, batch_norm=c.get("batch_norm", False))


def run_case(c: dict, bmg, device: str) -> dict:
    """Forward + backward of case `c` on `bmg` from seeded parameters; returns every output and parameter gradient."""
    torch.manual_seed(1234)
    model = _module(c).to(device).train()
    p = c.get("dropout", 0.0)
    if p:
        n = [0]

        def mask_fn(like):        # the same keep masks in every run: site k of the step draws from seed 99 + k
            g = torch.Generator(device=like.device).manual_seed(99 + n[0])
            n[0] += 1
            return (torch.rand(like.shape, generator=g, device=like.device) >= p).to(like.dtype)

        model._mask_fn = mask_fn
    g = torch.Generator().manual_seed(7)
    nV, nE, B = bmg.V.shape[0], bmg.E.shape[0], len(bmg)
    out = {}
    if c["module"].startswith("mpnn"):
        Y = torch.randn(B, 1, generator=g).to(device)
        loss = model.training_loss(bmg, Y)
        out["loss"] = loss.detach().reshape(1)
    elif c["module"].startswith("mab"):
        H_v, H_e = model(bmg)
        out["H_v"], out["H_e"] = H_v.detach(), H_e.detach()
        loss = (H_v * torch.randn(H_v.shape, generator=g).to(device)).sum() + (H_e * torch.randn(H_e.shape, generator=g).to(device)).sum()
    else:
        V_d = torch.randn(nV, c["d_vd"], generator=g).to(device) if c.get("d_vd") else None
        H = model(bmg, V_d)
        out["H"] = H.detach()
        loss = (H.float() * torch.randn(H.shape, generator=g).to(device)).sum()
    loss.backward()
    for k, prm in model.named_parameters():
        assert prm.grad is not None, k
        out["grad." + k] = prm.grad.detach()
    assert nE > 0
    return {k: v.cpu() for k, v in out.items()}


def assert_bit_identical(ref: dict, got: dict, what: str):
    """Every tensor of both runs finite, and equal bit for bit (as raw bytes: -0.0 vs +0.0 counts as a difference)."""
    assert ref.keys() == got.keys()
    bad = []
    for k in ref:
        a, b = ref[k], got[k]
        for name, t in (("zero-filled", a), (what, b)):
            if not bool(torch.isfinite(t.float()).all()):
                bad.append(f"{k}: {int((~torch.isfinite(t.float())).sum())} non-finite values ({name} run)")
        if a.shape != b.shape or not torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)):
            bad.append(f"{k}: differs")
    assert not bad, f"{what}: " + "; ".join(bad)
