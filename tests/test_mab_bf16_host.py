"""CPU tier: MABBond / MABAtomMessagePassing(precision="bf16") -- the host logic of engine.MABMPFunction (depth loop of the
bf16 tier, f32 read-outs, the per-edge W_eo head and the entry of its gradient into the depth loop's mirror) on the
emulated kernels of tests/emu.py + tests/emu_mab.py, against the MAB goldens and the oracle."""
from __future__ import annotations

import collections
import ctypes
import warnings

import numpy as np
import pytest
import torch

from chemprop_b200 import _lib, composed, engine
from tests import emu_mab
from tests.util import check_mab_case, golden_bmg, load_golden, params_of

BF16_GOLDENS = ("mab_bond_d3", "mab_bond_noedges", "mab_atom_d2_vertex_only", "mab_atom_d3_desc")


def _record(monkeypatch) -> collections.Counter:
    """Count the calls of the depth-step kernels, the f32 FMA GEMMs (with rows) and the composed tier."""
    calls = collections.Counter()
    for name in ("bond_step_fused", "bond_step_bwd_fused", "atom_step_fused", "atom_step_bwd_fused", "linear_tc_rows"):
        f = getattr(engine, name)
        monkeypatch.setattr(engine, name, (lambda f, n: lambda *a, **k: (calls.update([n]), f(*a, **k))[1])(f, name))
    for name in ("linear_fwd", "linear_wgrad"):
        f = getattr(engine, name)

        def rec(*a, _f=f, _n=name, **k):
            if k.get("R") is None or k["R"] > 0:           # a 0-row call launches nothing
                calls.update([_n])
            return _f(*a, **k)
        monkeypatch.setattr(engine, name, rec)
    fm = composed.mab_forward
    monkeypatch.setattr(composed, "mab_forward", lambda *a, **k: (calls.update(["composed"]), fm(*a, **k))[1])
    return calls


def _golden_module(g: dict, precision: str):
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing
    from tests.util import activation_arg

    cfg = g["config"]
    cls = MABBondMessagePassing if cfg["kind"] == "mab_bond" else MABAtomMessagePassing
    mp = cls(d_v=cfg.get("d_v", 72), d_e=cfg.get("d_e", 14), d_h=cfg["d_h"], bias=cfg.get("bias", False), depth=cfg["depth"],
             activation=activation_arg(cfg), undirected=cfg.get("undirected", False), d_vd=cfg.get("d_vd"),
             d_ed=cfg.get("d_ed"), return_vertex_embeddings=cfg.get("vertex", True),
             return_edge_embeddings=cfg.get("edge", True), precision=precision)
    mp.load_state_dict(params_of(g), strict=True)
    return mp


def _golden_run(g: dict, mp):
    from chemprop_b200.nn import MeanAggregation

    bmg = golden_bmg(g, "cpu")
    d = lambda k: torch.from_numpy(g[k]) if k in g else None  # noqa: E731
    H_v, H_e = mp(bmg, d("V_d"), d("E_d"))
    loss = 0.0
    if H_v is not None:
        loss = loss + (MeanAggregation()(H_v, bmg.batch) * d("G")).sum()
    if H_e is not None:
        loss = loss + (H_e * d("G_e")).sum()
    loss.backward()
    return H_v, H_e


def _close_bf16(got: torch.Tensor, ref, what: str, grad: bool = False, kinked: bool = False):
    """Outputs: max |err| <= 1e-2 max(1, max |ref|).  Gradients: max |err| <= 6e-2 max |ref|.  `kinked` (ReLU / LeakyReLU on a batch
    of a few molecules): bf16 storage moves pre-activations across zero and flips tau' there, noise that only averages out over
    large batches -- the bound of the bf16 golden tests of Bond / AtomMessagePassing (max 0.5, Frobenius 0.2) applies."""
    got = got.detach().double().cpu()
    ref = torch.as_tensor(ref).double()
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    if not got.numel():
        return
    err = (got - ref).abs().max().item()
    scale = ref.abs().max().item()
    if not grad:
        assert err <= 1e-2 * max(1.0, scale), (what, err, scale)
    elif kinked:
        fro = ((got - ref).norm() / max(1e-12, ref.norm().item())).item()
        assert err <= 0.5 * max(scale, 1e-3) and fro <= 0.2, (what, err, scale, fro)
    else:
        assert err <= 6e-2 * max(scale, 1e-6), (what, err, scale)


@pytest.mark.parametrize("name", BF16_GOLDENS)
def test_bf16_mab_matches_golden_through_emulation(name, monkeypatch):
    emu_mab.patch_engine(monkeypatch)
    calls = _record(monkeypatch)
    g = load_golden(name)
    cfg = g["config"]
    mp = _golden_module(g, "bf16")
    assert not mp.uses_composed_tier()
    with warnings.catch_warnings():
        warnings.simplefilter("error", RuntimeWarning)          # the eligible configurations run without a warning
        H_v, H_e = _golden_run(g, mp)
    assert calls["composed"] == 0 and calls["linear_fwd"] == 0 and calls["linear_wgrad"] == 0, calls
    loop = cfg["depth"] - 1 if g["E"].shape[0] > 0 else 0
    vertex, edge = cfg.get("vertex", True), cfg.get("edge", True)
    if cfg["kind"] == "mab_bond":
        assert (calls["bond_step_fused"], calls["bond_step_bwd_fused"]) == (loop, loop), calls
    else:
        # without an edge head the read-out's gradient gather runs on the fused kernel too (AtomMessagePassing's mirror)
        assert (calls["atom_step_fused"], calls["atom_step_bwd_fused"]) == (loop, loop + int(vertex and not edge)), calls
    # forward: W_vo and W_eo read-outs in f32; backward: one mirror-mode entry (edge head present and edges in the batch)
    assert calls["linear_tc_rows"] == int(vertex) + (2 * int(edge) if g["E"].shape[0] > 0 else 0), calls
    assert (H_v is None) == (not vertex) and (H_e is None) == (not edge)
    if H_v is not None:
        assert H_v.dtype == torch.float32
        _close_bf16(H_v, g["H_v"], "H_v")
    if H_e is not None:
        assert H_e.dtype == torch.float32
        _close_bf16(H_e, g["H_e"], "H_e")                       # caller's edge order
    grads = {k: p.grad for k, p in mp.named_parameters()}
    n = 0
    for k, v in g.items():
        if k.startswith("grad."):
            _close_bf16(grads[k[len("grad."):]], v, k, grad=True, kinked=cfg.get("activation", "relu") in ("relu", "leakyrelu"))
            n += 1
    assert n >= 3


def test_bf16_request_outside_the_tier_warns_and_runs_composed(monkeypatch):
    """undirected=True with PReLU, edge read-out only: the composed tier at fp32 accuracy, with a warning naming why."""
    emu_mab.patch_engine(monkeypatch)
    monkeypatch.setattr(engine, "_WARNED", set())
    calls = _record(monkeypatch)
    g = load_golden("mab_bond_edges_only")
    mp = _golden_module(g, "bf16")
    assert mp.uses_composed_tier() and "activation PReLU" == mp.composed_reason()
    with pytest.warns(RuntimeWarning, match=r"precision='bf16' requested, but this configuration \(activation PReLU\)"):
        H_v, H_e = _golden_run(g, mp)
    assert calls["composed"] == 1 and calls["linear_tc_rows"] == 0
    check_mab_case(g, mp, H_v, H_e, 2e-6)


@pytest.mark.parametrize("why, kw", [
    ("undirected=True", dict(undirected=True)),
    ("training-mode dropout", dict(dropout=0.2)),
    ("d_h = 320 > 304", dict(d_h=320)),
    ("d_h = 30 not a multiple of 4", dict(d_h=30)),
    ("GEMM inner dimensions", dict(d_v=300, d_h=160)),
])
def test_bf16_eligibility_reasons(why, kw):
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing

    for cls in (MABBondMessagePassing, MABAtomMessagePassing):
        mp = cls(precision="bf16", **kw)
        assert why in mp.composed_reason() and mp.uses_composed_tier()
        if "dropout" in why:
            mp.eval()
            assert mp.composed_reason() is None          # inference-mode dropout is the identity
    assert MABBondMessagePassing(precision="fp32").uses_composed_tier()
    assert MABBondMessagePassing(precision="bf16", activation="selu").composed_reason() == "activation SELU"


SWEEP = [
    # kind, depth, bias, act, vertex, edge, shuffled, cgr
    ("bond", 1, True, "relu", True, True, False, False),
    ("bond", 1, False, "tanh", False, True, True, False),
    ("bond", 2, False, "leakyrelu", True, False, True, False),
    ("bond", 3, True, "tanh", False, True, True, False),
    ("bond", 4, True, "elu", True, True, True, True),
    ("atom", 1, True, "tanh", True, True, True, False),
    ("atom", 1, False, "elu", False, True, False, True),
    ("atom", 2, True, "relu", False, True, False, False),
    ("atom", 3, False, "elu", True, True, True, True),
    ("atom", 4, True, "leakyrelu", True, False, True, False),
]


def sweep_case(kind, depth, bias, act, vertex, edge, shuffled, cgr, device="cpu", n_mols=7, d_h=48, seed=0):
    """One randomised configuration: the bf16 module on `device` against oracle/restatement.mab_forward in f64 (outputs and
    every parameter gradient of sum(mean_agg(H_v) G) + sum(H_e G_e))."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(seed)
    d_v, d_e = (106, 28) if cgr else (72, 14)
    mgs = make_molecules(n_mols, seed=seed + 3, mean_atoms=12 if not cgr else 30, std_atoms=4, shuffle_edges=shuffled,
                         d_v=d_v, d_e=d_e)
    cls = MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing
    mp = cls(d_v=d_v, d_e=d_e, d_h=d_h, bias=bias, depth=depth, activation=act, return_vertex_embeddings=vertex,
             return_edge_embeddings=edge, precision="bf16")
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    ref = BatchMolGraph(mgs)
    n_mols, nE = len(mgs), ref.E.shape[0]
    G = torch.randn(n_mols, d_h, dtype=torch.float64)
    G_e = torch.randn(nE, d_h, dtype=torch.float64) / 4
    Hv_ref, He_ref = R.mab_forward(kind, ref.V.double(), ref.E.double(), ref.edge_index, ref.rev_edge_index, P["W_i.weight"],
                                   P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"), P.get("W_vo.weight"),
                                   P.get("W_vo.bias"), P.get("W_eo.weight"), P.get("W_eo.bias"), depth, act,
                                   return_vertex=vertex, return_edge=edge)
    loss = 0.0
    if vertex:
        loss = loss + (R.aggregate(Hv_ref, ref.batch, "mean") * G).sum()
    if edge:
        loss = loss + (He_ref * G_e).sum()
    loss.backward()
    mp = mp.to(device)
    bmg = BatchMolGraph(mgs)
    bmg.to(device)
    assert not mp.uses_composed_tier()
    H_v, H_e = mp(bmg)
    loss = 0.0
    if vertex:
        loss = loss + (MeanAggregation()(H_v, bmg.batch) * G.float().to(device)).sum()
    if edge:
        loss = loss + (H_e * G_e.float().to(device)).sum()
    loss.backward()
    assert (H_v is None) == (not vertex) and (H_e is None) == (not edge)
    if vertex:
        _close_bf16(H_v, Hv_ref.detach(), "H_v")
    if edge:
        _close_bf16(H_e, He_ref.detach(), "H_e")
    for k, p in mp.named_parameters():
        ref_g = P[k].grad if P[k].grad is not None else torch.zeros_like(P[k])      # W_h at depth 1: unused, zero
        _close_bf16(p.grad, ref_g, k, grad=True, kinked=act in ("relu", "leakyrelu"))


@pytest.mark.parametrize("case", SWEEP, ids=lambda c: "-".join(map(str, c)))
def test_bf16_mab_random_sweep_vs_oracle(case, monkeypatch):
    emu_mab.patch_engine(monkeypatch)
    sweep_case(*case)


def test_hparams_round_trip():
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing

    for cls in (MABBondMessagePassing, MABAtomMessagePassing):
        mp = cls(d_h=64, depth=2, activation="tanh", d_ed=3, return_vertex_embeddings=False, precision="bf16")
        hp = dict(mp.hparams)
        assert hp["precision"] == "bf16" and hp["cls"] is cls
        back = hp.pop("cls")(**hp)
        assert type(back) is cls and back.precision == "bf16" and back.hparams == mp.hparams
        assert set(back.state_dict()) == set(mp.state_dict())
        assert cls().precision == "fp32" and cls().hparams["precision"] == "fp32"
    with pytest.raises(ValueError):
        MABBondMessagePassing(precision="fp16")


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_bf16_mab_modules_inside_the_reference_mol_atom_bond_mpnn(kind, monkeypatch):
    """chemprop.models.MolAtomBondMPNN (models/mol_atom_bond.py:215-238) wrapping the engine's bf16 MAB modules vs the
    all-reference model: molecule-, atom- and bond-level fingerprints at the bf16 bound, every gradient of a loss on all three
    within 6 % of its scale."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data.collate import BatchMolAtomBondGraph
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MolAtomBondMPNN
    from chemprop.nn.message_passing import MABAtomMessagePassing, MABBondMessagePassing

    import chemprop_b200.nn as ours
    from chemprop_b200.data import make_molecules

    emu_mab.patch_engine(monkeypatch)
    torch.manual_seed(4)
    bmg = BatchMolAtomBondGraph([RefMG(*m) for m in make_molecules(9, seed=6, mean_atoms=8, std_atoms=3, shuffle_edges=True)])
    kw = dict(d_h=32, depth=3, bias=True, activation="elu")
    ref_mp = (MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing)(**kw)
    our_mp = (ours.MABBondMessagePassing if kind == "bond" else ours.MABAtomMessagePassing)(precision="bf16", **kw)
    preds = lambda: dict(mol_predictor=ref_nn.RegressionFFN(input_dim=32), atom_predictor=ref_nn.RegressionFFN(input_dim=32),  # noqa: E731
                         bond_predictor=ref_nn.RegressionFFN(input_dim=64))
    ref = MolAtomBondMPNN(ref_mp, ref_nn.SumAggregation(), batch_norm=True, **preds())
    drop = MolAtomBondMPNN(our_mp, ours.SumAggregation(), batch_norm=True, **preds())
    drop.load_state_dict(ref.state_dict())
    results = []
    for model in (ref, drop):
        model.eval()                              # dropout-free, and the batch norm uses its running statistics
        model.zero_grad()
        H_g, H_v, H_e = model.fingerprint(bmg)
        assert H_v.dtype == H_e.dtype == torch.float32
        loss = H_g.square().mean() + H_v.tanh().mean() + (H_e * torch.linspace(-1, 1, 64)).mean()
        loss.backward()
        results.append(([t.detach() for t in (H_g, H_v, H_e)],
                        {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}))
    assert not our_mp.uses_composed_tier()
    for i, (a, b) in enumerate(zip(results[0][0], results[1][0])):
        _close_bf16(b, a, ("H_g", "H_v", "H_e")[i])
    assert set(results[0][1]) == set(results[1][1])
    for k in results[0][1]:
        _close_bf16(results[1][1][k], results[0][1][k], k, grad=True)


def test_rows_entry_point_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    fn = lib.dmpnn_linear_tc_rows_bf16
    p = ctypes.c_void_p(4096)                     # aligned, never dereferenced: every call below fails its host checks
    ok = dict(A=p, lda=64, R=10, K=64, W=p, N=64, bias=None, act=_lib.ACT_RELU, ap=0.0, Y=None, ldy=0, pre=0, orow=None,
              res=None, ldres=0, rrow=None, C=p, dt=_lib.F32, ldc=64)

    def call(**over):
        a = dict(ok, **over)
        return fn(a["A"], a["lda"], a["R"], a["K"], a["W"], a["N"], a["bias"], a["act"], a["ap"], a["Y"], a["ldy"], a["pre"],
                  a["orow"], a["res"], a["ldres"], a["rrow"], a["C"], a["dt"], a["ldc"], None)

    y, r = ctypes.c_void_p(8192), ctypes.c_void_p(12288)
    mirror = dict(Y=y, ldy=64, dt=_lib.BF16)
    bad = [dict(K=0), dict(K=449), dict(N=305), dict(act=9), dict(dt=5), dict(A=None), dict(lda=60), dict(lda=32),
           dict(A=ctypes.c_void_p(4098)), dict(ldc=62), dict(C=ctypes.c_void_p(4100)),
           dict(orow=p), dict(res=r, ldres=64), dict(pre=1),                         # mirror-only arguments in forward mode
           dict(mirror, dt=_lib.F32),                                                # the mirror stores bf16
           dict(mirror, bias=p),                                                     # ... and takes no bias
           dict(mirror, ldy=40), dict(mirror, Y=ctypes.c_void_p(8200)),              # Y stride / alignment
           dict(mirror, res=r, ldres=8), dict(mirror, res=p, ldres=64),              # residual stride; residual aliasing C
           dict(mirror, rrow=p),                                                     # res_row without a residual
           dict(mirror, C=y), dict(mirror, C=ctypes.c_void_p(4104)),                 # C aliasing Y; bf16 C alignment
           dict(dt=_lib.BF16, ldc=32)]
    for over in bad:
        assert call(**over) != 0, over
        assert b"linear_tc_rows" in lib.dmpnn_last_error(), over
    assert call(R=0) == 0                                                            # nothing to do
    assert call(R=0, **mirror) == 0
    with pytest.raises(_lib.DmpnnError):
        _lib.check(call(N=0), "dmpnn_linear_tc_rows_bf16")
