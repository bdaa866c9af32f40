"""GPU tier: the fused depth step on atoms of in-degree above four -- hypervalent S / P (degree 5-6) and condensed reaction
graphs, whose atoms carry the union of reactant and product bonds.  There the message warps leave the packed-bf16 sums
(<= 3 siblings, <= 4 neighbours) for an f32 loop with its own indexing, and the ATOM kernel's tiles hold more edge rows than
its staged neighbour table (512 entries), so the gather reads the global table.  Batches: make_molecule(max_deg=6) plus
complete graphs K_6 .. K_12 (in-degree 5 .. 11), shuffled edge order.  Kernels against torch with the kernel's rounding
points (tests/emu.py: packed bf16 for small in-degree, f32 with one rounding above), modules against the oracle and the
rounding-aware emulation."""
from __future__ import annotations

from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

RTOL, ATOL = 2 ** -6, 2e-2          # the tolerances of tests/test_gpu_fused_step.py


def _complete_graph(rng, k: int, d_v: int = 72, d_e: int = 14):
    """K_k as a MolGraph in the featuriser's edge convention (2i: u -> v, 2i + 1: v -> u), then shuffled."""
    from chemprop_b200.data.molgraph import MolGraph

    bonds = [(u, v) for u in range(k) for v in range(u + 1, k)]
    nb = len(bonds)
    ei = np.array([e for u, v in bonds for e in ((u, v), (v, u))], dtype=np.int64).T
    rev = np.arange(2 * nb, dtype=np.int64).reshape(-1, 2)[:, ::-1].ravel()
    V = np.zeros((k, d_v), dtype=np.float32)
    V[np.arange(k)[:, None], rng.integers(0, d_v - 1, size=(k, 7))] = 1.0
    V[:, -1] = rng.uniform(0.01, 0.4, size=k)
    E = np.repeat(rng.uniform(0.0, 1.0, size=(nb, d_e)).astype(np.float32), 2, axis=0)
    p = rng.permutation(2 * nb)
    inv = np.empty_like(p)
    inv[p] = np.arange(2 * nb)
    return MolGraph(V=V, E=E[p], edge_index=ei[:, p], rev_edge_index=inv[rev[p]])


def high_degree_molecules(n_mols: int, seed: int, kmax: int = 12, reps: int = 3, big: int = 0, d_v: int = 72, d_e: int = 14):
    """n_mols molecules of 6-30 atoms with atom degree up to 6, `reps` copies of each K_6 .. K_kmax, and `big` molecules of
    70-100 atoms with degree up to 6 (more than 128 directed edges); shuffled molecule order."""
    from chemprop_b200.data import make_molecule

    rng = np.random.default_rng(seed)
    mgs = [make_molecule(rng, int(rng.integers(6, 31)), d_v, d_e, ring_frac=0.25, max_deg=6, shuffle_edges=True)
           for _ in range(n_mols)]
    mgs += [_complete_graph(rng, k, d_v, d_e) for k in range(6, kmax + 1) for _ in range(reps)]
    mgs += [make_molecule(rng, int(rng.integers(70, 101)), d_v, d_e, ring_frac=0.25, max_deg=6, shuffle_edges=True)
            for _ in range(big)]
    return [mgs[i] for i in rng.permutation(len(mgs))]


def _layout(mgs):
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.engine import get_layout

    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    cpu = SimpleNamespace(E=lay.E, V=lay.V, rowptr=lay.rowptr.cpu(), dst_row=lay.dst_row.cpu(), rev_row=lay.rev_row.cpu(),
                          src_row=lay.src_row.cpu())
    return lay, cpu


def _hidden(rows, h, seed, relu=False):
    from chemprop_b200.engine import pad_hidden

    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.zeros(rows, pad_hidden(h), dtype=torch.bfloat16, device="cuda")
    x = torch.randn(rows, h, device="cuda", generator=g) * 0.7
    t[:, :h] = (torch.relu(x) if relu else x).bfloat16()
    return t


def _weights(h, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    return W, torch.randn(h, device="cuda", generator=g) * 0.1


def _close(got, ref, atol=ATOL):
    torch.testing.assert_close(got.float().cpu(), ref.float().cpu(), rtol=RTOL, atol=atol)


def _bond_ref_fwd(cpu, Hin, H0, W, b, h, first):
    from tests.emu import _bf, _sibling_sum_packed

    f = Hin[:, :h].float().cpu()
    if first:
        f = _bf(torch.relu(f))
    A = _sibling_sum_packed(f, cpu, through_rev=False)      # A row r = message of edge rev(r)
    M = torch.zeros_like(A)
    M[cpu.rev_row.long()] = A
    Z = M @ _bf(W.cpu()).t() + H0[:, :h].float().cpu() + b.cpu()
    return _bf(torch.relu(Z)), M


def _flagged_rows_with_high_indeg(lay, cpu):
    """(number of flagged windows, max in-degree of the destination atom over the rows of flagged windows)"""
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    if wf is None:
        return 0, 0
    n = int(nw.item())
    rows, flags = trp[: n + 1].cpu().numpy(), wf[:n].cpu().numpy()
    indeg = (cpu.rowptr[1:] - cpu.rowptr[:-1]).numpy()[cpu.dst_row.numpy()]
    hi = max((int(indeg[rows[i]:rows[i + 1]].max()) for i in range(n) if flags[i] and rows[i + 1] > rows[i]), default=0)
    return int(flags.sum()), hi


@pytest.mark.parametrize("windows", [False, True], ids=["tiles", "windows"])
@pytest.mark.parametrize("first", [True, False], ids=["first", "later"])
def test_bond_step_high_indegree(first, windows):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_fused, pack_weight_bf16

    h = 300
    mgs = high_degree_molecules(300, seed=1, kmax=12 if windows else 11, big=6 if windows else 0)
    lay, cpu = _layout(mgs)
    assert lay.max_indeg >= 5 and (lay.max_tile_rows > 128) == windows
    if windows:
        n_flag, hi = _flagged_rows_with_high_indeg(lay, cpu)
        assert n_flag >= 6 and hi >= 5, (n_flag, hi)
    H0, Hp = _hidden(lay.E, h, 2), _hidden(lay.E, h, 3, relu=True)
    W, b = _weights(h, 4)
    Hin = H0 if first else Hp
    Hn = torch.full_like(H0, float("nan"))
    M1 = torch.full_like(H0, float("nan")) if first else None
    bond_step_fused(Hin, H0, Hn, h, pack_weight_bf16(W), b, lay, _lib.ACT_RELU, 0.0, first, M_out=M1)
    torch.cuda.synchronize()
    ref, M = _bond_ref_fwd(cpu, Hin, H0, W, b, h, first)
    assert bool(torch.isfinite(Hn[:, :h].float()).all())
    _close(Hn[:, :h], ref)
    if first:
        _close(M1[:, :h], M)


@pytest.mark.parametrize("windows", [False, True], ids=["tiles", "windows"])
@pytest.mark.parametrize("mode,n_add", [("mask", 0), ("copy", 0), ("last", 0), ("last", 1), ("last", 2)])
def test_bond_mirror_high_indegree(mode, n_add, windows):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_bwd_fused, pack_weight_bf16
    from tests.emu import _bf, _dact, _sibling_sum_packed

    h = 300
    mgs = high_degree_molecules(300, seed=5, kmax=12 if windows else 11, big=6 if windows else 0)
    lay, cpu = _layout(mgs)
    assert lay.max_indeg >= 5 and (lay.max_tile_rows > 128) == windows
    if windows:
        n_flag, hi = _flagged_rows_with_high_indeg(lay, cpu)
        assert n_flag >= 6 and hi >= 5, (n_flag, hi)
    dZ, Y, H0 = _hidden(lay.E, h, 6), _hidden(lay.E, h, 7, relu=True), _hidden(lay.E, h, 8)
    adds = [_hidden(lay.E, h, 9 + i) for i in range(n_add)]
    W, _ = _weights(h, 10)
    out = torch.full_like(dZ, float("nan"))
    G = torch.full_like(dZ, float("nan"))
    Yk = {"mask": Y, "copy": None, "last": H0}[mode]
    bond_step_bwd_fused(dZ, Yk, out, h, pack_weight_bf16(W.t().contiguous()), lay, _lib.ACT_RELU, 0.0, G_out=G,
                        y_is_preact=(mode == "last"), addends=tuple(adds))
    torch.cuda.synchronize()
    Gref = _sibling_sum_packed(dZ[:, :h].float().cpu(), cpu, through_rev=True)
    D = Gref @ _bf(W.cpu())
    if Yk is not None:
        D = D * _dact(Yk[:, :h].float().cpu(), _lib.ACT_RELU, 0.0, mode == "last")
    for a in adds:
        D = D + a[:, :h].float().cpu()
    _close(G[:, :h], Gref)
    assert bool(torch.isfinite(out[:, :h].float()).all())
    _close(out[:, :h], _bf(D), atol=6.5e-2 if n_add else 3e-2)


def _atom_batch(seed):
    from chemprop_b200.engine import atom_tables

    mgs = high_degree_molecules(200, seed=seed, kmax=12, reps=20)
    lay, cpu = _layout(mgs)
    ta, te, info, _ = atom_tables(lay)
    indeg = (cpu.rowptr[1:] - cpu.rowptr[:-1])
    assert lay.max_tile_atoms <= 128 and int(indeg.max()) == 11 and int((indeg >= 5).sum()) >= 500
    assert int(info[1]) > 512, int(info[1])              # tiles with more edge rows than the staged neighbour table
    return lay, cpu


@pytest.mark.parametrize("first", [True, False], ids=["first", "later"])
def test_atom_step_high_indegree(first):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import atom_step_fused, pack_weight_bf16
    from tests.emu import _bf, _neighbour_sum_packed

    h = 300
    lay, cpu = _atom_batch(seed=11)
    H0, Hp = _hidden(lay.V, h, 12), _hidden(lay.V, h, 13, relu=True)
    W, b = _weights(h, 14)
    Hin = H0 if first else Hp
    Hn = torch.full_like(H0, float("nan"))
    N1 = torch.full_like(H0, float("nan")) if first else None
    atom_step_fused(Hin, H0, Hn, h, pack_weight_bf16(W), b, lay, _lib.ACT_RELU, 0.0, first, N_out=N1)
    torch.cuda.synchronize()
    f = Hin[:, :h].float().cpu()
    if first:
        f = _bf(torch.relu(f))
    N = _neighbour_sum_packed(f, cpu)
    ref = _bf(torch.relu(N @ _bf(W.cpu()).t() + H0[:, :h].float().cpu() + b.cpu()))
    assert bool(torch.isfinite(Hn[:, :h].float()).all())
    _close(Hn[:, :h], ref)
    if first:
        _close(N1[:, :h], N)


@pytest.mark.parametrize("mode", ["mask", "copy", "last"])
def test_atom_mirror_high_indegree(mode):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import atom_step_bwd_fused, pack_weight_bf16
    from tests.emu import _bf, _dact, _neighbour_sum_packed

    h = 300
    lay, cpu = _atom_batch(seed=15)
    dZ, Y, H0 = _hidden(lay.V, h, 16), _hidden(lay.V, h, 17, relu=True), _hidden(lay.V, h, 18)
    W, _ = _weights(h, 19)
    out = torch.full_like(dZ, float("nan"))
    G = torch.full_like(dZ, float("nan"))
    Yk = {"mask": Y, "copy": None, "last": H0}[mode]
    atom_step_bwd_fused(dZ, Yk, out, h, pack_weight_bf16(W.t().contiguous()), lay, _lib.ACT_RELU, 0.0, G_out=G,
                        y_is_preact=(mode == "last"))
    torch.cuda.synchronize()
    Gref = _neighbour_sum_packed(dZ[:, :h].float().cpu(), cpu)
    D = Gref @ _bf(W.cpu())
    if Yk is not None:
        D = D * _dact(Yk[:, :h].float().cpu(), _lib.ACT_RELU, 0.0, mode == "last")
    _close(G[:, :h], Gref)
    assert bool(torch.isfinite(out[:, :h].float()).all())
    _close(out[:, :h], _bf(D), atol=3e-2)


def _grad_close(got, ref, rel, what, rel_max=None):
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = max(1e-6, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    fro = ((got - ref).norm() / max(1e-12, ref.norm().item())).item()
    assert err <= (rel if rel_max is None else rel_max) * scale and fro <= rel, (what, err, scale, fro)


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_module_high_indegree_vs_oracle_and_emulation(kind):
    """Bond / AtomMessagePassing(precision="bf16") on a high-degree batch, forward + every weight gradient: against the f64
    oracle (hidden states within 1e-2 of their scale, gradients within 6 % in the Frobenius norm) and against the
    rounding-aware emulation of the same tier (gradients within 2 %, max and Frobenius).  The oracle's max-abs bound is 20 %:
    on this batch bf16 storage alone moves single entries that far -- the emulation, which rounds where the kernels store
    bf16, is 13 % off the oracle in the largest entry of the atom kind's W_i gradient (|H| reaches ~45 with 11 neighbours)."""
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.engine import get_layout
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation
    from oracle import restatement as R
    from tests import emu

    mgs = high_degree_molecules(400, seed=21, kmax=12, reps=4)
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    torch.manual_seed(3)
    state = {k: v.detach().clone() for k, v in cls(d_h=300, depth=3, bias=True).state_dict().items()}
    Gm = torch.randn(len(mgs), 300, generator=torch.Generator().manual_seed(5))

    def make(device):
        mp = cls(d_h=300, depth=3, bias=True, precision="bf16")
        mp.load_state_dict(state)
        return mp.to(device)

    loss_fn = lambda H, b: (MeanAggregation()(H, b.batch).float() * Gm.to(H.device)).sum()  # noqa: E731
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    assert lay.max_indeg >= 11
    mp = make("cuda")
    H = mp(bmg)
    loss_fn(H, bmg).backward()
    with pytest.MonkeyPatch.context() as mpatch:
        emu.patch_engine(mpatch)
        mpe, bme = make("cpu"), BatchMolGraph(mgs)
        He = mpe(bme)
        loss_fn(He, bme).backward()
    bm = BatchMolGraph(mgs)
    P = {k: v.double().requires_grad_(True) for k, v in state.items()}
    H_ref = R.message_passing_forward(kind, bm.V.double(), bm.E.double(), bm.edge_index, bm.rev_edge_index,
                                      P["W_i.weight"], P["W_i.bias"], P["W_h.weight"], P["W_h.bias"], P["W_o.weight"],
                                      P["W_o.bias"], 3)
    (R.aggregate(H_ref, bm.batch, "mean") * Gm.double()).sum().backward()
    tol = 1e-2 * max(1.0, H_ref.detach().abs().max().item())
    assert (H.detach().double().cpu() - H_ref.detach()).abs().max().item() <= tol
    for k, p in mp.named_parameters():
        _grad_close(p.grad, dict(mpe.named_parameters())[k].grad, 2e-2, (k, "vs emulation"))
        _grad_close(p.grad, P[k].grad, 6e-2, (k, "vs f64 oracle"), rel_max=0.2)
