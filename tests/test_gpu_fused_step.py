"""GPU tier: the fused wgmma depth-step kernel (dmpnn_bond_step_fused_bf16) against a plain
PyTorch fp32 reference of the same op that emulates its roundings (bf16 message, bf16 W_h, fp32
accumulate), and against the unfused fp32-accurate kernels."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _setup(n_mols, h, seed, shuffle=True, min_atoms=2, big=0):
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import get_layout, pad_hidden

    mgs = make_molecules(n_mols, seed=seed, shuffle_edges=shuffle, min_atoms=min_atoms)
    if big:        # molecules of ~130 .. 400 directed edges scattered through the batch: more rows than one 128-row tile
        bigs = make_molecules(big, seed=seed + 1, mean_atoms=110.0, std_atoms=40.0, min_atoms=66, max_atoms=200,
                              shuffle_edges=shuffle)
        step = max(1, len(mgs) // big)
        for i, m in enumerate(bigs):
            mgs.insert(min(len(mgs), i * step + 1), m)
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    hp = pad_hidden(h)
    g = torch.Generator(device="cuda").manual_seed(seed)
    H0 = torch.zeros(lay.E, hp, dtype=torch.bfloat16, device="cuda")
    H0[:, :h] = (torch.randn(lay.E, h, device="cuda", generator=g) * 0.7).bfloat16()
    Hp = torch.zeros_like(H0)
    Hp[:, :h] = torch.relu(torch.randn(lay.E, h, device="cuda", generator=g)).bfloat16()
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    return lay, H0, Hp, W, b, hp


def _torch_reference(lay, Hin, H0, W, b, h, act, first):
    """fp32 torch restatement of the fused op with the kernel's rounding points."""
    tau = {"relu": torch.relu, "tanh": torch.tanh}[act]
    X = Hin[:, :h].float()
    if first:
        X = tau(X)
    dst = lay.dst_row.long()
    A = torch.zeros(lay.V, h, device=X.device).index_add_(0, dst, X)       # per-atom sums over in-edges
    Mt = (A[dst] - X).bfloat16().float()                                    # row e' holds M[rev(e')] (bf16)
    Z = Mt @ W.bfloat16().float().t()
    rev = lay.rev_row.long()
    out = torch.zeros_like(Hin)
    z = Z + H0[rev, :h].float() + (b if b is not None else 0.0)
    out[rev, :h] = tau(z).bfloat16()
    return out


@pytest.mark.parametrize("h,first,act,bias", [
    (300, False, "relu", False), (300, True, "relu", False), (300, False, "tanh", True), (64, False, "relu", True),
    (128, True, "tanh", False), (200, False, "relu", False), (160, False, "relu", True), (16, False, "relu", False),
    (304, False, "relu", False),
])
def test_fused_step_vs_torch_reference(h, first, act, bias):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_fused, pack_weight_bf16

    lay, H0, Hp, W, b, hp = _setup(700, h, seed=h + int(first))
    assert lay.max_tile_rows <= 128
    Hin = H0 if first else Hp
    code = {"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    Wpk = pack_weight_bf16(W)
    Hn = torch.zeros_like(H0)
    Hn[:, :h] = float("nan")                   # every data column must be written; the row padding stays zero
    M1 = torch.full_like(H0, float("nan")) if first else None   # first step: the consumed message is also stored
    bond_step_fused(Hin, H0, Hn, h, Wpk, b if bias else None, lay, code, 0.0, first, M_out=M1)
    torch.cuda.synchronize()
    ref = _torch_reference(lay, Hin, H0, W, b if bias else None, h, act, first)
    if first:
        tau = {"relu": torch.relu, "tanh": torch.tanh}[act]
        X, dst, rev = tau(H0[:, :h].float()), lay.dst_row.long(), lay.rev_row.long()
        Mref = torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)[dst[rev]] - X[rev]   # M[e] (mixins.py:11-18)
        torch.testing.assert_close(M1[:, :h].float(), Mref.bfloat16().float(), rtol=2 ** -6, atol=2e-2)
    assert torch.isfinite(Hn.float()).all(), "rows/columns left unwritten"
    assert hp == h or float(Hn[:, h:].float().abs().max()) == 0.0, "row padding must stay zero"
    torch.testing.assert_close(Hn.float(), ref.float(), rtol=2 ** -6, atol=2e-2)   # a couple of bf16 ulps (message summed in packed bf16)
    assert (Hn.float() - ref.float()).abs().mean().item() <= 1e-3


def test_fused_step_matches_unfused_kernels():
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_message, bond_step_fused, linear_fwd, pack_weight_bf16

    h = 300
    lay, H0, Hp, W, b, hp = _setup(2500, h, seed=3)
    Hn = torch.zeros_like(H0)
    bond_step_fused(Hp, H0, Hn, h, pack_weight_bf16(W), b, lay, _lib.ACT_RELU, 0.0, False)
    M = torch.zeros_like(H0)
    bond_message(Hp, lay, h, M)
    Hu = torch.zeros_like(H0)
    linear_fwd(M, h, W.contiguous(), Hu, h, bias=b, res=H0, act=_lib.ACT_RELU, R=lay.E, pad_to=hp)
    torch.cuda.synchronize()
    err = (Hn.float() - Hu.float()).abs().max().item()
    assert err <= 5e-2, err      # bf16 W_h in the fused kernel vs f32 W_h in the SIMT kernel


def test_fused_step_many_tiles_and_single_atoms():
    """More tiles than SMs (persistent loop wraps) + 1-atom molecules (zero-row atoms inside tiles)."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_fused, pack_weight_bf16

    h = 96
    lay, H0, Hp, W, b, hp = _setup(4000, h, seed=9, min_atoms=1)
    assert lay.n_tiles > 132 * 2     # more than two waves of the H100's 132 SMs
    Hn = torch.zeros_like(H0)
    Hn[:, :h] = float("nan")
    bond_step_fused(Hp, H0, Hn, h, pack_weight_bf16(W), None, lay, _lib.ACT_RELU, 0.0, False)
    torch.cuda.synchronize()
    ref = _torch_reference(lay, Hp, H0, W, None, h, "relu", False)
    assert torch.isfinite(Hn.float()).all()
    torch.testing.assert_close(Hn.float(), ref.float(), rtol=2 ** -6, atol=2e-2)


def test_fused_rejects_unsupported():
    from chemprop_b200 import DmpnnError, _lib
    from chemprop_b200.engine import bond_step_fused

    lay, H0, Hp, W, b, hp = _setup(10, 64, seed=1)
    with pytest.raises(DmpnnError):
        bond_step_fused(Hp, H0, torch.zeros_like(H0), 400, torch.zeros(16, dtype=torch.uint8, device="cuda"), None,
                        lay, _lib.ACT_RELU, 0.0, False)


@pytest.mark.parametrize("h,act,masked", [(300, "relu", True), (300, "relu", False), (64, "tanh", True), (200, "relu", True)])
def test_fused_backward_step_vs_torch_reference(h, act, masked):
    """Autograd mirror of the depth step on the fused kernel: dOut = (S.P)(dZ . W_h) * tau'(Y)."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_bwd_fused, pack_weight_bf16

    lay, H0, Hp, W, b, hp = _setup(900, h, seed=17 + h)
    g = torch.Generator(device="cuda").manual_seed(5)
    dZ = torch.zeros_like(H0)
    dZ[:, :h] = torch.randn(lay.E, h, device="cuda", generator=g).bfloat16()
    Y = Hp if act == "relu" else torch.tanh(H0.float()).bfloat16()
    out = torch.zeros_like(H0)
    out[:, :h] = float("nan")
    code = {"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    Gk = torch.full_like(H0, float("nan"))
    bond_step_bwd_fused(dZ, Y if masked else None, out, h, pack_weight_bf16(W.t().contiguous()), lay, code, 0.0, G_out=Gk)
    torch.cuda.synchronize()
    # reference: dM = dZ . W_h ; dH[e] = sum_{x in seg(e)} dM[rev x] - dM[rev e] ; times tau'(Y)
    rev, dst = lay.rev_row.long(), lay.dst_row.long()
    X = dZ[:, :h].float()[rev]                                            # (P dZ)
    A = torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)
    torch.testing.assert_close(Gk[:, :h].float(), (A[dst] - X).bfloat16().float(), rtol=2 ** -6, atol=2e-2)   # (S.P) dZ
    # the GEMM's A operand as the kernel rounds it: packed-bf16 sibling sums (<= 2 roundings), tests/emu.py
    from types import SimpleNamespace

    from tests.emu import _sibling_sum_packed

    lay_cpu = SimpleNamespace(E=lay.E, V=lay.V, rowptr=lay.rowptr.cpu(), dst_row=lay.dst_row.cpu(), rev_row=lay.rev_row.cpu())
    SP = _sibling_sum_packed(dZ[:, :h].float().cpu(), lay_cpu, through_rev=True).cuda()
    G = SP @ W.bfloat16().float()                                         # ((S.P) dZ) . W_h   (W_h: out x in)
    if masked:
        y = Y[:, :h].float()
        G = G * ((y > 0).float() if act == "relu" else (1 - y * y))
    assert torch.isfinite(out.float()).all()
    torch.testing.assert_close(out[:, :h].float(), G.bfloat16().float(), rtol=2 ** -6, atol=2e-2)
    assert hp == h or float(out[:, h:].float().abs().max()) == 0.0


@pytest.mark.parametrize("h,act,n_add", [(300, "relu", 2), (300, "relu", 1), (64, "tanh", 2), (200, "relu", 0)])
def test_fused_backward_last_step_masks_from_preactivation_and_sums(h, act, n_add):
    """t = 1 mirror step: dH_0 = ((S.P) dZ . W_h) * tau'(H_0) + addends, one rounding after the f32 sum."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_bwd_fused, pack_weight_bf16

    lay, H0, Hp, W, b, hp = _setup(900, h, seed=29 + h)
    g = torch.Generator(device="cuda").manual_seed(7)

    def rnd():
        t = torch.zeros_like(H0)
        t[:, :h] = torch.randn(lay.E, h, device="cuda", generator=g).bfloat16()
        return t

    dZ = rnd()
    adds = [dZ, rnd()][:n_add]                      # the step's own input is one of the addends in the engine
    out = torch.full_like(H0, float("nan"))
    code = {"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    bond_step_bwd_fused(dZ, H0, out, h, pack_weight_bf16(W.t().contiguous()), lay, code, 0.0, y_is_preact=True,
                        addends=tuple(adds))
    torch.cuda.synchronize()
    rev, dst = lay.rev_row.long(), lay.dst_row.long()
    X = dZ[:, :h].float()[rev]
    A = torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)
    G = (A[dst] - X).bfloat16().float() @ W.bfloat16().float()
    z = H0[:, :h].float()
    G = (G * ((z > 0).float() if act == "relu" else (1 - torch.tanh(z) ** 2))).bfloat16().float()   # staged in bf16
    for a in adds:
        G = G + a[:, :h].float()
    torch.testing.assert_close(out[:, :h].float(), G.bfloat16().float(), rtol=2 ** -6, atol=6.5e-2)   # 2 ulp at |x| in [4, 8): cancelling terms
    pad16 = (h + 15) // 16 * 16
    assert pad16 == h or float(out[:, h:pad16].float().abs().max()) == 0.0
    with pytest.raises(Exception):                  # addends are a property of the pre-activation (last) mode
        bond_step_bwd_fused(dZ, Hp, out, h, pack_weight_bf16(W.t().contiguous()), lay, code, 0.0, addends=(dZ,))


@pytest.mark.parametrize("h,first,act", [(300, False, "relu"), (300, True, "relu"), (64, False, "tanh")])
def test_fused_step_molecules_larger_than_a_tile(h, first, act):
    """Molecules with more than 128 directed edges (condensed reaction graphs): their tiles run as 128-row windows of the
    same kernel, siblings / reverse edges outside the window gathered from global memory (Layout.step_tables)."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_fused, pack_weight_bf16

    lay, H0, Hp, W, b, hp = _setup(300, h, seed=41 + h, big=25)
    assert lay.max_tile_rows > 128
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    n_work = int(nw.item())
    rows = trp[: n_work + 1].cpu().numpy()
    assert n_work > nt and (np.diff(rows) <= 128).all() and (np.diff(rows) >= 0).all() and rows[-1] == lay.E
    assert int(wf[:n_work].sum()) >= 2 * 25 - 5
    Hin = H0 if first else Hp
    code = {"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    Hn = torch.zeros_like(H0)
    Hn[:, :h] = float("nan")
    M1 = torch.full_like(H0, float("nan")) if first else None
    bond_step_fused(Hin, H0, Hn, h, pack_weight_bf16(W), b, lay, code, 0.0, first, M_out=M1)
    torch.cuda.synchronize()
    ref = _torch_reference(lay, Hin, H0, W, b, h, act, first)
    assert torch.isfinite(Hn.float()).all(), "rows/columns left unwritten"
    torch.testing.assert_close(Hn.float(), ref.float(), rtol=2 ** -6, atol=2e-2)
    if first:
        tau = {"relu": torch.relu, "tanh": torch.tanh}[act]
        X, dst, rev = tau(H0[:, :h].float()), lay.dst_row.long(), lay.rev_row.long()
        Mref = torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)[dst[rev]] - X[rev]
        torch.testing.assert_close(M1[:, :h].float(), Mref.bfloat16().float(), rtol=2 ** -6, atol=2e-2)


def test_fused_backward_step_molecules_larger_than_a_tile():
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_bwd_fused, pack_weight_bf16

    h = 300
    lay, H0, Hp, W, b, hp = _setup(300, h, seed=77, big=25)
    assert lay.max_tile_rows > 128
    g = torch.Generator(device="cuda").manual_seed(5)
    dZ = torch.zeros_like(H0)
    dZ[:, :h] = torch.randn(lay.E, h, device="cuda", generator=g).bfloat16()
    out = torch.zeros_like(H0)
    out[:, :h] = float("nan")
    Gk = torch.full_like(H0, float("nan"))
    bond_step_bwd_fused(dZ, Hp, out, h, pack_weight_bf16(W.t().contiguous()), lay, _lib.ACT_RELU, 0.0, G_out=Gk)
    torch.cuda.synchronize()
    rev, dst = lay.rev_row.long(), lay.dst_row.long()
    X = dZ[:, :h].float()[rev]
    A = torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)
    torch.testing.assert_close(Gk[:, :h].float(), (A[dst] - X).bfloat16().float(), rtol=2 ** -6, atol=2e-2)
    G = ((A[dst] - X).bfloat16().float() @ W.bfloat16().float()) * (Hp[:, :h].float() > 0).float()
    assert torch.isfinite(out.float()).all()
    torch.testing.assert_close(out[:, :h].float(), G.bfloat16().float(), rtol=2 ** -6, atol=2e-2)


# ---- atom-granular step (ATOM instantiations of the same kernel: dmpnn_atom_step_fused_bf16) ---------------------------
def _atom_setup(n_mols, h, seed, cgr=False, mean_atoms=25.0):
    from chemprop_b200.data import BatchMolGraph, make_cgr_graphs, make_molecules
    from chemprop_b200.engine import get_layout, pad_hidden

    mgs = make_cgr_graphs(n_mols, seed=seed) if cgr else make_molecules(n_mols, seed=seed, shuffle_edges=True, min_atoms=1,
                                                                         mean_atoms=mean_atoms)
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    hp = pad_hidden(h)
    g = torch.Generator(device="cuda").manual_seed(seed)
    H0 = torch.zeros(lay.V, hp, dtype=torch.bfloat16, device="cuda")
    H0[:, :h] = (torch.randn(lay.V, h, device="cuda", generator=g) * 0.7).bfloat16()
    Hp = torch.zeros_like(H0)
    Hp[:, :h] = torch.relu(torch.randn(lay.V, h, device="cuda", generator=g)).bfloat16()
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    return lay, H0, Hp, W, b, hp


def _neighbour_sum(lay, X):
    """sum over the in-edges e of v of X[src(e)] with the kernel's rounding points: in slot order as packed bf16 (a rounding
    after every add) for in-degree <= 4, in f32 with one rounding beyond.  X: bf16-valued f32."""
    V, dev = lay.V, X.device
    rowptr, src = lay.rowptr.long(), lay.src_row.long()
    g0 = rowptr[:V]
    d = rowptr[1:V + 1] - g0
    acc = torch.zeros(V, X.shape[1], device=dev)
    for k in range(4):
        ok = (k < d) & (d <= 4)
        x = src[torch.clamp(g0 + k, max=max(lay.E - 1, 0))]
        acc = (acc + X[x] * ok.unsqueeze(1).float()).bfloat16().float()
    big = d > 4
    if bool(big.any()):
        s = torch.zeros(V, X.shape[1], device=dev).index_add_(0, lay.dst_row.long(), X[src])
        acc = torch.where(big.unsqueeze(1), s.bfloat16().float(), acc)
    return acc


@pytest.mark.parametrize("h,first,act,bias,cgr", [
    (300, False, "relu", False, False), (300, True, "relu", False, False), (300, False, "tanh", True, True),
    (64, False, "relu", True, False), (128, True, "tanh", False, True), (304, False, "relu", False, True),
    (16, True, "relu", True, False),
])
def test_atom_fused_step_vs_torch_reference(h, first, act, bias, cgr):
    """H_next[v] = tau(H_0[v] + b + W . sum_{e in in(v)} g(H[src e])): the ATOM gather (tile-local neighbour table, packed-bf16
    sums for in-degree <= 3, f32 beyond) + the shared GEMM / epilogue, against torch with the kernel's rounding points."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import atom_step_fused, pack_weight_bf16

    lay, H0, Hp, W, b, hp = _atom_setup(90 if cgr else 700, h, seed=h + int(first), cgr=cgr)
    assert lay.max_tile_atoms <= 128
    tau = {"relu": torch.relu, "tanh": torch.tanh}[act]
    code = {"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    Hin = H0 if first else Hp
    Hn = torch.full_like(H0, float("nan"))
    Hn[:, h:] = 0
    N1 = torch.full_like(H0, float("nan")) if first else None
    atom_step_fused(Hin, H0, Hn, h, pack_weight_bf16(W), b if bias else None, lay, code, 0.0, first, N_out=N1)
    torch.cuda.synchronize()
    X = Hin[:, :h].float()
    if first:
        X = tau(X).bfloat16().float()
    N = _neighbour_sum(lay, X)
    ref = tau(N @ W.bfloat16().float().t() + H0[:, :h].float() + (b if bias else 0.0)).bfloat16().float()
    assert torch.isfinite(Hn.float()).all(), "rows/columns left unwritten"
    assert hp == h or float(Hn[:, h:].float().abs().max()) == 0.0
    if first:
        torch.testing.assert_close(N1[:, :h].float(), N, rtol=2 ** -6, atol=2e-2)
    torch.testing.assert_close(Hn[:, :h].float(), ref, rtol=2 ** -6, atol=2e-2)


@pytest.mark.parametrize("mode", ["mask", "copy", "last"])
@pytest.mark.parametrize("cgr", [False, True])
def test_atom_fused_backward_step(mode, cgr):
    """Mirror: dOut = ((A dZ) . W) [* tau'(Y)], G_out = A dZ, with A the symmetric atom adjacency."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import atom_step_bwd_fused, pack_weight_bf16

    h = 300
    lay, Ypre, Yact, W, _, hp = _atom_setup(80 if cgr else 600, h, seed=11, cgr=cgr)
    g = torch.Generator(device="cuda").manual_seed(5)
    dZ = torch.zeros_like(Ypre)
    dZ[:, :h] = torch.randn(lay.V, h, device="cuda", generator=g).bfloat16()
    dOut = torch.full_like(Ypre, float("nan"))
    dOut[:, h:] = 0
    G = torch.full_like(Ypre, float("nan"))
    Y = None if mode == "copy" else (Ypre if mode == "last" else Yact)
    atom_step_bwd_fused(dZ, Y, dOut, h, pack_weight_bf16(W.t().contiguous()), lay, _lib.ACT_RELU, 0.0, G_out=G,
                        y_is_preact=(mode == "last"))
    torch.cuda.synchronize()
    Gref = _neighbour_sum(lay, dZ[:, :h].float())
    D = Gref @ W.bfloat16().float()
    if Y is not None:
        D = D * (Y[:, :h].float() > 0).float()
    torch.testing.assert_close(G[:, :h].float(), Gref, rtol=2 ** -6, atol=2e-2)
    torch.testing.assert_close(dOut[:, :h].float(), D.bfloat16().float(), rtol=2 ** -6, atol=3e-2)


def test_atom_tiles_cover_the_batch():
    """dmpnn_tiles_build with the atom limits: tiles are runs of whole molecules, <= 128 atoms each, covering every atom once;
    the greedy rule (restarted every 1024 molecules) checked against a host walk."""
    from chemprop_b200.engine import atom_tables

    lay, *_ = _atom_setup(2500, 64, seed=3, mean_atoms=30.0)
    ta, te, info, _ = atom_tables(lay)
    n = int(info[0])
    ta, te = ta[: n + 1].cpu().numpy(), te[: n + 1].cpu().numpy()
    mol_a, mol_r = lay.mol_atom_ptr.cpu().numpy(), lay.mol_row_ptr.cpu().numpy()
    exp_a, B, m = [], lay.B, 0
    while m < B:
        stop = min(B, (m // 1024 + 1) * 1024)
        j = m + 1
        while j < stop and mol_a[j + 1] - mol_a[m] <= 128 and mol_r[j + 1] - mol_r[m] <= 1024:
            j += 1
        exp_a.append(mol_a[m])
        m = j
    exp_a.append(mol_a[B])
    assert ta.tolist() == exp_a
    assert ta[0] == 0 and ta[-1] == lay.V and te[-1] == lay.E and int(info[2]) <= 128
    rowptr = lay.rowptr.cpu().numpy()
    assert (te == rowptr[ta]).all()
