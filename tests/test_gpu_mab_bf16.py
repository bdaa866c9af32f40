"""GPU tier: MABBond / MABAtomMessagePassing(precision="bf16") on the real kernels -- dmpnn_linear_tc_rows_bf16 against torch
in both modes, then the modules against the goldens, the oracle, the rounding-aware emulation and themselves (bit-for-bit) and
a training step captured with CudaGraphStep."""
from __future__ import annotations

import pytest
import torch

from chemprop_b200 import _lib, engine
from tests.test_gpu_fused_activations import U, _check_bound, _dtau64, _lip, _tau64
from tests.test_mab_bf16_host import BF16_GOLDENS, _close_bf16, _golden_module, sweep_case
from tests.util import load_golden

pytestmark = pytest.mark.gpu

ACTS = [(_lib.ACT_NONE, 0.0), (_lib.ACT_RELU, 0.0), (_lib.ACT_LEAKYRELU, 0.1), (_lib.ACT_TANH, 0.0), (_lib.ACT_ELU, 1.0)]
_NAME = {_lib.ACT_NONE: "none", _lib.ACT_RELU: "relu", _lib.ACT_LEAKYRELU: "leakyrelu", _lib.ACT_TANH: "tanh",
         _lib.ACT_ELU: "elu"}


def _act(x, act, p):
    return {_lib.ACT_NONE: lambda: x, _lib.ACT_RELU: lambda: torch.relu(x), _lib.ACT_LEAKYRELU: lambda: torch.where(x > 0, x, p * x),
            _lib.ACT_TANH: lambda: torch.tanh(x), _lib.ACT_ELU: lambda: torch.where(x > 0, x, p * torch.expm1(x))}[act]()


@pytest.mark.parametrize("N", [40, 64, 300])
@pytest.mark.parametrize("act, ap", ACTS)
def test_rows_kernel_forward_mode(N, act, ap):
    """C = act(A . W^T + b) with f32 and bf16 stores; R = 300 (not a multiple of the 128-row tile), K = 14 + N."""
    g = torch.Generator().manual_seed(N + act)
    R, K = 300, 14 + N
    A = torch.randn(R, K, generator=g).to(torch.bfloat16)
    W, b = torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g)
    Ad = torch.zeros(R, (K + 15) // 16 * 16, dtype=torch.bfloat16, device="cuda")
    Ad[:, :K] = A.cuda()
    Wpk = engine.pack_weight_tc(W.cuda())
    out32 = torch.full((R, N), float("nan"), device="cuda")
    engine.linear_tc_rows(Ad, K, Wpk, N, out32, bias=b.cuda(), act=act, act_param=ap)
    n16 = (N + 15) // 16 * 16
    out16 = torch.full((R, engine.pad_hidden(N)), float("nan"), dtype=torch.bfloat16, device="cuda")
    engine.linear_tc_rows(Ad, K, Wpk, N, out16, bias=b.cuda(), act=act, act_param=ap)
    # float64 with the kernel's rounding points (tests/test_gpu_fused_activations.py): the f32 accumulation, tau in f32, and
    # half a bf16 ulp for the bf16 store
    a64, w64, b64 = A.double(), W.to(torch.bfloat16).double(), b.double()
    Z = a64 @ w64.t()
    y = _tau64(_NAME[act], ap, Z + b64)
    delta = _lip(_NAME[act], ap) * (2 * K * U * (a64.abs() @ w64.abs().t()) + 3 * U * (Z.abs() + b64.abs())) + 8 * U * y.abs()
    _check_bound(out32.cpu(), y, delta, f"rows forward f32 N={N} act={act}", bf16_out=False)
    _check_bound(out16[:, :N].cpu(), y, delta, f"rows forward bf16 N={N} act={act}")
    assert bool((out16[:, N:n16] == 0).all())


@pytest.mark.parametrize("N", [40, 64, 300])
@pytest.mark.parametrize("act, ap", ACTS)
@pytest.mark.parametrize("pre", [False, True])
def test_rows_kernel_mirror_mode(N, act, ap, pre):
    """C[out_row[r]] = (A . W^T + res[res_row[r]]) * tau'(Y[out_row[r]]): a random permutation as out_row, a residual map with
    repeats, tau' from the activation output or from the pre-activation; rows of C outside out_row are left alone."""
    g = torch.Generator().manual_seed(7 * N + act + int(pre))
    R, K, Rc, Rres = 300, N, 340, 37
    hp = engine.pad_hidden(N)
    A = torch.randn(R, K, generator=g).to(torch.bfloat16)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    out_row = torch.randperm(Rc, generator=g)[:R].to(torch.int32)
    res_row = torch.randint(0, Rres, (R,), generator=g, dtype=torch.int32)
    res = torch.randn(Rres, N, generator=g).to(torch.bfloat16)
    z = torch.randn(Rc, N, generator=g)
    Y = (z if pre else _act(z, act, ap)).to(torch.bfloat16)
    q, s = out_row.long(), res_row.long()
    a64, w64 = A.double(), W.to(torch.bfloat16).double()
    D, Ua = a64 @ w64.t(), a64.abs() @ w64.abs().t()

    def bound_check(got, r, Yq, what):
        """(D + r) * tau'(Yq) in float64, bounded by the f32 accumulation, the f32 residual add and tau', and half a bf16 ulp."""
        d = _dtau64(_NAME[act], ap, Yq.double(), pre)
        ref = (D + r) * d
        delta = d.abs() * (2 * K * U * Ua + 2 * U * (D.abs() + r.abs())) + 8 * U * (1 + d.abs()) * (D + r).abs()
        _check_bound(got, ref, delta, f"rows mirror {what} N={N} act={act} pre={pre}")

    dev = lambda x, cols: torch.cat([x, torch.zeros(x.shape[0], cols - x.shape[1], dtype=x.dtype)], 1).cuda()  # noqa: E731
    out = torch.full((Rc, hp), 7.0, dtype=torch.bfloat16, device="cuda")
    engine.linear_tc_rows(dev(A, hp), K, engine.pack_weight_tc(W.cuda()), N, out, act=act, act_param=ap, Y=dev(Y, hp),
                          from_preact=pre, out_row=out_row.cuda(), res=dev(res, hp), res_row=res_row.cuda())
    out = out.cpu()
    bound_check(out[q, :N], res.double()[s], Y[q], "with maps")
    assert bool((out[q, N:(N + 15) // 16 * 16] == 0).all())
    untouched = torch.ones(Rc, dtype=torch.bool)
    untouched[q] = False
    assert bool((out[untouched] == 7.0).all())
    # without maps or residual: identity rows
    out2 = torch.zeros((R, hp), dtype=torch.bfloat16, device="cuda")
    engine.linear_tc_rows(dev(A, hp), K, engine.pack_weight_tc(W.cuda()), N, out2, act=act, act_param=ap, Y=dev(Y[:R], hp),
                          from_preact=pre)
    bound_check(out2[:, :N].cpu(), torch.zeros_like(D), Y[:R], "identity rows")


@pytest.mark.parametrize("name", BF16_GOLDENS)
def test_bf16_mab_matches_golden(name):
    g = load_golden(name)
    mp = _golden_module(g, "bf16").cuda()
    assert not mp.uses_composed_tier()
    H_v, H_e = _golden_run_cuda(g, mp)
    kinked = g["config"].get("activation", "relu") in ("relu", "leakyrelu")
    if H_v is not None:
        assert H_v.dtype == torch.float32
        _close_bf16(H_v, g["H_v"], "H_v")
    if H_e is not None:
        assert H_e.dtype == torch.float32
        _close_bf16(H_e, g["H_e"], "H_e")
    grads = {k: p.grad for k, p in mp.named_parameters()}
    for k, v in g.items():
        if k.startswith("grad."):
            _close_bf16(grads[k[len("grad."):]], v, k, grad=True, kinked=kinked)


def _golden_run_cuda(g, mp):
    from chemprop_b200.nn import MeanAggregation
    from tests.util import golden_bmg

    bmg = golden_bmg(g, "cuda")
    d = lambda k: torch.from_numpy(g[k]).cuda() if k in g else None  # noqa: E731
    H_v, H_e = mp(bmg, d("V_d"), d("E_d"))
    loss = 0.0
    if H_v is not None:
        loss = loss + (MeanAggregation()(H_v, bmg.batch) * d("G")).sum()
    if H_e is not None:
        loss = loss + (H_e * d("G_e")).sum()
    loss.backward()
    return H_v, H_e


@pytest.mark.parametrize("case", [("bond", 3, True, "tanh", True, True, True, False),
                                  ("atom", 2, True, "elu", True, True, True, True),
                                  ("bond", 1, False, "elu", True, True, True, True),
                                  ("atom", 1, True, "tanh", False, True, False, False)], ids=lambda c: "-".join(map(str, c)))
def test_bf16_mab_random_cases_vs_oracle(case):
    sweep_case(*case, device="cuda", n_mols=20, d_h=64, seed=2)


def _big_batch_run(make_module, mgs, device, Gm, Ge):
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.nn import MeanAggregation

    mp = make_module().to(device)
    bmg = BatchMolGraph(mgs)
    bmg.to(device)
    H_v, H_e = mp(bmg)
    ((MeanAggregation()(H_v, bmg.batch) * Gm.to(device)).sum() + (H_e * Ge.to(device)).sum()).backward()
    return mp, H_v.detach().float().cpu(), H_e.detach().float().cpu(), {k: p.grad.detach().float().cpu() for k, p in mp.named_parameters()}


def _grad_close(got, ref, rel, what):
    got, ref = got.double(), ref.double()
    scale = max(1e-6, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    fro = ((got - ref).norm() / max(1e-12, ref.norm().item())).item()
    assert err <= rel * scale and fro <= rel, (what, err, scale, fro)


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_bf16_mab_1500_molecules_vs_oracle_and_rounding_aware_emulation(kind):
    """1 500 molecules, d_h = 300, depth 3, ReLU, both read-outs: outputs within the bf16 bound of the oracle, every
    gradient within 6 % of its scale; against the rounding-aware emulation of the same tier (tests/emu_mab.py): 2 %."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing
    from oracle import restatement as R
    from tests import emu_mab

    torch.manual_seed(11)
    mgs = make_molecules(1500, seed=21, shuffle_edges=True)
    cls = MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing
    state = cls(d_h=300, depth=3, bias=True).state_dict()
    make = lambda: (lambda m: (m.load_state_dict(state), m)[1])(cls(d_h=300, depth=3, bias=True, precision="bf16"))  # noqa: E731
    nE = sum(m.E.shape[0] for m in mgs)
    gen = torch.Generator().manual_seed(5)
    Gm, Ge = torch.randn(1500, 300, generator=gen), torch.randn(nE, 300, generator=gen) / 50
    mp, H_v, H_e, grads = _big_batch_run(make, mgs, "cuda", Gm, Ge)
    assert not mp.uses_composed_tier()
    with pytest.MonkeyPatch.context() as mpatch:
        emu_mab.patch_engine(mpatch)
        _, eH_v, eH_e, egrads = _big_batch_run(make, mgs, "cpu", Gm, Ge)
    _close_bf16(H_v, eH_v, "H_v vs emulation")
    _close_bf16(H_e, eH_e, "H_e vs emulation")
    for k in grads:
        _grad_close(grads[k], egrads[k], 2e-2, k)
    P = {k: v.detach().clone().requires_grad_(True) for k, v in state.items()}
    ref = BatchMolGraph(mgs)
    Hv_r, He_r = R.mab_forward(kind, ref.V, ref.E, ref.edge_index, ref.rev_edge_index, P["W_i.weight"], P["W_i.bias"],
                               P["W_h.weight"], P["W_h.bias"], P["W_vo.weight"], P["W_vo.bias"], P["W_eo.weight"],
                               P["W_eo.bias"], 3, "relu")
    ((R.aggregate(Hv_r, ref.batch, "mean") * Gm).sum() + (He_r * Ge).sum()).backward()
    _close_bf16(H_v, Hv_r.detach(), "H_v")
    _close_bf16(H_e, He_r.detach(), "H_e")
    for k in grads:
        _close_bf16(grads[k], P[k].grad, k, grad=True)


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_bf16_mab_cgr_batch(kind):
    """Condensed-reaction graphs (~170 directed edges per molecule, d_v = 106, d_e = 28): the bond kind on the fused step's
    128-row window path, the atom kind on the fused atom step; against the oracle."""
    from chemprop_b200.data import BatchMolGraph, make_cgr_graphs
    from chemprop_b200.engine import get_layout
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(3)
    mgs = make_cgr_graphs(40, seed=4)
    cls = MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing
    mp = cls(d_v=106, d_e=28, d_h=300, depth=3, activation="tanh", precision="bf16")
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    mp = mp.cuda()
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    assert lay.max_tile_rows > 128 and lay.max_tile_atoms <= engine.ATOM_TILE_ATOMS
    engine.STEP_EVENTS = []
    try:
        H_v, H_e = mp(bmg)
        tags = {t for t, _, _ in engine.STEP_EVENTS}
    finally:
        engine.STEP_EVENTS = None
    assert tags == ({"fused_first", "fused"} if kind == "bond" else {"atom_fused_first", "atom_fused"}), tags
    gen = torch.Generator().manual_seed(1)
    Gm, Ge = torch.randn(40, 300, generator=gen, dtype=torch.float64), torch.randn(bmg.E.shape[0], 300, generator=gen, dtype=torch.float64)
    ((MeanAggregation()(H_v, bmg.batch) * Gm.float().cuda()).sum() + (H_e * Ge.float().cuda()).sum()).backward()
    ref = BatchMolGraph(mgs)
    Hv_r, He_r = R.mab_forward(kind, ref.V.double(), ref.E.double(), ref.edge_index, ref.rev_edge_index, P["W_i.weight"], None,
                               P["W_h.weight"], None, P["W_vo.weight"], P["W_vo.bias"], P["W_eo.weight"], P["W_eo.bias"], 3, "tanh")
    ((R.aggregate(Hv_r, ref.batch, "mean") * Gm).sum() + (He_r * Ge).sum()).backward()
    _close_bf16(H_v, Hv_r.detach(), "H_v")
    _close_bf16(H_e, He_r.detach(), "H_e")
    for k, p in mp.named_parameters():
        _close_bf16(p.grad, P[k].grad, k, grad=True)


def _mab_step_setup(kind):
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import MABAtomMessagePassing, MABBondMessagePassing

    torch.manual_seed(6)
    cls = MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing
    mp = cls(d_h=96, depth=3, bias=True, activation="relu", precision="bf16").cuda()
    bmg = BatchMolGraph(make_molecules(200, seed=8, shuffle_edges=True))
    bmg.to("cuda")
    gen = torch.Generator().manual_seed(2)
    Gm = torch.randn(200, 96, generator=gen).cuda()
    Ge = torch.randn(bmg.E.shape[0], 96, generator=gen).cuda()
    return mp, bmg, Gm, Ge


def _mab_loss(mp, bmg, Gm, Ge):
    from chemprop_b200.nn import MeanAggregation

    H_v, H_e = mp(bmg)
    return (MeanAggregation()(H_v, bmg.batch) * Gm).sum() + (H_e * Ge).sum(), H_v, H_e


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_bf16_mab_bitwise_reproducible(kind):
    mp, bmg, Gm, Ge = _mab_step_setup(kind)
    runs = []
    for _ in range(2):
        mp.zero_grad(set_to_none=True)
        loss, H_v, H_e = _mab_loss(mp, bmg, Gm, Ge)
        loss.backward()
        runs.append((H_v.detach().clone(), H_e.detach().clone(), {k: p.grad.clone() for k, p in mp.named_parameters()}))
    (a_v, a_e, a_g), (b_v, b_e, b_g) = runs
    assert torch.equal(a_v, b_v) and torch.equal(a_e, b_e)
    for k in a_g:
        assert torch.equal(a_g[k], b_g[k]), k


def _eager_step(mp, bmg, Gm, Ge):
    """One eager training step; returns (loss, grads) detached.  Its autograd graph is gone when this returns: a graph kept
    alive would keep the parameters' gradient-accumulation nodes, which were created on the (legacy) default stream, and a
    later capture that reuses them would have to wait on that stream (cudaErrorStreamCaptureImplicit)."""
    mp.zero_grad(set_to_none=True)
    loss, _, _ = _mab_loss(mp, bmg, Gm, Ge)
    loss.backward()
    return loss.detach().clone(), {k: p.grad.clone() for k, p in mp.named_parameters()}


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_bf16_mab_training_step_in_a_cuda_graph(kind):
    """A MAB training step captured with CudaGraphStep (no host synchronisation on the path) equals the eager step, bit for
    bit, on its first and its second replay."""
    from chemprop_b200.graph import CudaGraphStep

    mp, bmg, Gm, Ge = _mab_step_setup(kind)
    torch.cuda.set_sync_debug_mode("error")         # a synchronising torch op on the path raises
    try:
        eager_loss, eager_grads = _eager_step(mp, bmg, Gm, Ge)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for p in mp.parameters():
        p.grad = torch.zeros_like(p)

    def fn(b):
        for p in mp.parameters():
            p.grad.zero_()
        loss, _, _ = _mab_loss(mp, b, Gm, Ge)
        loss.backward()
        return loss

    step = CudaGraphStep(fn)
    for _ in range(2):
        out = step(bmg).clone()
        assert torch.equal(out, eager_loss)
        for k, p in mp.named_parameters():
            assert torch.equal(p.grad, eager_grads[k]), k
    assert step.captures == 1 and step.replays == 2 and step.last_launches > 0
