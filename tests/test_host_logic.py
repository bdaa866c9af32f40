"""CPU tier: the HOST logic of the engine -- the hand-written autograd mirrors (engine.py) and the composed tier
(composed.py) -- run with the kernel wrappers swapped for the torch emulations of tests/emu.py and compared with the
golden vectors of the real reference.  What this pins without a GPU: which op is called on which operand with
which index table, in which order, and that every gradient (incl. a learnable activation's) is wired through.  The
kernels themselves are checked on the H100 by the `-m gpu` tests."""
import numpy as np
import pytest
import torch

from tests import emu
from tests.util import (COMPOSED_GOLDENS, build_engine_module, check_mab_case, golden_bmg, golden_names, load_golden,
                        run_mab_case)

ATOL = 2e-6


def _run(g, mp=None):
    from chemprop_b200.nn import MeanAggregation, NormAggregation, SumAggregation

    mp = build_engine_module(g, "cpu", "fp32") if mp is None else mp
    bmg = golden_bmg(g, "cpu")
    V_d = torch.from_numpy(g["V_d"]) if "V_d" in g else None
    # one intra-op thread: the f32 reductions then sum in one fixed order on every host (with several threads the order, and
    # the last bits of the large-batch gradients compared with the goldens, depends on the core count)
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        H = mp(bmg, V_d)
        aggs = {n: a(H, bmg.batch) for n, a in (("mean", MeanAggregation()), ("sum", SumAggregation()),
                                                ("norm", NormAggregation()))}
        (aggs["mean"].float() * torch.from_numpy(g["G"])).sum().backward()
    finally:
        torch.set_num_threads(threads)
    return mp, bmg, H, aggs


def _check(g, mp, H, aggs):
    np.testing.assert_allclose(H.detach().numpy(), g["H_v"], rtol=1e-5, atol=ATOL)
    for n in ("mean", "sum", "norm"):
        np.testing.assert_allclose(aggs[n].detach().numpy(), g[f"agg_{n}"], rtol=1e-5, atol=ATOL)
    grads = {k: p.grad for k, p in mp.named_parameters()}
    n_checked = 0
    for k, v in g.items():
        if k.startswith("grad."):
            got = grads[k[len("grad."):]]
            assert got is not None, k
            np.testing.assert_allclose(got.numpy(), v, rtol=1e-4, atol=ATOL, err_msg=k)
            n_checked += 1
    assert n_checked >= 3


@pytest.mark.parametrize("name", [n for n in golden_names() if n not in COMPOSED_GOLDENS])
def test_monolithic_f32_tier_through_emulation(name, monkeypatch):
    """engine.BondMPFunction / AtomMPFunction (generic mirror) on emulated kernels == reference golden.  Doubles as
    the validation of the emulation: this host code is the one the GPU tests verify with the real kernels."""
    emu.patch_engine(monkeypatch)
    g = load_golden(name)
    mp, bmg, H, aggs = _run(g)
    assert not mp.uses_composed_tier()
    _check(g, mp, H, aggs)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", [n for n in golden_names() if n not in COMPOSED_GOLDENS])
def test_monolithic_bf16_tier_through_emulation(name, fused, monkeypatch):
    """The bf16 / tensor-core tier's host logic (bond_forward tc path, bond_backward_tc with the fused-step mirror, the
    atom tc path, and with `fused=False` the generic mirror on bf16 buffers) on emulated kernels, same bounds as
    tests/test_gpu_parity.py::test_bf16_tier_matches_reference_golden."""
    from chemprop_b200 import engine

    emu.patch_engine(monkeypatch)
    calls = {"fwd": 0, "bwd": 0}
    f_fwd, f_bwd = engine.bond_step_fused, engine.bond_step_bwd_fused
    monkeypatch.setattr(engine, "bond_step_fused", lambda *a, **k: (calls.__setitem__("fwd", calls["fwd"] + 1), f_fwd(*a, **k))[1])
    monkeypatch.setattr(engine, "bond_step_bwd_fused", lambda *a, **k: (calls.__setitem__("bwd", calls["bwd"] + 1), f_bwd(*a, **k))[1])
    g = load_golden(name)
    mp = build_engine_module(g, "cpu", "bf16", fused)
    mp, bmg, H, aggs = _run(g, mp)
    cfg = g["config"]
    expect_fused = (fused and cfg["kind"] == "bond" and cfg["depth"] > 1 and g["E"].shape[0] > 0
                    and cfg["d_h"] % 4 == 0 and (engine.UNDIRECTED_FUSED or not cfg.get("undirected")))      # molecules larger than a 128-row tile and undirected=True stay on the fused kernel too
    assert (calls["fwd"], calls["bwd"]) == ((cfg["depth"] - 1,) * 2 if expect_fused else (0, 0)), calls
    assert H.dtype == (torch.float32 if "V_d" in g else torch.bfloat16)      # W_d (torch, f32) follows the engine's part
    np.testing.assert_allclose(H.detach().float().numpy(), g["H_v"], rtol=0, atol=1e-2)
    np.testing.assert_allclose(aggs["mean"].detach().float().numpy(), g["agg_mean"], rtol=0, atol=1e-2)
    smooth = g["config"].get("activation", "relu") in ("tanh", "elu")
    grads = {k: p.grad for k, p in mp.named_parameters()}
    for k, v in g.items():
        if k.startswith("grad."):
            got = grads[k[len("grad."):]].float().numpy()
            scale = max(1e-3, float(np.abs(v).max()))
            fro = float(np.linalg.norm(got - v) / max(1e-6, np.linalg.norm(v)))
            lim = (2e-2, 2e-2) if smooth else (0.5, 0.2)
            assert np.abs(got - v).max() <= lim[0] * scale and fro <= lim[1], (k, np.abs(got - v).max(), scale, fro)


@pytest.mark.parametrize("name", COMPOSED_GOLDENS)
def test_composed_tier_matches_reference_golden(name, monkeypatch):
    """PReLU (with its own gradient), SELU, a user module (Softplus), AtomMP undirected: composed.py == reference."""
    emu.patch_engine(monkeypatch)
    g = load_golden(name)
    mp, bmg, H, aggs = _run(g)
    assert mp.uses_composed_tier()
    _check(g, mp, H, aggs)
    if "prelu" in name:
        assert "grad.tau.weight" in g and mp.tau.weight.grad is not None


@pytest.mark.parametrize("name", ["bond_d3_relu", "bond_d2_bias", "bond_d3_undirected", "bond_d3_tanh", "bond_d3_mixed",
                                  "bond_d3_noedges", "bond_d3_vd", "atom_d3_relu", "atom_d3_bias_tanh", "atom_d3_cgr",
                                  "atom_d3_noedges", "atom_d1", "bond_d1"])
def test_composed_tier_equals_monolithic_configurations(name, monkeypatch):
    """The composed tier forced onto configurations the monolithic tier also serves: same goldens."""
    emu.patch_engine(monkeypatch)
    g = load_golden(name)
    mp = build_engine_module(g, "cpu", "fp32")
    monkeypatch.setattr(type(mp), "uses_composed_tier", lambda self, lay=None: True)
    mp, bmg, H, aggs = _run(g, mp)
    _check(g, mp, H, aggs)


@pytest.mark.parametrize("kind,undirected,act", [("bond", False, "relu"), ("bond", True, "tanh"), ("atom", False, "elu"),
                                                 ("atom", True, "prelu")])
def test_training_dropout_mask_for_mask(kind, undirected, act, monkeypatch):
    """dropout > 0 in training (base.py:139, :182, :188): the composed tier applies the caller's dropout module at the
    reference's three sites; with the masks it drew mapped back to the caller's edge order, the oracle reproduces the
    run exactly (forward and every gradient)."""
    from tests.util import dropout_mask_for_mask

    emu.patch_engine(monkeypatch)
    dropout_mask_for_mask(kind, undirected, act, "cpu")


@pytest.mark.parametrize("name", golden_names(mab=True))
def test_mab_modules_match_reference_golden(name, monkeypatch):
    """MABBond / MABAtomMessagePassing (vertex + per-edge embeddings in the caller's edge order, extra atom / bond
    descriptors, edges-only / vertex-only) on the composed tier == the reference, outputs and every gradient."""
    emu.patch_engine(monkeypatch)
    g = load_golden(name)
    mp, H_v, H_e = run_mab_case(g, "cpu")
    check_mab_case(g, mp, H_v, H_e, ATOL)


def test_attentive_aggregation_matches_reference_fixture(monkeypatch):
    from tests.util import check_attentive

    emu.patch_engine(monkeypatch)
    check_attentive("cpu")


@pytest.mark.parametrize("depth,bias", [(3, True), (1, False), (2, False), (5, True)])
def test_training_dropout_on_the_fused_bf16_path(depth, bias, monkeypatch):
    """ReLU + dropout in training keeps the fused bf16 path (no 10x cliff onto the composed tier): masks are not stored,
    1 / (1 - p) is folded into the packed weights of the mirror -- checked mask for mask against the oracle."""
    from chemprop_b200 import engine
    from tests.util import fused_dropout_vs_oracle

    emu.patch_engine(monkeypatch)
    calls = {"n": 0}
    f = engine.bond_step_fused
    monkeypatch.setattr(engine, "bond_step_fused", lambda *a, **k: (calls.__setitem__("n", calls["n"] + 1), f(*a, **k))[1])
    fused_dropout_vs_oracle("cpu", depth=depth, bias=bias)
    assert calls["n"] == depth - 1


def test_constrainer_ffn_matches_reference_fixture(monkeypatch):
    from tests.util import check_constrainer

    emu.patch_engine(monkeypatch)
    check_constrainer("cpu")


def test_constrainer_ffn_trailing_molecules_without_rows(monkeypatch):
    from tests.util import check_constrainer_empty_trailing

    emu.patch_engine(monkeypatch)
    check_constrainer_empty_trailing("cpu")


def test_engine_mpnn_head_matches_reference_training_step(monkeypatch):
    """SURVEY.md 8f-2: agg -> batch norm -> FFN -> MSE on the engine == chemprop's MPNN.training_step (loss, gradients, running stats)."""
    from tests.util import check_mpnn_head

    emu.patch_engine(monkeypatch)
    check_mpnn_head("cpu")


def test_eval_mode_with_dropout_configured_stays_monolithic(monkeypatch):
    emu.patch_engine(monkeypatch)
    g = load_golden("bond_d3_dropout_eval")
    mp, bmg, H, aggs = _run(g)
    assert mp.dropout.p == 0.3 and not mp.training and not mp.uses_composed_tier()
    _check(g, mp, H, aggs)
    mp.train()
    assert mp.uses_composed_tier()


def test_tier_selection():
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing

    class MyReLU(torch.nn.ReLU):           # a subclass may override forward: not assumed to be ReLU
        pass

    assert not BondMessagePassing(d_h=8).uses_composed_tier()
    assert not BondMessagePassing(d_h=8, undirected=True, activation="elu").uses_composed_tier()
    assert BondMessagePassing(d_h=8, activation="prelu").uses_composed_tier()
    assert BondMessagePassing(d_h=8, activation="selu").uses_composed_tier()
    assert BondMessagePassing(d_h=8, activation=torch.nn.GELU()).uses_composed_tier()
    assert BondMessagePassing(d_h=8, activation=MyReLU()).uses_composed_tier()
    assert AtomMessagePassing(d_h=8, undirected=True).uses_composed_tier()
    assert not AtomMessagePassing(d_h=8).uses_composed_tier()
    mp = BondMessagePassing(d_h=8, dropout=0.1)
    assert mp.uses_composed_tier() and not mp.eval().uses_composed_tier()
    with pytest.raises(Exception, match="no CPU fallback|CUDA"):     # the composed tier has no CPU path either
        from chemprop_b200.data import BatchMolGraph, make_molecules
        BondMessagePassing(d_h=8, activation="prelu")(BatchMolGraph(make_molecules(2, seed=0)))


@pytest.mark.parametrize("seed", range(24))
def test_randomised_configurations_vs_oracle(seed, monkeypatch):
    """Random module configuration x random batch (1-atom molecules, shuffled edge order, occasionally a > 128-edge
    molecule or an edgeless batch): whichever tier serves it (monolithic f32 or composed) == the f64 oracle, forward
    and every gradient."""
    from chemprop_b200.data import BatchMolGraph, make_molecule, make_molecules
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation, NormAggregation, SumAggregation
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    rng = np.random.default_rng(1000 + seed)
    kind = ("bond", "atom")[int(rng.integers(2))]
    act = ("relu", "leakyrelu", "prelu", "tanh", "elu", "selu")[int(rng.integers(6))]
    depth, bias, undirected = int(rng.integers(1, 6)), bool(rng.integers(2)), bool(rng.integers(2))
    d_h, d_v, d_e = int(rng.choice([8, 20, 33, 64])), int(rng.choice([5, 72])), int(rng.choice([3, 14]))
    shape = int(rng.integers(4))
    if shape == 0:
        mgs = [make_molecule(rng, 1, d_v, d_e) for _ in range(3)]                                   # no edges at all
    elif shape == 1:
        mgs = make_molecules(7, seed=seed, mean_atoms=8, std_atoms=4, min_atoms=1, d_v=d_v, d_e=d_e, shuffle_edges=True)
    elif shape == 2:
        mgs = [make_molecule(rng, 3, d_v, d_e), make_molecule(rng, 80, d_v, d_e), make_molecule(rng, 1, d_v, d_e)]
    else:
        mgs = make_molecules(1, seed=seed, mean_atoms=20, d_v=d_v, d_e=d_e)
    torch.manual_seed(seed)
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_v=d_v, d_e=d_e, d_h=d_h, bias=bias, depth=depth, activation=act, undirected=undirected)
    bmg = BatchMolGraph(mgs)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward(kind, bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"),
                                      P["W_o.weight"], P["W_o.bias"], depth, act, undirected, prelu_weight=P.get("tau.weight"))
    agg_cls, mode = ((MeanAggregation, "mean"), (SumAggregation, "sum"), (NormAggregation, "norm"))[int(rng.integers(3))]
    G = torch.from_numpy(rng.normal(size=(len(mgs), d_h)))
    (R.aggregate(H_ref, bmg.batch, mode, n_mols=len(mgs)) * G).sum().backward()
    H = mp(bmg)
    (agg_cls()(H, bmg.batch) * G.float()).sum().backward()
    assert (H.detach().double() - H_ref.detach()).abs().max().item() <= 2e-5
    for k, p in mp.named_parameters():
        ref = torch.zeros_like(P[k]) if P[k].grad is None else P[k].grad      # e.g. W_h at depth 1: unused
        got = torch.zeros_like(ref) if p.grad is None else p.grad.double()
        assert (got - ref).abs().max().item() <= 2e-4 * max(1.0, ref.abs().max().item()), (k, kind, act, depth, shape)


@pytest.mark.parametrize("precision,dropout", [("bf16", 0.1), ("fp32", 0.0)])
def test_training_loop_through_the_loader_overfits(precision, dropout, monkeypatch):
    """README's training loop (PackedBatchLoader with side arrays + tile packing -> module -> aggregation -> head ->
    Adam; bf16 with dropout = the fused-path dropout), kernels emulated: the loss must collapse, as in the reference's
    "can it overfit" integration tests (tests/integration/test_regression_mol.py:56-89)."""
    from chemprop_b200.data import PackedBatchLoader, PackedMolGraphDataset, make_molecules
    from chemprop_b200.nn import BondMessagePassing, MeanAggregation
    from chemprop_b200.parallel import FlatGradAllReducer

    emu.patch_engine(monkeypatch)
    torch.manual_seed(0)
    mgs = make_molecules(120, seed=0, mean_atoms=8, std_atoms=2)
    targets = np.array([[mg.V.shape[0] / 8.0 - 1.0] for mg in mgs], dtype=np.float32)
    loader = PackedBatchLoader(PackedMolGraphDataset.from_molgraphs(mgs), batch_size=40, shuffle=True, seed=0,
                               transfer_dtype=torch.bfloat16 if precision == "bf16" else None, arrays={"y": targets})
    mp, agg, head = BondMessagePassing(d_h=32, precision=precision, dropout=dropout), MeanAggregation(), torch.nn.Linear(32, 1)
    params = list(mp.parameters()) + list(head.parameters())
    opt, reducer = torch.optim.Adam(params, 3e-3), FlatGradAllReducer(params)
    epoch_loss = []
    for _ in range(30):
        tot = 0.0
        for batch in loader:
            opt.zero_grad(set_to_none=True)
            pred = head(agg(mp(batch.bmg), batch.bmg.batch).float())
            loss = torch.nn.functional.mse_loss(pred, batch.extras["y"])
            loss.backward()
            reducer.allreduce_()
            opt.step()
            tot += loss.item()
        epoch_loss.append(tot / len(loader))
    assert epoch_loss[-1] < 0.1 * epoch_loss[0] and epoch_loss[-1] < 0.01, (epoch_loss[0], epoch_loss[-1])


@pytest.mark.parametrize("depth,d_e,bias", [(3, 28, False), (2, 28, True), (4, 0, True), (3, 14, True)])
def test_atom_bf16_tier_runs_on_the_fused_atom_step(depth, d_e, bias, monkeypatch):
    """AtomMessagePassing, bf16 tier: every depth step is ONE call of the fused atom step (forward: depth - 1; mirror: depth - 1
    step launches + the read-out launch on dY), the loop-invariant bond term is folded into H_0' (no bias left for the step when
    d_e > 0), and the result matches the oracle at the tier's tolerance; a molecule with more than 128 atoms sends the batch to the
    two-launch step with a one-time warning."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_cgr_graphs, make_molecules
    from chemprop_b200.nn import AtomMessagePassing
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    calls = []
    f0, b0 = engine.atom_step_fused, engine.atom_step_bwd_fused
    monkeypatch.setattr(engine, "atom_step_fused", lambda *a, **k: (calls.append(("f", a[5] is not None, a[9])), f0(*a, **k))[1])
    monkeypatch.setattr(engine, "atom_step_bwd_fused", lambda *a, **k: (calls.append(("b",)), b0(*a, **k))[1])
    torch.manual_seed(depth + d_e)
    mgs = make_cgr_graphs(5, seed=depth, d_v=106, d_e=d_e) if d_e else make_molecules(9, seed=depth, d_v=106, d_e=14, min_atoms=1)
    if d_e == 0:                                                         # bond-feature-less graphs: no term to fold into H_0'
        mgs = [type(m)(V=m.V, E=m.E[:, :0], edge_index=m.edge_index, rev_edge_index=m.rev_edge_index) for m in mgs]
    bmg = BatchMolGraph(mgs)
    mp = AtomMessagePassing(d_v=106, d_e=d_e, d_h=48, depth=depth, bias=bias, precision="bf16")
    H = mp(bmg)
    H.float().square().sum().backward()
    fwd = [c for c in calls if c[0] == "f"]
    assert len(fwd) == depth - 1 and [c[2] for c in fwd] == [True] + [False] * (depth - 2)          # first_step flags
    assert all(c[1] == (bias and d_e == 0) for c in fwd)                 # the step carries b_h only when nothing folded it into H_0'
    assert len([c for c in calls if c[0] == "b"]) == depth               # read-out launch + depth - 1 mirror steps
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    Hr = R.message_passing_forward("atom", bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index, P["W_i.weight"],
                                   P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"), P["W_o.weight"], P["W_o.bias"], depth)
    Hr.square().sum().backward()
    assert float((H.detach().double() - Hr.detach()).abs().max()) <= 1e-2 * max(1.0, float(Hr.detach().abs().max()))
    for k, p in mp.named_parameters():
        ref = P[k].grad
        assert float((p.grad.double() - ref).abs().max()) <= 6e-2 * max(1e-6, float(ref.abs().max())), k

    calls.clear()
    engine._WARNED.discard("atom_unfused")
    bigs = make_molecules(2, seed=1, mean_atoms=150.0, std_atoms=1.0, min_atoms=140, max_atoms=160, d_v=106, d_e=max(d_e, 1)) \
        + make_molecules(3, seed=2, d_v=106, d_e=max(d_e, 1))
    if d_e == 0:
        bigs = [type(m)(V=m.V, E=m.E[:, :0], edge_index=m.edge_index, rev_edge_index=m.rev_edge_index) for m in bigs]
    big = BatchMolGraph(bigs)
    with pytest.warns(RuntimeWarning, match="fused atom depth step"):
        mp(big)
    assert not calls


@pytest.mark.parametrize("kind,precision", [("bond", "fp32"), ("bond", "bf16"), ("atom", "bf16"), ("atom", "fp32")])
def test_second_backward_and_feature_gradients(kind, precision, monkeypatch):
    """The autograd node keeps its saved tensors: a second backward with `retain_graph=True` reproduces the first one's
    gradients exactly (torch's own behaviour; round 1 dropped them after the first backward).  And features that require grad are
    refused loudly -- the hand-written mirror produces parameter gradients only, a silent `None` would be wrong."""
    from chemprop_b200._lib import DmpnnError
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing

    emu.patch_engine(monkeypatch)
    torch.manual_seed(3)
    bmg = BatchMolGraph(make_molecules(12, seed=4))
    mp = (BondMessagePassing if kind == "bond" else AtomMessagePassing)(d_h=32, depth=3, precision=precision)
    loss = mp(bmg).float().square().sum()
    loss.backward(retain_graph=True)
    first = {k: p.grad.clone() for k, p in mp.named_parameters()}
    mp.zero_grad(set_to_none=True)
    loss.backward()
    for k, p in mp.named_parameters():
        assert torch.equal(p.grad, first[k]), k
    bmg2 = BatchMolGraph(make_molecules(3, seed=5))
    bmg2.V = bmg2.V.clone().requires_grad_(True)
    with pytest.raises(DmpnnError, match="require grad"):
        mp(bmg2)


def test_graph_step_reloads_a_new_batch_object_even_at_a_reused_address():
    """`CudaGraphStep.load` skips the copy into the graph's static inputs only for the very same, unmodified batch OBJECT.
    Batches of a fixed-signature loader are new objects whose `id()` is routinely the one of the batch just freed and whose
    tensors are all at version 0: an id / version stamp alone replayed stale inputs (host-only check of that logic)."""
    import gc

    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.graph import CudaGraphStep, _Captured

    mgs = make_molecules(6, seed=3)
    static = BatchMolGraph(mgs)
    static.V.zero_()
    cap = _Captured()
    cap.bmg, cap.last, cap.last_ref = static, None, None
    step = CudaGraphStep(lambda b: None)

    b1 = BatchMolGraph(mgs)
    step.load(cap, b1)
    assert torch.equal(static.V, b1.V)
    static.V.fill_(-1.0)
    step.load(cap, b1)                                   # same object, untouched: nothing copied
    assert bool((static.V == -1.0).all())
    b1.V.mul_(2.0)                                       # in-place change torch knows of: copied again
    step.load(cap, b1)
    assert torch.equal(static.V, b1.V)

    seen = set()
    for k in range(64):                                  # new objects, many of them at the address of the one just freed
        b = BatchMolGraph(mgs)
        b.V.fill_(float(k))
        seen.add(id(b))
        step.load(cap, b)
        assert bool((static.V == float(k)).all())
        del b
        gc.collect()
    assert len(seen) < 64                                # the allocator did hand out a reused id at least once


def test_cached_segment_tables_do_not_outlive_an_in_place_change_of_batch(monkeypatch):
    """`get_layout` leaves the molecule offsets on `bmg.batch` so that `Aggregation.forward(H, bmg.batch)` needs no device
    read-back; the attachment carries the tensor's version and is void once `batch` has been changed in place."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import BondMessagePassing, SumAggregation

    emu.patch_engine(monkeypatch)
    bmg = BatchMolGraph(make_molecules(5, seed=2))
    mp = BondMessagePassing(d_h=16, depth=2)
    H = mp(bmg).detach()
    assert getattr(bmg.batch, "_dmpnn_seg", None) is not None
    agg = SumAggregation()
    out5 = agg(H, bmg.batch)
    assert out5.shape[0] == 5
    merged = bmg.batch
    merged.clamp_(max=1)                                   # molecules 1..4 become one segment; the cache must not be used
    out2 = agg(H, merged)
    assert out2.shape[0] == 2
    assert torch.allclose(out2[1], out5[1:].sum(0), atol=1e-5) and torch.allclose(out2[0], out5[0], atol=1e-6)


@pytest.mark.parametrize("oracle", [True, False])
@pytest.mark.parametrize("kind,gen_kw", [("bond", dict(seed=4)), ("atom", dict(seed=6, cgr=True))])
def test_full_size_property_checks_through_emulation(kind, gen_kw, oracle, monkeypatch):
    """tests/util.full_size_checks (the oracle bound plus reproducibility, exact linearity of the mirror, checksum of
    checksums and molecule-order invariance; run at BASELINE sizes on the GPU) exercised here at a small size over the
    emulated kernel wrappers, so that the checks themselves are known to be sound before they meet hardware."""
    from tests.util import full_size_checks

    emu.patch_engine(monkeypatch)
    out = full_size_checks(kind, 60 if kind == "bond" else 12, "cpu", gen_kw=gen_kw, grad_tol=0.2,   # tiny batch: kink noise
                           oracle=oracle)
    assert out["rows"] > 0 and (("err_H" in out and out["err_H"] > 0) if oracle else "err_H" not in out)


@pytest.mark.parametrize("depth,bias,act,d_h", [(3, False, "relu", 64), (4, True, "tanh", 64), (3, True, "relu", 62)])
def test_undirected_bf16_tier_runs_on_the_fused_step(depth, bias, act, d_h, monkeypatch):
    """BondMessagePassing(undirected=True, precision="bf16") (base.py:202-203 averages H with its reverse before the message):
    the average is a prologue pass (dmpnn_rev_average, applying the first step's tau) and every depth step -- forward and
    mirror -- is ONE launch of the fused kernel on the averaged state; the W_h gradient contracts the mirror's gathered operand
    with the saved averaged state.  With d_h % 4 != 0 the step runs as message + dmpnn_linear_tc_bf16 (H_0 residual, bias and
    tau in the GEMM's epilogue).  Either way no GEMM of the tier touches the f32 FMA kernel, and the result matches the oracle
    at the tier's tolerance."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import BondMessagePassing
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    engine._WARNED.discard("unfused")
    calls = []
    for name, tag in (("linear_tc", "tc"), ("linear_fwd", "simt"), ("linear_wgrad", "simt"), ("bond_step_fused", "fused"),
                      ("bond_step_bwd_fused", "fused_bwd"), ("rev_average", "avg")):
        f0 = getattr(engine, name)
        monkeypatch.setattr(engine, name, lambda *a, _f=f0, _t=tag, **k: (
            calls.append((_t, k.get("res") is not None) if _t == "tc" else (_t,)), _f(*a, **k))[1])
    torch.manual_seed(depth)
    bmg = BatchMolGraph(make_molecules(14, seed=depth, shuffle_edges=True))
    mp = BondMessagePassing(d_h=d_h, depth=depth, bias=bias, activation=act, undirected=True, precision="bf16")
    H = mp(bmg)
    fwd = list(calls)
    fused = d_h % 4 == 0
    assert ("simt",) not in fwd, fwd
    assert fwd.count(("fused",)) == (depth - 1 if fused else 0) and fwd.count(("avg",)) == depth - 1
    assert fwd.count(("tc", True)) == (0 if fused else depth - 1) and fwd.count(("tc", False)) == 2     # W_h steps; W_i and W_o
    H.float().square().sum().backward()
    assert ("simt",) not in calls                                                        # the mirror's GEMMs too
    assert calls.count(("fused_bwd",)) == (depth - 1 if fused else 0) and calls.count(("avg",)) == 2 * (depth - 1)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    Hr = R.message_passing_forward("bond", bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index, P["W_i.weight"],
                                   P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"), P["W_o.weight"], P["W_o.bias"], depth,
                                   act, undirected=True)
    Hr.square().sum().backward()
    assert float((H.detach().double() - Hr.detach()).abs().max()) <= 1e-2 * max(1.0, float(Hr.detach().abs().max()))
    for k, p in mp.named_parameters():
        ref = P[k].grad
        assert float((p.grad.double() - ref).abs().max()) <= 6e-2 * max(1e-6, float(ref.abs().max())), k


@pytest.mark.parametrize("d_h,expect_x3", [(64, True), (62, False)])
def test_composed_tier_runs_its_plain_gemms_on_the_x3_tensor_core_kernels(d_h, expect_x3, monkeypatch):
    """Composed tier (here: PReLU): the W_h GEMM of every depth step -- an ungathered single-source product -- and its two
    mirror GEMMs go to the f32-accurate tensor-core kernels (dmpnn_linear_x3 / dmpnn_wgrad_x3) when d_h is a multiple of 4;
    otherwise, and for the gathered two-source W_i / W_o operands, the f32 FMA kernel runs.  Same results either way."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import BondMessagePassing
    from oracle import restatement as R

    from chemprop_b200 import composed

    emu.patch_engine(monkeypatch)
    monkeypatch.setitem(composed._X3_STATE, "ok", True)              # the first-use check has its own test below
    calls = []
    for name in ("linear_x3", "wgrad_x3", "linear_fwd", "linear_wgrad"):
        f0 = getattr(engine, name)
        monkeypatch.setattr(engine, name, lambda *a, _f=f0, _n=name, **k: (calls.append(_n), _f(*a, **k))[1])
    torch.manual_seed(3)
    bmg = BatchMolGraph(make_molecules(10, seed=3))
    depth = 3
    mp = BondMessagePassing(d_h=d_h, depth=depth, bias=True, activation="prelu")
    assert mp.uses_composed_tier()
    H = mp(bmg)
    assert calls.count("linear_x3") == ((depth - 1) if expect_x3 else 0)
    assert calls.count("linear_fwd") == (2 if expect_x3 else depth + 1)                  # W_i and W_o (+ W_h steps without x3)
    H.square().sum().backward()
    assert calls.count("wgrad_x3") == ((depth - 1) if expect_x3 else 0)
    assert calls.count("linear_x3") == (2 * (depth - 1) if expect_x3 else 0)             # + dX = dY . W_h per step
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    Hr = R.message_passing_forward("bond", bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index, P["W_i.weight"],
                                   P["W_i.bias"], P["W_h.weight"], P["W_h.bias"], P["W_o.weight"], P["W_o.bias"], depth, "prelu",
                                   prelu_weight=P["tau.weight"])
    Hr.square().sum().backward()
    assert float((H.detach().double() - Hr.detach()).abs().max()) <= 1e-5
    for k, p in mp.named_parameters():
        ref = P[k].grad
        assert float((p.grad.double() - ref).abs().max()) <= 1e-5 * max(1e-6, float(ref.abs().max())), k   # f32 sums vs f64


@pytest.mark.parametrize("seed", range(16))
def test_randomised_bf16_bond_configurations_fused_vs_unfused_vs_oracle(seed, monkeypatch):
    """bf16 tier of BondMessagePassing over random configurations (directed / undirected, depth 1-5, bias, the four fused
    activations) and batch shapes (edgeless, 1-atom molecules, a molecule of more than 128 directed edges, shuffled edge order):
    the path on the fused depth step and the path with `fused=False` (separate message / GEMM kernels, generic mirror) are two
    host-side compositions of the same arithmetic -- they must agree closely, and both sit within the tier's bound of the f64
    oracle.  Smooth activations carry the tight gradient bound; with ReLU-like kinks bf16 storage flips derivatives near zero."""
    from chemprop_b200.data import BatchMolGraph, make_molecule, make_molecules
    from chemprop_b200.nn import BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    rng = np.random.default_rng(7000 + seed)
    act = ("relu", "leakyrelu", "tanh", "elu")[int(rng.integers(4))]
    depth, bias, undirected = int(rng.integers(1, 6)), bool(rng.integers(2)), bool(seed % 2)
    d_h = int(rng.choice([16, 48, 64, 100]))
    shape = int(rng.integers(4))
    if shape == 0:
        mgs = [make_molecule(rng, 1, 72, 14) for _ in range(3)]
    elif shape == 1:
        mgs = make_molecules(9, seed=seed, mean_atoms=8, std_atoms=4, min_atoms=1, shuffle_edges=True)
    elif shape == 2:
        mgs = [make_molecule(rng, 3, 72, 14), make_molecule(rng, 80, 72, 14), make_molecule(rng, 1, 72, 14)]
    else:
        mgs = make_molecules(12, seed=seed, mean_atoms=20)
    torch.manual_seed(seed)
    mp = BondMessagePassing(d_h=d_h, bias=bias, depth=depth, activation=act, undirected=undirected, precision="bf16")
    bmg = BatchMolGraph(mgs)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward("bond", bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"),
                                      P["W_o.weight"], P["W_o.bias"], depth, act, undirected)
    G = torch.from_numpy(rng.normal(size=(len(mgs), d_h)))
    (R.aggregate(H_ref, bmg.batch, "mean", n_mols=len(mgs)) * G).sum().backward()
    runs = {}
    for fused in (True, False):
        mp.fused = fused
        mp.zero_grad(set_to_none=True)
        b = BatchMolGraph(mgs)
        H = mp(b)
        (MeanAggregation()(H, b.batch) * G.float()).sum().backward()
        runs[fused] = (H.detach().double(), {k: (torch.zeros_like(P[k]) if p.grad is None else p.grad.double())
                                             for k, p in mp.named_parameters()})
    scale = max(1.0, float(H_ref.detach().abs().max()))
    smooth = act in ("tanh", "elu")
    for fused, (H, grads) in runs.items():
        assert float((H - H_ref.detach()).abs().max()) <= 1e-2 * scale, (fused, act, depth, undirected, shape)
        for k, g in grads.items():
            ref = torch.zeros_like(P[k]) if P[k].grad is None else P[k].grad
            lim = 3e-2 if smooth else 0.5
            assert float((g - ref).abs().max()) <= lim * max(1e-3, float(ref.abs().max())), (fused, k, act, depth, undirected, shape)
    assert float((runs[True][0] - runs[False][0]).abs().max()) <= 1.6e-2 * scale
    if smooth:
        for k in runs[True][1]:
            a, b_ = runs[True][1][k], runs[False][1][k]
            assert float((a - b_).abs().max()) <= 3e-2 * max(1e-3, float(b_.abs().max())), (k, act, depth, undirected, shape)


@pytest.mark.parametrize("broken", [False, True])
def test_composed_tier_checks_its_x3_gemm_on_first_use(broken, monkeypatch):
    """The composed tier's first 3xTF32 product in a process is cross-checked against the f32 FMA kernel (one extra launch and
    one sync, once).  Agreement: x3 from then on.  Disagreement (here: a kernel that returns garbage): a RuntimeWarning, x3
    off for the process, and the results -- this call's included -- come from the FMA kernel, so they are still right."""
    from chemprop_b200 import composed, engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import BondMessagePassing
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    monkeypatch.setitem(composed._X3_STATE, "ok", None)
    calls = []
    good = engine.linear_x3

    def x3(*a, **k):
        calls.append("x3")
        good(*a, **k)
        if broken:
            a[4].mul_(1.5)                                           # `out`: a wrong product

    simt0 = engine.linear_fwd
    monkeypatch.setattr(engine, "linear_x3", x3)
    monkeypatch.setattr(engine, "linear_fwd", lambda *a, **k: (calls.append("simt"), simt0(*a, **k))[1])
    torch.manual_seed(1)
    bmg = BatchMolGraph(make_molecules(8, seed=1))
    mp = BondMessagePassing(d_h=32, depth=3, activation="selu")
    if broken:
        with pytest.warns(RuntimeWarning, match="3xTF32 GEMM disagrees"):
            H = mp(bmg)
        assert composed._X3_STATE["ok"] is False and calls.count("x3") == 1        # tried once, never again
    else:
        H = mp(bmg)
        assert composed._X3_STATE["ok"] is True and calls.count("x3") == 2 and calls.count("simt") == 3   # W_i, check, W_o
    H.square().sum().backward()
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    Hr = R.message_passing_forward("bond", bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index, P["W_i.weight"],
                                   None, P["W_h.weight"], None, P["W_o.weight"], P["W_o.bias"], 3, "selu")
    Hr.square().sum().backward()
    assert float((H.detach().double() - Hr.detach()).abs().max()) <= 1e-5
    for k, p in mp.named_parameters():
        ref = P[k].grad
        assert float((p.grad.double() - ref).abs().max()) <= 1e-5 * max(1e-6, float(ref.abs().max())), k
