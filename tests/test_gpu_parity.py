"""GPU tier: the CUDA path (through the C ABI) against the golden vectors of the real
reference and against oracle/restatement.py on seeded inputs.
Tolerances (BASELINE.json north_star): indices bit-exact; hidden states <= 1e-5 in the fp32 tier,
<= 1e-2 in the bf16 tier."""
import numpy as np
import pytest
import torch

from tests.util import (COMPOSED_GOLDENS, build_engine_module, golden_bmg, golden_names, load_golden,
                        oracle_forward)

pytestmark = pytest.mark.gpu

FP32_ATOL = 1e-5
BF16_ATOL = 1e-2
# goldens served by the monolithic (tau-fused) tiers; the composed-tier goldens run in tests/test_gpu_zcomposed.py
MONOLITHIC_GOLDENS = [n for n in golden_names() if n not in COMPOSED_GOLDENS]


def _engine_run(g, precision, fused=True):
    from chemprop_b200.nn import MeanAggregation, NormAggregation, SumAggregation

    mp = build_engine_module(g, "cuda", precision, fused)
    bmg = golden_bmg(g, "cuda")
    V_d = torch.from_numpy(g["V_d"]).cuda() if "V_d" in g else None
    H = mp(bmg, V_d)
    aggs = {n: a(H, bmg.batch) for n, a in (("mean", MeanAggregation()), ("sum", SumAggregation()),
                                            ("norm", NormAggregation()))}
    loss = (aggs["mean"].float() * torch.from_numpy(g["G"]).cuda()).sum()
    loss.backward()
    grads = {k: p.grad for k, p in mp.named_parameters() if p.grad is not None}
    return mp, bmg, H, aggs, loss, grads


@pytest.mark.parametrize("name", golden_names() + golden_names(mab=True))
def test_layout_bit_exact(name):
    from chemprop_b200.engine import get_layout
    from oracle import layout_np

    g = load_golden(name)
    bmg = golden_bmg(g, "cuda")
    lay = get_layout(bmg)
    L = layout_np.build_layout(g["edge_index"], g["rev_edge_index"], g["batch"], int(g["n_mols"]))
    for k in ("perm", "inv_perm", "rowptr", "src_row", "dst_row", "rev_row", "mol_atom_ptr", "mol_row_ptr"):
        got = getattr(lay, k).cpu().numpy()
        assert got.dtype == np.int32 and np.array_equal(got, L[k]), k
    assert lay.n_tiles == L["n_tiles"]
    for k in ("tile_mol_ptr", "tile_row_ptr", "tile_atom_ptr"):
        assert np.array_equal(getattr(lay, k).cpu().numpy()[: L["n_tiles"] + 1], L[k]), k
    assert lay.flags == L["flags"] and lay.max_indeg == L["max_indeg"]
    assert lay.max_tile_rows == L["max_tile_rows"] and lay.max_tile_atoms == L["max_tile_atoms"]


@pytest.mark.parametrize("name", MONOLITHIC_GOLDENS)
def test_fp32_tier_matches_reference_golden(name):
    g = load_golden(name)
    mp, bmg, H, aggs, loss, grads = _engine_run(g, "fp32")
    assert H.dtype == torch.float32 and tuple(H.shape) == g["H_v"].shape
    np.testing.assert_allclose(H.detach().cpu().numpy(), g["H_v"], rtol=0, atol=FP32_ATOL)
    for n in ("mean", "sum", "norm"):
        np.testing.assert_allclose(aggs[n].detach().cpu().numpy(), g[f"agg_{n}"], rtol=1e-5, atol=FP32_ATOL)
    for k, v in g.items():
        if k.startswith("grad."):
            got = grads[k[len("grad."):]].cpu().numpy()
            np.testing.assert_allclose(got, v, rtol=1e-4, atol=FP32_ATOL, err_msg=k)


def _emulated_run(make_module, make_bmg, V_d=None, loss_fn=None):
    """The same module / batch through tests/emu.py on the CPU: engine.py's host logic over torch emulations of the
    kernels that round to bf16 exactly where the kernels store bf16 (the fused step's packed-bf16 message sums included).
    A rounding-aware stand-in for the hardware run: ReLU kink flips caused by bf16 storage happen identically in both, so
    the hand-written mirror can be held to a tight bound."""
    from tests import emu

    with pytest.MonkeyPatch.context() as mpatch:
        emu.patch_engine(mpatch)
        mp = make_module()
        bmg = make_bmg()
        H = mp(bmg, V_d)
        loss = loss_fn(H, bmg)
        loss.backward()
        return H.detach().float(), {k: p.grad.detach().float() for k, p in mp.named_parameters() if p.grad is not None}


def _grad_close(got, ref, rel, what):
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = max(1e-6, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    fro = ((got - ref).norm() / max(1e-12, ref.norm().item())).item()
    assert err <= rel * scale and fro <= rel, (what, err, scale, fro)


@pytest.mark.parametrize("name", MONOLITHIC_GOLDENS)
def test_bf16_tier_matches_reference_golden(name):
    from chemprop_b200.nn import MeanAggregation

    g = load_golden(name)
    mp, bmg, H, aggs, loss, grads = _engine_run(g, "bf16")
    np.testing.assert_allclose(H.detach().float().cpu().numpy(), g["H_v"], rtol=0, atol=BF16_ATOL)
    np.testing.assert_allclose(aggs["mean"].detach().float().cpu().numpy(), g["agg_mean"], rtol=0, atol=BF16_ATOL)
    # Gradients.  (1) Against the rounding-aware emulation of this very tier (same bf16 storage points): <= 2 %, whatever
    # the activation -- this is the check that can see a wrong or mis-scaled term of the hand-written mirror.
    V_d = torch.from_numpy(g["V_d"]) if "V_d" in g else None
    G = torch.from_numpy(g["G"])
    _, egrads = _emulated_run(lambda: build_engine_module(g, "cpu", "bf16"), lambda: golden_bmg(g, "cpu"), V_d,
                              lambda H, b: (MeanAggregation()(H, b.batch).float() * G).sum())
    for k, v in egrads.items():
        _grad_close(grads[k].float(), v, 2e-2, (name, k, "vs emulation"))
    # (2) Against the fp32 reference golden.  Smooth activations: 2 %.  ReLU-like kinks: bf16 storage flips the derivative of
    # the pre-activations that sit within rounding distance of zero; on these 6-molecule batches that is a several-percent
    # random walk on the summed weight gradient (tools/diag_bf16.py), so this comparison is a sanity bound only -- (1) and
    # test_bf16_mirror_vs_rounding_aware_emulation carry the proof.
    smooth = g["config"].get("activation", "relu") in ("tanh", "elu")
    for k, v in g.items():
        if k.startswith("grad."):
            got = grads[k[len("grad."):]].float().cpu().numpy()
            scale = max(1e-3, float(np.abs(v).max()))
            fro = float(np.linalg.norm(got - v) / max(1e-6, np.linalg.norm(v)))
            lim = (2e-2, 2e-2) if smooth else (0.5, 0.2)
            assert np.abs(got - v).max() <= lim[0] * scale and fro <= lim[1], (k, np.abs(got - v).max(), scale, fro)


@pytest.mark.parametrize("act,depth,bias,dropout", [("relu", 3, False, 0.0), ("relu", 3, True, 0.25), ("leakyrelu", 4, True, 0.0),
                                                    ("relu", 2, False, 0.0)])
def test_bf16_mirror_vs_rounding_aware_emulation(act, depth, bias, dropout):
    """The benchmarked backward (engine.bond_backward_tc: fused mirror steps, G / M^1 weight-gradient operands, per-term
    dW_i, dropout scale folded into the packed weights) on 1 500 molecules at h = 300, against the rounding-aware
    emulation of the same tier: every gradient <= 2 % (max-abs relative to the tensor's scale, and Frobenius); and against
    the f64 oracle: <= 6 % of the tensor's scale (bf16 kink noise averages out over ~75 k edges)."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(11)
    mgs = make_molecules(1500, seed=21)
    proto = BondMessagePassing(d_h=300, depth=depth, bias=bias, activation=act, dropout=dropout, precision="bf16")
    state = {k: v.detach().clone() for k, v in proto.state_dict().items()}
    gen = torch.Generator().manual_seed(5)
    Gm = torch.randn(1500, 300, generator=gen)

    def keep_mask(like):
        # deterministic {0,1} keep mask from the element index alone: identical on the GPU and in the emulation
        n = like.numel()
        i = torch.arange(n, dtype=torch.int64, device=like.device)
        hsh = (i * 2654435761 + 12345) % 4294967296
        m = ((hsh >> 8) % 1000 >= int(dropout * 1000)).to(like.dtype)
        return m.view_as(like)

    def make(device):
        mp = BondMessagePassing(d_h=300, depth=depth, bias=bias, activation=act, dropout=dropout, precision="bf16")
        mp.load_state_dict(state)
        mp = mp.to(device)
        mp.train()
        if dropout > 0:
            mp._mask_fn = keep_mask
        return mp

    loss_fn = lambda H, b: (MeanAggregation()(H, b.batch).float() * Gm.to(H.device)).sum()
    H_e, egrads = _emulated_run(lambda: make("cpu"), lambda: BatchMolGraph(mgs), None, loss_fn)
    mp = make("cuda")
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    H = mp(bmg)
    from chemprop_b200.engine import get_layout
    assert not mp.uses_composed_tier(get_layout(bmg))
    loss_fn(H, bmg).backward()
    assert (H.detach().float().cpu() - H_e).abs().max().item() <= 4e-2   # a few bf16 ulps where an f32 sum order differs
    assert ((H.detach().float().cpu() - H_e).abs() > 1e-3).float().mean().item() <= 1e-2
    for k, p in mp.named_parameters():
        _grad_close(p.grad.float(), egrads[k], 2e-2, (k, "vs emulation"))
    if dropout == 0.0:
        bm = BatchMolGraph(mgs)
        P = {k: v.double().requires_grad_(True) for k, v in state.items()}
        H_ref = R.message_passing_forward("bond", bm.V.double(), bm.E.double(), bm.edge_index, bm.rev_edge_index,
                                          P["W_i.weight"], P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"),
                                          P["W_o.weight"], P["W_o.bias"], depth, act)
        (R.aggregate(H_ref, bm.batch, "mean") * Gm.double()).sum().backward()
        for k, p in mp.named_parameters():
            _grad_close(p.grad.float(), P[k].grad, 6e-2, (k, "vs f64 oracle"))


@pytest.mark.parametrize("n_mols,min_atoms", [(3000, 1), (1024, 2), (1025, 2), (5000, 2)])
def test_layout_bit_exact_many_molecules(n_mols, min_atoms):
    """More molecules than one packing chunk (1024): chunk-boundary tile breaks, bit-exact vs numpy."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import get_layout
    from oracle import layout_np

    bmg = BatchMolGraph(make_molecules(n_mols, seed=n_mols, shuffle_edges=True, min_atoms=min_atoms))
    L = layout_np.build_layout(bmg.edge_index.numpy(), bmg.rev_edge_index.numpy(), bmg.batch.numpy(), n_mols)
    bmg.to("cuda")
    lay = get_layout(bmg)
    for k in ("perm", "inv_perm", "rowptr", "src_row", "dst_row", "rev_row", "mol_atom_ptr", "mol_row_ptr"):
        assert np.array_equal(getattr(lay, k).cpu().numpy(), L[k]), k
    assert lay.n_tiles == L["n_tiles"]
    for k in ("tile_mol_ptr", "tile_row_ptr", "tile_atom_ptr"):
        assert np.array_equal(getattr(lay, k).cpu().numpy()[: L["n_tiles"] + 1], L[k]), k
    assert (lay.flags, lay.max_indeg, lay.max_tile_rows, lay.max_tile_atoms) == (
        L["flags"], L["max_indeg"], L["max_tile_rows"], L["max_tile_atoms"])


@pytest.mark.parametrize("n_mols,kw", [(6, {}), (1500, dict(shuffle_edges=True, min_atoms=1)),
                                        (40, dict(mean_atoms=90, std_atoms=20, max_atoms=150))])
def test_host_meta_words_equal_device_meta_words(n_mols, kw):
    """The meta words our collate computes on the host (dmpnn_batch_meta_host; they let the step skip the device
    read-back) are the ones dmpnn_layout_build writes on the device."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import get_layout

    bmg = BatchMolGraph(make_molecules(n_mols, seed=n_mols, **kw))
    host_words = list(bmg._meta_host)
    bmg.to("cuda")
    assert bmg._meta_host == host_words
    lay = get_layout(bmg)
    assert lay._meta_host == host_words                      # taken from the host, no read-back
    assert lay.meta.tolist()[:5] == host_words[:5]           # and identical to the device's


def test_inputs_not_mutated():
    """tests/integration/test_regression_mol.py:143-226 of the reference."""
    g = load_golden("bond_d3_graphtf")
    mp = build_engine_module(g, "cuda", "fp32")
    bmg = golden_bmg(g, "cuda")
    before = [t.clone() for t in (bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch)]
    with torch.no_grad():
        mp(bmg)
    for a, b in zip(before, (bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch)):
        assert torch.equal(a, b)


def test_invalid_vd_shape_raises():
    from chemprop_b200.exceptions import InvalidShapeError

    g = load_golden("bond_d3_vd")
    mp = build_engine_module(g, "cuda", "fp32")
    bmg = golden_bmg(g, "cuda")
    with pytest.raises(InvalidShapeError):
        mp(bmg, torch.zeros(bmg.V.shape[0], 7, device="cuda"))


@pytest.mark.parametrize("kind,precision,n_mols,d_h,depth", [
    ("bond", "fp32", 1500, 300, 3), ("bond", "bf16", 1500, 300, 3), ("atom", "fp32", 800, 300, 3),
    ("atom", "bf16", 800, 128, 4), ("bond", "fp32", 300, 600, 6),
])
def test_medium_batch_vs_oracle(kind, precision, n_mols, d_h, depth):
    """Seeded synthetic batch: CUDA path vs the oracle restatement (CPU, fp64 accumulate reference)."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(0)
    mgs = make_molecules(n_mols, seed=5, shuffle_edges=(kind == "bond"))
    bmg = BatchMolGraph(mgs)
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_h=d_h, depth=depth, bias=True, precision=precision)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward(kind, bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], P["W_i.bias"], P["W_h.weight"], P["W_h.bias"],
                                      P["W_o.weight"], P["W_o.bias"], depth)
    a_ref = R.aggregate(H_ref, bmg.batch, "mean")
    a_ref.square().sum().backward()
    mp = mp.cuda()
    bmg.to("cuda")
    H = mp(bmg)
    a = MeanAggregation()(H, bmg.batch)
    a.float().square().sum().backward()
    tol = FP32_ATOL if precision == "fp32" else BF16_ATOL
    if precision == "fp32" and depth >= 6:
        tol = 5e-5  # fp32 round-off grows with depth x width (reference itself is only fp32-accurate here)
    if precision == "bf16":
        # 1e-2 is relative to the hidden-state scale: with |H| up to 2.5 (atom, depth 4) one bf16 ulp of the stored
        # output alone is 1.6e-2, so the bound scales with max|H| once that exceeds 1
        tol = tol * max(1.0, H_ref.detach().abs().max().item())
    assert (H.detach().double().cpu() - H_ref.detach()).abs().max().item() <= tol
    assert (a.detach().double().cpu() - a_ref.detach()).abs().max().item() <= tol
    for k, p in mp.named_parameters():
        ref = P[k].grad
        scale = max(1e-6, ref.abs().max().item())
        err = (p.grad.double().cpu() - ref).abs().max().item()
        assert err <= (2e-4 if precision == "fp32" else 6e-2) * scale, (k, err, scale)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_tile_packed_molecule_order_vs_oracle(precision):
    """bench.py's batch: molecules ordered by the loader's tile packing (dmpnn_tile_pack_order) -> nearly full 128-row
    tiles, 3-4 molecules in many of them.  Same parity bar as any other order, forward and gradients."""
    from chemprop_b200 import _lib
    from chemprop_b200.data import BatchMolGraph, make_molecules, tile_packing_order_of
    from chemprop_b200.nn import BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(0)
    mgs = make_molecules(1500, seed=8)
    plain_tiles = BatchMolGraph(mgs)._meta_host[_lib.META_N_TILES]
    mgs = [mgs[i] for i in tile_packing_order_of(mgs)]
    bmg = BatchMolGraph(mgs)
    tiles = bmg._meta_host[_lib.META_N_TILES]
    assert tiles < 0.9 * plain_tiles and bmg.E.shape[0] / (128 * tiles) > 0.9
    mp = BondMessagePassing(d_h=300, depth=3, precision=precision)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward("bond", bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], None, P["W_h.weight"], None, P["W_o.weight"], P["W_o.bias"], 3)
    a_ref = R.aggregate(H_ref, bmg.batch, "mean")
    a_ref.square().sum().backward()
    mp = mp.cuda()
    bmg.to("cuda")
    H = mp(bmg)
    a = MeanAggregation()(H, bmg.batch)
    a.float().square().sum().backward()
    tol = FP32_ATOL if precision == "fp32" else BF16_ATOL * max(1.0, H_ref.detach().abs().max().item())
    assert (H.detach().double().cpu() - H_ref.detach()).abs().max().item() <= tol
    assert (a.detach().double().cpu() - a_ref.detach()).abs().max().item() <= tol
    for k, p in mp.named_parameters():
        ref = P[k].grad
        scale = max(1e-6, ref.abs().max().item())
        assert (p.grad.double().cpu() - ref).abs().max().item() <= (2e-4 if precision == "fp32" else 6e-2) * scale, k


def test_aggregation_without_cached_segments():
    """Aggregation.forward(H, batch) called with a bare `batch` tensor (agg.py:39-59 contract)."""
    from chemprop_b200.nn import MeanAggregation, SumAggregation
    from oracle import restatement as R

    torch.manual_seed(1)
    batch = torch.tensor([0, 0, 0, 2, 2, 3, 5, 5, 5, 5])          # molecules 1 and 4 are empty
    H = torch.randn(10, 33, requires_grad=True)
    ref = R.aggregate(H, batch, "mean")
    Hc = H.detach().cuda().requires_grad_(True)
    out = MeanAggregation()(Hc, batch.cuda())
    torch.testing.assert_close(out.cpu(), ref.detach(), rtol=1e-6, atol=1e-6)
    assert out.shape == (6, 33) and float(out[1].abs().sum()) == 0.0   # empty graph -> zero row (agg.py:44-45)
    G = torch.randn(6, 33)
    (ref * G).sum().backward()
    (out * G.cuda()).sum().backward()
    torch.testing.assert_close(Hc.grad.cpu(), H.grad, rtol=1e-6, atol=1e-6)
    out_s = SumAggregation()(Hc.detach(), batch.cuda())
    torch.testing.assert_close(out_s.cpu(), R.aggregate(H.detach(), batch, "sum"), rtol=1e-6, atol=1e-6)


def test_reference_style_batchmolgraph_object():
    """A plain object exposing the reference's five tensors + __len__ works (no layout cache slot)."""
    g = load_golden("bond_d3_relu")

    class RefLike:
        __slots__ = ("V", "E", "edge_index", "rev_edge_index", "batch", "n")

        def __len__(self):
            return self.n

    b = RefLike()
    b.V, b.E = torch.from_numpy(g["V"]).cuda(), torch.from_numpy(g["E"]).cuda()
    b.edge_index, b.rev_edge_index = torch.from_numpy(g["edge_index"]).cuda(), torch.from_numpy(g["rev_edge_index"]).cuda()
    b.batch, b.n = torch.from_numpy(g["batch"]).cuda(), int(g["n_mols"])
    mp = build_engine_module(g, "cuda", "fp32")
    with torch.no_grad():
        H = mp(b)
    np.testing.assert_allclose(H.cpu().numpy(), g["H_v"], rtol=0, atol=FP32_ATOL)


def test_broken_reverse_map_is_rejected():
    from chemprop_b200 import DmpnnError

    g = load_golden("bond_d3_relu")
    bmg = golden_bmg(g, "cuda")
    bad = bmg.rev_edge_index.clone()
    bad[0], bad[1] = bad[1].item(), bad[0].item()
    bmg.rev_edge_index = bad
    mp = build_engine_module(g, "cuda", "fp32")
    with pytest.raises(DmpnnError, match="reverse-edge"):
        mp(bmg)


@pytest.mark.parametrize("kind,precision", [("atom", "bf16"), ("bond", "bf16"), ("atom", "fp32")])
def test_cgr_dims_vs_oracle(kind, precision):
    """BASELINE config 4 shapes: ~80-atom condensed reaction graphs, d_v = 106, d_e = 28 (readout K = 406 > 384:
    seven k slabs in the tensor-core GEMMs; graphs with > 128 directed edges take the unfused depth step)."""
    from chemprop_b200.data import BatchMolGraph, make_cgr_graphs
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(0)
    bmg = BatchMolGraph(make_cgr_graphs(120, seed=9))
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_v=106, d_e=28, d_h=300, depth=3, precision=precision)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward(kind, bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], None, P["W_h.weight"], None, P["W_o.weight"], P["W_o.bias"], 3)
    a_ref = R.aggregate(H_ref, bmg.batch, "mean")
    a_ref.square().sum().backward()
    mp = mp.cuda()
    bmg.to("cuda")
    from chemprop_b200 import engine
    engine.STEP_EVENTS = []
    try:
        H = mp(bmg)
        tags = {t for t, _, _ in engine.STEP_EVENTS}
    finally:
        engine.STEP_EVENTS = None
    if kind == "bond" and precision == "bf16":
        # ~170 directed edges per graph: every molecule is larger than a 128-row tile and still runs on the fused kernel
        assert engine.get_layout(bmg).max_tile_rows > 128 and tags == {"fused_first", "fused"}, tags
    if kind == "atom" and precision == "bf16":
        # ~80-atom graphs: every depth step of the atom path is one launch of the fused kernel's ATOM instantiation
        assert tags == {"atom_fused_first", "atom_fused"}, tags
    a = MeanAggregation()(H, bmg.batch)
    a.float().square().sum().backward()
    tol = FP32_ATOL if precision == "fp32" else BF16_ATOL * max(1.0, H_ref.detach().abs().max().item())
    assert (H.detach().double().cpu() - H_ref.detach()).abs().max().item() <= tol
    assert (a.detach().double().cpu() - a_ref.detach()).abs().max().item() <= tol
    for k, p in mp.named_parameters():
        ref = P[k].grad
        scale = max(1e-6, ref.abs().max().item())
        err = (p.grad.double().cpu() - ref).abs().max().item()
        # fp32: W_i's gradient sums ~10 k atom rows of 80-atom graphs in a different order than the f64 oracle
        assert err <= (1e-3 if precision == "fp32" else 6e-2) * scale, (k, err, scale)
