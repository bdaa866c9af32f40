"""CPU tier: EngineMulticomponentMessagePassing / EngineMulticomponentMPNN (chemprop_b200/nn/multi.py), the multicomponent
collate and MulticomponentPackedDataset under PackedBatchLoader, through the torch emulations of the kernel wrappers
(tests/emu.py), against the reference's own `MulticomponentMPNN.training_step` (tests/golden/fixture_mc_*.npz, written by
tools/make_golden_multicomponent.py).  `build_model`, `fixture_batches` and `check_fixture` are shared with
tests/test_gpu_multicomponent.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from oracle.ref_shim import reference_available
from tests import emu
from tests.test_classification_host import patch_classification
from tests.util import load_golden

CASES = ("shared_reg", "unshared_bn_xd", "shared_bin_edgeless")
N_COMP = 2


def build_model(case: str, g: dict, precision: str = "fp32"):
    """EngineMulticomponentMPNN of the fixture's configuration (tools/make_golden_multicomponent.py) holding its initial
    state: a strict load of the reference's state dict minus the criterion's torchmetrics states."""
    import chemprop_b200.nn as N

    if case == "shared_reg":
        blocks, agg = [N.BondMessagePassing(d_h=32, precision=precision)], N.MeanAggregation()
    elif case == "unshared_bn_xd":
        blocks = [N.BondMessagePassing(d_h=32, precision=precision),
                  N.AtomMessagePassing(d_h=24, activation="elu", bias=True, precision=precision)]
        agg = N.SumAggregation()
    else:
        blocks, agg = [N.BondMessagePassing(d_h=32, activation="tanh", bias=True, precision=precision)], N.NormAggregation(norm=20.0)
    mcmp = N.EngineMulticomponentMessagePassing(blocks, n_components=N_COMP, shared=case != "unshared_bn_xd")
    d_fp = mcmp.output_dim + (3 if "X_d" in g else 0)
    kw = dict(n_tasks=2, input_dim=d_fp, hidden_dim=24, n_layers=2)
    pred = N.EngineBinaryClassificationFFN(**kw) if case == "shared_bin_edgeless" else N.EngineRegressionFFN(**kw)
    xdt = N.ScaleTransform([0.0] * 3, [1.0] * 3) if "X_d" in g else None
    model = N.EngineMulticomponentMPNN(mcmp, agg, pred, batch_norm=bool(g["batch_norm"]), X_d_transform=xdt)
    state = {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")}
    res = model.load_state_dict({k: v for k, v in state.items() if not k.endswith(("total_loss", "num_samples"))},
                                strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model


def split_molgraphs(V, E, edge_index, rev_edge_index, batch, n_mols: int):
    """The MolGraphs of a collated batch (edges of a molecule are contiguous in a collate)."""
    from chemprop_b200.data import MolGraph

    atom_ptr = np.zeros(n_mols + 1, np.int64)
    np.cumsum(np.bincount(batch, minlength=n_mols), out=atom_ptr[1:])
    mol_of_edge = batch[edge_index[0]] if edge_index.shape[1] else np.zeros(0, np.int64)
    edge_ptr = np.zeros(n_mols + 1, np.int64)
    np.cumsum(np.bincount(mol_of_edge, minlength=n_mols), out=edge_ptr[1:])
    out = []
    for m in range(n_mols):
        a0, a1, e0, e1 = atom_ptr[m], atom_ptr[m + 1], edge_ptr[m], edge_ptr[m + 1]
        out.append(MolGraph(V[a0:a1], E[e0:e1], edge_index[:, e0:e1] - a0, rev_edge_index[e0:e1] - e0))
    return out


def fixture_molgraphs(g: dict) -> list:
    """Per component, the fixture's molecules."""
    n = int(g["n_dp"])
    return [split_molgraphs(g[f"V.{c}"], g[f"E.{c}"], g[f"edge_index.{c}"], g[f"rev_edge_index.{c}"], g[f"batch.{c}"], n)
            for c in range(N_COMP)]


def fixture_batches(g: dict, union: bool, device: str):
    """The fixture's batch: a list of the components' batches (as the reference saw them), or the interleaved union."""
    from chemprop_b200.data import BatchMolGraph

    if union:
        comps = fixture_molgraphs(g)
        bmg = BatchMolGraph([comps[c][m] for m in range(int(g["n_dp"])) for c in range(N_COMP)])
        bmg.to(device)
        return bmg
    out = []
    for c in range(N_COMP):
        b = BatchMolGraph.from_tensors(*(torch.from_numpy(g[f"{k}.{c}"]) for k in ("V", "E", "edge_index", "rev_edge_index",
                                                                                   "batch")), int(g["n_dp"]))
        b.to(device)
        out.append(b)
    return out


def check_fixture(case: str, union: bool, device: str, precision: str = "fp32", fp_tol: float = 1e-5,
                  rtol: float = 2e-4, atol: float = 2e-6):
    """Fingerprint, train-mode predictions, loss, every gradient, batch-norm statistics and eval-mode predictions of the
    engine model against the reference's `MulticomponentMPNN.training_step` on the same weights."""
    g = load_golden(f"fixture_mc_{case}")
    X_d = torch.from_numpy(g["X_d"]).to(device) if "X_d" in g else None
    Y, w = torch.from_numpy(g["Y"]).to(device), torch.from_numpy(g["w"]).to(device)
    bmgs = fixture_batches(g, union, device)
    model = build_model(case, g, precision).to(device)
    model.train()
    bn0 = {k: v.clone() for k, v in model.bn.state_dict().items()}
    with torch.no_grad():
        fp = model.fingerprint(bmgs, None, X_d)
        preds = model.predictor.train_step(fp)
    assert fp.shape == g["fingerprint"].shape
    np.testing.assert_allclose(fp.float().cpu().numpy(), g["fingerprint"], rtol=0, atol=fp_tol)
    np.testing.assert_allclose(preds.float().cpu().numpy(), g["preds_train"], rtol=1e-4, atol=max(fp_tol, 1e-5))
    model.bn.load_state_dict(bn0)
    model.zero_grad()
    loss = model.training_loss(bmgs, Y, w, None, X_d)
    loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy(), g["loss"], rtol=max(rtol, 1e-4), atol=atol)
    names = {k for k, _ in model.named_parameters()}
    assert names == {k[len("grad."):] for k in g if k.startswith("grad.")}
    for k, p in model.named_parameters():
        np.testing.assert_allclose(p.grad.cpu().numpy(), g["grad." + k], rtol=rtol, atol=atol, err_msg=k)
    if bool(g["batch_norm"]):
        for k in ("running_mean", "running_var", "num_batches_tracked"):
            np.testing.assert_allclose(getattr(model.bn, k).cpu().numpy(), g["after.bn." + k], rtol=1e-5, atol=1e-6)
    model.eval()
    with torch.no_grad():
        out = model(bmgs, None, X_d)
    np.testing.assert_allclose(out.float().cpu().numpy(), g["preds_eval"], rtol=1e-4, atol=max(fp_tol, 1e-5))


PATHS = [(c, False) for c in CASES] + [(c, True) for c in CASES if c != "unshared_bn_xd"]


@pytest.mark.parametrize("case,union", PATHS)
def test_engine_multicomponent_mpnn_matches_reference_training_step(case, union, monkeypatch):
    patch_classification(monkeypatch)
    check_fixture(case, union, "cpu")


def test_shared_union_and_list_paths_agree(monkeypatch):
    patch_classification(monkeypatch)
    g = load_golden("fixture_mc_shared_reg")
    res = []
    for union in (False, True):
        model = build_model("shared_reg", g)
        model.train()
        loss = model.training_loss(fixture_batches(g, union, "cpu"), torch.from_numpy(g["Y"]), torch.from_numpy(g["w"]))
        loss.backward()
        res.append((loss.detach(), {k: p.grad.clone() for k, p in model.named_parameters()}))
    torch.testing.assert_close(res[1][0], res[0][0], rtol=1e-6, atol=1e-7)
    for k in res[0][1]:
        torch.testing.assert_close(res[1][1][k], res[0][1][k], rtol=1e-5, atol=1e-7, msg=k)


def test_container_mirrors_the_reference_and_validates_its_inputs():
    import chemprop_b200.nn as N
    from chemprop_b200.data import BatchMolGraph, make_molecules

    b = N.BondMessagePassing(d_h=16)
    shared = N.EngineMulticomponentMessagePassing([b], n_components=3, shared=True)
    assert len(shared) == 3 and shared.output_dim == 48 and all(blk is b for blk in shared.blocks)
    assert [k for k in shared.state_dict() if k.endswith("W_h.weight")] == [f"blocks.{c}.W_h.weight" for c in range(3)]
    assert set(shared.hparams) == {"cls", "blocks", "n_components", "shared"} and shared.hparams["cls"] is type(shared)
    with pytest.raises(ValueError, match="empty"):
        N.EngineMulticomponentMessagePassing([], n_components=2)
    with pytest.raises(ValueError, match="n_components"):
        N.EngineMulticomponentMessagePassing([b], shared=True)
    unshared = N.EngineMulticomponentMessagePassing([b, N.AtomMessagePassing(d_h=8)], n_components=2)
    assert unshared.output_dim == 24
    union = BatchMolGraph(make_molecules(4, seed=1))
    with pytest.raises(ValueError, match="shared"):
        unshared(union)
    with pytest.raises(ValueError, match="3 components"):
        shared([union, union])
    model = N.EngineMulticomponentMPNN(shared, N.MeanAggregation())
    assert model.predictor.ffn[0][0].in_features == 48
    with pytest.raises(ValueError, match="whole number"):
        model.fingerprint(BatchMolGraph(make_molecules(4, seed=2)))


@pytest.mark.parametrize("shared", [False, True])
def test_reference_state_dict_loads_strictly(shared):
    """A reference MulticomponentMPNN's state dict (shared: with its duplicated `blocks.<c>.*` keys), without `metrics.*`,
    loads into EngineMulticomponentMPNN with strict=True (the fixtures' states were taken from the reference model)."""
    case = "shared_reg" if shared else "unshared_bn_xd"
    g = load_golden(f"fixture_mc_{case}")
    model = build_model(case, g)
    ref_keys = {k[len("param."):] for k in g if k.startswith("param.") and not k.endswith(("total_loss", "num_samples"))}
    assert set(model.state_dict()) == ref_keys
    assert ("message_passing.blocks.1.W_h.weight" in ref_keys)


@pytest.mark.skipif(not reference_available(), reason="needs the unmodified reference package (CHEMPROP_REFERENCE_ROOT)")
@pytest.mark.parametrize("shared", [False, True])
def test_reference_checkpoint_round_trip_rebuilds_the_engine_container(shared, tmp_path):
    """chemprop.models.utils.save_model / load_model(multicomponent=True) (models/multi.py:68-109 rebuilds every block and
    the container from hparams["cls"]): a model saved with the engine's container and blocks comes back with them."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.models import MulticomponentMPNN
    from chemprop.models.utils import load_model, save_model

    import chemprop_b200.nn as ours

    torch.manual_seed(3)
    blocks = ([ours.BondMessagePassing(d_h=16, precision="bf16", activation="tanh")] if shared else
              [ours.BondMessagePassing(d_h=16), ours.AtomMessagePassing(d_h=8, depth=4, bias=True)])
    mcmp = ours.EngineMulticomponentMessagePassing(blocks, n_components=2, shared=shared)
    model = MulticomponentMPNN(mcmp, ours.SumAggregation(), ref_nn.RegressionFFN(input_dim=mcmp.output_dim))
    path = tmp_path / "model.pt"
    save_model(path, model)
    back = load_model(path, multicomponent=True)
    mp = back.message_passing
    assert type(mp) is ours.EngineMulticomponentMessagePassing and mp.shared == shared and mp.n_components == 2
    assert [type(b) for b in mp.blocks] == [type(b) for b in mcmp.blocks]
    if shared:
        assert mp.blocks[0] is mp.blocks[1] and mp.blocks[0].precision == "bf16"
    else:
        assert mp.blocks[1].depth == 4 and mp.blocks[1].W_i.bias is not None
    assert type(back.agg) is ours.SumAggregation
    for (ka, a), (kb, b) in zip(model.state_dict().items(), back.state_dict().items()):
        assert ka == kb and torch.equal(a, b)


def _datum(mg, rng):
    from chemprop_b200.data import Datum

    return Datum(mg, rng.normal(size=(mg.V.shape[0], 2)).astype(np.float32), rng.normal(size=3).astype(np.float32),
                 rng.normal(size=2).astype(np.float32), float(rng.uniform(0.5, 2)), None, None)


def test_collate_multicomponent_union_is_interleaved_and_per_component_as_the_reference():
    from chemprop_b200.data import BatchMolGraph, collate_batch, collate_multicomponent, make_molecules

    rng = np.random.default_rng(0)
    solutes = make_molecules(7, seed=11, mean_atoms=9, std_atoms=3)
    solvents = make_molecules(7, seed=12, mean_atoms=2, std_atoms=1, min_atoms=1, max_atoms=4)
    data = [[_datum(a, rng), _datum(b, rng)] for a, b in zip(solutes, solvents)]
    per = collate_multicomponent(data)
    uni = collate_multicomponent(data, union=True)
    ref0 = collate_batch([d[0] for d in data])
    for a, b in zip(per[2:], ref0[2:]):
        assert (a is None and b is None) or torch.equal(a, b)
    for a, b in zip(uni[2:], ref0[2:]):
        assert (a is None and b is None) or torch.equal(a, b)
    assert isinstance(per.bmgs, list) and len(per.bmgs) == 2 and isinstance(uni.bmgs, BatchMolGraph)
    u = uni.bmgs
    assert len(u) == 14 and u._meta_host is not None
    mgs = split_molgraphs(u.V.numpy(), u.E.numpy(), u.edge_index.numpy(), u.rev_edge_index.numpy(), u.batch.numpy(), 14)
    for m in range(7):
        for c, comp in enumerate((solutes, solvents)):
            got, want = mgs[m * 2 + c], comp[m]
            for x, y in zip(got, want):
                np.testing.assert_array_equal(np.asarray(x), np.asarray(y))
    want_Vd = np.concatenate([d[c].V_d for d in data for c in range(2)])
    np.testing.assert_array_equal(uni.V_ds.numpy(), want_Vd)
    for c in range(2):
        np.testing.assert_array_equal(per.V_ds[c].numpy(), np.concatenate([d[c].V_d for d in data]))


def _mc_dataset(n=41, union=True):
    from chemprop_b200.data import MulticomponentPackedDataset, PackedMolGraphDataset, make_molecules

    solutes = make_molecules(n, seed=21, mean_atoms=12, std_atoms=4)
    solvents = make_molecules(n, seed=22, mean_atoms=2, std_atoms=1.5, min_atoms=1, max_atoms=5)
    packed = [PackedMolGraphDataset.from_molgraphs(m) for m in (solutes, solvents)]
    return MulticomponentPackedDataset(packed, union=union), (solutes, solvents), packed


@pytest.mark.parametrize("world", [1, 3])
@pytest.mark.parametrize("pack", [False, True])
def test_loader_draws_the_packed_batch_loader_datapoints_in_interleaved_order(world, pack):
    """Same seed -> the same data points per batch as PackedBatchLoader over one component (the samplers, the rank split and
    drop_last are its own); each union batch is the interleaved collate of those data points; the extras follow them."""
    from chemprop_b200.data import BatchMolGraph, PackedBatchLoader

    mc, (solutes, solvents), packed = _mc_dataset()
    y = np.arange(len(mc), dtype=np.float32)
    for rank in range(world):
        kw = dict(batch_size=8, shuffle=True, seed=5, rank=rank, world=world, pack_tiles=pack, arrays={"y": y})
        ref = PackedBatchLoader(packed[0], **kw)
        lo = PackedBatchLoader(mc, **kw)
        assert len(lo) == len(ref)
        for _epoch in range(2):
            n = 0
            for a, b in zip(lo, ref):                        # host batches are views of the loader's ring: check each now
                n += 1
                assert sorted(a.ids.tolist()) == sorted(b.ids.tolist())
                np.testing.assert_array_equal(a.extras["y"].numpy(), y[a.ids])
                exp = BatchMolGraph([(solutes, solvents)[c][m] for m in a.ids for c in range(2)])
                for t, s in zip((a.bmg.V, a.bmg.E, a.bmg.edge_index, a.bmg.rev_edge_index, a.bmg.batch),
                                (exp.V, exp.E, exp.edge_index, exp.rev_edge_index, exp.batch)):
                    assert torch.equal(t, s)
                assert a.bmg._meta_host == exp._meta_host
            assert n == len(ref)


def test_loader_packs_data_points_by_summed_size_and_meta_words_match_the_layout_build():
    from chemprop_b200.data import tile_packing_order

    mc, _, packed = _mc_dataset(60)
    ids = np.random.default_rng(3).permutation(60)[:25]
    order = mc.packed_order(ids)
    na = sum(d.n_atoms(ids) for d in packed)
    ne = sum(d.n_edges(ids) for d in packed)
    np.testing.assert_array_equal(order, ids[tile_packing_order(na, ne)])
    bmg = mc.batch(order)
    np.testing.assert_array_equal(np.bincount(bmg.batch.numpy(), minlength=50)[0::2], packed[0].n_atoms(order))
    np.testing.assert_array_equal(np.bincount(bmg.batch.numpy(), minlength=50)[1::2], packed[1].n_atoms(order))
    emu.build_layout(bmg.edge_index, bmg.rev_edge_index, bmg.batch, len(bmg), bmg._meta_host)   # asserts the meta words


def test_unshared_loader_yields_the_components_batches_of_the_same_ids():
    from chemprop_b200.data import BatchMolGraph, PackedBatchLoader

    mc, comps, _ = _mc_dataset(union=False)
    for b in PackedBatchLoader(mc, batch_size=16, shuffle=True, seed=1):
        assert isinstance(b.bmg, list) and len(b.bmg) == 2
        for c in range(2):
            exp = BatchMolGraph([comps[c][m] for m in b.ids])
            assert torch.equal(b.bmg[c].V, exp.V) and torch.equal(b.bmg[c].edge_index, exp.edge_index)
            assert b.bmg[c]._meta_host == exp._meta_host


def test_union_mode_holds_the_features_once():
    """In union mode only the stacked copy is kept (and moved by `to`): the components' arrays are not referenced."""
    import gc
    import weakref

    mc, _, packed = _mc_dataset()
    refs = [weakref.ref(d) for d in packed]
    del packed
    gc.collect()
    assert all(r() is None for r in refs) and mc.components is None
    assert mc.stacked.V_all.shape[0] == int(mc._atoms.sum())
    moved = mc.to("cpu")
    assert moved.stacked is not None and moved.components is None and len(moved) == len(mc) == 41


def test_union_needs_components_of_one_feature_width():
    from chemprop_b200.data import MulticomponentPackedDataset, PackedMolGraphDataset, make_molecules

    a = PackedMolGraphDataset.from_molgraphs(make_molecules(5, seed=1))
    b = PackedMolGraphDataset.from_molgraphs(make_molecules(5, seed=2, d_v=40))
    with pytest.raises(ValueError, match="feature widths"):
        MulticomponentPackedDataset([a, b], union=True)
    MulticomponentPackedDataset([a, b], union=False)
    with pytest.raises(ValueError, match="equal lengths"):
        MulticomponentPackedDataset([a, PackedMolGraphDataset.from_molgraphs(make_molecules(4, seed=3))])


def test_replicate_is_the_concatenation_of_copies():
    from chemprop_b200.data import PackedMolGraphDataset, make_molecules

    ds = PackedMolGraphDataset.from_molgraphs(make_molecules(9, seed=4))
    r = ds.replicate(3)
    assert len(r) == 27
    for i in (0, 8, 9, 17, 26):
        for x, y in zip(r.molgraph(i), ds.molgraph(i % 9)):
            np.testing.assert_array_equal(np.asarray(x), np.asarray(y))
