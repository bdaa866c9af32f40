"""CPU tier: host-side mirror of the reference module interface (constructor, hparams,
state-dict keys, error behaviour) -- and that the product path has NO CPU fallback."""
import copy

import numpy as np
import pytest
import torch

from chemprop_b200 import DmpnnError
from chemprop_b200.data import BatchMolGraph, Datum, collate_batch, make_molecules
from chemprop_b200.nn import (AggregationRegistry, AtomMessagePassing, BondMessagePassing, MeanAggregation,
                              NormAggregation, SumAggregation)
from tests.util import load_golden, params_of


def test_state_dict_keys_and_shapes_match_reference_checkpoint():
    """Keys/shapes of tests/data/example_model_v2_regression_mol.pt (golden `bond_d3_trained`)."""
    g = load_golden("bond_d3_trained")
    mp = BondMessagePassing()
    sd = mp.state_dict()
    ref = params_of(g)
    assert set(sd) == set(ref) == {"W_i.weight", "W_h.weight", "W_o.weight", "W_o.bias"}
    for k in sd:
        assert tuple(sd[k].shape) == tuple(ref[k].shape)
    mp.load_state_dict(ref)
    assert mp.output_dim == 300


@pytest.mark.parametrize("cls", [BondMessagePassing, AtomMessagePassing])
def test_constructor_contract(cls):
    mp = cls(d_v=10, d_e=4, d_h=32, bias=True, depth=4, activation="tanh", undirected=False, d_vd=3)
    hp = mp.hparams
    for k in ("d_v", "d_e", "d_h", "bias", "depth", "dropout", "activation", "undirected", "d_vd",
              "V_d_transform", "graph_transform", "cls"):
        assert k in hp
    assert hp["cls"] is cls
    rebuilt = hp["cls"](**{k: v for k, v in hp.items() if k != "cls"})   # models/model.py:267-271
    assert type(rebuilt) is cls and rebuilt.depth == 4 and isinstance(rebuilt.tau, torch.nn.Tanh)
    assert mp.W_d.in_features == 35 and mp.output_dim == 35
    assert mp.W_i.in_features == (14 if cls is BondMessagePassing else 10)
    assert mp.W_h.in_features == (32 if cls is BondMessagePassing else 36)
    assert mp.W_o.bias is not None and mp.W_i.bias is not None


def test_aggregation_registry_and_hparams():
    assert AggregationRegistry["mean"] is MeanAggregation and AggregationRegistry["sum"] is SumAggregation
    agg = AggregationRegistry["norm"](norm=50.0)
    assert isinstance(agg, NormAggregation) and agg.hparams == {"dim": 0, "cls": NormAggregation, "norm": 50.0}


def test_no_cpu_fallback():
    bmg = BatchMolGraph(make_molecules(3, seed=0))
    mp = BondMessagePassing(d_h=16)
    with pytest.raises(DmpnnError, match="no CPU fallback|CUDA"):
        mp(bmg)
    with pytest.raises(DmpnnError):
        MeanAggregation()(torch.zeros(5, 4), torch.tensor([0, 0, 1, 1, 2]))


def test_batchmolgraph_surface():
    mgs = make_molecules(5, seed=1)
    bmg = BatchMolGraph(mgs)
    assert len(bmg) == 5
    assert bmg.to("cpu") is None                       # in place, returns None (collate.py:68-73)
    c = copy.copy(bmg)
    c.V = c.V * 2
    assert not torch.equal(c.V, bmg.V) and c.edge_index is bmg.edge_index


def test_collate_batch_contract():
    mgs = make_molecules(2, seed=2)
    data = [Datum(mg, np.ones((mg.V.shape[0], 2)), np.array([1.0, 2.0]), np.array([0.5]), 2.0,
                  np.array([True]), np.array([False])) for mg in mgs]
    tb = collate_batch(data)
    assert isinstance(tb.bmg, BatchMolGraph) and tb.V_d.shape == (tb.bmg.V.shape[0], 2)
    assert tb.X_d.shape == (2, 2) and tb.Y.shape == (2, 1) and tb.w.tolist() == [[2.0], [2.0]]
    assert tb.lt_mask.dtype == torch.bool


def test_collate_batch_tile_packing_reorders_every_field_alike():
    from chemprop_b200 import _lib

    mgs = make_molecules(600, seed=4)
    data = [Datum(mg, np.full((mg.V.shape[0], 1), i, dtype=np.float32), np.array([float(i)]), np.array([float(i)]), float(i),
                  None, None) for i, mg in enumerate(mgs)]
    plain, packed = collate_batch(data), collate_batch(data, pack_tiles=True)
    order = packed.Y[:, 0].long()
    assert torch.equal(torch.sort(order).values, torch.arange(600)) and not torch.equal(order, torch.arange(600))
    assert torch.equal(packed.w[:, 0].long(), order) and torch.equal(packed.X_d[:, 0].long(), order)
    ref = BatchMolGraph([mgs[i] for i in order.tolist()])
    assert torch.equal(packed.bmg.V, ref.V) and torch.equal(packed.bmg.edge_index, ref.edge_index)
    assert torch.equal(packed.V_d[:, 0].long(), order[packed.bmg.batch])            # per-atom descriptors follow their molecule
    assert packed.bmg._meta_host[_lib.META_N_TILES] < 0.9 * plain.bmg._meta_host[_lib.META_N_TILES]
    assert torch.equal(plain.Y[:, 0].long(), torch.arange(600))


def test_compact_transfer_staging_is_the_rounded_batch():
    """transfer_dtype=bfloat16 stages bf16 features / int32 indices next to the public f32 / int64 view."""
    mgs = make_molecules(40, seed=3)
    plain, compact = BatchMolGraph(mgs), BatchMolGraph(mgs, transfer_dtype=torch.bfloat16)
    assert compact.V.dtype == torch.float32 and compact.edge_index.dtype == torch.int64      # public view unchanged
    assert torch.equal(compact.V, plain.V) and torch.equal(compact.edge_index, plain.edge_index)
    Vb, Eb, ei, rv, bt = compact._xfer
    assert (Vb.dtype, Eb.dtype, ei.dtype, rv.dtype, bt.dtype) == (torch.bfloat16, torch.bfloat16, torch.int32, torch.int32, torch.int32)
    assert torch.equal(Vb, plain.V.bfloat16()) and torch.equal(Eb, plain.E.bfloat16())
    assert torch.equal(ei.long(), plain.edge_index) and torch.equal(rv.long(), plain.rev_edge_index)
    assert torch.equal(bt.long(), plain.batch)
    assert compact.transfer_nbytes() * 2 == plain.transfer_nbytes()
    with pytest.raises(ValueError):
        BatchMolGraph(mgs, transfer_dtype=torch.float16)


def test_collate_extension_and_ctypes_paths_agree():
    """BatchMolGraph built through the CPython collate extension == through the ctypes C-ABI path, including dtype /
    layout coercion of the inputs (float64, Fortran-ordered, int32 indices) and the compact transfer copy."""
    from chemprop_b200.data import MolGraph
    from chemprop_b200.data.collate import _collate_ext

    mgs = make_molecules(60, seed=12, shuffle_edges=True, min_atoms=1)
    odd = [MolGraph(np.asfortranarray(mg.V.astype(np.float64)), mg.E[:, ::1].astype(np.float64), mg.edge_index.astype(np.int32),
                    mg.rev_edge_index.astype(np.int32)) for mg in mgs[:10]] + list(mgs[10:])
    ref = BatchMolGraph(mgs, transfer_dtype=torch.bfloat16, use_extension=False)
    for src in (mgs, odd, tuple(mgs)):
        for ext in (True, False):
            got = BatchMolGraph(src, transfer_dtype=torch.bfloat16, use_extension=ext)
            for k in ("V", "E", "edge_index", "rev_edge_index", "batch"):
                assert torch.equal(getattr(got, k), getattr(ref, k)), (k, ext)
            for a, b in zip(got._xfer, ref._xfer):
                assert a.dtype == b.dtype and torch.equal(a.float() if a.is_floating_point() else a,
                                                          b.float() if b.is_floating_point() else b)
    assert len(BatchMolGraph([])) == 0 and BatchMolGraph([]).V.shape[0] == 0
    if _collate_ext() is None:
        pytest.skip("collate extension not built here (ctypes path covered)")
    m0 = next(mg for mg in mgs if mg.E.shape[0] > 0)
    bad = [MolGraph(m0.V, m0.E[:-1], m0.edge_index, m0.rev_edge_index)]
    for ext in (True, False):
        with pytest.raises(ValueError, match="MolGraph.E has"):
            BatchMolGraph(bad, use_extension=ext)


def _np_meta(bmg):
    from chemprop_b200 import _lib
    from oracle import layout_np

    L = layout_np.build_layout(bmg.edge_index.numpy(), bmg.rev_edge_index.numpy(), bmg.batch.numpy(), len(bmg))
    m = [0] * _lib.META_WORDS
    m[_lib.META_N_TILES], m[_lib.META_FLAGS], m[_lib.META_MAX_INDEG] = L["n_tiles"], L["flags"], L["max_indeg"]
    m[_lib.META_MAX_TILE_ROWS], m[_lib.META_MAX_TILE_ATOMS] = L["max_tile_rows"], L["max_tile_atoms"]
    return m


@pytest.mark.parametrize("n_mols,kw", [(0, {}), (1, {}), (7, dict(min_atoms=1)), (300, dict(shuffle_edges=True)),
                                        (1024, {}), (1025, dict(min_atoms=1)), (3000, dict(shuffle_edges=True, min_atoms=1)),
                                        (40, dict(mean_atoms=90, std_atoms=20, max_atoms=150))])
def test_host_meta_bit_exact_vs_numpy_layout(n_mols, kw):
    """dmpnn_batch_meta_host (what lets the training step skip the device read-back of the layout meta words) against
    oracle/layout_np.py -- which the GPU tests in turn hold bit-exact against dmpnn_layout_build."""
    bmg = BatchMolGraph(make_molecules(n_mols, seed=n_mols + 3, **kw))
    assert bmg._meta_host == _np_meta(bmg)
    moved = BatchMolGraph.from_tensors(bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch, len(bmg))
    assert moved._meta_host == bmg._meta_host
    c = copy.copy(bmg)
    assert c._meta_host == bmg._meta_host
    if n_mols >= 7:
        assert bmg._meta_host[0] >= 1 and bmg._meta_host[1] == 7


def test_host_meta_flags_on_invalid_batches_and_invalidation():
    from chemprop_b200 import _lib
    from chemprop_b200.data.collate import host_meta

    bmg = BatchMolGraph(make_molecules(20, seed=8))
    ei, rev, bt = bmg.edge_index.clone(), bmg.rev_edge_index.clone(), bmg.batch.clone()
    bad_rev = rev.clone()
    bad_rev[0] = 2                                                      # edge 0's reverse is edge 1
    f = host_meta(ei, bad_rev, bt, 20)[_lib.META_FLAGS]
    assert f & _lib.FLAG_INDEX_IN_RANGE and not f & _lib.FLAG_REV_INVOLUTION and f & _lib.FLAG_BATCH_SORTED
    bad_bt = bt.clone()
    bad_bt[0], bad_bt[-1] = bt[-1].item(), bt[0].item()
    f = host_meta(ei, rev, bad_bt, 20)[_lib.META_FLAGS]
    assert f & _lib.FLAG_INDEX_IN_RANGE and not f & _lib.FLAG_BATCH_SORTED
    bad_ei = ei.clone()
    bad_ei[0, 3] = bmg.V.shape[0]
    assert host_meta(bad_ei, rev, bt, 20)[_lib.META_FLAGS] == 0
    for bad in ((ei, bad_rev, bt), (ei, rev, bad_bt), (bad_ei, rev, bt)):
        b = BatchMolGraph.from_tensors(bmg.V, bmg.E, *bad, 20)
        assert b._meta_host == _np_meta(b) or b._meta_host[_lib.META_FLAGS] == _np_meta(b)[_lib.META_FLAGS] != 7
    # replacing an index tensor drops the host words (and the cached layout): the engine re-derives them on the device
    assert bmg._meta_host is not None
    bmg.rev_edge_index = bad_rev
    assert bmg._meta_host is None and bmg._layout is None
    assert host_meta(ei.int(), rev, bt, 20) is None                     # not the reference's int64: no host words


def test_batchmolgraph_pickles_with_its_staging_copy_and_meta_words():
    """DataLoader worker processes hand batches over by pickling (chemprop/cli/common.py:35 `num_workers`)."""
    import pickle

    b = BatchMolGraph(make_molecules(5, seed=0), transfer_dtype=torch.bfloat16)
    c = pickle.loads(pickle.dumps(b))
    assert len(c) == 5 and torch.equal(c.edge_index, b.edge_index) and torch.equal(c.V, b.V)
    assert c._meta_host == b._meta_host and c._xfer is not None and c._layout is None


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    """No silent fallback: without libdmpnn_sm90.so every entry into the engine raises, naming the build command."""
    from chemprop_b200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", tmp_path / "libdmpnn_sm90.so")
    with pytest.raises(DmpnnError, match="chemprop_b200.build.*no CPU / PyTorch fallback"):
        _lib.load()
    with pytest.raises(DmpnnError, match="not found"):
        BatchMolGraph(make_molecules(2, seed=0), use_extension=False)          # the host collate is a library call too


def test_product_path_never_imports_the_oracle_or_the_reference():
    """oracle/ is test infrastructure: nothing under chemprop_b200/ may import it (or chemprop, or tests) -- checked on the
    syntax trees, so that comments and docstrings citing the oracle do not count."""
    import ast
    import pathlib

    root = pathlib.Path(__file__).resolve().parents[1] / "chemprop_b200"
    banned = {"oracle", "tests"}
    optional = {"chemprop"}                       # only integrate.py may import the reference, inside a function, on request
    for path in sorted(root.rglob("*.py")):
        tree = ast.parse(path.read_text(), filename=str(path))
        for node in ast.walk(tree):
            names = []
            if isinstance(node, ast.Import):
                names = [a.name for a in node.names]
            elif isinstance(node, ast.ImportFrom) and node.level == 0 and node.module:
                names = [node.module]
            for n in names:
                top = n.split(".")[0]
                assert top not in banned, (str(path), n)
                if top in optional:
                    assert path.name == "integrate.py", (str(path), n)


def test_collate_batch_in_dataloader_worker_processes():
    """The reference runs `collate_batch` in CPU-only DataLoader worker processes (chemprop/data/dataloader.py:88-96,
    `num_workers`): the batch object crosses a process boundary by pickle and must arrive whole -- tensors, size and the
    host-computed layout meta words (without them the training step would fall back to a device read-back)."""
    import pickle

    from chemprop_b200.data.collate import Datum

    mgs = make_molecules(12, seed=2)
    data = [Datum(m, None, None, np.array([float(i)], dtype=np.float32), 1.0, None, None) for i, m in enumerate(mgs)]
    direct = [collate_batch(data[:6]), collate_batch(data[6:])]
    dl = torch.utils.data.DataLoader(data, batch_size=6, collate_fn=collate_batch, num_workers=2)
    got = list(dl)
    assert len(got) == 2
    for a, b in zip(got, direct):
        for k in ("V", "E", "edge_index", "rev_edge_index", "batch"):
            assert torch.equal(getattr(a.bmg, k), getattr(b.bmg, k)), k
        assert len(a.bmg) == len(b.bmg) == 6 and a.bmg._meta_host == b.bmg._meta_host is not None
        assert torch.equal(a.Y, b.Y) and torch.equal(a.w, b.w)
    c = pickle.loads(pickle.dumps(direct[0].bmg))
    assert c._meta_host == direct[0].bmg._meta_host and c._layout is None and torch.equal(c.E, direct[0].bmg.E)
