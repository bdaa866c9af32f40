"""CPU tier of tests/test_gpu_layout_scale.py: the packing restatement of oracle/layout_np.py against a brute-force walk,
dmpnn_batch_meta_host against the oracle on the same index-only batches (valid ones, and ones with out-of-range indices,
which only the host may see: on the device k_rev_rows would read `perm` entries nobody wrote), the work table's
restatement on tiles of more than 128 atoms, and Layout.step_tables' decision to build it."""
import numpy as np
import pytest
import torch

from tests.test_gpu_layout_scale import (BATCHES, _batch, _chunks, _scan_blocks, fragment_batch, host_meta,
                                         index_batch, invalid_batch, INVALID_IN_RANGE)


def _brute_force_tiles(ap, rp, row_limit, atom_limit, chunk=1024):
    """The greedy rule walked molecule by molecule (the form dmpnn_batch_meta_host uses)."""
    B = len(ap) - 1
    starts, t = [], 0
    for m in range(B):
        if m > t and (m % chunk == 0 or rp[m + 1] - rp[t] > row_limit or ap[m + 1] - ap[t] > atom_limit):
            starts.append(t)
            t = m
    if B > 0:
        starts.append(t)
    tm = np.array(starts + [B], np.int64)
    mr = int(np.diff(np.asarray(rp)[tm]).max()) if B else 0
    ma = int(np.diff(np.asarray(ap)[tm]).max()) if B else 0
    return tm, mr, ma


@pytest.mark.parametrize("seed", range(12))
def test_pack_tiles_matches_brute_force_walk(seed):
    """pack_tiles (bisection per tile start, as the kernel does) against the molecule-by-molecule walk on random offset
    arrays: empty and oversized molecules, limits from 1 to beyond the batch, 0 .. 3000 molecules."""
    from oracle import layout_np

    rng = np.random.default_rng(seed)
    B = int(rng.choice([0, 1, 2, 1023, 1024, 1025, 2049, 3000]))
    na = rng.integers(0, 200 if seed % 3 == 0 else 40, size=B)
    nr = rng.integers(0, 300 if seed % 2 == 0 else 60, size=B)
    na[rng.random(B) < 0.1] = 0
    nr[rng.random(B) < 0.1] = 0
    ap = np.concatenate([[0], np.cumsum(na)]).astype(np.int32)
    rp = np.concatenate([[0], np.cumsum(nr)]).astype(np.int32)
    for rl, al in ((128, 128), (1, 1), (64, 128), (4096, 1), (1024, 128), (10 ** 6, 10 ** 6)):
        tm, mr, ma = layout_np.pack_tiles(ap, rp, rl, al)
        btm, bmr, bma = _brute_force_tiles(ap, rp, rl, al)
        assert tm.tolist() == btm.tolist() and (mr, ma) == (bmr, bma), (B, rl, al)


def test_batches_reach_the_boundaries():
    """The GPU file's batch list reaches what it is for: more than 1024 scan blocks and tile chunks, exactly 1024 / 1025
    scan blocks, one and two chunks around B = 1024."""
    sizes = {n: (_batch(n)["batch"].shape[0], _batch(n)["B"]) for n in
             ("million-tiny", "V+1=2048*1024", "V+1=2048*1024+1", "B=1024", "B=1025")}
    assert _scan_blocks(sizes["million-tiny"][0]) > 1024 and _chunks(sizes["million-tiny"][1]) > 1024
    assert _scan_blocks(sizes["V+1=2048*1024"][0]) == 1024 and _chunks(sizes["V+1=2048*1024"][1]) == 1024
    assert _scan_blocks(sizes["V+1=2048*1024+1"][0]) == 1025
    assert _chunks(sizes["B=1024"][1]) == 1 and _chunks(sizes["B=1025"][1]) == 2


@pytest.mark.parametrize("name", BATCHES)
def test_batch_meta_host_matches_oracle(name):
    """dmpnn_batch_meta_host (the words the sync-free training step trusts) equals the restatement on every batch of the
    GPU file, the million-molecule ones and the chunk boundaries included."""
    from chemprop_b200 import _lib
    from oracle import layout_np

    b = _batch(name)
    L = layout_np.build_layout(b["edge_index"], b["rev_edge_index"], b["batch"], b["B"])
    want = [0] * _lib.META_WORDS
    want[_lib.META_N_TILES], want[_lib.META_FLAGS], want[_lib.META_MAX_INDEG] = L["n_tiles"], L["flags"], L["max_indeg"]
    want[_lib.META_MAX_TILE_ROWS], want[_lib.META_MAX_TILE_ATOMS] = L["max_tile_rows"], L["max_tile_atoms"]
    assert L["flags"] == 7
    assert host_meta(b).tolist() == want


def _out_of_range(case):
    b = index_batch(np.full(1500, 20), seed=2)
    ei, rev, batch = b["edge_index"].copy(), b["rev_edge_index"].copy(), b["batch"].copy()
    V, E = batch.shape[0], rev.shape[0]
    if case == "src-too-large":
        ei[0, 17] = V
    elif case == "dst-negative":
        ei[1, E - 1] = -1
    elif case == "rev-too-large":
        rev[5] = E
    elif case == "rev-negative":
        rev[0] = -3
    elif case == "batch-too-large":
        batch[-1] = b["B"]
    elif case == "batch-negative":
        batch[0] = -1
    return dict(edge_index=ei, rev_edge_index=rev, batch=batch, B=b["B"])


@pytest.mark.parametrize("case", ["src-too-large", "dst-negative", "rev-too-large", "rev-negative", "batch-too-large",
                                  "batch-negative"] + INVALID_IN_RANGE)
def test_batch_meta_host_flags_of_invalid_batches(case):
    """Invalid batches, out-of-range indices included: dmpnn_batch_meta_host's flags word equals the restatement's (0 with
    an index out of range), and the engine refuses a batch carrying those words before it launches anything."""
    from chemprop_b200 import _lib, engine
    from oracle import layout_np

    b = invalid_batch(case) if case in INVALID_IN_RANGE else _out_of_range(case)
    want = layout_np.layout_flags(b["edge_index"], b["rev_edge_index"], b["batch"], b["B"])
    assert want != 7 and (want == 0) == (case not in INVALID_IN_RANGE), want
    meta = host_meta(b)
    assert int(meta[_lib.META_FLAGS]) == want
    with pytest.raises(_lib.DmpnnError):
        engine.check_flags(int(meta[_lib.META_FLAGS]))


def test_work_table_restatement_flags_tiles_of_more_than_128_atoms():
    """On the layout of the fragment batch (140-atom / 40-row and 300-atom / 100-row molecules first, in the middle and
    last of 2 000), the restated work table keeps one item per tile and flags exactly the tiles of more than 128 atoms;
    C2-sized tiles are left unflagged and oversized-row tiles are cut into 128-row windows."""
    from chemprop_b200.data import BatchMolGraph
    from oracle import layout_np

    mgs, at = fragment_batch(5)
    bmg = BatchMolGraph(mgs)
    L = layout_np.build_layout(bmg.edge_index.numpy(), bmg.rev_edge_index.numpy(), bmg.batch.numpy(), len(mgs))
    assert L["max_tile_atoms"] == 300 and L["max_tile_rows"] <= 128
    W = layout_np.work_table(L["tile_row_ptr"], L["tile_atom_ptr"])
    na = np.diff(L["tile_atom_ptr"])
    assert W["n_work"] == L["n_tiles"] and np.array_equal(W["work_row_ptr"], L["tile_row_ptr"])
    assert np.array_equal(np.flatnonzero(W["work_flag"]), np.flatnonzero(na > 128)) and int(W["work_flag"].sum()) == 6
    tiles_of = L["tile_mol_ptr"]
    assert all(np.flatnonzero(tiles_of == m).size == 1 for m in at)       # every fragment molecule opens a tile of its own
    # a tile of 300 rows: three windows, all flagged
    W = layout_np.work_table(np.array([0, 40, 340, 400], np.int32), np.array([0, 30, 190, 200], np.int32))
    assert W["n_work"] == 5 and W["work_row_ptr"].tolist() == [0, 40, 168, 296, 340, 400]
    assert W["work_flag"].tolist() == [0, 1, 1, 1, 0] and W["work_atom_ptr"].tolist() == [0, 30, 30, 30, 190, 200]


class _FakeLib:
    def __init__(self):
        self.calls = 0

    def dmpnn_work_table_build(self, *a):
        self.calls += 1
        return 0


@pytest.mark.parametrize("rows,atoms,builds", [(128, 128, False), (129, 60, True), (40, 129, True), (200, 300, True),
                                               (0, 0, False)])
def test_step_tables_builds_the_work_table_for_oversized_tiles(rows, atoms, builds, monkeypatch):
    """Layout.step_tables reads both limits from the (host) meta words: a layout whose largest tile holds more than 128 rows
    or more than 128 atoms gets the work table, one launch; any other passes its tiles as they are, with no launch."""
    from chemprop_b200 import _lib, engine

    fake = _FakeLib()
    monkeypatch.setattr(_lib, "load", lambda: fake)
    monkeypatch.setattr(engine, "_stream", lambda: 0)
    meta = [0] * _lib.META_WORDS
    meta[_lib.META_N_TILES], meta[_lib.META_FLAGS] = 3, 7
    meta[_lib.META_MAX_TILE_ROWS], meta[_lib.META_MAX_TILE_ATOMS] = rows, atoms
    z = torch.zeros(8, dtype=torch.int32)
    lay = engine.Layout(10, 40, 3, z, z, z, z, z, z, z, z, z, z, z, torch.tensor(meta, dtype=torch.int32), list(meta))
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    assert fake.calls == int(builds) and (wf is not None) == builds and (nw is not None) == builds
    assert nt == 3 and (dr is lay.dst_row if builds else dr is None)
    if not builds:
        assert trp is lay.tile_row_ptr and tap is lay.tile_atom_ptr
    lay.step_tables()
    assert fake.calls == int(builds)                  # built once per batch


def test_fragment_molecule_shape():
    from tests.test_gpu_layout_scale import fragment_molecule

    rng = np.random.default_rng(0)
    for a, r in ((140, 40), (300, 100)):
        m = fragment_molecule(rng, a, r)
        assert m.V.shape[0] == a and m.edge_index.shape[1] == r and m.E.shape[0] == r
        assert int(m.edge_index.max()) > 256 or a < 256
        ei, rev = m.edge_index, m.rev_edge_index
        assert np.array_equal(rev[rev], np.arange(r)) and np.array_equal(ei[0, rev], ei[1])
