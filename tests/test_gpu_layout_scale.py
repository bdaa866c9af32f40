"""GPU tier: the index kernels of csrc/layout.cu at batch scale, bit-exact against oracle/layout_np.py, and the fused bond
step on molecules with more atoms than a tile holds.

The batches are index-only (`index_batch`): numpy edge_index / rev_edge_index / batch built directly, no features, so a
batch of a million molecules takes seconds.  They reach what the goldens (a few hundred atoms) cannot: more than one block
of the row-pointer scan (2048 atoms per block) and more than 1024 of them (the carry loop of k_scan_bsums), more than one
tile-packing chunk (1024 molecules) and more than 1024 of them (the `c >= 1024` branch of k_tiles_gather), work tables of
more than 1024 tiles, tiles closed at exactly 128 rows / atoms, oversized molecules at warp and chunk boundaries of the tile
index, zero-atom and edgeless molecules, hub atoms of in-degree up to 5000 and shuffled edge order.

Every output buffer is filled with a poison value and followed by a sentinel tail: an entry the kernel should write and
did not, or a write past the end, fails the comparison.  The CPU half (dmpnn_batch_meta_host against the oracle, the
packing restatement against a brute-force walk, the work table's decision in Layout.step_tables) is in
tests/test_layout_scale_host.py.  This module imports nothing CUDA at import."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest
import torch

POISON = -0x5A5A5A5B        # what an output entry holds until a kernel writes it
SENTINEL = 0x7E57AB1E       # the tail past an output's declared size: never written
TAIL = 64


# ---- index-only batches ------------------------------------------------------------------------------------------
def index_batch(n_atoms, linked=None, star=None, loops=None, ring_frac=0.06, shuffle_edges=False, seed=0) -> dict:
    """A batch of B molecules in the reference featuriser's edge order (bond k: edges 2k u->v, 2k+1 v->u, rev = e ^ 1), from
    per-molecule sizes.  Atom j >= 1 of molecule m with j < linked[m] bonds to one of atoms j-3 .. j-1 (to atom 0 when
    star[m]: a hub of in-degree linked[m] - 1); the atoms from linked[m] on are isolated; a share ring_frac of the atoms
    j >= 5 close a ring to atom j - 5; loops[m] adds a self-loop edge (its own reverse) on atom 0.  Returns edge_index
    (2 x E), rev_edge_index, batch (int64 numpy) and B."""
    rng = np.random.default_rng(seed)
    n_atoms = np.asarray(n_atoms, dtype=np.int64)
    B = n_atoms.shape[0]
    linked = n_atoms if linked is None else np.asarray(linked, dtype=np.int64)
    star = np.zeros(B, bool) if star is None else np.asarray(star, bool)
    loops = np.zeros(B, bool) if loops is None else np.asarray(loops, bool)
    ap = np.zeros(B + 1, np.int64)
    np.cumsum(n_atoms, out=ap[1:])
    V = int(ap[-1])
    batch = np.repeat(np.arange(B, dtype=np.int64), n_atoms)
    v = np.arange(V, dtype=np.int64)
    j = v - ap[batch]
    inside = j < linked[batch]
    tree = (j >= 1) & inside
    step = 1 + np.floor(rng.random(V) * np.minimum(3, np.maximum(j, 1))).astype(np.int64)
    parent = np.where(star[batch], ap[batch], v - step)
    ring = (j >= 5) & inside & ~star[batch] & (rng.random(V) < ring_frac)
    bu = np.concatenate([parent[tree], v[ring] - 5])
    bv = np.concatenate([v[tree], v[ring]])
    o = np.argsort(bv, kind="stable")                   # bonds in molecule order
    bu, bv = bu[o], bv[o]
    nb = bu.shape[0]
    src = np.empty(2 * nb, np.int64)
    dst = np.empty(2 * nb, np.int64)
    src[0::2], dst[0::2], src[1::2], dst[1::2] = bu, bv, bv, bu
    rev = np.arange(2 * nb, dtype=np.int64) ^ 1
    la = ap[:B][loops]
    src, dst = np.concatenate([src, la]), np.concatenate([dst, la])
    rev = np.concatenate([rev, 2 * nb + np.arange(la.shape[0])])
    q = np.argsort(batch[src] if V else src, kind="stable")     # every molecule's edges together, in molecule order
    ei, rev = np.stack([src[q], dst[q]]), _inverse(q)[rev[q]]
    out = dict(edge_index=ei, rev_edge_index=rev, batch=batch, B=B)
    return shuffle(out, seed + 1) if shuffle_edges else out


def _inverse(p):
    inv = np.empty_like(p)
    inv[p] = np.arange(p.shape[0])
    return inv


def shuffle(b: dict, seed: int) -> dict:
    """The same batch with its edges in random order (rev remapped)."""
    E = b["rev_edge_index"].shape[0]
    p = np.random.default_rng(seed).permutation(E)          # new position j holds old edge p[j]
    return dict(b, edge_index=b["edge_index"][:, p], rev_edge_index=_inverse(p)[b["rev_edge_index"][p]])


def reorder_molecules(b: dict, order) -> dict:
    """The same molecules in the order `order` (new molecule k is old molecule order[k]); edges follow their molecule."""
    order = np.asarray(order, np.int64)
    B, batch, ei = b["B"], b["batch"], b["edge_index"]
    na = np.bincount(batch, minlength=B)
    ap = np.concatenate([[0], np.cumsum(na)])
    lens = na[order]
    old = np.repeat(ap[order] - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()))
    new_of_old = _inverse(old)
    rank = _inverse(order)
    q = np.argsort(rank[batch[ei[0]]], kind="stable")
    return dict(edge_index=new_of_old[ei[:, q]], rev_edge_index=_inverse(q)[b["rev_edge_index"][q]],
                batch=np.repeat(np.arange(B, dtype=np.int64), lens), B=B)


def tile_packed(b: dict) -> dict:
    """The batch in the loader's tile-packing molecule order (dmpnn_tile_pack_order, as bench.py feeds it)."""
    from chemprop_b200 import _lib

    B = b["B"]
    na = np.bincount(b["batch"], minlength=B).astype(np.int64)
    ne = np.bincount(b["batch"][b["edge_index"][0]], minlength=B).astype(np.int64)
    order = np.empty(B, np.int64)
    _lib.check(_lib.load().dmpnn_tile_pack_order(B, na.ctypes.data, ne.ctypes.data, order.ctypes.data), "tile_pack_order")
    return reorder_molecules(b, order)


def _normal_sizes(rng, n, mean, std, lo, hi):
    return np.clip(np.rint(rng.normal(mean, std, size=n)), lo, hi).astype(np.int64)


def _menu_batch(seed, n=3000):
    """Molecules drawn from a menu of sizes at the tile limits: exactly 128 / 127 / 129 rows (65-atom chains, a self-loop
    for the odd counts), 64 + 64 rows, 128 / 129 atoms with few rows, 64 isolated atoms, single atoms."""
    rng = np.random.default_rng(seed)
    #          atoms, linked, loop
    menu = [(65, 65, False), (65, 65, True), (64, 64, True), (33, 33, False), (32, 32, False), (2, 2, False),
            (128, 10, False), (129, 10, False), (64, 0, False), (1, 1, False), (128, 65, False), (63, 63, True)]
    pick = rng.integers(0, len(menu), size=n)
    a, lk, lp = (np.array([menu[i][k] for i in pick]) for k in range(3))
    return index_batch(a, linked=lk, loops=lp, ring_frac=0.0, seed=seed)


def _oversized_at(positions, n=1100, seed=0):
    """n molecules of exactly 128 rows (one tile each, so tile index == molecule index) with oversized molecules at
    `positions`: alternately 300 atoms / ~600 rows (cut into windows) and 140 atoms / 40 rows (one window, > 128 atoms)."""
    a, lk = np.full(n, 65), np.full(n, 65)
    for i, p in enumerate(positions):
        a[p], lk[p] = (300, 300) if i % 2 == 0 else (140, 21)
    return index_batch(a, linked=lk, ring_frac=0.0, seed=seed)


def _batch(name: str) -> dict:
    rng = np.random.default_rng(sum(map(ord, name)))
    if name in ("C2", "C2-packed", "C2-shuffled", "C5", "C5-packed"):
        n = 25_000 if name.startswith("C5") else 10_000
        b = index_batch(_normal_sizes(rng, n, 25, 5, 2, 60), seed=n, shuffle_edges=name == "C2-shuffled")
        return tile_packed(b) if name.endswith("packed") else b
    if name in ("C4", "C4-packed"):
        b = index_batch(_normal_sizes(rng, 10_000, 80, 10, 20, 120), ring_frac=0.03, seed=4)
        return tile_packed(b) if name.endswith("packed") else b
    if name.startswith("B="):
        n = int(name[2:])
        return index_batch(_normal_sizes(rng, n, 12, 6, 1, 40), seed=n, shuffle_edges=n % 2 == 1)
    if name == "million-tiny":         # > 1024 * 1024 molecules of 1-3 atoms, V + 1 > 2048 * 1024
        return index_batch(rng.integers(1, 4, size=1024 * 1024 + 50_000), ring_frac=0.0, seed=5)
    if name == "V+1=2048*1024":        # exactly 1024 scan blocks, exactly 1024 chunks
        a = np.full(1024 * 1024, 2)
        a[-1] = 1
        return index_batch(a, ring_frac=0.0, seed=6)
    if name == "V+1=2048*1024+1":      # 1025 scan blocks
        return index_batch(np.full(1024 * 1024, 2), ring_frac=0.0, seed=7)
    if name.startswith("V="):          # V + 1 around 2048 k
        V = int(name[2:])
        a = np.full(V // 7, 7)
        return index_batch(np.append(a, V - a.sum()) if V % 7 else a, seed=V)
    if name == "menu":
        return _menu_batch(8)
    if name == "menu-shuffled":
        return shuffle(_menu_batch(9), 9)
    if name == "oversized-31-32":
        return _oversized_at([31, 32, 63, 64])
    if name == "oversized-1023-1024":
        return _oversized_at([1023, 1024, 1055, 1056])
    if name == "edgeless-chunk":       # molecules 1000 .. 2199 single atoms: chunk 1 (1024 .. 2047) is edgeless throughout
        a = _normal_sizes(rng, 3000, 25, 5, 2, 60)
        a[1000:2200] = 1
        return index_batch(a, seed=10)
    if name == "zero-atom":            # zero-atom molecules first, in the middle, at chunk boundaries and last
        a = _normal_sizes(rng, 2500, 25, 5, 2, 60)
        a[[0, 1, 500, 501, 502, 1023, 1024, 2047]] = 0
        a[-40:] = 0
        return index_batch(a, seed=11)
    if name == "hubs":                 # star molecules: hub atoms of in-degree 64 / 300 / 5000, shuffled edges
        a = _normal_sizes(rng, 1500, 25, 5, 2, 60)
        star = np.zeros(1500, bool)
        for p, k in ((10, 64), (700, 300), (1400, 5000)):
            a[p], star[p] = k + 1, True
        return index_batch(a, star=star, seed=12, shuffle_edges=True)
    if name == "empty":                # V = 0, E = 0, B = 0
        return index_batch(np.zeros(0, np.int64))
    if name == "atoms-no-edges":       # E = 0
        return index_batch(np.ones(3000, np.int64))
    if name == "molecules-no-atoms":   # V = 0, B > 0 (every molecule empty)
        return index_batch(np.zeros(2100, np.int64))
    raise KeyError(name)


BATCHES = ["C2", "C2-packed", "C2-shuffled", "C4", "C4-packed", "C5", "C5-packed", "B=1023", "B=1024", "B=1025",
           "B=2048", "B=2049", "million-tiny", "V+1=2048*1024", "V+1=2048*1024+1", "V=2046", "V=2047", "V=2048",
           "V=4095", "V=4096", "V=4097", "menu", "menu-shuffled", "oversized-31-32", "oversized-1023-1024",
           "edgeless-chunk", "zero-atom", "hubs", "empty", "atoms-no-edges", "molecules-no-atoms"]

ARRAYS = ("perm", "inv_perm", "rowptr", "src_row", "dst_row", "rev_row", "mol_atom_ptr", "mol_row_ptr", "tile_mol_ptr",
          "tile_row_ptr", "tile_atom_ptr")


def host_meta(b: dict) -> np.ndarray:
    """dmpnn_batch_meta_host of a batch (all DMPNN_META_WORDS words)."""
    from chemprop_b200 import _lib

    ei, rev, batch = (np.ascontiguousarray(b[k]) for k in ("edge_index", "rev_edge_index", "batch"))
    E, V = rev.shape[0], batch.shape[0]
    meta = np.full(_lib.META_WORDS, POISON, np.int32)
    _lib.check(_lib.load().dmpnn_batch_meta_host(ei.ctypes.data if E else None, rev.ctypes.data if E else None,
                                                 batch.ctypes.data if V else None, V, E, b["B"], meta.ctypes.data),
               "dmpnn_batch_meta_host")
    return meta


# ---- device helpers ----------------------------------------------------------------------------------------------
def _out(n: int) -> torch.Tensor:
    t = torch.full((n + TAIL,), POISON, dtype=torch.int32, device="cuda")
    t[n:] = SENTINEL
    return t


def _tail_ok(t: torch.Tensor, n: int, what):
    assert bool((t[n:] == SENTINEL).all()), (what, "wrote past its end")


def device_layout(b: dict) -> dict:
    """dmpnn_layout_build straight through the C ABI into poisoned, sentinel-tailed buffers of exactly the declared sizes
    (E, V + 1, B + 1, DMPNN_META_WORDS); the workspace is poisoned too (the build must clear what it uses)."""
    from chemprop_b200 import _lib

    lib = _lib.load()
    ei = torch.from_numpy(np.ascontiguousarray(b["edge_index"])).cuda()
    rev = torch.from_numpy(np.ascontiguousarray(b["rev_edge_index"])).cuda()
    batch = torch.from_numpy(np.ascontiguousarray(b["batch"])).cuda()
    E, V, B = rev.shape[0], batch.shape[0], b["B"]
    sizes = dict(perm=E, inv_perm=E, rowptr=V + 1, src_row=E, dst_row=E, rev_row=E, mol_atom_ptr=B + 1, mol_row_ptr=B + 1,
                 tile_mol_ptr=B + 1, tile_row_ptr=B + 1, tile_atom_ptr=B + 1, meta=_lib.META_WORDS)
    bufs = {k: _out(n) for k, n in sizes.items()}
    nbytes = C.c_size_t(0)
    _lib.check(lib.dmpnn_layout_workspace_bytes(V, E, B, C.byref(nbytes)), "dmpnn_layout_workspace_bytes")
    ws = torch.full((max(nbytes.value, 1),), 0xA5, dtype=torch.uint8, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.dmpnn_layout_build(ei.data_ptr(), rev.data_ptr(), batch.data_ptr(), V, E, B,
                                      *(bufs[k].data_ptr() for k in ARRAYS + ("meta",)), ws.data_ptr(), s),
               "dmpnn_layout_build")
    torch.cuda.synchronize()
    for k, n in sizes.items():
        _tail_ok(bufs[k], n, k)
    return {k: bufs[k][:sizes[k]].cpu().numpy() for k in sizes}


def _scan_blocks(V):
    return (V + 1 + 2047) // 2048


def _chunks(B):
    return (B + 1023) // 1024


@pytest.fixture(scope="module")
def layouts():
    """name -> (batch, oracle layout, device layout), built once for the module's tests."""
    from oracle import layout_np

    cache = {}

    def get(name):
        if name not in cache:
            b = _batch(name)
            L = layout_np.build_layout(b["edge_index"], b["rev_edge_index"], b["batch"], b["B"])
            cache.clear()                  # keep one batch of up to 2 M atoms in memory at a time
            cache[name] = (b, L, device_layout(b))
        return cache[name]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("name", BATCHES)
def test_layout_build_bit_exact_at_scale(name, layouts):
    """All eleven arrays and the meta words of dmpnn_layout_build against the restatement, nothing written past them, the
    tile tables untouched past n_tiles + 1; and dmpnn_batch_meta_host's words equal to the device's."""
    from chemprop_b200 import _lib

    b, L, D = layouts(name)
    V, E, B = b["batch"].shape[0], b["rev_edge_index"].shape[0], b["B"]
    nt = L["n_tiles"]
    print(f"[layout-scale] {name}: B = {B}, V = {V}, E = {E}, scan blocks {_scan_blocks(V)}, tile chunks {_chunks(B)}, "
          f"tiles {nt}, max tile rows {L['max_tile_rows']}, max tile atoms {L['max_tile_atoms']}, "
          f"max in-degree {L['max_indeg']}")
    assert L["flags"] == 7
    for k in ARRAYS[:8]:
        assert D[k].dtype == np.int32 and np.array_equal(D[k], L[k]), k
    for k in ARRAYS[8:]:
        assert np.array_equal(D[k][:nt + 1], L[k]), k
        assert bool((D[k][nt + 1:] == POISON).all()), (k, "written past n_tiles + 1")
    want = [0] * _lib.META_WORDS
    want[_lib.META_N_TILES], want[_lib.META_FLAGS], want[_lib.META_MAX_INDEG] = nt, L["flags"], L["max_indeg"]
    want[_lib.META_MAX_TILE_ROWS], want[_lib.META_MAX_TILE_ATOMS] = L["max_tile_rows"], L["max_tile_atoms"]
    assert D["meta"].tolist() == want
    assert host_meta(b).tolist() == want          # the sync-free step trusts these words instead of the device's


# ---- dmpnn_tiles_build, dmpnn_work_table_build, dmpnn_sorted_index_to_ptr -----------------------------------------
TILES_BATCHES = ["C2", "C4", "B=1025", "B=2049", "million-tiny", "menu", "oversized-1023-1024", "edgeless-chunk",
                 "zero-atom", "hubs", "empty", "molecules-no-atoms"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", TILES_BATCHES)
def test_tiles_build_every_limit(name, layouts):
    """dmpnn_tiles_build at row limits {1, 64, 128, 4096} x atom limits {1, 128} against the restatement: tile offsets
    (n_tiles + 1 entries, nothing written past them) and info = (n_tiles, max rows, max atoms, 0)."""
    from chemprop_b200 import _lib
    from oracle import layout_np

    lib = _lib.load()
    b, L, _ = layouts(name)
    B = b["B"]
    ap = torch.from_numpy(L["mol_atom_ptr"]).cuda()
    rp = torch.from_numpy(L["mol_row_ptr"]).cuda()
    nbytes = C.c_size_t(0)
    _lib.check(lib.dmpnn_tiles_workspace_bytes(B, C.byref(nbytes)), "dmpnn_tiles_workspace_bytes")
    ws = torch.full((nbytes.value,), 0xA5, dtype=torch.uint8, device="cuda")
    for rl in (1, 64, 128, 4096):
        for al in (1, 128):
            T = layout_np.tiles_build(L["mol_atom_ptr"], L["mol_row_ptr"], rl, al)
            trp, tap, info = _out(B + 1), _out(B + 1), _out(4)
            _lib.check(lib.dmpnn_tiles_build(ap.data_ptr(), rp.data_ptr(), B, rl, al, trp.data_ptr(), tap.data_ptr(),
                                             info.data_ptr(), ws.data_ptr(), torch.cuda.current_stream().cuda_stream),
                       "dmpnn_tiles_build")
            torch.cuda.synchronize()
            for t, n in ((trp, B + 1), (tap, B + 1), (info, 4)):
                _tail_ok(t, n, (name, rl, al))
            n = int(T["info"][0])
            assert info[:4].tolist() == T["info"].tolist(), (name, rl, al)
            assert trp[:n + 1].tolist() == T["tile_row_ptr"].tolist(), (name, rl, al)
            assert tap[:n + 1].tolist() == T["tile_atom_ptr"].tolist(), (name, rl, al)
            assert bool((trp[n + 1:B + 1] == POISON).all()) and bool((tap[n + 1:B + 1] == POISON).all()), (name, rl, al)


def _work_table_device(trp: np.ndarray, tap: np.ndarray):
    from chemprop_b200 import _lib

    n_tiles = trp.shape[0] - 1
    E = int(trp[-1]) if n_tiles > 0 else 0
    cap = n_tiles + E // 128 + 2                         # Layout.step_tables' capacity
    wr, wa, nw = _out(cap + 1), _out(cap + 1), _out(1)
    wf = torch.full((cap + 1 + TAIL,), 0x5B, dtype=torch.int8, device="cuda")
    wf[cap + 1:] = 0x3C
    tr, ta = torch.from_numpy(np.ascontiguousarray(trp)).cuda(), torch.from_numpy(np.ascontiguousarray(tap)).cuda()
    _lib.check(_lib.load().dmpnn_work_table_build(tr.data_ptr(), ta.data_ptr(), n_tiles, wr.data_ptr(), wa.data_ptr(),
                                                  wf.data_ptr(), nw.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "dmpnn_work_table_build")
    torch.cuda.synchronize()
    for t, n in ((wr, cap + 1), (wa, cap + 1), (nw, 1)):
        _tail_ok(t, n, "work table")
    assert bool((wf[cap + 1:] == 0x3C).all()), "work_flag written past its capacity"
    n = int(nw[0])
    assert bool((wr[n + 1:cap + 1] == POISON).all()) and bool((wf[n:cap + 1] == 0x5B).all())
    return wr[:n + 1].cpu().numpy(), wa[:n + 1].cpu().numpy(), wf[:n].cpu().numpy(), n


def _check_work_table(trp, tap, what):
    from oracle import layout_np

    W = layout_np.work_table(trp, tap)
    wr, wa, wf, n = _work_table_device(trp, tap)
    assert n == W["n_work"], (what, n, W["n_work"])
    assert np.array_equal(wr, W["work_row_ptr"]) and np.array_equal(wa, W["work_atom_ptr"]), what
    assert np.array_equal(wf, W["work_flag"]), what
    return W


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["C2", "C4", "oversized-31-32", "oversized-1023-1024", "menu", "hubs", "million-tiny",
                                  "empty"])
def test_work_table_of_layouts(name, layouts):
    """dmpnn_work_table_build on the layout's own tiles against the restatement: 128-row windows of the tiles over 128 rows,
    and flag 1 on those windows and on every tile of more than 128 atoms."""
    b, L, _ = layouts(name)
    W = _check_work_table(L["tile_row_ptr"], L["tile_atom_ptr"], name)
    print(f"[layout-scale] work table {name}: n_tiles {L['n_tiles']}, n_work {W['n_work']}, flagged "
          f"{int(W['work_flag'].sum())}")
    if name.startswith("oversized"):
        assert int(W["work_flag"].sum()) > 2 and L["n_tiles"] > 1024


@pytest.mark.gpu
@pytest.mark.parametrize("n_tiles", [0, 1, 31, 32, 33, 1023, 1024, 1025, 2049])
def test_work_table_tile_counts(n_tiles):
    """Synthetic tile tables around the kernel's warp (32) and chunk (1024) boundaries: tiles of 0 .. 700 rows and 0 .. 300
    atoms, with the large ones on lanes 0, 31 and 32 and on the last tile."""
    rng = np.random.default_rng(n_tiles)
    nr = rng.integers(0, 129, size=n_tiles)
    na = rng.integers(0, 129, size=n_tiles)
    for i in (0, 31, 32, 1023, 1024, n_tiles - 1):
        if 0 <= i < n_tiles:
            nr[i], na[i] = (rng.integers(129, 700), rng.integers(1, 300)) if i % 2 == 0 else (rng.integers(0, 129), 200)
    big = rng.random(n_tiles) < 0.05
    nr[big] = rng.integers(129, 520, size=int(big.sum()))
    trp = np.concatenate([[0], np.cumsum(nr)]).astype(np.int32)
    tap = np.concatenate([[0], np.cumsum(na)]).astype(np.int32)
    _check_work_table(trp, tap, n_tiles)


SEG_CASES = {
    "C2": lambda: _batch("C2")["batch"],
    "million-tiny": lambda: _batch("million-tiny")["batch"],
    "zero-atom": lambda: _batch("zero-atom")["batch"],
    "empty": lambda: np.zeros(0, np.int64),
    "single": lambda: np.zeros(1, np.int64),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SEG_CASES))
@pytest.mark.parametrize("extra", [0, 1, 5])
def test_sorted_index_to_ptr(name, extra):
    """dmpnn_sorted_index_to_ptr with n_seg = max + 1 + extra (trailing empty segments): ptr bit-exact, status 0, nothing
    written past n_seg + 1."""
    from oracle import layout_np

    idx = SEG_CASES[name]()
    n_seg = (int(idx.max()) + 1 if idx.size else 0) + extra
    want, st = layout_np.sorted_index_to_ptr(idx, n_seg)
    ptr, status = _sorted_index_to_ptr_device(idx, n_seg)
    assert st == 0 and status == 0
    assert np.array_equal(ptr, want)


def _sorted_index_to_ptr_device(idx: np.ndarray, n_seg: int):
    from chemprop_b200 import _lib

    x = torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int64)).cuda()
    ptr, status = _out(n_seg + 1), _out(1)
    _lib.check(_lib.load().dmpnn_sorted_index_to_ptr(x.data_ptr(), x.shape[0], n_seg, ptr.data_ptr(), status.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream), "dmpnn_sorted_index_to_ptr")
    torch.cuda.synchronize()
    _tail_ok(ptr, n_seg + 1, "ptr")
    _tail_ok(status, 1, "status")
    return ptr[:n_seg + 1].cpu().numpy(), int(status[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["decreasing", "negative", "too-large", "decreasing-and-too-large"])
def test_sorted_index_to_ptr_status(case):
    """An index that decreases or leaves [0, n_seg) sets the status bits the restatement names (ptr is then unspecified,
    but nothing is written past n_seg + 1)."""
    from oracle import layout_np

    idx = np.repeat(np.arange(3000, dtype=np.int64), 3)
    n_seg = 3000
    if "decreasing" in case:
        idx[4000], idx[4001] = idx[4001], idx[4000] - 1
    if case == "negative":
        idx[0] = -1
    if "too-large" in case:
        idx[-1] = n_seg
    _, st = layout_np.sorted_index_to_ptr(idx, n_seg)
    _, status = _sorted_index_to_ptr_device(idx, n_seg)
    assert st != 0 and status == st, (status, st)


# ---- invalid batches: indices in range, so the device build stays in bounds ---------------------------------------
def invalid_batch(case: str) -> dict:
    b = index_batch(_normal_sizes(np.random.default_rng(3), 2100, 25, 5, 2, 60), seed=3)
    ei, rev, batch = b["edge_index"].copy(), b["rev_edge_index"].copy(), b["batch"].copy()
    if case == "rev-not-involution":
        rev[[100, 1500]] = rev[[1500, 100]]
    elif case == "rev-wrong-endpoints":           # rev[rev[e]] == e, but e and rev[e] are not reverses of each other
        rev[[0, 1, 2, 3]] = [2, 3, 0, 1]
    elif case == "batch-decreasing":
        a = int(np.flatnonzero(np.diff(batch) > 0)[700])
        batch[a + 1] = batch[a] - 1
    elif case == "cross-molecule-edge":           # one bond moved to join two molecules; rev stays a proper involution
        e = 2 * 500
        far = int(np.flatnonzero(batch == batch[ei[0, e]] + 40)[0])
        ei[1, e], ei[0, e + 1] = far, far
    else:
        raise KeyError(case)
    return dict(edge_index=ei, rev_edge_index=rev, batch=batch, B=b["B"])


INVALID_IN_RANGE = ["rev-not-involution", "rev-wrong-endpoints", "batch-decreasing", "cross-molecule-edge"]


class _Graph:
    """The index tensors of a BatchMolGraph, without features or host meta words."""

    def __init__(self, b):
        self.edge_index = torch.from_numpy(b["edge_index"]).cuda()
        self.rev_edge_index = torch.from_numpy(b["rev_edge_index"]).cuda()
        self.batch = torch.from_numpy(b["batch"]).cuda()
        self.n = b["B"]

    def __len__(self):
        return self.n


@pytest.mark.gpu
@pytest.mark.parametrize("case", INVALID_IN_RANGE)
def test_invalid_batch_flags(case):
    """A batch whose indices are all in range but which breaks one rule: the device's flags word equals the restatement's and
    dmpnn_batch_meta_host's, and the engine refuses the batch."""
    from chemprop_b200 import _lib, engine
    from chemprop_b200._lib import DmpnnError
    from oracle import layout_np

    b = invalid_batch(case)
    want = layout_np.layout_flags(b["edge_index"], b["rev_edge_index"], b["batch"], b["B"])
    assert want & _lib.FLAG_INDEX_IN_RANGE and want != 7, want
    D = device_layout(b)
    assert int(D["meta"][_lib.META_FLAGS]) == want
    assert int(host_meta(b)[_lib.META_FLAGS]) == want
    with pytest.raises(DmpnnError):
        engine.get_layout(_Graph(b))


@pytest.mark.gpu
def test_work_table_adds_no_launch_without_oversized_molecules():
    """Layout.step_tables launches dmpnn_work_table_build only for a batch with a tile of more than 128 rows or atoms: a C2
    batch adds no launch, a batch with one 140-atom / 40-row molecule adds exactly one and gets that tile flagged."""
    from chemprop_b200 import _lib, engine

    lib = _lib.load()
    for name, want_launch in (("C2", False), ("oversized-atoms", True)):
        if name == "C2":
            b = _batch("C2")
        else:
            a, lk = np.full(2000, 25), np.full(2000, 25)
            a[1000], lk[1000] = 140, 21
            b = index_batch(a, linked=lk, ring_frac=0.0, seed=13)
        g = _Graph(b)
        lay = engine.get_layout(g)
        assert (lay.max_tile_atoms > 128) == want_launch and lay.max_tile_rows <= 128
        n0 = lib.dmpnn_launch_count()
        trp, tap, nt, wf, nw, dr = lay.step_tables()
        torch.cuda.synchronize()
        assert lib.dmpnn_launch_count() - n0 == int(want_launch), name
        assert (wf is not None) == want_launch
        if want_launch:
            n = int(nw.item())
            assert n == nt
            flagged = np.flatnonzero(wf[:n].cpu().numpy())
            assert flagged.size == 1
            t = int(flagged[0])
            assert int(tap[t + 1] - tap[t]) == 140 and int(trp[t + 1] - trp[t]) == 40


# ---- the fused bond step on tiles of more than 128 atoms ----------------------------------------------------------
def fragment_molecule(rng, n_atoms: int, rows: int, d_v: int = 72, d_e: int = 14):
    """A molecule of n_atoms atoms and `rows` directed edges: a tree of rows / 2 + 1 atoms and isolated atoms, in random atom
    order (so the bonded atoms lie anywhere in the molecule's atom range, past atom 256 too)."""
    from chemprop_b200.data import MolGraph, make_molecule

    m = make_molecule(rng, rows // 2 + 1, d_v, d_e, ring_frac=0.0, shuffle_edges=True)
    iso = make_molecule(rng, n_atoms - (rows // 2 + 1), d_v, d_e, ring_frac=0.0)
    V = np.concatenate([m.V, iso.V])
    p = rng.permutation(n_atoms)                 # new atom j is old atom p[j]
    return MolGraph(V=V[p], E=m.E, edge_index=_inverse(p)[m.edge_index], rev_edge_index=m.rev_edge_index)


FRAGMENTS = ((140, 40), (300, 100))


def fragment_batch(seed: int, n_mols: int = 2000, d_v: int = 72, d_e: int = 14):
    """n_mols molecules: ~25-atom ones, with a 140-atom / 40-row and a 300-atom / 100-row molecule first, in the middle and
    last (the middle and last ones reach the kernel through the next-tile prefetch of its row-pointer slice).  Returns the
    molecules and the indices of the fragment molecules."""
    from chemprop_b200.data import make_molecules

    rng = np.random.default_rng(seed)
    n_small = n_mols - 3 * len(FRAGMENTS)
    small = make_molecules(n_small, seed=seed, d_v=d_v, d_e=d_e, shuffle_edges=True)
    frag = lambda: [fragment_molecule(rng, a, r, d_v, d_e) for a, r in FRAGMENTS]  # noqa: E731
    mgs = frag() + small[: n_small // 2] + frag() + small[n_small // 2:] + frag()
    k = len(FRAGMENTS)
    at = list(range(k)) + list(range(k + n_small // 2, 2 * k + n_small // 2)) + list(range(n_mols - k, n_mols))
    return mgs, at


def _check_fragment_layout(lay):
    """The batch reaches the kernel as it should: tiles over 128 atoms but none over 128 rows, each flagged in the work
    table as one window."""
    assert lay.max_tile_atoms == 300 and lay.max_tile_rows <= 128, (lay.max_tile_atoms, lay.max_tile_rows)
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    assert wf is not None and int(nw.item()) == nt
    flagged = np.flatnonzero(wf[:nt].cpu().numpy())
    na = np.diff(tap[: nt + 1].cpu().numpy())
    assert np.array_equal(flagged, np.flatnonzero(na > 128)) and flagged.size == 3 * len(FRAGMENTS)


@pytest.mark.gpu
@pytest.mark.parametrize("first,act", [(False, "relu"), (True, "relu"), (False, "tanh")])
def test_fused_step_tiles_of_more_than_128_atoms(first, act):
    """dmpnn_bond_step_fused_bf16 and its mirror on a batch whose fragment molecules have more atoms than the kernel's staged
    row-pointer slice holds: every row against torch with the kernel's rounding points (tests/test_gpu_fused_step.py)."""
    from chemprop_b200 import _lib
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.engine import bond_step_bwd_fused, bond_step_fused, get_layout, pad_hidden, pack_weight_bf16
    from tests.test_gpu_fused_step import _torch_reference

    h = 300
    mgs, _ = fragment_batch(31 + int(first))
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    _check_fragment_layout(lay)
    hp = pad_hidden(h)
    g = torch.Generator(device="cuda").manual_seed(7)
    H0 = torch.zeros(lay.E, hp, dtype=torch.bfloat16, device="cuda")
    H0[:, :h] = (torch.randn(lay.E, h, device="cuda", generator=g) * 0.7).bfloat16()
    Hp = torch.zeros_like(H0)
    Hp[:, :h] = torch.relu(torch.randn(lay.E, h, device="cuda", generator=g)).bfloat16()
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    code = {"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    Hin = H0 if first else Hp
    Hn = torch.zeros_like(H0)
    Hn[:, :h] = float("nan")
    bond_step_fused(Hin, H0, Hn, h, pack_weight_bf16(W), b, lay, code, 0.0, first)
    torch.cuda.synchronize()
    assert torch.isfinite(Hn.float()).all(), "rows/columns left unwritten"
    torch.testing.assert_close(Hn.float(), _torch_reference(lay, Hin, H0, W, b, h, act, first).float(), rtol=2 ** -6,
                               atol=2e-2)
    # the mirror: dOut = ((S.P) dZ) . W_h * tau'(Y), G = (S.P) dZ
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
    Gref = (A[dst] - X).bfloat16().float()
    torch.testing.assert_close(Gk[:, :h].float(), Gref, rtol=2 ** -6, atol=2e-2)
    # the GEMM of the operand the kernel gathered (G_out is that operand): Gref's f32 sibling sums differ from the kernel's
    # packed-bf16 ones by an ulp here and there, and over 100 k rows W_h's 300-term sums carry such a difference past 2e-2
    ref = ((Gk[:, :h].float() @ W.bfloat16().float()) * (Hp[:, :h].float() > 0).float()).bfloat16().float()
    assert torch.isfinite(out.float()).all()
    torch.testing.assert_close(out[:, :h].float(), ref, rtol=2 ** -6, atol=2e-2)


def _projection(n_mols, d, at, seed):
    """The loss projection G: the fragment molecules' rows weigh 30 times the others', so that their share of every weight
    gradient is far above the bars."""
    G = torch.randn(n_mols, d, generator=torch.Generator().manual_seed(seed))
    G[at] *= 30.0
    return G


@pytest.mark.gpu
@pytest.mark.parametrize("undirected", [False, True])
def test_bond_message_passing_tiles_of_more_than_128_atoms_vs_f64(undirected, monkeypatch):
    """BondMessagePassing(precision="bf16") on the fused depth step over the fragment batch: H_v, the aggregate and every
    gradient against oracle/restatement.py in float64 and against the rounding-aware emulation, at the bars of
    tests/test_gpu_zy_paths.py for batches without K_k (float64: 1e-2 * max(1, max|H|), gradients 6 %; emulation: 4e-2 per
    element, gradients 2 %)."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.nn import MeanAggregation
    from tests.test_gpu_parity import _emulated_run
    from tests.test_gpu_zy_paths import _close_grad, _close_h, _f64_oracle, _initial_state, _module_factory, _report

    name = f"fragments-bond-{'undirected' if undirected else 'directed'}"
    c = dict(kind="bond", precision="bf16", d_h=300, depth=3, act="relu", bias=True, undirected=undirected)
    seed = 61 + int(undirected)
    mgs, at = fragment_batch(seed)
    state = _initial_state(c, seed)
    make = _module_factory(c, state)
    Gm = _projection(len(mgs), c["d_h"], at, seed)
    loss_fn = lambda H, b: (MeanAggregation()(H, b.batch).float() * Gm.to(H.device)).sum()  # noqa: E731
    H_ref, a_ref, g_ref = _f64_oracle(c, mgs, state, Gm)

    plans = []
    plan0 = engine.plan
    monkeypatch.setattr(engine, "plan", lambda *a: (plans.append(p := plan0(*a)), p)[1])
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = engine.get_layout(bmg)
    _check_fragment_layout(lay)
    mp = make("cuda")
    assert not mp.uses_composed_tier(lay)
    H = mp(bmg)
    a = MeanAggregation()(H, bmg.batch)
    (a.float() * Gm.cuda()).sum().backward()
    torch.cuda.synchronize()
    assert [p.fused for p in plans] == [True], plans
    grads = {k: p.grad for k, p in mp.named_parameters()}
    hmax = max(1.0, H_ref.abs().max().item())
    worst = {"H_v vs f64": _close_h(name, "H_v vs f64", H.detach(), H_ref, 1e-2 * hmax),
             "agg vs f64": _close_h(name, "agg vs f64", a.detach(), a_ref, 1e-2 * hmax),
             "grads vs f64": max(_close_grad(name, f"{k} vs f64", grads[k], g_ref[k], 6e-2, 6e-2) for k in grads)}
    H_e, egrads = _emulated_run(lambda: make("cpu"), lambda: BatchMolGraph(mgs), None, loss_fn)
    dH = (H.detach().float().cpu() - H_e).abs()
    bar = 4e-2 * (H_e.abs() / 2).clamp_min(1.0)
    worst["H_v vs emulation"] = _report(name, "H_v vs emulation (of the element's bar)", (dH / bar).max().item(), 1.0)
    assert bool((dH <= bar).all()), dH.max().item()
    assert (dH > 1e-3).float().mean().item() <= 1e-2
    worst["grads vs emulation"] = max(_close_grad(name, f"{k} vs emulation", grads[k], egrads[k], 2e-2, 2e-2) for k in grads)
    print(f"[layout-scale] {name}: worst fraction of each bar " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.gpu
def test_mab_bond_tiles_of_more_than_128_atoms_vs_f64(monkeypatch):
    """MABBondMessagePassing(precision="bf16") (the mab_bond path: fused depth step, W_vo and W_eo read-outs) over the
    fragment batch: H_v, H_e and every gradient against restatement.mab_forward in float64 at the bars of
    tests/test_gpu_zy_mab_paths.py for batches without K_k (1e-2 * max(1, max|H|); gradients 6 %)."""
    from chemprop_b200 import engine
    from tests.test_gpu_zy_mab_paths import _D, _f64_oracle, _inputs, _run, make_module
    from tests.test_gpu_zy_paths import _close_grad, _close_h

    name = "fragments-mab-bond"
    c = dict(_D, kind="bond")
    seed = 67
    mgs, at = fragment_batch(seed)
    torch.manual_seed(seed)
    state = {k: v.detach().clone() for k, v in make_module(c).state_dict().items()}
    V_d, E_d, _, G_e = _inputs(c, mgs, seed)
    G = _projection(len(mgs), c["d_h"], at, seed)
    plans = []
    plan0 = engine.plan
    monkeypatch.setattr(engine, "plan", lambda *a: (plans.append(p := plan0(*a)), p)[1])
    mp = make_module(c, "cuda", state)
    mp.train()
    bmg, H_v, H_e, grads = _run(mp, mgs, "cuda", V_d, E_d, G, G_e)
    torch.cuda.synchronize()
    _check_fragment_layout(engine.get_layout(bmg))
    assert [p.fused for p in plans if p.forward is not None] == [True], plans
    H_v_ref, H_e_ref, g_ref = _f64_oracle(c, mgs, state, V_d, E_d, G, G_e, None, "cuda")
    assert set(grads) == set(g_ref)
    worst = {}
    for w, got, ref in (("H_v", H_v, H_v_ref), ("H_e", H_e, H_e_ref)):
        worst[f"{w} vs f64"] = _close_h(name, f"{w} vs f64", got, ref, 1e-2 * max(1.0, ref.abs().max().item()))
    worst["grads vs f64"] = max(_close_grad(name, f"{k} vs f64", grads[k], g_ref[k], 6e-2, 6e-2) for k in grads)
    print(f"[layout-scale] {name}: worst fraction of each bar " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
