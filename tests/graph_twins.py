"""TEST INFRASTRUCTURE ONLY.  Same-signature twins of a batch, for the CUDA-graph replay tests
(tests/test_graph_signature_host.py, tests/test_gpu_graph_replay.py).

`CudaGraphStep` replays one graph for every batch of one `batch_signature`: V, d_v, E, d_e, B and the layout meta words.
A twin is a batch of that signature with different contents, built by transformations that cannot move a meta word:

  * `relabel`: the atoms of each molecule relabelled and its directed edges reordered, reverse maps kept involutions (per
    molecule sizes and degree multisets unchanged).  `paired=True` keeps each bond's two edges at 2i, 2i + 1 (what the
    mol-atom-bond pair mean needs) and shuffles bonds and their directions instead;
  * `tile_shuffle`: the molecules after the first of each tile of the layout (<= 128 rows and <= 128 atoms) permuted
    inside the tile, so the greedy packing closes every tile where it did, and the oversized molecules (one tile each)
    permuted among themselves;
  * `window_molecules`: two oversized molecules that trade bonds -- the same atom counts and the same total of rows, but a
    different number of 128-row windows (a chain of 70 atoms against a branched ring system of 70 atoms).

`facts` restates the layout of a molecule list with oracle/layout_np.py; `differences` names what two batches of one
signature differ in:
  (a) the atom-tile count (dmpnn_tiles_build at engine.ATOM_TILE_ATOMS / ATOM_TILE_EDGES: n_tiles_dev of atom_tables);
  (b) the fused step's window count (dmpnn_work_table_build: n_work_dev of Layout.step_tables);
  (c) where the atoms of in-degree > 4 and the edgeless molecules sit;
  (d) mol_atom_ptr (the per-molecule targets and aggregation segments)."""
from __future__ import annotations

import numpy as np

from chemprop_b200.data import MolGraph
from oracle import layout_np

ATOM_TILE_ATOMS, ATOM_TILE_EDGES = 128, 1024     # chemprop_b200.engine.ATOM_TILE_* (asserted in the CPU test)


def relabel(mg: MolGraph, rng: np.random.Generator, paired: bool = False) -> MolGraph:
    n, ne = mg.V.shape[0], mg.edge_index.shape[1]
    p = rng.permutation(n)                          # new atom j is old atom p[j]
    new_of = np.empty(n, np.int64)
    new_of[p] = np.arange(n)
    ei = new_of[np.asarray(mg.edge_index, np.int64)]
    rev = np.asarray(mg.rev_edge_index, np.int64)
    if paired:
        assert ne % 2 == 0 and np.array_equal(rev, np.arange(ne) ^ 1), "paired relabel needs rev[e] = e ^ 1"
        flip = rng.integers(0, 2, size=ne // 2)
        pairs = rng.permutation(ne // 2)
        q = np.stack([2 * pairs + flip, 2 * pairs + 1 - flip], 1).ravel()
    else:
        q = rng.permutation(ne)                     # new edge j is old edge q[j]
    qi = np.empty(ne, np.int64)
    qi[q] = np.arange(ne)
    return MolGraph(V=mg.V[p], E=mg.E[q], edge_index=ei[:, q], rev_edge_index=qi[rev[q]] if ne else rev)


def _ptrs(mgs) -> tuple:
    na = np.array([m.V.shape[0] for m in mgs], np.int64)
    ne = np.array([m.edge_index.shape[1] for m in mgs], np.int64)
    return np.concatenate([[0], np.cumsum(na)]), np.concatenate([[0], np.cumsum(ne)]), na, ne


def tile_shuffle(mgs: list, rng: np.random.Generator) -> list:
    ap, rp, na, ne = _ptrs(mgs)
    tm, _, _ = layout_np.pack_tiles(ap, rp)
    order = np.arange(len(mgs))
    big = np.nonzero((ne > layout_np.TILE_ROWS) | (na > layout_np.TILE_ATOMS))[0]
    order[big] = rng.permutation(big)
    for s, e in zip(tm[:-1], tm[1:]):             # a tile's first molecule stays: it is what closes the tile before
        if e - s > 2:
            order[s + 1:e] = s + 1 + rng.permutation(e - s - 1)
    return [mgs[i] for i in order]


def twin(mgs: list, seed: int, paired: bool = False) -> list:
    rng = np.random.default_rng(seed)
    return tile_shuffle([relabel(m, rng, paired) for m in mgs], rng)


def bond_graph(rng: np.random.Generator, n_atoms: int, n_bonds: int, d_v: int, d_e: int, chain: bool = False,
               max_deg: int = 4) -> MolGraph:
    """n_atoms atoms, exactly n_bonds bonds, degree <= max_deg: a chain (or a random tree) plus random ring closures;
    edges in the featuriser's order (2i: u -> v, 2i + 1: v -> u)."""
    deg = np.zeros(n_atoms, np.int64)
    bonds = []
    for v in range(1, n_atoms):
        cand = [v - 1] if chain else [u for u in range(v) if deg[u] < max_deg]
        u = int(cand[rng.integers(len(cand))])
        bonds.append((u, v))
        deg[u] += 1
        deg[v] += 1
    have = set(bonds)
    while len(bonds) < n_bonds:
        u, v = sorted(int(x) for x in rng.integers(0, n_atoms, size=2))
        if u == v or (u, v) in have or deg[u] >= max_deg or deg[v] >= max_deg:
            continue
        bonds.append((u, v))
        have.add((u, v))
        deg[u] += 1
        deg[v] += 1
    assert len(bonds) == n_bonds
    V = np.zeros((n_atoms, d_v), np.float32)
    V[np.arange(n_atoms)[:, None], rng.integers(0, d_v - 1, size=(n_atoms, 7))] = 1.0
    V[:, -1] = rng.uniform(0.01, 0.4, size=n_atoms)
    Eb = np.zeros((n_bonds, max(d_e, 1)), np.float32)
    Eb[np.arange(n_bonds)[:, None], rng.integers(0, max(d_e, 1), size=(n_bonds, 3))] = 1.0
    ei = np.array([[a for u, v in bonds for a in (u, v)], [a for u, v in bonds for a in (v, u)]], np.int64)
    return MolGraph(V=V, E=np.repeat(Eb, 2, axis=0)[:, :d_e], edge_index=ei,
                    rev_edge_index=np.arange(2 * n_bonds, dtype=np.int64) ^ 1)


def window_molecules(seed: int, d_v: int, d_e: int) -> tuple:
    """(pair A, pair B, the largest): pair A is a 70-atom chain (138 rows: 2 windows) and 100 atoms with 130 bonds (260 rows:
    3 windows); pair B is 70 atoms with 100 bonds (200 rows: 2 windows) and a 100-atom tree (198 rows: 2 windows); the same
    atoms and rows, one window fewer.  The third molecule (300 rows) holds the batch's largest tile in both."""
    rng = np.random.default_rng(seed)
    a = [bond_graph(rng, 70, 69, d_v, d_e, chain=True), bond_graph(rng, 100, 130, d_v, d_e)]
    b = [bond_graph(rng, 70, 100, d_v, d_e), bond_graph(rng, 100, 99, d_v, d_e)]
    return a, b, bond_graph(rng, 110, 150, d_v, d_e)


def edgeless_molecules(n_mols: int, seed: int, d_v: int, d_e: int) -> list:
    """n_mols molecules of 1-3 atoms without bonds (salts, single heavy atoms)."""
    rng = np.random.default_rng(seed)
    out = []
    for k in rng.integers(1, 4, size=n_mols):
        V = np.zeros((k, d_v), np.float32)
        V[np.arange(k)[:, None], rng.integers(0, d_v - 1, size=(k, 7))] = 1.0
        V[:, -1] = rng.uniform(0.01, 0.4, size=k)
        out.append(MolGraph(V=V, E=np.zeros((0, d_e), np.float32), edge_index=np.zeros((2, 0), np.int64),
                            rev_edge_index=np.zeros(0, np.int64)))
    return out


def collate(mgs: list) -> tuple:
    """(edge_index, rev_edge_index, batch) of the batch of `mgs`, as numpy int64."""
    ap, rp, na, ne = _ptrs(mgs)
    ei = np.concatenate([np.asarray(m.edge_index, np.int64) + a for m, a in zip(mgs, ap)], 1) if mgs else np.zeros((2, 0))
    rev = np.concatenate([np.asarray(m.rev_edge_index, np.int64) + r for m, r in zip(mgs, rp)])
    return ei.astype(np.int64), rev, np.repeat(np.arange(len(mgs)), na)


def facts(mgs: list) -> dict:
    ei, rev, batch = collate(mgs)
    L = layout_np.build_layout(ei, rev, batch, len(mgs))
    meta = (L["n_tiles"], L["flags"], L["max_indeg"], L["max_tile_rows"], L["max_tile_atoms"], 0, 0, 0)
    at = layout_np.tiles_build(L["mol_atom_ptr"], L["mol_row_ptr"], ATOM_TILE_EDGES, ATOM_TILE_ATOMS)
    return dict(signature=(int(batch.shape[0]), int(mgs[0].V.shape[1]), int(ei.shape[1]), int(mgs[0].E.shape[1]),
                           len(mgs), tuple(int(x) for x in meta)),
                atom_tiles=int(at["info"][0]), windows=layout_np.work_table(L["tile_row_ptr"], L["tile_atom_ptr"])["n_work"],
                high_degree=np.nonzero(np.diff(L["rowptr"]) > 4)[0], edgeless=np.nonzero(np.diff(L["mol_row_ptr"]) == 0)[0],
                mol_atom_ptr=L["mol_atom_ptr"], rowptr=L["rowptr"], perm=L["perm"])


def differences(a: dict, b: dict) -> set:
    """Which of (a)-(d) two batches' `facts` differ in; asserts they have one signature and different index tables."""
    assert a["signature"] == b["signature"], (a["signature"], b["signature"])
    assert not all(np.array_equal(a[k], b[k]) for k in ("rowptr", "perm", "mol_atom_ptr")), "not a twin: the same layout"
    out = set()
    if a["atom_tiles"] != b["atom_tiles"]:
        out.add("a")
    if a["windows"] != b["windows"]:
        out.add("b")
    if len(a["high_degree"]) + len(a["edgeless"]) and not (np.array_equal(a["high_degree"], b["high_degree"])
                                                           and np.array_equal(a["edgeless"], b["edgeless"])):
        out.add("c")
    if not np.array_equal(a["mol_atom_ptr"], b["mol_atom_ptr"]):
        out.add("d")
    return out


def twins(mgs: list, want: dict, seed: int, paired: bool = False, windows: tuple | None = None, tries: int = 64) -> list:
    """[A, B, C]: A = `mgs`, B and C twins of it.  `want` = {"B": "abd", "C": "cd"}: the differences from A each twin must
    show (asserted); seeds are tried in order until they do.  `windows` = (index, pair B): B holds pair B at
    [index, index + 1] in place of A's pair (before its shuffle)."""
    fa = facts(mgs)
    out = [mgs]
    for name, k in (("B", 1), ("C", 2)):
        for s in range(tries):
            base = list(mgs)
            if windows is not None and name == "B":
                i, pair = windows
                base[i:i + 2] = pair
            t = twin(base, seed + 1000 * k + s, paired)
            if set(want[name]) <= differences(fa, facts(t)):
                out.append(t)
                break
        else:
            raise AssertionError(f"no twin {name} differing in {want[name]} within {tries} seeds")
    return out
