"""TEST INFRASTRUCTURE ONLY.  numpy restatement of the engine's integer layout
(dmpnn_layout_build): stable sort of edges by destination atom, per-row src / dst / rev, molecule
offsets and the greedy molecule-aligned tile table; and of the other index kernels of csrc/layout.cu
(dmpnn_tiles_build, dmpnn_work_table_build, dmpnn_sorted_index_to_ptr).  Integer work -> the CUDA
output must be bit-exact with this."""
from __future__ import annotations

import numpy as np

TILE_ROWS = 128
TILE_ATOMS = 128
TILE_CHUNK = 1024   # greedy packing restarts every TILE_CHUNK molecules (chunks are packed independently)
WINDOW_ROWS = 128   # the fused step's work items hold <= 128 rows


def pack_tiles(mol_atom_ptr: np.ndarray, mol_row_ptr: np.ndarray, row_limit: int = TILE_ROWS,
               atom_limit: int = TILE_ATOMS) -> tuple[np.ndarray, int, int]:
    """Greedy molecule-aligned packing: a tile opened at molecule t0 takes the following molecules while its rows stay
    <= row_limit and its atoms <= atom_limit (its first molecule always, whatever its size), and every TILE_CHUNK-th
    molecule opens a new tile.  Returns (tile_mol_ptr [n_tiles + 1] int32 with the sentinel B, max rows, max atoms of a tile).
    Both offset arrays are non-decreasing, so the closing molecule of every tile start is found by bisection (as the kernel
    does); only the chain of tile starts is walked."""
    ap = np.asarray(mol_atom_ptr, dtype=np.int64)
    rp = np.asarray(mol_row_ptr, dtype=np.int64)
    B = ap.shape[0] - 1
    if B <= 0:
        return np.zeros(1, np.int32), 0, 0
    t0 = np.arange(B)
    # first i > t0 with rp[i + 1] > rp[t0] + row_limit (or the same for atoms), capped at the end of t0's chunk
    i_r = np.searchsorted(rp, rp[:B] + row_limit, side="right") - 1
    i_a = np.searchsorted(ap, ap[:B] + atom_limit, side="right") - 1
    chunk_end = np.minimum((t0 // TILE_CHUNK + 1) * TILE_CHUNK, B)
    nxt = np.maximum(np.minimum(np.minimum(i_r, i_a), chunk_end), t0 + 1)
    starts, t = [], 0
    while t < B:
        starts.append(t)
        t = int(nxt[t])
    tile_mol_ptr = np.array(starts + [B], dtype=np.int32)
    return tile_mol_ptr, int(np.diff(rp[tile_mol_ptr]).max()), int(np.diff(ap[tile_mol_ptr]).max())


def tiles_build(mol_atom_ptr: np.ndarray, mol_row_ptr: np.ndarray, row_limit: int, atom_limit: int) -> dict:
    """dmpnn_tiles_build: the tile starts' row / atom offsets and info = (n_tiles, max rows, max atoms, 0)."""
    tm, mr, ma = pack_tiles(mol_atom_ptr, mol_row_ptr, row_limit, atom_limit)
    return dict(tile_row_ptr=np.asarray(mol_row_ptr, np.int32)[tm], tile_atom_ptr=np.asarray(mol_atom_ptr, np.int32)[tm],
                info=np.array([len(tm) - 1, mr, ma, 0], np.int32))


def work_table(tile_row_ptr: np.ndarray, tile_atom_ptr: np.ndarray) -> dict:
    """dmpnn_work_table_build: every tile of more than 128 rows cut into ceil(rows / 128) windows of 128 consecutive rows
    (the last one shorter), every other tile one work item; flag 1 on the windows of a cut tile and on a tile of more than
    128 atoms (the fused step's shared-memory row-pointer slice holds 129 entries), 0 elsewhere."""
    rp = np.asarray(tile_row_ptr, dtype=np.int64)
    ap = np.asarray(tile_atom_ptr, dtype=np.int64)
    n_tiles = rp.shape[0] - 1
    if n_tiles <= 0:
        return dict(work_row_ptr=np.zeros(1, np.int32), work_atom_ptr=np.zeros(1, np.int32),
                    work_flag=np.zeros(0, np.int8), n_work=0)
    nr, na = np.diff(rp), np.diff(ap)
    cnt = np.where(nr > WINDOW_ROWS, (nr + WINDOW_ROWS - 1) // WINDOW_ROWS, 1)
    tile = np.repeat(np.arange(n_tiles), cnt)
    k = np.arange(tile.shape[0]) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    far = (cnt > 1) | (na > TILE_ATOMS)
    return dict(work_row_ptr=np.append(rp[tile] + WINDOW_ROWS * k, rp[-1]).astype(np.int32),
                work_atom_ptr=np.append(ap[tile], ap[-1]).astype(np.int32),
                work_flag=far[tile].astype(np.int8), n_work=int(tile.shape[0]))


def sorted_index_to_ptr(index: np.ndarray, n_seg: int) -> tuple[np.ndarray | None, int]:
    """dmpnn_sorted_index_to_ptr: (ptr [n_seg + 1] int32, status).  ptr[s] = first i with index[i] >= s, ptr[n_seg] = n,
    so trailing segments without rows come out empty.  status: bit 0 = an index outside [0, n_seg), bit 2 = index
    decreases somewhere.  ptr is None when status != 0 (the kernel's ptr is then unspecified)."""
    index = np.asarray(index, dtype=np.int64)
    status = (1 if index.size and (index.min() < 0 or index.max() >= n_seg) else 0) | \
             (4 if index.size > 1 and bool((np.diff(index) < 0).any()) else 0)
    if status:
        return None, status
    return np.searchsorted(index, np.arange(n_seg + 1), side="left").astype(np.int32), 0


def layout_flags(edge_index: np.ndarray, rev: np.ndarray, batch: np.ndarray, n_mols: int) -> int:
    """DMPNN_META_FLAGS of a batch: bit 0 rev is an involution with swapped endpoints, bit 1 batch non-decreasing and every
    edge inside a molecule, bit 2 every index in range (the other two bits require it)."""
    src, dst = np.asarray(edge_index[0], np.int64), np.asarray(edge_index[1], np.int64)
    rev, batch = np.asarray(rev, np.int64), np.asarray(batch, np.int64)
    E, V, B = src.shape[0], batch.shape[0], int(n_mols)
    in_range = bool(E == 0 or (src.min() >= 0 and src.max() < V and dst.min() >= 0 and dst.max() < V
                               and rev.min() >= 0 and rev.max() < E))
    in_range = in_range and bool(V == 0 or (batch.min() >= 0 and batch.max() < B))
    invol = in_range and bool(E == 0 or (np.array_equal(rev[rev], np.arange(E)) and np.array_equal(src[rev], dst)
                                         and np.array_equal(dst[rev], src)))
    sorted_ = in_range and bool(np.all(np.diff(batch) >= 0)) and bool(E == 0 or np.array_equal(batch[src], batch[dst]))
    return (1 if invol else 0) | (2 if sorted_ else 0) | (4 if in_range else 0)


def build_layout(edge_index: np.ndarray, rev: np.ndarray, batch: np.ndarray, n_mols: int) -> dict:
    src, dst = edge_index[0].astype(np.int64), edge_index[1].astype(np.int64)
    rev = np.asarray(rev, dtype=np.int64)
    E, V, B = src.shape[0], batch.shape[0], int(n_mols)
    perm = np.argsort(dst, kind="stable").astype(np.int32)
    inv_perm = np.empty(E, dtype=np.int32)
    inv_perm[perm] = np.arange(E, dtype=np.int32)
    rowptr = np.zeros(V + 1, dtype=np.int32)
    np.cumsum(np.bincount(dst, minlength=V), out=rowptr[1:])
    src_row = src[perm].astype(np.int32)
    dst_row = dst[perm].astype(np.int32)
    rev_row = inv_perm[rev[perm]].astype(np.int32) if E else np.zeros(0, np.int32)
    mol_atom_ptr = np.searchsorted(batch, np.arange(B + 1), side="left").astype(np.int32)
    mol_row_ptr = rowptr[mol_atom_ptr].astype(np.int32)
    tile_mol_ptr, max_rows, max_atoms = pack_tiles(mol_atom_ptr, mol_row_ptr, TILE_ROWS, TILE_ATOMS)
    n_tiles = len(tile_mol_ptr) - 1
    tile_row_ptr = mol_row_ptr[tile_mol_ptr].astype(np.int32)
    tile_atom_ptr = mol_atom_ptr[tile_mol_ptr].astype(np.int32)
    flags = layout_flags(edge_index, rev, batch, B)
    max_indeg = int(np.diff(rowptr).max()) if V else 0
    return dict(perm=perm, inv_perm=inv_perm, rowptr=rowptr, src_row=src_row, dst_row=dst_row, rev_row=rev_row,
                mol_atom_ptr=mol_atom_ptr, mol_row_ptr=mol_row_ptr, tile_mol_ptr=tile_mol_ptr, tile_row_ptr=tile_row_ptr,
                tile_atom_ptr=tile_atom_ptr, n_tiles=n_tiles,
                flags=flags, max_indeg=max_indeg, max_tile_rows=max_rows, max_tile_atoms=max_atoms)
