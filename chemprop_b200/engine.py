"""Host side of the engine: device layout, thin wrappers over the C ABI (raw pointers in, nothing
allocated inside the library) and the autograd functions the nn modules call.

PyTorch here is plumbing only: it owns device memory (caching allocator), streams and the
autograd graph; every arithmetic step on the path is a kernel of libdmpnn_sm90.so.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass

import torch
from torch import Tensor

from . import _lib
from ._lib import (ACT_ELU, ACT_LEAKYRELU, ACT_NONE, ACT_RELU, ACT_TANH, BF16, F32, SCALE_DIV_CONST,
                   SCALE_INV_COUNT, SCALE_NONE, DmpnnError)

# True: a BatchMolGraph that carries host-computed layout meta words (our collate: dmpnn_batch_meta_host) is trusted
# and the step never synchronises on the device copy; False: always read the device-computed words (one sync per batch)
HOST_META = os.environ.get("DMPNN_HOST_META", "1") != "0"      # DMPNN_HOST_META=0: A/B switch for measurements

HIDDEN_ALIGN = 64  # hidden row stride padded to 64 elements: bf16 rows start on 128-byte lines (one TMA request per box row)

# Kernel limits (`plan` decides from them which path a message-passing call takes)
MAX_TC_HIDDEN = 304   # d_h of the fused depth step and of the bf16 tensor-core linear kernels
MAX_TC_K = 448        # inner dimension K of the bf16 tensor-core linear kernels
MAX_X3_DIM = 4096     # every dimension of the 3xTF32 GEMMs

# Optional device-side timing of the depth step (bench.py's roofline): when a list, every depth step
# appends (tag, start_event, end_event) recorded on the launching stream.
STEP_EVENTS: list | None = None


class _StepTimer:
    def __init__(self, tag: str | None):      # None: nothing is timed
        self.tag = tag

    def __enter__(self):
        if STEP_EVENTS is not None and self.tag is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record(torch.cuda.current_stream())
        return self

    def __exit__(self, *exc):
        if STEP_EVENTS is not None and self.tag is not None:
            self.e1.record(torch.cuda.current_stream())
            STEP_EVENTS.append((self.tag, self.e0, self.e1))
        return False


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)
_raw_device = getattr(torch._C, "_cuda_getDevice", None)


def _stream() -> int:
    """cudaStream_t of torch's current stream on the current device.  Called once per kernel launch (~60 per training step):
    the raw accessors cost ~0.3 us, `torch.cuda.current_stream().cuda_stream` ~15 us (0.45 ms of host time per step)."""
    if _raw_stream is not None and _raw_device is not None:
        return _raw_stream(_raw_device())
    return torch.cuda.current_stream().cuda_stream


def _dt(t: Tensor) -> int:
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise DmpnnError(f"unsupported dtype {t.dtype}")


def _ptr(t: Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def _ld(t: Tensor) -> int:
    assert t.dim() == 2 and (t.stride(1) == 1 or t.shape[1] <= 1), "rows must be contiguous"
    return max(int(t.stride(0)), int(t.shape[1]))


def _require_cuda(*ts: Tensor):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise DmpnnError(
                "chemprop_b200 runs on CUDA (sm_90a) only; got a CPU tensor. There is no CPU fallback: "
                "move the BatchMolGraph and the module to the GPU."
            )


def pad_hidden(h: int) -> int:
    return (h + HIDDEN_ALIGN - 1) // HIDDEN_ALIGN * HIDDEN_ALIGN


# ----------------------------------------------------------------------------------------------
# layout
# ----------------------------------------------------------------------------------------------
@dataclass
class Layout:
    V: int
    E: int
    B: int
    perm: Tensor
    inv_perm: Tensor
    rowptr: Tensor
    src_row: Tensor
    dst_row: Tensor
    rev_row: Tensor
    mol_atom_ptr: Tensor
    mol_row_ptr: Tensor
    tile_mol_ptr: Tensor
    tile_row_ptr: Tensor
    tile_atom_ptr: Tensor
    meta: Tensor
    _meta_host: list | None = None
    _work: tuple | None = None
    _atom_work: tuple | None = None
    _mab: tuple | None = None

    def _host(self):
        if self._meta_host is None:
            self._meta_host = self.meta.tolist()  # one small D2H sync per batch
        return self._meta_host

    @property
    def n_tiles(self) -> int:
        return self._host()[_lib.META_N_TILES]

    @property
    def flags(self) -> int:
        return self._host()[_lib.META_FLAGS]

    @property
    def max_indeg(self) -> int:
        return self._host()[_lib.META_MAX_INDEG]

    @property
    def max_tile_rows(self) -> int:
        return self._host()[_lib.META_MAX_TILE_ROWS]

    @property
    def max_tile_atoms(self) -> int:
        return self._host()[_lib.META_MAX_TILE_ATOMS]

    def validate(self):
        check_flags(self.flags)

    def step_tables(self):
        """(tile_row_ptr, tile_atom_ptr, n_tiles, work_flag, n_work_dev, dst_row) for the fused depth step.  Batches whose
        molecules all fit a tile of 128 rows and 128 atoms pass the layout's tile tables as they are; a batch with larger
        molecules (condensed reaction graphs; a molecule of many fragments) gets the work table of dmpnn_work_table_build:
        oversized tiles cut into 128-row windows that gather from global memory, built once per batch on the device (no host
        read-back: the kernel reads the window count from device memory)."""
        if self.max_tile_rows <= 128 and self.max_tile_atoms <= 128:
            return self.tile_row_ptr, self.tile_atom_ptr, self.n_tiles, None, None, None
        if self._work is None:
            lib = _lib.load()
            dev = self.rowptr.device
            cap = self.n_tiles + self.E // 128 + 2
            wr = torch.empty(cap + 1, dtype=torch.int32, device=dev)
            wa = torch.empty(cap + 1, dtype=torch.int32, device=dev)
            wf = torch.zeros(cap + 1, dtype=torch.int8, device=dev)
            nw = torch.zeros(1, dtype=torch.int32, device=dev)
            _lib.check(lib.dmpnn_work_table_build(self.tile_row_ptr.data_ptr(), self.tile_atom_ptr.data_ptr(), self.n_tiles,
                                                  wr.data_ptr(), wa.data_ptr(), wf.data_ptr(), nw.data_ptr(), _stream()),
                       "dmpnn_work_table_build")
            self._work = (wr, wa, wf, nw)
        wr, wa, wf, nw = self._work
        return wr, wa, self.n_tiles, wf, nw, self.dst_row


def check_flags(f: int):
    if not f & _lib.FLAG_INDEX_IN_RANGE:
        raise DmpnnError("BatchMolGraph indices out of range (edge_index / rev_edge_index / batch)")
    if not f & _lib.FLAG_BATCH_SORTED:
        raise DmpnnError("BatchMolGraph.batch must be non-decreasing and edges must stay inside a molecule")
    if not f & _lib.FLAG_REV_INVOLUTION:
        raise DmpnnError(
            "rev_edge_index is not a proper reverse-edge map (rev[rev[e]]==e with swapped endpoints); "
            "the engine requires it (every featuriser-made graph satisfies it)"
        )


def build_layout(edge_index: Tensor, rev_edge_index: Tensor, batch: Tensor, n_mols: int,
                 meta_host: list | None = None) -> Layout:
    """dmpnn_layout_build on the current stream.  Inputs are the reference's int64 index tensors.
    `meta_host`: the meta words already computed on the host for this very batch (dmpnn_batch_meta_host, by our
    collate): the layout then never reads `meta` back from the device -- no sync in the training step."""
    _require_cuda(edge_index, rev_edge_index, batch)
    lib = _lib.load()
    dev = edge_index.device
    edge_index = edge_index.contiguous()
    rev_edge_index = rev_edge_index.contiguous()
    batch = batch.contiguous()
    if edge_index.dtype != torch.int64 or rev_edge_index.dtype != torch.int64 or batch.dtype != torch.int64:
        raise DmpnnError("edge_index / rev_edge_index / batch must be int64 (as in the reference BatchMolGraph)")
    E = int(edge_index.shape[1])
    V = int(batch.shape[0])
    B = int(n_mols)
    i32 = dict(dtype=torch.int32, device=dev)
    perm = torch.empty(max(E, 1), **i32)
    inv_perm = torch.empty(max(E, 1), **i32)
    rowptr = torch.empty(V + 1, **i32)
    src_row = torch.empty(max(E, 1), **i32)
    dst_row = torch.empty(max(E, 1), **i32)
    rev_row = torch.empty(max(E, 1), **i32)
    # the zero-initialised outputs are views of ONE buffer (one memset instead of six fill launches per step)
    sizes = (B + 1, B + 1, B + 2, B + 2, B + 2, _lib.META_WORDS)
    zbuf = torch.zeros(sum(sizes), **i32)
    mol_atom_ptr, mol_row_ptr, tile_mol_ptr, tile_row_ptr, tile_atom_ptr, meta = torch.split(zbuf, sizes)
    nbytes = C.c_size_t(0)
    _lib.check(lib.dmpnn_layout_workspace_bytes(V, E, B, C.byref(nbytes)), "dmpnn_layout_workspace_bytes")
    ws = torch.empty(max(nbytes.value, 256), dtype=torch.uint8, device=dev)
    rc = lib.dmpnn_layout_build(
        edge_index.data_ptr(), rev_edge_index.data_ptr(), batch.data_ptr(), V, E, B,
        perm.data_ptr(), inv_perm.data_ptr(), rowptr.data_ptr(), src_row.data_ptr(), dst_row.data_ptr(),
        rev_row.data_ptr(), mol_atom_ptr.data_ptr(), mol_row_ptr.data_ptr(), tile_mol_ptr.data_ptr(),
        tile_row_ptr.data_ptr(), tile_atom_ptr.data_ptr(), meta.data_ptr(), ws.data_ptr(), _stream(),
    )
    _lib.check(rc, "dmpnn_layout_build")
    return Layout(V, E, B, perm[:E], inv_perm[:E], rowptr, src_row[:E], dst_row[:E], rev_row[:E], mol_atom_ptr,
                  mol_row_ptr, tile_mol_ptr, tile_row_ptr, tile_atom_ptr, meta,
                  None if meta_host is None else list(meta_host))


def get_layout(bmg) -> Layout:
    """Layout of a BatchMolGraph (ours or the reference's), cached on the object when it allows it."""
    lay = getattr(bmg, "_layout", None)
    if lay is not None and lay.rowptr.device == bmg.edge_index.device:
        return lay
    meta_host = getattr(bmg, "_meta_host", None) if HOST_META else None
    if meta_host is not None:
        check_flags(meta_host[_lib.META_FLAGS])      # an invalid batch is refused before anything is launched
        lay = build_layout(bmg.edge_index, bmg.rev_edge_index, bmg.batch, len(bmg), meta_host)
    else:
        lay = build_layout(bmg.edge_index, bmg.rev_edge_index, bmg.batch, len(bmg))
    lay.validate()
    try:
        bmg._layout = lay
    except AttributeError:  # reference BatchMolGraph is a slots dataclass: rebuild per call
        pass
    # let Aggregation.forward(H, bmg.batch) find the molecule offsets without a device sync
    try:
        bt = bmg.batch
        bt._dmpnn_seg, bt._dmpnn_seg_v = (lay.mol_atom_ptr, bt.to(torch.int32), lay.B), bt._version
    except Exception:
        pass
    return lay


def segments_of(batch: Tensor, n_seg: int | None = None):
    """(ptr int32 [B+1], seg_of_row int32 [V], B) for a sorted int64 `batch` (agg.py:74-75).  `n_seg`: the segment count
    is given by the caller (nn/ffn.py:123 sizes by the constraints' rows): trailing segments without rows come out empty
    (`ptr[s] == ptr[s+1]`), an index >= n_seg is an error."""
    seg = getattr(batch, "_dmpnn_seg", None)          # attached by get_layout / an earlier call; void after an in-place change
    if (seg is not None and getattr(batch, "_dmpnn_seg_v", None) == batch._version and seg[0].device == batch.device
            and (n_seg is None or seg[2] == n_seg)):
        return seg
    _require_cuda(batch)
    lib = _lib.load()
    n = int(batch.shape[0])
    if n_seg is None:
        B = int(batch.max().item()) + 1 if n > 0 else 0   # same device sync as the reference (agg.py:75)
    else:
        B = int(n_seg)
    ptr = torch.zeros(B + 1, dtype=torch.int32, device=batch.device)
    status = torch.zeros(1, dtype=torch.int32, device=batch.device)
    bc = batch.contiguous()
    _lib.check(lib.dmpnn_sorted_index_to_ptr(bc.data_ptr(), n, B, ptr.data_ptr(), status.data_ptr(), _stream()),
               "dmpnn_sorted_index_to_ptr")
    st = int(status.item())
    if st & 1:       # V_RANGE of csrc/layout.cu
        raise DmpnnError(f"`batch` holds a molecule index outside [0, {B})")
    if st != 0:
        raise DmpnnError("Aggregation: `batch` must be non-decreasing (atoms of a molecule contiguous)")
    seg = (ptr, bc.to(torch.int32), B)
    if n_seg is None:
        try:
            batch._dmpnn_seg, batch._dmpnn_seg_v = seg, batch._version
        except Exception:
            pass
    return seg


# ----------------------------------------------------------------------------------------------
# op wrappers (tensors in, launches on the current stream)
# ----------------------------------------------------------------------------------------------
def linear_fwd(X1: Tensor, K1: int, W: Tensor, out: Tensor, N: int, *, idx1: Tensor | None = None,
               X2: Tensor | None = None, K2: int = 0, idx2: Tensor | None = None, bias: Tensor | None = None,
               res: Tensor | None = None, act: int = ACT_NONE, act_param: float = 0.0, R: int | None = None,
               pad_to: int | None = None):
    lib = _lib.load()
    R = out.shape[0] if R is None else R
    assert W.dtype == torch.float32 and (W.stride(1) == 1 or W.shape[1] == 1) and W.shape[0] == N and W.shape[1] == K1 + K2
    rc = lib.dmpnn_linear_fwd(
        X1.data_ptr(), _dt(X1), _ld(X1), _ptr(idx1), K1,
        _ptr(X2), _dt(X2) if X2 is not None else F32, _ld(X2) if X2 is not None else 0, _ptr(idx2), K2,
        W.data_ptr(), W.stride(0), _ptr(bias),
        _ptr(res), _dt(res) if res is not None else F32, _ld(res) if res is not None else 0,
        act, float(act_param), out.data_ptr(), _dt(out), _ld(out), pad_to if pad_to is not None else min(_ld(out), out.shape[1]),
        R, N, _stream(),
    )
    _lib.check(rc, "dmpnn_linear_fwd")


def linear_wgrad(dY: Tensor, X1: Tensor, K1: int, dW: Tensor, N: int, *, idx1: Tensor | None = None,
                 X2: Tensor | None = None, K2: int = 0, idx2: Tensor | None = None, dbias: Tensor | None = None,
                 accumulate: bool = False, R: int | None = None):
    lib = _lib.load()
    R = dY.shape[0] if R is None else R
    assert dW.dtype == torch.float32 and dW.stride(1) == 1
    nbytes = C.c_size_t(0)
    _lib.check(lib.dmpnn_linear_wgrad_workspace_bytes(R, N, K1 + K2, C.byref(nbytes)), "wgrad_workspace_bytes")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dY.device)
    rc = lib.dmpnn_linear_wgrad(
        dY.data_ptr(), _dt(dY), _ld(dY), X1.data_ptr(), _dt(X1), _ld(X1), _ptr(idx1), K1,
        _ptr(X2), _dt(X2) if X2 is not None else F32, _ld(X2) if X2 is not None else 0, _ptr(idx2), K2,
        dW.data_ptr(), dW.stride(0), _ptr(dbias), 1 if accumulate else 0, R, N, ws.data_ptr(), _stream(),
    )
    _lib.check(rc, "dmpnn_linear_wgrad")


def segment_sum(X: Tensor, ptr: Tensor, n_seg: int, Ccols: int, out: Tensor, *, idx: Tensor | None = None,
                act: int = ACT_NONE, act_param: float = 0.0, scale_mode: int = SCALE_NONE, scale: float = 1.0,
                pad_to: int | None = None):
    lib = _lib.load()
    rc = lib.dmpnn_segment_sum(
        X.data_ptr(), _dt(X), _ld(X), _ptr(idx), ptr.data_ptr(), n_seg, Ccols, act, float(act_param),
        scale_mode, float(scale), out.data_ptr(), _dt(out), _ld(out),
        pad_to if pad_to is not None else min(_ld(out), out.shape[1]), _stream(),
    )
    _lib.check(rc, "dmpnn_segment_sum")


def segment_bcast(G: Tensor, seg_of_row: Tensor, ptr: Tensor | None, R: int, Ccols: int, out: Tensor, *,
                  scale_mode: int = SCALE_NONE, scale: float = 1.0, n_seg: int = 0):
    """n_seg > 0: rows of segment s are [ptr[s], ptr[s+1]) -- walk segments instead of looking every row up."""
    lib = _lib.load()
    rc = lib.dmpnn_segment_bcast(G.data_ptr(), _dt(G), _ld(G), seg_of_row.data_ptr(), _ptr(ptr),
                                 n_seg if ptr is not None else 0, R, Ccols,
                                 scale_mode, float(scale), out.data_ptr(), _dt(out), _ld(out), _stream())
    _lib.check(rc, "dmpnn_segment_bcast")


def bond_message(X: Tensor, lay: Layout, Ccols: int, out: Tensor, *, act: int = ACT_NONE, act_param: float = 0.0,
                 permute_on_read: bool = False):
    lib = _lib.load()
    if lay.E == 0:
        return
    rc = lib.dmpnn_bond_message(X.data_ptr(), _dt(X), _ld(X), lay.rowptr.data_ptr(), lay.rev_row.data_ptr(),
                                lay.V, Ccols, act, float(act_param), 1 if permute_on_read else 0,
                                out.data_ptr(), _dt(out), _ld(out), _stream())
    _lib.check(rc, "dmpnn_bond_message")


def rev_average(X: Tensor, lay: Layout, Ccols: int, out: Tensor, *, act: int = ACT_NONE, act_param: float = 0.0):
    lib = _lib.load()
    if lay.E == 0:
        return
    rc = lib.dmpnn_rev_average(X.data_ptr(), _dt(X), _ld(X), lay.rev_row.data_ptr(), lay.E, Ccols, act,
                               float(act_param), out.data_ptr(), _dt(out), _ld(out), _stream())
    _lib.check(rc, "dmpnn_rev_average")


def act_bwd(G: Tensor, Yact: Tensor, R: int, Ccols: int, *, act: int, act_param: float = 0.0,
            gidx: Tensor | None = None, from_preact: bool = False, dZ: Tensor | None = None,
            acc: Tensor | None = None):
    lib = _lib.load()
    if R == 0:
        return
    rc = lib.dmpnn_act_bwd(
        G.data_ptr(), _dt(G), _ld(G), _ptr(gidx), Yact.data_ptr(), _dt(Yact), _ld(Yact),
        1 if from_preact else 0, act, float(act_param),
        _ptr(dZ), _dt(dZ) if dZ is not None else F32, _ld(dZ) if dZ is not None else 0,
        _ptr(acc), _dt(acc) if acc is not None else F32, _ld(acc) if acc is not None else 0,
        R, Ccols, _stream(),
    )
    _lib.check(rc, "dmpnn_act_bwd")


# ----------------------------------------------------------------------------------------------
# message passing: forward / backward drivers
# ----------------------------------------------------------------------------------------------
@dataclass
class MPConfig:
    depth: int
    act: int
    act_param: float
    undirected: bool
    hidden_dtype: torch.dtype  # torch.float32 (<=1e-5 tier) or torch.bfloat16 (<=1e-2 tier)
    fused: bool = True         # use the fused wgmma depth-step kernel when applicable
    dropout_p: float = 0.0     # > 0: active nn.Dropout -- on the fused bf16 / ReLU path (Plan.dropout_ok), or forward-only
    mask_fn: object = None     # keep-mask source `f(like) -> {0,1} tensor like `like``; None = torch's bernoulli_
    forward_only: bool = False  # no backward follows (Monte Carlo dropout): dropout runs on every bond path, any activation


def _hidden(rows: int, hp: int, dtype, dev) -> Tensor:
    return torch.zeros((max(rows, 1), hp), dtype=dtype, device=dev)


UNDIRECTED_FUSED = os.environ.get("DMPNN_UNDIRECTED_FUSED", "1") != "0"   # DMPNN_UNDIRECTED_FUSED=0: A/B switch (message + GEMM launches)


_WARNED: set = set()


def _warn_once(key: str, msg: str):
    if key not in _WARNED:
        _WARNED.add(key)
        import warnings

        warnings.warn(msg, RuntimeWarning, stacklevel=3)


_FUSED_STATE: dict = {}


def _fused_available() -> bool:
    if "ok" not in _FUSED_STATE:
        lib = _lib.load()
        n = C.c_size_t(0)
        _FUSED_STATE["ok"] = lib.dmpnn_pack_weight_bf16_bytes(MAX_TC_HIDDEN, MAX_TC_HIDDEN, C.byref(n)) == 0
    return _FUSED_STATE["ok"]


def pack_weight_bf16(W: Tensor) -> Tensor:
    lib = _lib.load()
    N, K = W.shape
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_pack_weight_bf16_bytes(N, K, C.byref(n)), "dmpnn_pack_weight_bf16_bytes")
    out = torch.empty(n.value, dtype=torch.uint8, device=W.device)
    Wc = W.detach().contiguous().float()
    _lib.check(lib.dmpnn_pack_weight_bf16(Wc.data_ptr(), Wc.stride(0), N, K, out.data_ptr(), _stream()),
               "dmpnn_pack_weight_bf16")
    return out


def pack_weight_tc(W: Tensor, transpose: bool = False) -> Tensor:
    """Pack an nn.Linear weight (N x K; or, with transpose, a K x N matrix used as B[n][k] = W[k][n]) for
    dmpnn_linear_tc_bf16."""
    lib = _lib.load()
    Wc = W.detach().float()
    if Wc.stride(1) != 1:
        Wc = Wc.contiguous()
    N, K = (Wc.shape[1], Wc.shape[0]) if transpose else (Wc.shape[0], Wc.shape[1])
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_pack_weight_tc_bytes(N, K, C.byref(n)), "dmpnn_pack_weight_tc_bytes")
    out = torch.empty(n.value, dtype=torch.uint8, device=W.device)
    _lib.check(lib.dmpnn_pack_weight_tc(Wc.data_ptr(), Wc.stride(0), N, K, 1 if transpose else 0, out.data_ptr(),
                                        _stream()), "dmpnn_pack_weight_tc")
    return out


def linear_tc(A: Tensor, K: int, Wpk: Tensor, N: int, out: Tensor, *, bias: Tensor | None = None,
              res: Tensor | None = None, act: int = ACT_NONE, act_param: float = 0.0, R: int | None = None):
    """out = act(A[:, :K] . W^T + bias + res) on the tensor cores (bf16 operands, f32 accumulate)."""
    lib = _lib.load()
    R = out.shape[0] if R is None else R
    assert A.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and (res is None or res.dtype == torch.bfloat16)
    rc = lib.dmpnn_linear_tc_bf16(A.data_ptr(), _ld(A), R, K, Wpk.data_ptr(), N, _ptr(bias), _ptr(res),
                                  _ld(res) if res is not None else 0, act, float(act_param),
                                  out.data_ptr(), _ld(out), _stream())
    _lib.check(rc, "dmpnn_linear_tc_bf16")


def linear_tc_rows(A: Tensor, K: int, Wpk: Tensor, N: int, out: Tensor, *, R: int | None = None, bias: Tensor | None = None,
                   act: int = ACT_NONE, act_param: float = 0.0, Y: Tensor | None = None, from_preact: bool = False,
                   out_row: Tensor | None = None, res: Tensor | None = None, res_row: Tensor | None = None):
    """dmpnn_linear_tc_rows_bf16, acc = A[r, :K] . W^T.  Forward mode (Y None): out[r] = act(acc + bias), f32 or bf16 `out`.
    Mirror mode: out[out_row[r]] = (acc + res[res_row[r]]) * tau'(Y[out_row[r]]) in bf16 (tau' of `act`, from the
    pre-activation when `from_preact`); a missing map is the identity."""
    lib = _lib.load()
    R = A.shape[0] if R is None else R
    assert A.dtype == torch.bfloat16 and (Y is None or Y.dtype == torch.bfloat16) and (res is None or res.dtype == torch.bfloat16)
    rc = lib.dmpnn_linear_tc_rows_bf16(A.data_ptr(), _ld(A), R, K, Wpk.data_ptr(), N, _ptr(bias), act, float(act_param),
                                       _ptr(Y), _ld(Y) if Y is not None else 0, 1 if from_preact else 0, _ptr(out_row),
                                       _ptr(res), _ld(res) if res is not None else 0, _ptr(res_row),
                                       out.data_ptr(), _dt(out), _ld(out), _stream())
    _lib.check(rc, "dmpnn_linear_tc_rows_bf16")


def wgrad_tc(dY: Tensor, X: Tensor, R: int, N: int, K: int, dW: Tensor, *, accumulate: bool = False):
    """dW[n, :K] (+)= sum_r dY[r, n] X[r, :K] on the tensor cores (bf16 operands)."""
    lib = _lib.load()
    assert dY.dtype == torch.bfloat16 and X.dtype == torch.bfloat16 and dW.dtype == torch.float32
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_wgrad_tc_workspace_bytes(N, K, C.byref(n)), "dmpnn_wgrad_tc_workspace_bytes")
    ws = torch.empty(n.value, dtype=torch.uint8, device=dW.device)
    rc = lib.dmpnn_wgrad_tc_bf16(dY.data_ptr(), _ld(dY), X.data_ptr(), _ld(X), R, N, K, dW.data_ptr(), dW.stride(0),
                                 1 if accumulate else 0, ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_wgrad_tc_bf16")


def wgrad_tc_multi(dYs: list, X: Tensor, R: int, N: int, K: int, dW: Tensor, *, accumulate: bool = False):
    """dW[n, :K] (+)= sum_t sum_r dY_t[r, n] X[r, :K]: up to three terms per launch share the X stream; longer lists are
    issued in groups, accumulating."""
    lib = _lib.load()
    nxb = ((K + 15) // 16 * 16 + 63) // 64             # X boxes of a stage (csrc/wgrad_tc.cu: 2 * terms + nxb <= 9)
    per = max(1, min(3, (9 - nxb) // 2))
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_wgrad_tc_workspace_bytes(N, K, C.byref(n)), "dmpnn_wgrad_tc_workspace_bytes")
    ws = torch.empty(n.value, dtype=torch.uint8, device=dW.device)
    for i in range(0, len(dYs), per):
        grp = dYs[i:i + per]
        assert all(t.dtype == torch.bfloat16 and _ld(t) == _ld(grp[0]) for t in grp) and X.dtype == torch.bfloat16
        arr = (C.c_void_p * len(grp))(*[t.data_ptr() for t in grp])
        rc = lib.dmpnn_wgrad_tc_multi_bf16(C.cast(arr, C.c_void_p), len(grp), _ld(grp[0]), X.data_ptr(), _ld(X), R, N, K,
                                           dW.data_ptr(), dW.stride(0), 1 if (accumulate or i > 0) else 0, ws.data_ptr(), _stream())
        _lib.check(rc, "dmpnn_wgrad_tc_multi_bf16")


# ---- fp32-accurate tensor-core GEMMs (3xTF32, csrc/gemm_x3.cu) -------------------------------------------------
X3_ENABLED = os.environ.get("DMPNN_X3", "1") != "0"          # DMPNN_X3=0: A/B switch (fp32 tier on the SIMT f32 GEMMs)


def pack_weight_x3(W: Tensor, transpose: bool = False) -> Tensor:
    """nn.Linear weight (N x K; with transpose: a K x N matrix used as B[n][k] = W[k][n]) split into tf32 hi / lo parts and
    laid out for dmpnn_linear_x3."""
    lib = _lib.load()
    Wc = W.detach()
    if Wc.dtype != torch.float32 or Wc.stride(1) != 1:
        Wc = Wc.float().contiguous()
    N, K = (Wc.shape[1], Wc.shape[0]) if transpose else (Wc.shape[0], Wc.shape[1])
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_pack_weight_x3_bytes(N, K, C.byref(n)), "dmpnn_pack_weight_x3_bytes")
    out = torch.empty(n.value, dtype=torch.uint8, device=W.device)
    _lib.check(lib.dmpnn_pack_weight_x3(Wc.data_ptr(), Wc.stride(0), N, K, 1 if transpose else 0, out.data_ptr(), _stream()),
               "dmpnn_pack_weight_x3")
    return out


def linear_x3(A: Tensor, K: int, Wpk: Tensor, N: int, out: Tensor, *, idx: Tensor | None = None, bias: Tensor | None = None,
              res: Tensor | None = None, act: int = ACT_NONE, act_param: float = 0.0, R: int | None = None,
              pad_to: int | None = None):
    """out[:, :N] = act(A[idx][:, :K] . W^T + bias + res) with f32 accuracy on the tensor cores; columns [N, pad_to) zeroed."""
    lib = _lib.load()
    R = out.shape[0] if R is None else R
    assert A.dtype == torch.float32 and out.dtype == torch.float32 and (res is None or res.dtype == torch.float32)
    pad_to = min(_ld(out), out.shape[1]) if pad_to is None else pad_to
    rc = lib.dmpnn_linear_x3(A.data_ptr(), _ld(A), _ptr(idx), R, K, Wpk.data_ptr(), N, _ptr(bias), _ptr(res),
                             _ld(res) if res is not None else 0, act, float(act_param), out.data_ptr(), _ld(out),
                             max(N, min(pad_to, (N + 15) // 16 * 16)), _stream())
    _lib.check(rc, "dmpnn_linear_x3")


def wgrad_x3(dY: Tensor, X: Tensor, R: int, N: int, K: int, dW: Tensor, *, accumulate: bool = False):
    """dW[n, :K] (+)= sum_r dY[r, n] X[r, :K] with f32 accuracy on the tensor cores."""
    lib = _lib.load()
    assert dY.dtype == torch.float32 and X.dtype == torch.float32 and dW.dtype == torch.float32
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_wgrad_x3_workspace_bytes(N, K, C.byref(n)), "dmpnn_wgrad_x3_workspace_bytes")
    ws = torch.empty(n.value, dtype=torch.uint8, device=dW.device)
    rc = lib.dmpnn_wgrad_x3(dY.data_ptr(), _ld(dY), X.data_ptr(), _ld(X), R, N, K, dW.data_ptr(), dW.stride(0),
                            1 if accumulate else 0, ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_wgrad_x3")


# ---- molecule-level head (csrc/head.cu) ------------------------------------------------------------------------
def bn_train_fwd(X: Tensor, gamma, beta, running_mean, running_var, eps: float, momentum: float, Y: Tensor, Xhat: Tensor,
                 mean: Tensor, invstd: Tensor):
    lib = _lib.load()
    B, d = X.shape
    rc = lib.dmpnn_bn_train_fwd(X.data_ptr(), X.stride(0), B, d, _ptr(gamma), _ptr(beta), float(eps), float(momentum),
                                _ptr(running_mean), _ptr(running_var), Y.data_ptr(), Y.stride(0), Xhat.data_ptr(),
                                Xhat.stride(0), mean.data_ptr(), invstd.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_bn_train_fwd")


def bn_bwd(dY: Tensor, Xhat: Tensor, gamma, invstd: Tensor, dX: Tensor, dgamma, dbeta):
    lib = _lib.load()
    B, d = dY.shape
    rc = lib.dmpnn_bn_bwd(dY.data_ptr(), dY.stride(0), Xhat.data_ptr(), Xhat.stride(0), B, d, _ptr(gamma), invstd.data_ptr(),
                          dX.data_ptr(), dX.stride(0), _ptr(dgamma), _ptr(dbeta), _stream())
    _lib.check(rc, "dmpnn_bn_bwd")


def mse_loss(P: Tensor, Y: Tensor, w, tw, loss: Tensor, dP: Tensor):
    lib = _lib.load()
    B, T = P.shape
    rc = lib.dmpnn_mse_loss(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w), _ptr(tw), B, T,
                            loss.data_ptr(), dP.data_ptr(), dP.stride(0) if B else T, _stream())
    _lib.check(rc, "dmpnn_mse_loss")


def bce_loss(P: Tensor, Y: Tensor, w, tw, loss: Tensor, dP: Tensor):
    lib = _lib.load()
    B, T = P.shape
    rc = lib.dmpnn_bce_loss(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w), _ptr(tw), B, T,
                            loss.data_ptr(), dP.data_ptr(), dP.stride(0) if B else T, _stream())
    _lib.check(rc, "dmpnn_bce_loss")


def ce_loss(P: Tensor, Y: Tensor, w, tw, C: int, loss: Tensor, dP: Tensor):
    """P: B x (T*C) logits (task t in columns [t*C, (t+1)*C)), Y: B x T class labels."""
    lib = _lib.load()
    B, TC = P.shape
    T = Y.shape[1]
    rc = lib.dmpnn_ce_loss(P.data_ptr(), P.stride(0) if B else TC, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w), _ptr(tw), B,
                           T, C, loss.data_ptr(), dP.data_ptr(), dP.stride(0) if B else TC, _stream())
    _lib.check(rc, "dmpnn_ce_loss")


def class_probs(P: Tensor, C: int, softmax: bool, out: Tensor):
    """out = sigmoid(P) (softmax=False) or the softmax of every group of C columns of P (B x (T*C))."""
    lib = _lib.load()
    B, TC = P.shape
    rc = lib.dmpnn_class_probs(P.data_ptr(), P.stride(0) if B else TC, B, TC // C, C, 1 if softmax else 0, out.data_ptr(),
                               out.stride(0) if B else TC, _stream())
    _lib.check(rc, "dmpnn_class_probs")


def pred_transform(X: Tensor, kind: int, u: int, mean, scale, out: Tensor):
    """out (B x T*u, read as B x T x u) = the predictor output of `kind` (_lib.PRED_*) from the raw MLP output X (B x T*u);
    mean / scale (T entries each, or None) apply UnscaleTransform's eval mode."""
    lib = _lib.load()
    B, Tu = X.shape
    rc = lib.dmpnn_pred_transform(X.data_ptr(), X.stride(0) if B else Tu, B, Tu // u, kind, u, _ptr(mean), _ptr(scale),
                                  out.data_ptr(), out.stride(0) if B else Tu, _stream())
    _lib.check(rc, "dmpnn_pred_transform")


def pred_transform_bwd(X: Tensor, dOut: Tensor, kind: int, u: int, scale, dX: Tensor):
    lib = _lib.load()
    B, Tu = X.shape
    rc = lib.dmpnn_pred_transform_bwd(X.data_ptr(), X.stride(0) if B else Tu, dOut.data_ptr(), dOut.stride(0) if B else Tu, B,
                                      Tu // u, kind, u, _ptr(scale), dX.data_ptr(), dX.stride(0) if B else Tu, _stream())
    _lib.check(rc, "dmpnn_pred_transform_bwd")


def _uq_args(P: Tensor, Y: Tensor, u: int):
    B, Tu = P.shape
    T = Y.shape[1]
    return P.data_ptr(), P.stride(0) if B else Tu, Y.data_ptr(), Y.stride(0) if B else T, B, T


def mve_loss(P: Tensor, Y: Tensor, w, tw, loss: Tensor, dP: Tensor):
    """P: B x (T*2) = (mean, var) per task, Y: B x T."""
    lib = _lib.load()
    p, ldp, y, ldy, B, T = _uq_args(P, Y, 2)
    rc = lib.dmpnn_mve_loss(p, ldp, y, ldy, _ptr(w), _ptr(tw), B, T, loss.data_ptr(), _ptr(dP), ldp, _stream())
    _lib.check(rc, "dmpnn_mve_loss")


def evidential_loss(P: Tensor, Y: Tensor, w, tw, v_kl: float, eps: float, loss: Tensor, dP: Tensor):
    """P: B x (T*4) = (mean, v, alpha, beta) per task, Y: B x T."""
    lib = _lib.load()
    p, ldp, y, ldy, B, T = _uq_args(P, Y, 4)
    rc = lib.dmpnn_evidential_loss(p, ldp, y, ldy, _ptr(w), _ptr(tw), B, T, float(v_kl), float(eps), loss.data_ptr(),
                                   _ptr(dP), ldp, _stream())
    _lib.check(rc, "dmpnn_evidential_loss")


def quantile_loss(P: Tensor, Y: Tensor, w, tw, alpha: float, loss: Tensor, dP: Tensor):
    """P: B x (T*2) = (mean, interval) per task, Y: B x T."""
    lib = _lib.load()
    p, ldp, y, ldy, B, T = _uq_args(P, Y, 2)
    rc = lib.dmpnn_quantile_loss(p, ldp, y, ldy, _ptr(w), _ptr(tw), B, T, float(alpha), loss.data_ptr(), _ptr(dP), ldp,
                                 _stream())
    _lib.check(rc, "dmpnn_quantile_loss")


def dirichlet_loss(P: Tensor, Y: Tensor, w, tw, C: int, v_kl: float, loss: Tensor, dP: Tensor):
    """P: B x (T*C) = alpha per task and class, Y: B x T class labels."""
    lib = _lib.load()
    p, ldp, y, ldy, B, T = _uq_args(P, Y, C)
    rc = lib.dmpnn_dirichlet_loss(p, ldp, y, ldy, _ptr(w), _ptr(tw), B, T, C, float(v_kl), loss.data_ptr(), _ptr(dP), ldp,
                                  _stream())
    _lib.check(rc, "dmpnn_dirichlet_loss")


def regression_loss(P: Tensor, Y: Tensor, w, tw, lt_mask, gt_mask, kind: int, loss: Tensor, dP: Tensor):
    """MSE / MAE / RMSE (_lib.LOSS_*) on P, Y (B x T); lt_mask / gt_mask (B x T uint8 with Y's row stride, or None) give
    the bounded variants."""
    lib = _lib.load()
    B, T = P.shape
    ldm = T
    for m in (lt_mask, gt_mask):
        if m is not None:
            assert m.dtype == torch.uint8 and m.shape == (B, T) and m.is_contiguous(), "masks: contiguous B x T uint8"
    rc = lib.dmpnn_regression_loss(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w),
                                   _ptr(tw), _ptr(lt_mask), _ptr(gt_mask), ldm, B, T, kind, loss.data_ptr(), _ptr(dP),
                                   dP.stride(0) if B else T, _stream())
    _lib.check(rc, "dmpnn_regression_loss")


def enrichment_loss(P: Tensor, Y: Tensor, w, tw, d: float, method: int, zscale: float, zinterval: float, loss: Tensor,
                    dP: Tensor):
    """NLogProbEnrichment on P (B x 1, the predicted enrichment) and Y (B x 2 counts k1, k2; NaN = masked); tw has 2
    entries, d = n2 / n1, method by _lib.ENRICH_METHODS."""
    lib = _lib.load()
    B = P.shape[0]
    rc = lib.dmpnn_enrichment_loss(P.data_ptr(), P.stride(0) if B else 1, Y.data_ptr(), Y.stride(0) if B else 2, _ptr(w),
                                   _ptr(tw), B, float(d), method, float(zscale), float(zinterval), loss.data_ptr(), _ptr(dP),
                                   dP.stride(0) if B else 1, _stream())
    _lib.check(rc, "dmpnn_enrichment_loss")


def spectral_transform(X: Tensor, act: int, out: Tensor):
    """out (B x T) = a(a(X)) normalised per row, a = softplus or exp (_lib.SPEC_*)."""
    lib = _lib.load()
    B, T = X.shape
    rc = lib.dmpnn_spectral_transform(X.data_ptr(), X.stride(0) if B else T, B, T, act, out.data_ptr(),
                                      out.stride(0) if B else T, _stream())
    _lib.check(rc, "dmpnn_spectral_transform")


def spectral_transform_bwd(X: Tensor, dOut: Tensor, act: int, dX: Tensor):
    lib = _lib.load()
    B, T = X.shape
    rc = lib.dmpnn_spectral_transform_bwd(X.data_ptr(), X.stride(0) if B else T, dOut.data_ptr(), dOut.stride(0) if B else T,
                                          B, T, act, dX.data_ptr(), dX.stride(0) if B else T, _stream())
    _lib.check(rc, "dmpnn_spectral_transform_bwd")


def _spectral_loss(fn: str, P: Tensor, Y: Tensor, w, tw, threshold, loss: Tensor, dP: Tensor):
    lib = _lib.load()
    B, T = P.shape
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_spectral_loss_workspace_bytes(B, C.byref(n)), "dmpnn_spectral_loss_workspace_bytes")
    ws = torch.empty(max(n.value, 1), dtype=torch.uint8, device=P.device)
    thr = float("nan") if threshold is None else float(threshold)
    rc = getattr(lib, fn)(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w), _ptr(tw), B,
                          T, thr, loss.data_ptr(), _ptr(dP), dP.stride(0) if B else T, ws.data_ptr(), _stream())
    _lib.check(rc, fn)


def sid_loss(P: Tensor, Y: Tensor, w, tw, threshold, loss: Tensor, dP: Tensor):
    """SID on spectra P and targets Y (B x T, NaN = masked bin); threshold None = no clamp."""
    _spectral_loss("dmpnn_sid_loss", P, Y, w, tw, threshold, loss, dP)


def wasserstein_loss(P: Tensor, Y: Tensor, w, tw, threshold, loss: Tensor, dP: Tensor):
    """Wasserstein (earth mover's) distance of the cumulative spectra; arguments as sid_loss."""
    _spectral_loss("dmpnn_wasserstein_loss", P, Y, w, tw, threshold, loss, dP)


# ---- atom- and bond-level heads (csrc/row_head.cu) ----------------------------------------------------------------
def edge_pair_mean(P: Tensor, rev: Tensor, out: Tensor):
    """out (E/2 x C) = (P[2i] + P[2i+1]) / 2 of P (E x C), NaN rows where rev[2i] != 2i+1 (rev: int32, E)."""
    lib = _lib.load()
    E, Cc = P.shape
    rc = lib.dmpnn_edge_pair_mean(P.data_ptr(), P.stride(0) if E else Cc, rev.data_ptr(), E, Cc, out.data_ptr(),
                                  out.stride(0) if E else Cc, _stream())
    _lib.check(rc, "dmpnn_edge_pair_mean")


def edge_pair_mean_bwd(G: Tensor, dP: Tensor):
    """dP (E x C): rows 2i and 2i+1 both G[i] / 2."""
    lib = _lib.load()
    E, Cc = dP.shape
    rc = lib.dmpnn_edge_pair_mean_bwd(G.data_ptr(), G.stride(0) if E else Cc, E, Cc, dP.data_ptr(), dP.stride(0) if E else Cc,
                                      _stream())
    _lib.check(rc, "dmpnn_edge_pair_mean_bwd")


def _rows_workspace(fn: str, B: int, T: int, dev) -> Tensor:
    lib = _lib.load()
    n = C.c_size_t(0)
    _lib.check(getattr(lib, fn + "_workspace_bytes")(B, T, C.byref(n)), fn + "_workspace_bytes")
    return torch.empty(max(n.value, 1), dtype=torch.uint8, device=dev)


def regression_loss_rows(P: Tensor, Y: Tensor, w, tw, lt_mask, gt_mask, kind: int, loss: Tensor, dP: Tensor):
    """regression_loss over the whole grid (dmpnn_regression_loss_rows): same arguments and results, for V or E rows."""
    lib = _lib.load()
    B, T = P.shape
    for m in (lt_mask, gt_mask):
        if m is not None:
            assert m.dtype == torch.uint8 and m.shape == (B, T) and m.is_contiguous(), "masks: contiguous B x T uint8"
    ws = _rows_workspace("dmpnn_regression_loss_rows", B, T, P.device)
    rc = lib.dmpnn_regression_loss_rows(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T,
                                        _ptr(w), _ptr(tw), _ptr(lt_mask), _ptr(gt_mask), T, B, T, kind, loss.data_ptr(),
                                        _ptr(dP), dP.stride(0) if B else T, ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_regression_loss_rows")


def bce_loss_rows(P: Tensor, Y: Tensor, w, tw, loss: Tensor, dP: Tensor):
    """bce_loss over the whole grid (dmpnn_bce_loss_rows)."""
    lib = _lib.load()
    B, T = P.shape
    ws = _rows_workspace("dmpnn_bce_loss_rows", B, T, P.device)
    rc = lib.dmpnn_bce_loss_rows(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w),
                                 _ptr(tw), B, T, loss.data_ptr(), _ptr(dP), dP.stride(0) if B else T, ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_bce_loss_rows")


def pinball_loss_rows(P: Tensor, Y: Tensor, w, tw, alpha: float, loss: Tensor, dP: Tensor):
    """PointQuantileLoss at `alpha` over the whole grid (dmpnn_pinball_loss_rows), for molecule, atom or bond rows."""
    lib = _lib.load()
    B, T = P.shape
    ws = _rows_workspace("dmpnn_pinball_loss_rows", B, T, P.device)
    rc = lib.dmpnn_pinball_loss_rows(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w),
                                     _ptr(tw), B, T, float(alpha), loss.data_ptr(), _ptr(dP), dP.stride(0) if B else T,
                                     ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_pinball_loss_rows")


def ce_loss_rows(P: Tensor, Y: Tensor, w, tw, C_: int, loss: Tensor, dP: Tensor):
    """ce_loss over the whole grid (dmpnn_ce_loss_rows); P: B x (T*C) logits, Y: B x T class labels."""
    lib = _lib.load()
    B, TC = P.shape
    T = Y.shape[1]
    ws = _rows_workspace("dmpnn_ce_loss_rows", B, T, P.device)
    rc = lib.dmpnn_ce_loss_rows(P.data_ptr(), P.stride(0) if B else TC, Y.data_ptr(), Y.stride(0) if B else T, _ptr(w),
                                _ptr(tw), B, T, C_, loss.data_ptr(), _ptr(dP), dP.stride(0) if B else TC, ws.data_ptr(),
                                _stream())
    _lib.check(rc, "dmpnn_ce_loss_rows")


# ---- ConstrainerFFN (csrc/constrain.cu) --------------------------------------------------------------------------
def constrain_fwd(Kl: Tensor, P: Tensor, ptr: Tensor, Cn: Tensor, out: Tensor, status: Tensor):
    """out (R x t) = P adjusted so that each molecule's constrained columns sum to Cn's row (ffn.py:119-141); Kl: R x n_c
    MLP output, ptr: int32 m + 1 molecule row offsets, Cn: m x t constraints (NaN in row 0 = unconstrained column).
    status (int32, 1): 0, or the constrained column count when (n_c, that count) is a shape the reference rejects."""
    lib = _lib.load()
    R, n_c = Kl.shape
    m, t = Cn.shape
    rc = lib.dmpnn_constrain_fwd(Kl.data_ptr(), Kl.stride(0) if R else n_c, n_c, P.data_ptr(), P.stride(0) if R else t,
                                 ptr.data_ptr(), m, Cn.data_ptr(), Cn.stride(0) if m else t, t, out.data_ptr(),
                                 out.stride(0) if R else t, status.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_constrain_fwd")


def constrain_bwd(G: Tensor, Kl: Tensor, P: Tensor, ptr: Tensor, Cn: Tensor, dP: Tensor, dKl: Tensor):
    """dP (R x t) and dKl (R x n_c) of constrain_fwd given G = dL/dout; arguments as constrain_fwd."""
    lib = _lib.load()
    R, n_c = Kl.shape
    m, t = Cn.shape
    rc = lib.dmpnn_constrain_bwd(G.data_ptr(), G.stride(0) if R else t, Kl.data_ptr(), Kl.stride(0) if R else n_c, n_c,
                                 P.data_ptr(), P.stride(0) if R else t, ptr.data_ptr(), m, Cn.data_ptr(),
                                 Cn.stride(0) if m else t, t, dP.data_ptr(), dP.stride(0) if R else t, dKl.data_ptr(),
                                 dKl.stride(0) if R else n_c, _stream())
    _lib.check(rc, "dmpnn_constrain_bwd")


# ---- validation / test metrics (csrc/metrics.cu) ------------------------------------------------------------------
def _metric_workspace(B: int, T: int, C_: int, dev) -> Tensor:
    lib = _lib.load()
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_metric_workspace_bytes(B, T, C_, C.byref(n)), "dmpnn_metric_workspace_bytes")
    return torch.empty(max(n.value, 1), dtype=torch.uint8, device=dev)


def _masks_ok(B: int, T: int, *ms):
    for m in ms:
        if m is not None:
            assert m.dtype == torch.uint8 and m.shape == (B, T) and m.is_contiguous(), "masks: contiguous B x T uint8"


def metric_accumulate(kind: int, P: Tensor, Y: Tensor, mask, w, tw, lt_mask, gt_mask, fstate, istate, status):
    """Adds one batch to a metric's state (_lib.METRIC_*): P, Y B x T f32; mask / lt_mask / gt_mask B x T uint8 or None
    (mask None: the finite targets); w (B) / tw (T) f32 or None; fstate f64, istate int64, status int32 (device)."""
    lib = _lib.load()
    B, T = Y.shape
    _masks_ok(B, T, mask, lt_mask, gt_mask)
    ws = _metric_workspace(B, T, 1, P.device)
    rc = lib.dmpnn_metric_accumulate(kind, P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T,
                                     _ptr(mask), _ptr(w), _ptr(tw), _ptr(lt_mask), _ptr(gt_mask), T, B, T, _ptr(fstate),
                                     _ptr(istate), _ptr(status), ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_metric_accumulate")


def metric_multiclass_mcc(P: Tensor, Y: Tensor, mask, w, C_: int, fstate: Tensor, status: Tensor):
    """Adds one batch to the multiclass MCC's T x (2C + 2) f64 state; P: B x (T*C) f32 class scores, Y: B x T labels."""
    lib = _lib.load()
    B, T = Y.shape
    _masks_ok(B, T, mask)
    ws = _metric_workspace(B, T, C_, P.device)
    rc = lib.dmpnn_metric_multiclass_mcc(P.data_ptr(), P.stride(0) if B else T * C_, Y.data_ptr(), Y.stride(0) if B else T,
                                         _ptr(mask), T, _ptr(w), B, T, C_, fstate.data_ptr(), status.data_ptr(),
                                         ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_metric_multiclass_mcc")


def metric_rank_format(P: Tensor, Y: Tensor, mask, score: Tensor, label: Tensor, keep: Tensor, status: Tensor):
    """One update of AUROC / AUPRC: writes score (f32), label and keep (uint8), B * T entries each."""
    lib = _lib.load()
    B, T = Y.shape
    _masks_ok(B, T, mask)
    ws = _metric_workspace(B, T, 1, P.device)
    rc = lib.dmpnn_metric_rank_format(P.data_ptr(), P.stride(0) if B else T, Y.data_ptr(), Y.stride(0) if B else T,
                                      _ptr(mask), T, B, T, score.data_ptr(), label.data_ptr(), keep.data_ptr(),
                                      status.data_ptr(), ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_metric_rank_format")


def rank_curve(score: Tensor, label: Tensor, keep: Tensor, out: Tensor):
    """out (f64, 2) = AUROC, AUPRC of the kept entries of the formatted updates (dmpnn_rank_curve)."""
    lib = _lib.load()
    n = score.numel()
    nb = C.c_size_t(0)
    _lib.check(lib.dmpnn_rank_curve_workspace_bytes(n, C.byref(nb)), "dmpnn_rank_curve_workspace_bytes")
    ws = torch.empty(max(nb.value, 1), dtype=torch.uint8, device=out.device)
    rc = lib.dmpnn_rank_curve(_ptr(score), _ptr(label), _ptr(keep), n, out.data_ptr(), ws.data_ptr(), nb.value, _stream())
    _lib.check(rc, "dmpnn_rank_curve")


def column_sum(Y: Tensor, R: int, N: int, out: Tensor, *, accumulate: bool = False):
    lib = _lib.load()
    n = C.c_size_t(0)
    _lib.check(lib.dmpnn_linear_wgrad_workspace_bytes(R, N, 1, C.byref(n)), "wgrad_workspace_bytes")
    ws = torch.empty(n.value, dtype=torch.uint8, device=out.device)
    rc = lib.dmpnn_column_sum(Y.data_ptr(), _dt(Y), _ld(Y), R, N, out.data_ptr(), 1 if accumulate else 0,
                              ws.data_ptr(), _stream())
    _lib.check(rc, "dmpnn_column_sum")


def bond_message_bwd_masked(dM: Tensor, Yact: Tensor, lay: Layout, Ccols: int, out: Tensor, *, act: int,
                            act_param: float = 0.0):
    lib = _lib.load()
    if lay.E == 0:
        return
    rc = lib.dmpnn_bond_message_bwd_masked(dM.data_ptr(), _dt(dM), _ld(dM), lay.rowptr.data_ptr(),
                                           lay.rev_row.data_ptr(), lay.V, Ccols, Yact.data_ptr(), _ld(Yact), act,
                                           float(act_param), out.data_ptr(), _ld(out), _stream())
    _lib.check(rc, "dmpnn_bond_message_bwd_masked")


def sum_act_bwd(Zs: list, G: Tensor | None, Ypre: Tensor | None, out: Tensor, R: int, Ccols: int, *, act: int,
                act_param: float = 0.0):
    """out = sum(Zs) + G * tau'(Ypre) in one pass (<= 8 addends per call; longer lists are folded)."""
    lib = _lib.load()
    if R == 0:
        return
    Zs = list(Zs)
    while len(Zs) > 8:   # fold the first eight into one buffer
        tmp = torch.empty_like(Zs[0])
        sum_act_bwd(Zs[:8], None, None, tmp, R, Ccols, act=act, act_param=act_param)
        Zs = [tmp] + Zs[8:]
    ref = Zs[0] if Zs else G
    arr = (C.c_void_p * 8)(*[z.data_ptr() for z in Zs] + [None] * (8 - len(Zs)))
    rc = lib.dmpnn_sum_act_bwd(C.cast(arr, C.c_void_p), len(Zs), _ld(ref), _ptr(G), _ld(G) if G is not None else 0,
                               _ptr(Ypre), _ld(Ypre) if Ypre is not None else 0, _dt(ref), act, float(act_param),
                               out.data_ptr(), _dt(out), _ld(out), R, Ccols, _stream())
    _lib.check(rc, "dmpnn_sum_act_bwd")


def concat_bf16(X1: Tensor, K1: int, out: Tensor, R: int, *, idx1: Tensor | None = None, X2: Tensor | None = None,
                K2: int = 0, idx2: Tensor | None = None, width: int | None = None):
    lib = _lib.load()
    width = out.shape[1] if width is None else width
    rc = lib.dmpnn_concat_bf16(X1.data_ptr(), _dt(X1), _ld(X1), _ptr(idx1), K1,
                               _ptr(X2), _dt(X2) if X2 is not None else F32, _ld(X2) if X2 is not None else 0,
                               _ptr(idx2), K2, out.data_ptr(), _ld(out), width, R, _stream())
    _lib.check(rc, "dmpnn_concat_bf16")


def dropout_keep_bits(rows: int, h: int, cfg: "MPConfig", like: Tensor) -> Tensor:
    """uint16 [rows, pad16(h) / 16] keep bits for one dropout site of the fused path (dmpnn_dropout_bits: Philox4x32-10 keyed
    by the device generator's seed and current offset, so `torch.manual_seed` governs the masks as in the reference; the
    offset is then advanced).  `cfg.mask_fn` (test hook) supplies a {0, 1} tensor instead, which is packed into the same words."""
    nj = (h + 15) // 16
    dev = like.device
    if cfg.mask_fn is not None:
        M = cfg.mask_fn(like)[:rows, : nj * 16].to(torch.int32).reshape(rows, nj, 16)
        w = (M << torch.arange(16, device=dev, dtype=torch.int32)).sum(-1)
        return w.to(torch.uint16).contiguous()
    if torch.cuda.is_current_stream_capturing():
        raise DmpnnError("training-mode dropout inside a captured CUDA graph is not supported (the Philox offset is host state)")
    lib = _lib.load()
    gen = torch.cuda.default_generators[dev.index if dev.index is not None else torch.cuda.current_device()]
    seed, off = int(gen.initial_seed()) & (2 ** 64 - 1), int(gen.get_offset())
    gen.set_offset(off + 4)
    bits = torch.empty((max(rows, 1), nj), dtype=torch.uint16, device=dev)
    _lib.check(lib.dmpnn_dropout_bits(bits.data_ptr(), rows, nj, float(cfg.dropout_p), seed, off, _stream()), "dmpnn_dropout_bits")
    return bits


def concat_f32(X1: Tensor, K1: int, out: Tensor, R: int, *, idx1: Tensor | None = None, X2: Tensor | None = None,
               K2: int = 0, idx2: Tensor | None = None, width: int | None = None):
    lib = _lib.load()
    width = out.shape[1] if width is None else width
    assert out.dtype == torch.float32
    rc = lib.dmpnn_concat_f32(X1.data_ptr(), _dt(X1), _ld(X1), _ptr(idx1), K1,
                              _ptr(X2), _dt(X2) if X2 is not None else F32, _ld(X2) if X2 is not None else 0,
                              _ptr(idx2), K2, out.data_ptr(), _ld(out), width, R, _stream())
    _lib.check(rc, "dmpnn_concat_f32")


def bond_step_fused(H_prev: Tensor, H0: Tensor, H_next: Tensor, h: int, Wpk: Tensor, bias: Tensor | None,
                    lay: Layout, act: int, act_param: float, first_step: bool, M_out: Tensor | None = None,
                    drop_bits: Tensor | None = None, drop_scale: float = 1.0):
    """One fused depth step; M_out (first step only) also receives the message M^1 the step consumed; `drop_bits`
    (dropout_keep_bits) applies training-mode dropout with scale `drop_scale` in the epilogue."""
    lib = _lib.load()
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    rc = lib.dmpnn_bond_step_fused_bf16(
        H_prev.data_ptr(), H0.data_ptr(), H_next.data_ptr(), _ld(H0), H0.shape[0], h, Wpk.data_ptr(), _ptr(bias),
        lay.rowptr.data_ptr(), lay.rev_row.data_ptr(), trp.data_ptr(), tap.data_ptr(),
        nt, act, float(act_param), 1 if first_step else 0, _ptr(M_out), _ptr(wf), _ptr(nw), _ptr(dr), _ptr(drop_bits),
        float(drop_scale), _stream(),
    )
    _lib.check(rc, "dmpnn_bond_step_fused_bf16")


def _empty_hidden(rows: int, hp: int, dtype, dev) -> Tensor:
    """Uninitialised hidden buffer: only for producers that write every column below pad16(h)."""
    return torch.empty((max(rows, 1), hp), dtype=dtype, device=dev)


def scale_mask_(X: Tensor, M: Tensor, scale: float):
    """X <- X * M * scale in place over the whole (contiguous) buffer -- dmpnn_scale_mask."""
    lib = _lib.load()
    assert X.is_contiguous() and M.is_contiguous() and X.shape == M.shape and X.dtype == M.dtype
    rc = lib.dmpnn_scale_mask(X.data_ptr(), M.data_ptr(), X.data_ptr(), _dt(X), X.numel(), float(scale), _stream())
    _lib.check(rc, "dmpnn_scale_mask")


def _dropout_(X: Tensor, cfg: MPConfig):
    """nn.Dropout(p) in training mode on a hidden buffer (base.py:139, :182): keep mask from torch's RNG stream (so
    torch.manual_seed governs it, as in the reference), applied with the exact f32 scale 1 / (1 - p)."""
    keep = 1.0 - cfg.dropout_p
    M = cfg.mask_fn(X) if cfg.mask_fn is not None else torch.empty_like(X).bernoulli_(keep)
    scale_mask_(X, M, 1.0 / keep)


def bond_step_bwd_fused(dZ: Tensor, Yact: Tensor | None, dOut: Tensor, h: int, WpkT: Tensor, lay: Layout, act: int,
                        act_param: float, G_out: Tensor | None = None, y_is_preact: bool = False,
                        addends: tuple = ()):
    """dOut = (S.P)(dZ . W_h) [* tau'(Yact)] in one fused launch (WpkT = pack_weight_bf16(W_h.t()));
    G_out also receives (S.P) dZ, the left operand of this step's W_h gradient."""
    lib = _lib.load()
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    rc = lib.dmpnn_bond_step_bwd_fused_bf16(
        dZ.data_ptr(), _ptr(Yact), dOut.data_ptr(), _ld(dZ), dZ.shape[0], h, WpkT.data_ptr(),
        lay.rowptr.data_ptr(), lay.rev_row.data_ptr(), trp.data_ptr(), tap.data_ptr(),
        nt, act, float(act_param), 1 if y_is_preact else 0,
        addends[0].data_ptr() if len(addends) > 0 else None, addends[1].data_ptr() if len(addends) > 1 else None,
        _ptr(G_out), _ptr(wf), _ptr(nw), _ptr(dr), _stream())
    _lib.check(rc, "dmpnn_bond_step_bwd_fused_bf16")


# ---- atom-granular fused step (AtomMessagePassing; the ATOM instantiations of the fused kernel) ------------------------
ATOM_FUSED_ENABLED = os.environ.get("DMPNN_ATOM_FUSED", "1") != "0"      # DMPNN_ATOM_FUSED=0: A/B switch (gather + GEMM launches)
ATOM_TILE_ATOMS, ATOM_TILE_EDGES = 128, 1024


def atom_tables(lay: Layout):
    """(tile_atom_ptr, tile_edge_ptr, n_tiles_dev, n_tiles_max) of the ATOM tiles of a batch: runs of whole molecules with
    <= 128 atoms (and <= 1024 edge rows, what the kernel's staged neighbour table holds), built once per batch on the device
    (dmpnn_tiles_build; the kernel reads the tile count from device memory: no host read-back)."""
    if lay._atom_work is None:
        lib = _lib.load()
        dev = lay.rowptr.device
        i32 = dict(dtype=torch.int32, device=dev)
        ta = torch.empty(lay.B + 2, **i32)
        te = torch.empty(lay.B + 2, **i32)
        info = torch.zeros(4, **i32)
        n = C.c_size_t(0)
        _lib.check(lib.dmpnn_tiles_workspace_bytes(lay.B, C.byref(n)), "dmpnn_tiles_workspace_bytes")
        ws = torch.empty(max(n.value, 16), dtype=torch.uint8, device=dev)
        _lib.check(lib.dmpnn_tiles_build(lay.mol_atom_ptr.data_ptr(), lay.mol_row_ptr.data_ptr(), lay.B, ATOM_TILE_EDGES,
                                         ATOM_TILE_ATOMS, te.data_ptr(), ta.data_ptr(), info.data_ptr(), ws.data_ptr(), _stream()),
                   "dmpnn_tiles_build")
        lay._atom_work = (ta, te, info, max(lay.B, 1))
    return lay._atom_work


def atom_step_fused(H_prev: Tensor, H0: Tensor, H_next: Tensor, h: int, Wpk: Tensor, bias: Tensor | None, lay: Layout,
                    act: int, act_param: float, first_step: bool, N_out: Tensor | None = None):
    """H_next[v] = act(H0[v] + bias + W . sum_{e in in(v)} g(H_prev[src(e)])) in one launch (dmpnn_atom_step_fused_bf16)."""
    lib = _lib.load()
    ta, te, info, nmax = atom_tables(lay)
    rc = lib.dmpnn_atom_step_fused_bf16(
        H_prev.data_ptr(), H0.data_ptr(), H_next.data_ptr(), _ld(H0), H0.shape[0], h, Wpk.data_ptr(), _ptr(bias),
        lay.rowptr.data_ptr(), lay.src_row.data_ptr(), ta.data_ptr(), te.data_ptr(), info.data_ptr(), nmax, act,
        float(act_param), 1 if first_step else 0, _ptr(N_out), _stream())
    _lib.check(rc, "dmpnn_atom_step_fused_bf16")


def atom_step_bwd_fused(dZ: Tensor, Yact: Tensor | None, dOut: Tensor, h: int, WpkT: Tensor, lay: Layout, act: int,
                        act_param: float, G_out: Tensor | None = None, y_is_preact: bool = False, addends: tuple = ()):
    """dOut[v] = ((sum_{e in in(v)} dZ[src(e)]) . W) [* act'(Yact[v])] [+ addends (y_is_preact only)]; G_out also receives
    the gathered operand."""
    lib = _lib.load()
    ta, te, info, nmax = atom_tables(lay)
    rc = lib.dmpnn_atom_step_bwd_fused_bf16(
        dZ.data_ptr(), _ptr(Yact), dOut.data_ptr(), _ld(dZ), dZ.shape[0], h, WpkT.data_ptr(), lay.rowptr.data_ptr(),
        lay.src_row.data_ptr(), ta.data_ptr(), te.data_ptr(), info.data_ptr(), nmax, act, float(act_param),
        1 if y_is_preact else 0, addends[0].data_ptr() if len(addends) > 0 else None,
        addends[1].data_ptr() if len(addends) > 1 else None, _ptr(G_out), _stream())
    _lib.check(rc, "dmpnn_atom_step_bwd_fused_bf16")


def _readout_pad(d_v: int, h: int) -> int:
    """Column at which M_v starts inside the read-out operand [V || M_v]: d_v rounded up to 8 columns (16-byte aligned bf16 rows
    for the vectorised segment sum that writes M_v in place; d_v = 106 of the reaction graphs left it on the scalar kernel:
    1.2 ms per step at C4), unless that would exceed the GEMM's K limit."""
    dvp = (d_v + 7) // 8 * 8
    return dvp if dvp + h <= MAX_TC_K else d_v


def _wo_padded(Wo: Tensor, d_v: int, dvp: int) -> Tensor:
    """W_o with zero columns for the padding between V and M_v"""
    if dvp == d_v:
        return Wo
    return torch.cat([Wo[:, :d_v], Wo.new_zeros((Wo.shape[0], dvp - d_v)), Wo[:, d_v:]], 1)


def _wo_unpadded(dWo_p: Tensor, d_v: int, dvp: int) -> Tensor:
    return dWo_p if dvp == d_v else torch.cat([dWo_p[:, :d_v], dWo_p[:, dvp:]], 1)


def _readout_operand(lay: Layout, V: Tensor, Hprev: Tensor, first: bool, h: int, cfg: MPConfig, idx: Tensor | None, dvp: int,
                     ones: bool):
    """The bf16 read-out operand [V || 0-pad to dvp || M_v || 0-pad to pad16(h) || 1] (the torch.cat of base.py:180), M_v
    (base.py:208-211) written in place by the segment sum of Hprev: over the in-edge rows of each atom (`idx` None: bonds) or
    over the rows idx[e] of its in-edges e (atoms: `src_row`).  `ones`: the last column holds ones when K = dvp + pad16(h) + 1
    fits the GEMM, and the W_o weight-gradient GEMM then delivers db_o (the column sums of dY) as its last column -- no
    column-sum pass over V x h.  Returns (XO, ones_col), ones_col None without the ones column; _readout_grads decodes it."""
    hc = (h + 15) // 16 * 16       # M_v zero-padded to pad16(h): 16-byte stores in the segment sum
    # columns beyond the K a GEMM asks for are clipped by its TMA descriptor
    XO = torch.empty((max(lay.V, 1), (dvp + hc + 1 + 15) // 16 * 16), dtype=cfg.hidden_dtype, device=V.device)
    concat_bf16(V, V.shape[1], XO, lay.V, width=dvp)
    segment_sum(Hprev, lay.rowptr, lay.V, h, XO[:, dvp:dvp + h], idx=idx, act=(cfg.act if first else ACT_NONE),
                act_param=cfg.act_param, pad_to=hc)
    ones_col = dvp + hc if ones and dvp + hc + 1 <= MAX_TC_K else None
    if ones_col is not None:
        XO[:, ones_col].fill_(1.0)
    return XO, ones_col


def _readout_grads(dY: Tensor, saved: dict, nV: int, h: int, d_v: int, bias: bool):
    """(dW_o, db_o) of the bf16 mirrors from dY and the read-out operand saved["XO"] of _readout_operand: one weight-gradient
    GEMM whose columns of the padding after V are dropped from dW_o; db_o is its ones column when the forward added one, else
    a column sum of dY (None without `bias`)."""
    dvp, oc = saved["dvp"], saved["ones_col"] if bias else None
    K = dvp + h if oc is None else oc + 1
    dWo_p = torch.empty((h, K), dtype=torch.float32, device=dY.device)
    wgrad_tc(dY, saved["XO"], nV, h, K, dWo_p)
    dWo = _wo_unpadded(dWo_p[:, :dvp + h], d_v, dvp)
    if oc is not None:
        return dWo, dWo_p[:, oc]
    dbo = None
    if bias:
        dbo = torch.zeros(h, dtype=torch.float32, device=dY.device)
        column_sum(dY, nV, h, dbo)
    return dWo, dbo


TC, X3, SIMT = "tc", "x3", "simt"     # GEMM families: bf16 tensor cores, 3xTF32 tensor cores, f32 FMA pipes


@dataclass(frozen=True)
class Plan:
    """How one message-passing call runs (see `plan`)."""
    gemm: str | None           # TC, X3 or SIMT
    fused: bool                # the depth loop runs on the fused step
    forward: object            # (lay, V, E, W_i, b_i, W_h, b_h, W_o, b_o, cfg, plan, ...) -> (H_v, saved)
    mirror: object             # (lay, V, E, W_i, W_h, W_o, cfg, plan, saved, gH_v, need_bias, ...) -> six gradients
    dropout_ok: bool = False   # training-mode dropout can stay on this path (bond kinds)
    reason: str | None = None  # mol-atom-bond kinds: why the bf16 path does not apply (None: it does)


@dataclass(frozen=True)
class Rows:
    """The operand [X1[idx1] || X2[idx2]] of a SIMT GEMM, read in place by dmpnn_linear_fwd / _wgrad: X1 gives its first
    X1.shape[1] columns, X2 the rest of the GEMM's K (an index None: rows in order)."""
    X1: Tensor
    idx1: Tensor | None = None
    X2: Tensor | None = None
    idx2: Tensor | None = None


def _sources(A, K: int) -> tuple:
    """(X1, K1, the two-source keywords) of a SIMT operand: a Rows, or a tensor whose first K columns are the operand."""
    if isinstance(A, Rows):
        K1 = A.X1.shape[1]
        return A.X1, K1, dict(idx1=A.idx1, X2=A.X2, K2=K - K1, idx2=A.idx2)
    return A, K, {}


class _Gemm:
    """The GEMM family of Plan.gemm == SIMT (f32 FMA pipes), and the interface of all three: what the generic bond path
    (bond_forward / bond_backward) and composed.GatherLinear need to state each GEMM once.  A family owns its kernels'
    argument order and padding rules, its weight image, its operand formats, its output buffers and where its bias gradient
    comes from.  Methods call the op wrappers through the module globals at call time (the tests substitute them)."""
    timer = None      # _StepTimer tag of the unfused depth step's W_h GEMM

    def pack(self, W: Tensor, transpose: bool = False):
        """The weight image of W (N x K), or with `transpose` of a K x N matrix used as B[n][k] = W[k][n]."""
        return W.t().contiguous() if transpose else W

    def product(self, A, K: int, Wp, N: int, out: Tensor, *, pad_to: int | None = None, **epilogue):
        """out[:R, :N] = act(A[:, :K] . W^T + bias + res), columns [N, pad_to) zeroed; `epilogue`: R, bias, res, act and
        act_param of the op wrappers."""
        X1, K1, src = _sources(A, K)
        linear_fwd(X1, K1, Wp, out, N, **src, pad_to=pad_to, **epilogue)

    def wgrad(self, dY: Tensor, X, R: int, N: int, K: int, dW: Tensor, db: Tensor | None = None, accumulate: bool = False):
        """dW (+)= dY[:R, :N]^T . X[:R, :K] and, with `db`, db (+)= the column sums of dY."""
        X1, K1, src = _sources(X, K)
        linear_wgrad(dY, X1, K1, dW, N, **src, dbias=db, accumulate=accumulate, R=R)

    def hidden(self, rows: int, hp: int, dtype, dev) -> Tensor:
        """A hidden-width (hp columns) GEMM output."""
        return _hidden(rows, hp, dtype, dev)

    def output(self, rows: int, N: int, dtype, dev) -> tuple:
        """(the read-out GEMM's output buffer, H_v: its rows [0, rows) and first N columns)."""
        out = torch.empty((rows, N), dtype=dtype, device=dev)
        return out, out

    def wi_operand(self, V: Tensor, E: Tensor, lay: Layout):
        """W_i's operand [V[src] || E] over the dst-sorted edge rows (mixins.py:8-9)."""
        return Rows(V, lay.src_row, E, lay.perm)

    def wo_operand(self, lay: Layout, V: Tensor, Hprev: Tensor, first: bool, h: int, cfg: MPConfig, ones: bool) -> tuple:
        """(W_o's operand [V || M_v], M_v = sum_{dst(e)=v} H[e] of Hprev, tau applied on load when `first` (base.py:180,
        208-211); the operand's ones column or None).  `ones` asks for a ones column when the family takes one."""
        Mv = _hidden(lay.V, pad_hidden(h), cfg.hidden_dtype, V.device)
        segment_sum(Hprev, lay.rowptr, lay.V, h, Mv, act=(cfg.act if first else ACT_NONE), act_param=cfg.act_param,
                    pad_to=Mv.shape[1])
        return Rows(V, X2=Mv), None


class _X3Gemm(_Gemm):
    """Plan.gemm == X3: 3xTF32 on the tensor cores (f32-accurate); every dimension a multiple of 4 (16-byte rows), the
    operands materialised in f32."""
    timer = "x3_gemm"

    def pack(self, W: Tensor, transpose: bool = False):
        return pack_weight_x3(W, transpose=transpose)

    def product(self, A, K: int, Wp, N: int, out: Tensor, *, pad_to: int | None = None, **epilogue):
        # A carries zero columns up to the next multiple of 4 (wi_operand)
        linear_x3(A, (K + 3) // 4 * 4, Wp, N, out, pad_to=pad_to, **epilogue)

    def wgrad(self, dY: Tensor, X, R: int, N: int, K: int, dW: Tensor, db: Tensor | None = None, accumulate: bool = False):
        K4 = (K + 3) // 4 * 4       # W_i's operand: dW computed over its zero padding columns, then copied out
        dW4 = dW if K4 == K else torch.empty((N, K4), dtype=torch.float32, device=dW.device)
        wgrad_x3(dY, X, R, N, K4, dW4, accumulate=accumulate)
        if dW4 is not dW:
            dW.copy_(dW4[:, :K])
        if db is not None:
            column_sum(dY, R, N, db, accumulate=accumulate)

    def wi_operand(self, V: Tensor, E: Tensor, lay: Layout):
        d_v, d_e = V.shape[1], E.shape[1]
        X0 = torch.empty((lay.E, (d_v + d_e + 3) // 4 * 4), dtype=torch.float32, device=V.device)
        concat_f32(V, d_v, X0, lay.E, idx1=lay.src_row, X2=E, K2=d_e, idx2=lay.perm)
        return X0

    def wo_operand(self, lay: Layout, V: Tensor, Hprev: Tensor, first: bool, h: int, cfg: MPConfig, ones: bool) -> tuple:
        # the torch.cat of base.py:180 assembled once: V copied in, M_v written in place by the segment sum
        d_v = V.shape[1]
        XO = torch.empty((lay.V, d_v + h), dtype=cfg.hidden_dtype, device=V.device)
        XO[:, :d_v].copy_(V)
        segment_sum(Hprev, lay.rowptr, lay.V, h, XO[:, d_v:], act=(cfg.act if first else ACT_NONE), act_param=cfg.act_param,
                    pad_to=h)
        return XO, None


class _TcGemm(_Gemm):
    """Plan.gemm == TC: bf16 operands on the tensor cores, f32 accumulate; its epilogues store pad16(N) columns."""

    def pack(self, W: Tensor, transpose: bool = False):
        return pack_weight_tc(W, transpose=transpose)

    def product(self, A, K: int, Wp, N: int, out: Tensor, *, pad_to: int | None = None, **epilogue):
        linear_tc(A, K, Wp, N, out, **epilogue)

    def wgrad(self, dY: Tensor, X, R: int, N: int, K: int, dW: Tensor, db: Tensor | None = None, accumulate: bool = False):
        dYb = dY
        if dY.dtype == torch.float32:      # an f32 accumulator (dH_0): the GEMM takes its bf16 image, the bias its f32 sums
            dYb = torch.empty((R, dY.shape[1]), dtype=torch.bfloat16, device=dY.device)
            concat_bf16(dY, N, dYb, R)
        wgrad_tc(dYb, X, R, N, K, dW, accumulate=accumulate)
        if db is not None:
            column_sum(dY, R, N, db, accumulate=accumulate)

    def hidden(self, rows: int, hp: int, dtype, dev) -> Tensor:
        return _empty_hidden(rows, hp, dtype, dev)

    def output(self, rows: int, N: int, dtype, dev) -> tuple:
        out = _empty_hidden(rows, pad_hidden(N), dtype, dev)
        return out, out[:rows, :N]

    def wi_operand(self, V: Tensor, E: Tensor, lay: Layout):
        d_v, d_e = V.shape[1], E.shape[1]
        X0 = torch.empty((lay.E, (d_v + d_e + 15) // 16 * 16), dtype=torch.bfloat16, device=V.device)
        concat_bf16(V, d_v, X0, lay.E, idx1=lay.src_row, X2=E, K2=d_e, idx2=lay.perm)
        return X0

    def wo_operand(self, lay: Layout, V: Tensor, Hprev: Tensor, first: bool, h: int, cfg: MPConfig, ones: bool) -> tuple:
        return _readout_operand(lay, V, Hprev, first, h, cfg, None, V.shape[1], ones)


GEMMS = {TC: _TcGemm(), X3: _X3Gemm(), SIMT: _Gemm()}     # the family of each Plan.gemm value


def plan(kind: str, cfg: MPConfig, lay: Layout | None, h: int, d_v: int, d_e: int) -> Plan:
    """The execution path of one message-passing call.  `kind`: "bond" / "atom" (Bond / AtomMPFunction and the export op's
    bonds), "mab_bond" / "mab_atom" (MABMPFunction), "export_atom" (the export op's atoms: never on the fused atom step).
    The only place that knows the kernels' limits, and the only one that warns, once per process and reason, when a bf16
    call leaves a fast path.  `lay` None (mol-atom-bond kinds): only `reason` is filled in, the eligibility of a module
    before it sees a batch."""
    reason = None
    if kind in ("mab_bond", "mab_atom"):
        Ks = (d_v + d_e, d_v + h, d_e + h) if kind == "mab_bond" else (d_v, h + d_e, d_v + h, d_e + h)   # + W_eo's K
        reason = (f"d_h = {h} > {MAX_TC_HIDDEN}" if h > MAX_TC_HIDDEN else f"d_h = {h} not a multiple of 4" if h % 4 != 0 else
                  "d_e = 0" if d_e == 0 else f"GEMM inner dimensions {Ks} above {MAX_TC_K}" if max(Ks) > MAX_TC_K else
                  "tensor-core kernels unavailable" if not _fused_available() else None)
        if lay is None:
            return Plan(None, False, None, None, reason=reason)
    bond = kind in ("bond", "mab_bond")
    bf16 = cfg.fused and cfg.hidden_dtype == torch.bfloat16
    Ks = (d_v + d_e, d_v + h) if bond else (d_v, h + d_e, d_v + h)
    tc = bf16 and h <= MAX_TC_HIDDEN and max(Ks) <= MAX_TC_K and _fused_available()
    # Training-mode dropout stays on the fused bf16 path (dropout_ok) for ReLU on directed bonds -- tau' of the post-dropout
    # state is the keep mask times tau' of the pre-dropout one, so no mask is stored and 1 / (1 - p) folds into the mirror's
    # packed weights -- with every GEMM on the tensor cores and every depth step fused.  Of a bond call with dropout only the
    # GEMM limits are warned about, and only when they alone keep it off that path (it then runs on the composed tier).
    # A forward-only call (cfg.forward_only: Monte Carlo dropout) stores no mask for a mirror, so its dropout runs wherever the
    # call would run without it: keep bits in every fused bond step, dmpnn_scale_mask everywhere else (bond_forward).
    train_drop = cfg.dropout_p > 0 and not cfg.forward_only
    drop_shape = cfg.act == ACT_RELU and not cfg.undirected and lay.E > 0 and h % 4 == 0
    if not tc and bf16 and not (bond and train_drop and not drop_shape) and _fused_available():
        _warn_once("tc_limits", f"chemprop_b200: precision='bf16' with d_h = {h}, GEMM inner dimensions {Ks}: outside the "
                   f"tensor-core kernels' limits (d_h <= {MAX_TC_HIDDEN}, d_v + d_e and d_v + d_h <= {MAX_TC_K}); the linear "
                   "layers run on the f32 FMA pipes with bf16 storage (the fp32 tier's 3xTF32 tensor-core GEMMs take d_h up "
                   f"to {MAX_X3_DIM})")
    if bond:
        # fp32 tier on the tensor cores: every GEMM dimension a multiple of 4 (16-byte operand rows), atoms to run on
        x3 = (X3_ENABLED and cfg.fused and cfg.hidden_dtype == torch.float32 and lay.V > 0
              and all(d % 4 == 0 and 0 < d <= MAX_X3_DIM for d in (h, d_v + h)) and _fused_available())
        # the fused depth step: molecules of any size (those with more than 128 directed edges run as 128-row windows,
        # Layout.step_tables); undirected bonds too, the reverse-edge average being a prologue pass (bond_forward)
        step = (bf16 and h <= MAX_TC_HIDDEN and lay.E > 0 and (not cfg.undirected or (UNDIRECTED_FUSED and h % 4 == 0))
                and _fused_available())
        if cfg.depth > 1 and not step and bf16 and lay.E > 0 and not train_drop:
            why = (f"d_h = {h} > {MAX_TC_HIDDEN}" if h > MAX_TC_HIDDEN else
                   "undirected=True with d_h % 4 != 0" if cfg.undirected else "kernel unavailable")
            _warn_once("unfused", f"chemprop_b200: this batch leaves the fused depth-step kernel ({why}): the depth loop runs "
                       "as separate message + GEMM launches")
        fused = cfg.depth > 1 and step
        # the tensor-core mirror needs the fused forward's saved M^1 and X_0: directed, edges, d_h % 4 == 0; otherwise the
        # generic mirror (which recomputes the M^t the fused forward did not keep)
        tc_mirror = kind == "mab_bond" or (tc and not cfg.undirected and lay.E > 0 and h % 4 == 0)
        return Plan(TC if tc else X3 if x3 else SIMT, fused, bond_forward, bond_backward_tc if tc_mirror else bond_backward,
                    dropout_ok=drop_shape and tc and (cfg.depth == 1 or fused), reason=reason)
    # atoms: the tensor-core path needs d_h % 4 == 0 and atoms to run on; a mol-atom-bond call is on it by `reason`
    atom_tc = tc and h % 4 == 0
    on_tc = kind == "mab_atom" or (atom_tc and lay.V > 0)
    fused = False
    if on_tc and kind != "export_atom":
        # the fused atom step: directed, depth > 1, no training dropout, and every molecule within one atom tile (a tile is a
        # run of whole molecules: max_tile_atoms exceeds the tile only for a single oversized molecule)
        fused = (ATOM_FUSED_ENABLED and cfg.depth > 1 and not cfg.undirected and cfg.dropout_p == 0 and lay.V > 0 and lay.E > 0
                 and atom_tc and lay.max_tile_atoms <= ATOM_TILE_ATOMS)
        if not fused and ATOM_FUSED_ENABLED and cfg.depth > 1 and lay.E > 0 and atom_tc:
            why = ("undirected=True" if cfg.undirected else "training dropout" if cfg.dropout_p > 0 else
                   f"a molecule with more than {ATOM_TILE_ATOMS} atoms")
            _warn_once("atom_unfused", f"chemprop_b200: this batch leaves the fused atom depth step ({why}): neighbour sum and "
                       "GEMM run as separate launches")
    if fused:
        return Plan(TC, True, atom_forward_fused, atom_backward_fused, reason=reason)
    if on_tc:
        return Plan(TC, False, atom_forward_tc, atom_backward_tc, reason=reason)
    return Plan(SIMT, False, atom_forward, atom_backward, reason=reason)


def bond_forward(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, bi, Wh: Tensor, bh, Wo: Tensor | None, bo,
                 cfg: MPConfig, path: Plan, for_backward: bool = False, readout_f32: bool = False):
    """BondMessagePassing.forward up to W_o (chemprop/nn/message_passing/base.py:196-212 with
    mixins.py:8-18 and base.py:135-141, 180-182) on `path`.  Returns (H_v, saved-for-backward).  `Wo` None: the
    depth loop only (H_v None); `readout_f32` (tensor-core path): the W_o epilogue stores H_v in f32."""
    dev = V.device
    h = Wh.shape[0]
    hp = pad_hidden(h)
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nE, nV = lay.E, lay.V
    a, ap = cfg.act, cfg.act_param
    gemm = GEMMS[path.gemm]
    egemm = gemm if nE > 0 else GEMMS[SIMT]    # the edge GEMMs of a batch without edges: empty launches of the SIMT kernel
    # H_0 = W_i([V[src] || E])   (mixins.py:8-9); rows in dst-sorted order.  The operand serves the W_i gradient too
    X0 = egemm.wi_operand(V, E, lay)
    H0 = egemm.hidden(nE, hp, T, dev)
    egemm.product(X0, d_v + d_e, egemm.pack(Wi), h, H0, R=nE, bias=bi, pad_to=hp)
    Hs, Ms, Hbars = [], [], []
    Hprev, first = H0, True  # H^0 = tau(H_0) is applied on load (base.py:200)
    use_fused = path.fused
    Wpk = pack_weight_bf16(Wh) if use_fused else None
    # off the fused kernel the W_h GEMM takes the H_0 residual, bias and tau in its epilogue
    Whp = egemm.pack(Wh) if (not use_fused and cfg.depth > 1) else None
    for _ in range(1, cfg.depth):
        if use_fused:
            Hn = _empty_hidden(nE, hp, T, dev)
            src_in, first_in = Hprev, first
            if cfg.undirected:
                # H~ = (H + H[rev]) / 2 (base.py:202-203) as a prologue pass; the first step's tau(H_0) is applied by it, so the
                # fused step always sees an activation.  H~^{t-1} is kept: it is the right factor of this step's W_h
                # gradient (dZ^T . M^t = ((S.P) dZ)^T . H~^{t-1}, bond_backward).  Zero-filled: the step's TMA boxes read
                # the padding columns up to the 64-column slab edge
                Hbar = _hidden(nE, hp, T, dev)
                rev_average(Hprev, lay, h, Hbar, act=(a if first else ACT_NONE), act_param=ap)
                Hbars.append(Hbar)
                src_in, first_in = Hbar, False
            # training: the first step also stores M^1 (it is tau(H_0)-gathered, which no later kernel can rebuild
            # from a stored activation); the later steps' W_h gradients use (S.P) dZ from the backward kernel instead
            M1 = _empty_hidden(nE, hp, T, dev) if (first_in and for_backward) else None
            # base.py:139 (active dropout): keep bits from Philox, applied in the step's epilogue -- no pass over E x h
            bits = dropout_keep_bits(nE, h, cfg, Hn) if cfg.dropout_p > 0 else None
            with _StepTimer("fused_first" if first else "fused"):
                bond_step_fused(src_in, H0, Hn, h, Wpk, bh, lay, a, ap, first_in, M_out=M1, drop_bits=bits,
                                drop_scale=1.0 / (1.0 - cfg.dropout_p) if bits is not None else 1.0)
            Ms.append(M1)
        else:
            if cfg.dropout_p > 0 and not cfg.forward_only:
                raise DmpnnError("training-mode dropout on the monolithic tier needs the fused depth step (see Plan.dropout_ok)")
            src_in, fa = Hprev, (a if first else ACT_NONE)
            if cfg.undirected:  # H = (H + H[rev]) / 2   (base.py:202-203)
                Hbar = _hidden(nE, hp, T, dev)
                rev_average(src_in, lay, h, Hbar, act=fa, act_param=ap)
                Hbars.append(Hbar)
                src_in, fa = Hbar, ACT_NONE
            M = _hidden(nE, hp, T, dev)
            Hn = _hidden(nE, hp, T, dev)
            with _StepTimer("unfused_first" if first else "unfused"):
                bond_message(src_in, lay, h, M, act=fa, act_param=ap)           # mixins.py:11-18
                with _StepTimer(egemm.timer):
                    egemm.product(M, h, Whp, h, Hn, R=nE, bias=bh, res=H0, act=a, act_param=ap, pad_to=hp)  # base.py:135-141
                if cfg.dropout_p > 0:
                    _dropout_(Hn, cfg)                                                 # base.py:139
            Ms.append(M)
        Hs.append(Hn)
        Hprev, first = Hn, False
    XO = Hv = ones_col = None
    if Wo is not None:
        if cfg.dropout_p > 0 and path.gemm != TC and not cfg.forward_only:
            raise DmpnnError("training-mode dropout on the monolithic tier needs the tensor-core path (see Plan.dropout_ok)")
        # H_v = tau(W_o([V || M_v]))   (base.py:180-182)
        XO, ones_col = gemm.wo_operand(lay, V, Hprev, first, h, cfg, for_backward and bo is not None)
        if readout_f32:
            Hv = torch.empty((max(nV, 1), h), dtype=torch.float32, device=dev)[:nV]
            linear_tc_rows(XO, d_v + h, pack_weight_tc(Wo), h, Hv, R=nV, bias=bo, act=a, act_param=ap)
            if cfg.dropout_p > 0 and nV > 0:
                _dropout_(Hv, cfg)                                                     # mol_atom_bond.py vertex_finalize
        else:
            Hvp, Hv = gemm.output(nV, h, T, dev)
            gemm.product(XO, d_v + h, gemm.pack(Wo), h, Hvp, R=nV, bias=bo, act=a, act_param=ap, pad_to=h)
            if cfg.dropout_p > 0:
                _dropout_(Hvp, cfg)                                                    # base.py:182
    saved = dict(H0=H0, Hs=Hs, Ms=Ms, Hbars=Hbars, Hv=Hv, X0=X0, XO=XO, dvp=d_v, ones_col=ones_col)
    return Hv, saved


def bond_backward(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, Wh: Tensor, Wo: Tensor, cfg: MPConfig, path: Plan,
                  saved: dict, gHv: Tensor, need_bias: tuple[bool, bool, bool]):
    """Hand-written autograd mirror (SURVEY.md 8a-7) of bond_forward on `path`.  Returns
    (dWi, dbi, dWh, dbh, dWo, dbo)."""
    dev = V.device
    h = Wh.shape[0]
    hp = pad_hidden(h)
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nE, nV = lay.E, lay.V
    a, ap = cfg.act, cfg.act_param
    H0, Hs, Ms, Hbars, Hv = saved["H0"], saved["Hs"], saved["Ms"], saved["Hbars"], saved["Hv"]
    f32 = dict(dtype=torch.float32, device=dev)
    dWi = torch.zeros_like(Wi, dtype=torch.float32)
    dWh = torch.zeros_like(Wh, dtype=torch.float32)
    dWo = torch.zeros_like(Wo, dtype=torch.float32)
    dbi = torch.zeros(h, **f32) if need_bias[0] else None
    dbh = torch.zeros(h, **f32) if need_bias[1] else None
    dbo = torch.zeros(h, **f32) if need_bias[2] else None
    gemm = GEMMS[path.gemm]
    if gHv.stride(1) != 1:
        gHv = gHv.contiguous()
    # readout: dY = g * tau'(Y); dW_o = dY^T [V || M_v]; dM_v = dY . W_o[:, d_v:]
    dY = _hidden(nV, hp, T, dev)
    act_bwd(gHv, Hv, nV, h, act=a, act_param=ap, dZ=dY)
    gemm.wgrad(dY, saved["XO"], nV, h, d_v + h, dWo, dbo)
    dMv = gemm.hidden(nV, hp, T, dev)
    gemm.product(dY, h, gemm.pack(Wo[:, d_v:], transpose=True), h, dMv, R=nV, pad_to=hp)
    dH0 = torch.zeros((max(nE, 1), hp), **f32)  # f32 accumulator of dH_0 over all depth steps
    if nE > 0:
        if cfg.depth == 1:
            # dH^0[e] = dM_v[dst(e)];  dH_0 = dH^0 * tau'(H_0)
            act_bwd(dMv, H0, nE, h, act=a, act_param=ap, gidx=lay.dst_row, from_preact=True, acc=dH0)
        else:
            WhT = gemm.pack(Wh, transpose=True)
            dZ = _hidden(nE, hp, T, dev)
            act_bwd(dMv, Hs[-1], nE, h, act=a, act_param=ap, gidx=lay.dst_row, dZ=dZ, acc=dH0)
            # undirected steps that ran on the fused kernel (they saved no M^t): their mirror on the fused kernel too
            fused_undirected = cfg.undirected and path.fused and path.gemm == TC
            WhT_f = pack_weight_bf16(Wh.t().contiguous()) if fused_undirected else None
            for t in range(cfg.depth - 1, 0, -1):
                # inputs of step t: Hin = H^{t-1} (or tau(H_0) when t == 1)
                first = t == 1
                Hin = H0 if first else Hs[t - 2]
                if fused_undirected:
                    # dH~^{t-1} = (S.P)(dZ . W_h) = ((S.P) dZ) . W_h, unmasked; the gathered operand G = (S.P) dZ is the left
                    # factor of the W_h gradient (dZ^T . M^t = G^T . H~^{t-1}, H~^{t-1} saved by the forward's prologue)
                    if dbh is not None:
                        column_sum(dZ, nE, h, dbh, accumulate=True)
                    G = _empty_hidden(nE, hp, T, dev)
                    dHbar = _empty_hidden(nE, hp, T, dev)
                    bond_step_bwd_fused(dZ, None, dHbar, h, WhT_f, lay, a, ap, G_out=G)
                    wgrad_tc(G, Hbars[t - 1], nE, h, h, dWh, accumulate=True)
                    dHin = _hidden(nE, hp, T, dev)
                    rev_average(dHbar, lay, h, dHin)
                else:
                    M = Ms[t - 1]
                    if M is None:  # fused forward did not materialise M^t: recompute it
                        M = _hidden(nE, hp, T, dev)
                        if cfg.undirected:
                            bond_message(Hbars[t - 1], lay, h, M)
                        else:
                            bond_message(Hin, lay, h, M, act=(a if first else ACT_NONE), act_param=ap)
                    gemm.wgrad(dZ, M, nE, h, h, dWh, dbh, accumulate=True)
                    dM = gemm.hidden(nE, hp, T, dev)
                    gemm.product(dZ, h, WhT, h, dM, R=nE, pad_to=hp)
                    dHin = _hidden(nE, hp, T, dev)
                    bond_message(dM, lay, h, dHin, permute_on_read=True)
                    if cfg.undirected:
                        tmp = _hidden(nE, hp, T, dev)
                        rev_average(dHin, lay, h, tmp)
                        dHin = tmp
                if first:
                    act_bwd(dHin, H0, nE, h, act=a, act_param=ap, from_preact=True, acc=dH0)
                else:
                    dZ = _hidden(nE, hp, T, dev)
                    act_bwd(dHin, Hin, nE, h, act=a, act_param=ap, dZ=dZ, acc=dH0)
        gemm.wgrad(dH0, saved["X0"], nE, h, d_v + d_e, dWi, dbi)
    return dWi, dbi, dWh, dbh, dWo, dbo


def bond_backward_tc(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, Wh: Tensor, Wo: Tensor, cfg: MPConfig, path: Plan,
                     saved: dict, gHv: Tensor | None, need_bias: tuple[bool, bool, bool], entry=None):
    """bf16-tier autograd mirror of bond_forward on the fused depth step (directed bonds).  Differences from the generic
    mirror: every GEMM is on the tensor cores (wgmma); each depth step's mirror is one launch of the fused kernel (_fused_mirror);
    dH_0 is never formed -- its terms stay in bf16 and are contracted with X_0 by one multi-term weight-gradient launch.
    `gHv` None: no read-out (dW_o, db_o None).  `entry(dMv, Y, from_preact, out)` (the mol-atom-bond edge head) replaces the
    pass that starts the loop, out = dM_v[dst(r)] * tau'(Y[r]): it writes out = (its own term + dM_v[dst(r)]) * tau'(Y[r]),
    dMv None when there is no read-out."""
    dev = V.device
    h = Wh.shape[0]
    hp = pad_hidden(h)
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nE, nV = lay.E, lay.V
    a, ap = cfg.act, cfg.act_param
    # pure streaming passes run over the 16-padded width (16-byte vectors; padding columns only ever feed
    # consumers that clip at h); the gather kernels keep 8-byte lanes (75 of 96 lanes busy beats 38 of 64)
    hc = (h + 15) // 16 * 16
    H0, Hs, Hv = saved["H0"], saved["Hs"], saved["Hv"]
    f32 = dict(dtype=torch.float32, device=dev)
    # every weight gradient is WRITTEN by its first GEMM (no zero fill + accumulate); zeros only where no GEMM runs
    no_e = nE == 0
    dWi = torch.zeros_like(Wi, dtype=torch.float32) if no_e else torch.empty_like(Wi, dtype=torch.float32)
    dWh = torch.zeros_like(Wh, dtype=torch.float32) if (no_e or cfg.depth == 1) else torch.empty_like(Wh, dtype=torch.float32)
    dWo = dbo = None
    dbi = torch.zeros(h, **f32) if need_bias[0] else None
    dbh = torch.zeros(h, **f32) if need_bias[1] else None
    # Training-mode dropout (cfg.dropout_p > 0; ReLU only, Plan.dropout_ok): a gradient that crosses a dropout site is
    # multiplied by the keep mask and by s = 1 / (1 - p).  With ReLU the mask is already in tau' of the stored POST-dropout
    # state ([H_post > 0] = mask * [H_pre > 0]), and s, a scalar, folds into the packed weight of the GEMM that produces
    # the gradient arriving at the site (or, for W_o's own gradient, into the result).
    s_drop = 1.0 / (1.0 - cfg.dropout_p) if cfg.dropout_p > 0 else 1.0
    s_v = s_drop                                      # site after W_o (base.py:182)
    s_e = s_drop if cfg.depth > 1 else 1.0            # site on H^{T-1} (base.py:139); H^0 = tau(H_0) has none
    if gHv is not None:
        if gHv.stride(1) != 1:
            gHv = gHv.contiguous()
        dY = _empty_hidden(nV, hp, T, dev)
        act_bwd(gHv, Hv, nV, h, act=a, act_param=ap, dZ=dY)      # dY / s_v
        dWo, dbo = _readout_grads(dY, saved, nV, h, d_v, need_bias[2])
        if s_v != 1.0:
            dWo.mul_(s_v)
            if dbo is not None:
                dbo.mul_(s_v)
    if nE == 0:
        return dWi, dbi, dWh, dbh, dWo, dbo
    dMv = None
    if gHv is not None:
        dMv = _empty_hidden(nV, hp, T, dev)
        Wo_m = Wo[:, d_v:] if s_v * s_e == 1.0 else Wo[:, d_v:] * (s_v * s_e)
        linear_tc(dY, h, pack_weight_tc(Wo_m, transpose=True), h, dMv, R=nV)
    if cfg.depth == 1:
        dH0b = _empty_hidden(nE, hp, T, dev)
        if entry is not None:
            entry(dMv, H0, True, dH0b)
        else:
            act_bwd(dMv, H0, nE, hc, act=a, act_param=ap, gidx=lay.dst_row, from_preact=True, dZ=dH0b)
        terms = [dH0b]
    else:
        WhT = pack_weight_bf16(Wh.t().contiguous())
        # mirror steps whose result arrives at a dropout site (every one but the last, which lands on H^0) carry s
        WhT_s = WhT if s_drop == 1.0 else pack_weight_bf16((Wh * s_drop).t().contiguous())
        dZ = _empty_hidden(nE, hp, T, dev)
        if entry is not None:
            entry(dMv, Hs[-1], False, dZ)
        else:
            act_bwd(dMv, Hs[-1], nE, hc, act=a, act_param=ap, gidx=lay.dst_row, dZ=dZ)    # dZ^{T-1}
        M1 = saved["Ms"][0]
        assert M1 is not None, "M^1 is saved by the fused forward step whenever a weight needs a gradient"
        terms = _fused_mirror(bond_step_bwd_fused, dZ, H0, Hs, M1, WhT, WhT_s, dWh, dbh, nE, h, lay, cfg)
    # dH_0 = sum_t dZ^t + dH^0 * tau'(H_0) is only ever contracted with X_0 (and summed for the bias): the terms stay apart and
    # the W_i gradient takes them all in one weight-gradient launch (X_0 read once), instead of a summing pass over E x h
    wgrad_tc_multi(terms, saved["X0"], nE, h, d_v + d_e, dWi)
    if dbi is not None:
        for i, P in enumerate(terms):
            column_sum(P, nE, h, dbi, accumulate=i > 0)
    return dWi, dbi, dWh, dbh, dWo, dbo


def _fused_mirror(step, dZ: Tensor, H0: Tensor, Hs: list, first_op: Tensor, WT1: Tensor, WT: Tensor, dWh: Tensor,
                  dbh: Tensor | None, R: int, h: int, lay: Layout, cfg: MPConfig) -> list:
    """The depth loop of the fused bf16 mirrors (DESIGN.md section 5), bonds and atoms alike.  `step` is the mirror mode of the
    fused depth step (bond_step_bwd_fused / atom_step_bwd_fused): dH^{t-1} = (B dZ^t) . W_h [* tau'], B the sibling gather
    S.P of bonds or the adjacency A of atoms, with its gathered operand G^t = B dZ^t written out.  G^t is the left factor of the
    step's W_h gradient (dZ^T . M^t = G^T . H^{t-1}); t = 1 has no stored tau(H_0) and contracts dZ^1 with `first_op`, the M^1 /
    N^1 the forward saved.  `WT1` is the packed W_h^T of the t = 1 step, `WT` that of the others (for bonds it carries the
    dropout scale).  dW_h is written by its first GEMM, db_h accumulated.  From dZ = dZ^{T-1}, returns the dH_0 terms
    [dZ^{T-1}, ..., dZ^1, dH^0 * tau'(H_0)]."""
    a, ap = cfg.act, cfg.act_param
    hp, T, dev = pad_hidden(h), cfg.hidden_dtype, dZ.device
    terms = [dZ]
    for t in range(cfg.depth - 1, 0, -1):
        accumulate = t < cfg.depth - 1
        if dbh is not None:
            column_sum(dZ, R, h, dbh, accumulate=True)
        if t == 1:
            wgrad_tc(dZ, first_op, R, h, h, dWh, accumulate=accumulate)
            dH0 = _empty_hidden(R, hp, T, dev)
            step(dZ, H0, dH0, h, WT1, lay, a, ap, y_is_preact=True)                          # dH^0 * tau'(H_0)
            terms.append(dH0)
        else:
            Hin = Hs[t - 2]
            dZn = _empty_hidden(R, hp, T, dev)
            G = _empty_hidden(R, hp, T, dev)
            step(dZ, Hin, dZn, h, WT, lay, a, ap, G_out=G)                                   # dZ^{t-1}
            wgrad_tc(G, Hin, R, h, h, dWh, accumulate=accumulate)
            dZ = dZn
            terms.append(dZ)
    return terms


def _refuse_feature_grads(ctx):
    """The hand-written mirrors produce the six parameter gradients only.  chemprop never asks for d/dV or d/dE (features
    come out of the featuriser), but a caller who does (learned atom embeddings, input saliency) must not get a silent
    `None` where the reference's autograd would deliver a gradient."""
    if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
        raise DmpnnError(
            "bmg.V / bmg.E require grad: the engine's hand-written backward produces parameter gradients only "
            "(d/dV, d/dE are not implemented); detach the features, or use the reference module for input attribution")


def _mp_inputs(ctx, V: Tensor, E: Tensor, params: tuple) -> tuple:
    """Start of every message-passing Function's forward: CUDA tensors only, no feature gradients, and the features and the
    (weight, bias) pairs of `params` (None stays None) as f32 contiguous tensors detached from autograd.  Records on `ctx`
    which biases are present and the dtype of each parameter's gradient (its weight's)."""
    _require_cuda(V, E, *params[0::2])
    _refuse_feature_grads(ctx)
    ctx.has_bias = tuple(b is not None for b in params[1::2])
    ctx.gdtypes = tuple(None if w is None else w.dtype for w in params[0::2] for _ in range(2))
    f32 = lambda t: None if t is None else t.detach().contiguous().float()  # noqa: E731
    return V.contiguous().float(), E.contiguous().float(), [f32(t) for t in params]


def _mp_save(ctx, lay: Layout, cfg: MPConfig, path: Plan, V: Tensor, E: Tensor, W: tuple, saved: dict, Hv: Tensor | None):
    """What the mirror needs.  `Hv` is the tensor autograd turns into this node's output: keeping THAT object in ctx.saved
    would be a reference cycle (node -> saved -> Hv -> grad_fn = node) and the step's activations would live until Python's
    cyclic GC runs (GBs per step, cudaMalloc on every step); a detached alias shares the storage without the back edge."""
    saved["Hv"] = None if Hv is None else Hv.detach()
    ctx.lay, ctx.cfg, ctx.plan, ctx.saved, ctx.VE, ctx.W = lay, cfg, path, saved, (V, E), W


def _mp_grads(ctx, grads: tuple, n_after: int) -> tuple:
    """backward's return: None for V and E, the parameter gradients in their weights' dtypes, None for the `n_after`
    non-tensor inputs.  ctx.saved stays until autograd frees the node: a second backward (retain_graph=True) works like
    torch's own."""
    cast = tuple(None if (g is None or d is None) else g.to(d) for g, d in zip(grads, ctx.gdtypes))
    return (None, None) + cast + (None,) * n_after


class BondMPFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, V, E, Wi, bi, Wh, bh, Wo, bo, lay, cfg):
        V, E, (Wi, bi, Wh, bh, Wo, bo) = _mp_inputs(ctx, V, E, (Wi, bi, Wh, bh, Wo, bo))
        p = plan("bond", cfg, lay, Wh.shape[0], V.shape[1], E.shape[1])
        Hv, saved = p.forward(lay, V, E, Wi, bi, Wh, bh, Wo, bo, cfg, p, for_backward=any(ctx.needs_input_grad))
        _mp_save(ctx, lay, cfg, p, V, E, (Wi, Wh, Wo), saved, Hv)
        return Hv

    @staticmethod
    def backward(ctx, gHv):
        grads = ctx.plan.mirror(ctx.lay, *ctx.VE, *ctx.W, ctx.cfg, ctx.plan, ctx.saved, gHv, ctx.has_bias)
        return _mp_grads(ctx, grads, 2)


# ----------------------------------------------------------------------------------------------
# atom message passing (atom-granular: every edge row depends only on its source atom)
# ----------------------------------------------------------------------------------------------
def atom_forward(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, bi, Wh: Tensor, bh, Wo: Tensor, bo,
                 cfg: MPConfig, path: Plan):
    """AtomMessagePassing.forward up to W_o (base.py:196-212 with mixins.py:22-30), restated on atoms:
    the reference's H[e] equals Ha[src(e)], so M[e] = [sum_{u in N(src e)} Ha[u] || sum_in E]."""
    dev = V.device
    h = Wi.shape[0]
    hp = pad_hidden(h)
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nV = lay.V
    a, ap = cfg.act, cfg.act_param
    H0 = _hidden(nV, hp, T, dev)
    linear_fwd(V, d_v, Wi, H0, h, bias=bi, R=nV, pad_to=hp)                       # mixins.py:22-23
    SE = torch.zeros((max(nV, 1), max(d_e, 1)), dtype=torch.float32, device=dev)   # sum of in-edge bond features
    if d_e > 0:
        segment_sum(E, lay.rowptr, nV, d_e, SE, idx=lay.perm)
    Hs, Ns = [], []
    Hprev, first = H0, True
    for _ in range(1, cfg.depth):
        Nb = _hidden(nV, hp, T, dev)  # sum over in-neighbours u of Ha[u]   (mixins.py:25-30)
        segment_sum(Hprev, lay.rowptr, nV, h, Nb, idx=lay.src_row, act=(a if first else ACT_NONE), act_param=ap,
                    pad_to=hp)
        Hn = _hidden(nV, hp, T, dev)
        linear_fwd(Nb, h, Wh, Hn, h, X2=SE if d_e > 0 else None, K2=d_e, bias=bh, res=H0, act=a, act_param=ap,
                   R=nV, pad_to=hp)                                                  # base.py:135-141
        Hs.append(Hn)
        Ns.append(Nb)
        Hprev, first = Hn, False
    Mv = _hidden(nV, hp, T, dev)
    segment_sum(Hprev, lay.rowptr, nV, h, Mv, idx=lay.src_row, act=(a if first else ACT_NONE), act_param=ap,
                pad_to=hp)                                                           # base.py:208-211
    Hv = torch.empty((nV, h), dtype=T, device=dev)
    linear_fwd(V, d_v, Wo, Hv, h, X2=Mv, K2=h, bias=bo, act=a, act_param=ap, R=nV, pad_to=h)
    return Hv, dict(H0=H0, Hs=Hs, Ns=Ns, SE=SE, Mv=Mv, Hv=Hv)


def atom_backward(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, Wh: Tensor, Wo: Tensor, cfg: MPConfig, path: Plan,
                  saved: dict, gHv: Tensor, need_bias):
    dev = V.device
    h = Wi.shape[0]
    hp = pad_hidden(h)
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nV = lay.V
    a, ap = cfg.act, cfg.act_param
    H0, Hs, Ns, SE, Mv, Hv = saved["H0"], saved["Hs"], saved["Ns"], saved["SE"], saved["Mv"], saved["Hv"]
    f32 = dict(dtype=torch.float32, device=dev)
    dWi = torch.zeros_like(Wi, dtype=torch.float32)
    dWh = torch.zeros_like(Wh, dtype=torch.float32)
    dWo = torch.zeros_like(Wo, dtype=torch.float32)
    dbi = torch.zeros(h, **f32) if need_bias[0] else None
    dbh = torch.zeros(h, **f32) if need_bias[1] else None
    dbo = torch.zeros(h, **f32) if need_bias[2] else None
    gHv = gHv.contiguous()
    dY = _hidden(nV, hp, T, dev)
    act_bwd(gHv, Hv, nV, h, act=a, act_param=ap, dZ=dY)
    linear_wgrad(dY, V, d_v, dWo, h, X2=Mv, K2=h, dbias=dbo, R=nV)
    WoT = Wo[:, d_v:].t().contiguous()
    dMv = _hidden(nV, hp, T, dev)
    linear_fwd(dY, h, WoT, dMv, h, R=nV, pad_to=hp)
    # d(Ha^{T-1})[u] = sum_{e: src(e)=u} dM_v[dst(e)] = sum_{e' in in(u)} dM_v[src(e')]  (rev is an involution)
    dH0 = torch.zeros((max(nV, 1), hp), **f32)
    dHa = _hidden(nV, hp, T, dev)
    segment_sum(dMv, lay.rowptr, nV, h, dHa, idx=lay.src_row, pad_to=hp)
    WhT = Wh[:, :h].t().contiguous() if cfg.depth > 1 else None
    for t in range(cfg.depth - 1, 0, -1):
        first = t == 1
        dZ = _hidden(nV, hp, T, dev)
        act_bwd(dHa, Hs[t - 1], nV, h, act=a, act_param=ap, dZ=dZ, acc=dH0)
        linear_wgrad(dZ, Ns[t - 1], h, dWh, h, X2=SE if d_e > 0 else None, K2=d_e, dbias=dbh, accumulate=True, R=nV)
        dN = _hidden(nV, hp, T, dev)
        linear_fwd(dZ, h, WhT, dN, h, R=nV, pad_to=hp)
        dHa = _hidden(nV, hp, T, dev)
        segment_sum(dN, lay.rowptr, nV, h, dHa, idx=lay.src_row, pad_to=hp)
    act_bwd(dHa, H0, nV, h, act=a, act_param=ap, from_preact=True, acc=dH0)
    linear_wgrad(dH0, V, d_v, dWi, h, dbias=dbi, R=nV)
    return dWi, dbi, dWh, dbh, dWo, dbo


def _atom_readout_tc(lay: Layout, V: Tensor, Hprev: Tensor, first: bool, h: int, Wo: Tensor, bo, cfg: MPConfig, rows: int,
                     with_ones: bool, readout_f32: bool):
    """H_v = tau(W_o([V || M_v])) of the atom tiers (base.py:180-182, 208-211): returns (H_v, XO, dvp, ones_col).  `with_ones`:
    a ones column delivers db_o with dW_o's GEMM (_readout_operand)."""
    dev, T, nV = V.device, cfg.hidden_dtype, lay.V
    a, ap = cfg.act, cfg.act_param
    d_v = V.shape[1]
    dvp = _readout_pad(d_v, h)
    XO, ones_col = _readout_operand(lay, V, Hprev, first, h, cfg, lay.src_row, dvp, with_ones and bo is not None)
    Wpk = pack_weight_tc(_wo_padded(Wo, d_v, dvp))
    if readout_f32:
        Hv = torch.empty((rows, h), dtype=torch.float32, device=dev)[:nV]
        linear_tc_rows(XO, dvp + h, Wpk, h, Hv, R=nV, bias=bo, act=a, act_param=ap)
    else:
        Hvp = torch.empty((rows, pad_hidden(h)), dtype=T, device=dev)
        linear_tc(XO, dvp + h, Wpk, h, Hvp, bias=bo, act=a, act_param=ap, R=nV)         # base.py:180-182
        Hv = Hvp[:nV, :h]
    return Hv, XO, dvp, ones_col


def atom_forward_tc(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, bi, Wh: Tensor, bh, Wo: Tensor, bo, cfg: MPConfig,
                    path: Plan, readout_f32: bool = False):
    """bf16 tier of atom_forward on the tensor cores: every GEMM is dmpnn_linear_tc_bf16 (the H_0 residual of
    base.py:138 is added in its epilogue), the neighbour sums write straight into the GEMM's A operand.  `Wo` None: no
    read-out; `readout_f32`: H_v stored in f32."""
    dev = V.device
    h = Wi.shape[0]
    hp = pad_hidden(h)
    hc = (h + 15) // 16 * 16
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nV = lay.V
    a, ap = cfg.act, cfg.act_param
    rows = max(nV, 1)
    kv = (d_v + 15) // 16 * 16
    Xv = torch.empty((rows, kv), dtype=T, device=dev)
    concat_bf16(V, d_v, Xv, nV, width=kv)
    H0 = _empty_hidden(nV, hp, T, dev)
    linear_tc(Xv, d_v, pack_weight_tc(Wi), h, H0, bias=bi, R=nV)                              # mixins.py:22-23
    SE = None
    if d_e > 0:                                                                               # loop-invariant bond term
        SE = torch.zeros((rows, d_e), dtype=torch.float32, device=dev)
        segment_sum(E, lay.rowptr, nV, d_e, SE, idx=lay.perm)
    ka = (h + d_e + 15) // 16 * 16
    Whpk = pack_weight_tc(Wh) if cfg.depth > 1 else None
    Hs, XAs = [], []
    Hprev, first = H0, True
    for _ in range(1, cfg.depth):
        XA = torch.empty((rows, ka), dtype=T, device=dev)   # [sum_{u in N(v)} Ha[u] || sum_in E]   (mixins.py:25-30)
        with _StepTimer("atom_step_first" if first else "atom_step"):
            segment_sum(Hprev, lay.rowptr, nV, h, XA[:, :h], idx=lay.src_row, act=(a if first else ACT_NONE), act_param=ap,
                        pad_to=h)
            if d_e > 0:
                concat_bf16(SE, d_e, XA[:, h:], nV, width=d_e)
            Hn = _empty_hidden(nV, hp, T, dev)
            linear_tc(XA, h + d_e, Whpk, h, Hn, bias=bh, res=H0, act=a, act_param=ap, R=nV)   # base.py:135-141
        Hs.append(Hn)
        XAs.append(XA)
        Hprev, first = Hn, False
    Hv = XO = dvp = None
    if Wo is not None:
        Hv, XO, dvp, _ = _atom_readout_tc(lay, V, Hprev, first, h, Wo, bo, cfg, rows, False, readout_f32)
    return Hv, dict(H0=H0, Hs=Hs, XAs=XAs, XO=XO, Xv=Xv, Hv=Hv, dvp=dvp, ones_col=None)


def atom_backward_tc(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, Wh: Tensor, Wo: Tensor, cfg: MPConfig, path: Plan,
                     saved: dict, gHv: Tensor | None, need_bias, entry=None):
    """Autograd mirror of atom_forward_tc (wgmma GEMMs; dH_0 is kept as separate terms, one W_i GEMM each).  `gHv` None:
    no read-out.  `entry(dHa, Y, from_preact, out)` (the mol-atom-bond edge head) replaces the first tau' pass
    out = dHa * tau'(Y): it writes out = (its own term + dHa) * tau'(Y), dHa None when there is no read-out."""
    dev = V.device
    h = Wi.shape[0]
    hp = pad_hidden(h)
    hc = (h + 15) // 16 * 16
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nV = lay.V
    a, ap = cfg.act, cfg.act_param
    H0, Hs, XAs, Xv, Hv = saved["H0"], saved["Hs"], saved["XAs"], saved["Xv"], saved["Hv"]
    f32 = dict(dtype=torch.float32, device=dev)
    dWi = torch.zeros_like(Wi, dtype=torch.float32)
    dWh = torch.zeros_like(Wh, dtype=torch.float32)
    dWo = torch.zeros_like(Wo, dtype=torch.float32) if gHv is not None else None
    dbi = torch.zeros(h, **f32) if need_bias[0] else None
    dbh = torch.zeros(h, **f32) if need_bias[1] else None
    dbo = torch.zeros(h, **f32) if (need_bias[2] and gHv is not None) else None
    if nV == 0:
        return dWi, dbi, dWh, dbh, dWo, dbo
    dHa = None
    if gHv is not None:
        if gHv.stride(1) != 1:
            gHv = gHv.contiguous()
        dY = _empty_hidden(nV, hp, T, dev)
        act_bwd(gHv, Hv, nV, h, act=a, act_param=ap, dZ=dY)
        dWo, dbo = _readout_grads(dY, saved, nV, h, d_v, dbo is not None)
        dMv = _empty_hidden(nV, hp, T, dev)
        linear_tc(dY, h, pack_weight_tc(Wo[:, d_v:], transpose=True), h, dMv, R=nV)
        # d(Ha^{T-1})[u] = sum_{e' in in(u)} dM_v[src(e')]   (rev is an involution)
        dHa = _empty_hidden(nV, hp, T, dev)
        segment_sum(dMv, lay.rowptr, nV, h, dHa, idx=lay.src_row, pad_to=hc)
    WhT_pk = pack_weight_tc(Wh[:, :h], transpose=True) if cfg.depth > 1 else None
    terms = []
    for t in range(cfg.depth - 1, 0, -1):
        dZ = _empty_hidden(nV, hp, T, dev)
        if entry is not None and t == cfg.depth - 1:
            entry(dHa, Hs[t - 1], False, dZ)
        else:
            act_bwd(dHa, Hs[t - 1], nV, hc, act=a, act_param=ap, dZ=dZ)
        terms.append(dZ)
        wgrad_tc(dZ, XAs[t - 1], nV, h, h + d_e, dWh, accumulate=True)
        if dbh is not None:
            column_sum(dZ, nV, h, dbh, accumulate=True)
        dN = _empty_hidden(nV, hp, T, dev)
        linear_tc(dZ, h, WhT_pk, h, dN, R=nV)
        dHa = _empty_hidden(nV, hp, T, dev)
        segment_sum(dN, lay.rowptr, nV, h, dHa, idx=lay.src_row, pad_to=hc)
    dH0l = _empty_hidden(nV, hp, T, dev)
    if entry is not None and cfg.depth == 1:
        entry(dHa, H0, True, dH0l)
    else:
        act_bwd(dHa, H0, nV, hc, act=a, act_param=ap, from_preact=True, dZ=dH0l)
    terms.append(dH0l)
    wgrad_tc_multi(terms, Xv, nV, h, d_v, dWi)       # dH_0 = sum_t dZ^t + dHa^0 * tau'(H_0), contracted term by term
    if dbi is not None:
        for i, P in enumerate(terms):
            column_sum(P, nV, h, dbi, accumulate=i > 0)
    return dWi, dbi, dWh, dbh, dWo, dbo


def atom_forward_fused(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, bi, Wh: Tensor, bh, Wo: Tensor, bo, cfg: MPConfig,
                       path: Plan, readout_f32: bool = False):
    """bf16 tier of atom_forward with ONE launch per depth step (dmpnn_atom_step_fused_bf16).  The reference's update
    (base.py:135-141) on atoms is tau(H_0 + b_h + W_h . [N^t || SE]) with N^t the neighbour sum of the previous state and SE the
    loop-invariant sum of the incoming bond features: W_h[:, h:] . SE + b_h is added to H_0 ONCE (a K = d_e GEMM with H_0 as
    the residual of its epilogue), which gives the step the bond step's shape  tau(H_0' + W_h[:, :h] . N^t)  -- gather, GEMM
    and epilogue in the fused kernel, with the gathered operand of the first step saved for the W_h gradient."""
    dev = V.device
    h = Wi.shape[0]
    hp = pad_hidden(h)
    hc = (h + 15) // 16 * 16
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nV = lay.V
    a, ap = cfg.act, cfg.act_param
    rows = max(nV, 1)
    # [V || sum_in E] side by side in ONE bf16 operand (16-column blocks): W_i reads its first d_v columns, the H_0' GEMM the
    # second block, and the mirror contracts the dZ^t terms with both in one weight-gradient launch
    kv = (d_v + 15) // 16 * 16
    ke = (d_e + 15) // 16 * 16 if d_e > 0 else 0
    Xv = torch.empty((rows, kv + ke), dtype=T, device=dev)
    concat_bf16(V, d_v, Xv, nV, width=kv)
    H0 = _empty_hidden(nV, hp, T, dev)
    linear_tc(Xv, d_v, pack_weight_tc(Wi), h, H0, bias=bi, R=nV)                              # mixins.py:22-23
    SEb, H0p, step_bias = None, H0, bh
    if d_e > 0:                                                                               # loop-invariant bond term
        SE = torch.zeros((rows, d_e), dtype=torch.float32, device=dev)
        segment_sum(E, lay.rowptr, nV, d_e, SE, idx=lay.perm)
        SEb = Xv[:, kv:kv + ke]
        concat_bf16(SE, d_e, SEb, nV, width=ke)
        H0p = _empty_hidden(nV, hp, T, dev)                                                   # H_0 + b_h + W_h[:, h:] . SE
        linear_tc(SEb, d_e, pack_weight_tc(Wh[:, h:]), h, H0p, bias=bh, res=H0, R=nV)
        step_bias = None
    Whpk = pack_weight_bf16(Wh[:, :h].contiguous())
    Hs, N1 = [], None
    Hprev, first = H0, True
    for _ in range(1, cfg.depth):
        Hn = _empty_hidden(nV, hp, T, dev)
        if first:
            N1 = _empty_hidden(nV, hp, T, dev)
        with _StepTimer("atom_fused_first" if first else "atom_fused"):
            atom_step_fused(Hprev, H0p, Hn, h, Whpk, step_bias, lay, a, ap, first, N_out=N1 if first else None)
        Hs.append(Hn)
        Hprev, first = Hn, False
    Hv = XO = dvp = ones_col = None
    if Wo is not None:          # db_o rides on dW_o's GEMM (ones column)
        Hv, XO, dvp, ones_col = _atom_readout_tc(lay, V, Hprev, first, h, Wo, bo, cfg, rows, True, readout_f32)
    return Hv, dict(H0=H0, Hs=Hs, N1=N1, SEb=SEb, XO=XO, Xv=Xv, Hv=Hv, dvp=dvp, ones_col=ones_col)


def atom_backward_fused(lay: Layout, V: Tensor, E: Tensor, Wi: Tensor, Wh: Tensor, Wo: Tensor, cfg: MPConfig, path: Plan,
                        saved: dict, gHv: Tensor | None, need_bias, entry=None):
    """Autograd mirror of atom_forward_fused.  With A the (symmetric) atom adjacency, N^t = A H^{t-1}:
    dH^{t-1} = ((A dZ^t) . W_h[:, :h]) * tau'(H^{t-1}) -- the mirror mode of the fused kernel, whose gathered operand
    G^t = A dZ^t is also the left factor of the step's weight gradient (dZ^T . N^t = G^T . H^{t-1}); t = 1 uses the N^1 the
    forward saved.  dW_h[:, h:] = (sum_t dZ^t)^T . SE and dW_i = (sum_t dZ^t + dH^0 tau'(H_0))^T . V as multi-term GEMMs."""
    dev = V.device
    h = Wi.shape[0]
    hp = pad_hidden(h)
    hc = (h + 15) // 16 * 16
    d_v, d_e = V.shape[1], E.shape[1]
    T = cfg.hidden_dtype
    nV = lay.V
    a, ap = cfg.act, cfg.act_param
    H0, Hs, N1, Xv, Hv = (saved[k] for k in ("H0", "Hs", "N1", "Xv", "Hv"))
    f32 = dict(dtype=torch.float32, device=dev)
    dWi = torch.empty_like(Wi, dtype=torch.float32)
    dWh = torch.empty_like(Wh, dtype=torch.float32)
    dWo = dbo = None
    dbi = torch.zeros(h, **f32) if need_bias[0] else None
    dbh = torch.zeros(h, **f32) if need_bias[1] else None
    if gHv is not None:
        if gHv.stride(1) != 1:
            gHv = gHv.contiguous()
        dY = _empty_hidden(nV, hp, T, dev)
        act_bwd(gHv, Hv, nV, h, act=a, act_param=ap, dZ=dY)
        if hc > h:
            # act_bwd writes h columns; the fused mirror below reads dY up to pad16(h), where a NaN left by the allocator
            # would reach every output column through the zero rows of the packed weight (0 * NaN = NaN)
            dY[:, h:hc].zero_()
        dWo, dbo = _readout_grads(dY, saved, nV, h, d_v, need_bias[2])
    # dZ^{T-1} = (A (dY . W_o[:, d_v:])) * tau'(H^{T-1}) = ((A dY) . W_o[:, d_v:]) * tau'(H^{T-1}): the read-out GEMM, the
    # neighbour gather of its result and the tau' pass are ONE mirror launch of the fused kernel on dY (three launches before)
    if entry is None:
        dZ = _empty_hidden(nV, hp, T, dev)
        atom_step_bwd_fused(dY, Hs[-1], dZ, h, pack_weight_bf16(Wo[:, d_v:].t().contiguous()), lay, a, ap)
    else:
        # zero-filled: the entry writes columns up to pad16(h), the next mirror step's TMA boxes read up to the 64-column edge
        dZ = _hidden(nV, hp, T, dev)
        # `entry(dHa, Y, from_preact, out)` (mol-atom-bond edge head): the read-out's term unmasked, as in atom_backward_tc
        # (dM_v = dY . W_o[:, d_v:], then its neighbour sum); the entry adds its own term and applies tau'
        dHa = None
        if gHv is not None:
            dMv = _empty_hidden(nV, hp, T, dev)
            linear_tc(dY, h, pack_weight_tc(Wo[:, d_v:], transpose=True), h, dMv, R=nV)
            dHa = _empty_hidden(nV, hp, T, dev)
            segment_sum(dMv, lay.rowptr, nV, h, dHa, idx=lay.src_row, pad_to=hc)
        entry(dHa, Hs[-1], False, dZ)
    WhT = pack_weight_bf16(Wh[:, :h].t().contiguous())
    terms = _fused_mirror(atom_step_bwd_fused, dZ, H0, Hs, N1, WhT, WhT, dWh[:, :h], dbh, nV, h, lay, cfg)
    if d_e > 0:
        # one pass over the dZ^t terms for both [V || sum_in E] blocks of Xv, then the dH^0 term for the V block alone
        kv = (d_v + 15) // 16 * 16
        dWx = torch.empty((h, kv + d_e), **f32)
        wgrad_tc_multi(terms[:-1], Xv, nV, h, kv + d_e, dWx)
        wgrad_tc(terms[-1], Xv, nV, h, d_v, dWx[:, :d_v], accumulate=True)
        dWi = dWx[:, :d_v]
        dWh[:, h:].copy_(dWx[:, kv:kv + d_e])
    else:
        wgrad_tc_multi(terms, Xv, nV, h, d_v, dWi)
    if dbi is not None:
        for i, P in enumerate(terms):
            column_sum(P, nV, h, dbi, accumulate=i > 0)
    return dWi, dbi, dWh, dbh, dWo, dbo


class AtomMPFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, V, E, Wi, bi, Wh, bh, Wo, bo, lay, cfg):
        V, E, (Wi, bi, Wh, bh, Wo, bo) = _mp_inputs(ctx, V, E, (Wi, bi, Wh, bh, Wo, bo))
        p = plan("atom", cfg, lay, Wi.shape[0], V.shape[1], E.shape[1])
        Hv, saved = p.forward(lay, V, E, Wi, bi, Wh, bh, Wo, bo, cfg, p)
        _mp_save(ctx, lay, cfg, p, V, E, (Wi, Wh, Wo), saved, Hv)
        return Hv

    @staticmethod
    def backward(ctx, gHv):
        grads = ctx.plan.mirror(ctx.lay, *ctx.VE, *ctx.W, ctx.cfg, ctx.plan, ctx.saved, gHv, ctx.has_bias)
        return _mp_grads(ctx, grads, 2)


# ----------------------------------------------------------------------------------------------
# mol-atom-bond message passing on the bf16 tier (chemprop/nn/message_passing/mol_atom_bond.py): the depth loop and the
# W_vo read-out of Bond / AtomMPFunction, plus the per-edge head H_e = tau(W_eo([E || H^{T-1}])) in the caller's edge order
# ----------------------------------------------------------------------------------------------
def mab_tables(lay: Layout):
    """(dst atom of caller edge e, src atom of caller edge e, caller edge of the reverse of dst-sorted row r) as int32, built
    once per batch: the residual map of the bond kind's mirror, the gather of the atom kind's edge operand, and the
    out-edge table of the atom kind's backward segment sum."""
    if lay._mab is None:
        ip = lay.inv_perm.long()
        lay._mab = (lay.dst_row.index_select(0, ip), lay.src_row.index_select(0, ip),
                    lay.perm.index_select(0, lay.rev_row.long()))
    return lay._mab


class MABMPFunction(torch.autograd.Function):
    """(H_v, H_e) of MABBond / MABAtomMessagePassing on the bf16 tier, both f32; an absent read-out (W_vo or W_eo None)
    gives an empty tensor in its place.

    Forward: the depth loop of bond_forward / atom_forward_fused (atom_forward_tc where the fused atom step does not apply),
    the W_vo read-out with an f32 store, and the edge head: X_e[e] = [E[e] || H^{T-1}(e)] assembled once in caller order
    (H^{T-1}(e) = H[inv_perm[e]] for bonds, H_a[src(e)] for atoms), then one tensor-core GEMM with bias, tau and the f32
    store in its epilogue.  Backward: dY_e = g_e * tau'(H_e); dW_eo, db_eo from X_e; the gradient dY_e . W_eo[:, d_e:]
    enters the depth loop's mirror at its first tau' (the `entry` of bond_backward_tc / the atom backward functions) through
    the mirror mode of dmpnn_linear_tc_rows_bf16; the rest of the mirror is unchanged."""

    @staticmethod
    def forward(ctx, V, E, Wi, bi, Wh, bh, Wvo, bvo, Weo, beo, lay, cfg, kind):
        V, E, (Wi_, bi_, Wh_, bh_, Wvo_, bvo_, Weo_, beo_) = _mp_inputs(ctx, V, E, (Wi, bi, Wh, bh, Wvo, bvo, Weo, beo))
        h = Wh_.shape[0]
        d_v, d_e = V.shape[1], E.shape[1]
        nE, nV = lay.E, lay.V
        dev, T = V.device, cfg.hidden_dtype
        a, ap = cfg.act, cfg.act_param
        p = plan("mab_" + kind, cfg, lay, h, d_v, d_e)
        if kind == "bond":
            Hv, saved = p.forward(lay, V, E, Wi_, bi_, Wh_, bh_, Wvo_, bvo_, cfg, p, for_backward=any(ctx.needs_input_grad),
                                  readout_f32=True)
            src_idx = lay.inv_perm
            if Weo_ is not None and nE > 0:
                mab_tables(lay)            # built here, on the forward's stream, for the backward's residual map
        else:
            Hv, saved = p.forward(lay, V, E, Wi_, bi_, Wh_, bh_, Wvo_, bvo_, cfg, p, readout_f32=True)
            src_idx = mab_tables(lay)[1] if nE > 0 else None
        He = Xe = None
        if Weo_ is not None:
            He = torch.empty((max(nE, 1), h), dtype=torch.float32, device=dev)[:nE]
            if nE > 0:
                Hfin = saved["Hs"][-1] if saved["Hs"] else None
                if Hfin is None:
                    # depth 1: H^0 = tau(H_0) is applied on load by every consumer and never stored -- the edge head needs the
                    # activated rows, so the W_i GEMM runs once more with tau in its epilogue
                    rows = nE if kind == "bond" else nV
                    Hfin = _empty_hidden(rows, pad_hidden(h), T, dev)
                    X, K = (saved["X0"], d_v + d_e) if kind == "bond" else (saved["Xv"], d_v)
                    linear_tc(X, K, pack_weight_tc(Wi_), h, Hfin, bias=bi_, act=a, act_param=ap, R=rows)
                Xe = torch.empty((nE, (d_e + h + 15) // 16 * 16), dtype=T, device=dev)
                concat_bf16(E, d_e, Xe, nE, X2=Hfin, K2=h, idx2=src_idx)
                linear_tc_rows(Xe, d_e + h, pack_weight_tc(Weo_), h, He, R=nE, bias=beo_, act=a, act_param=ap)
                if cfg.dropout_p > 0:
                    _dropout_(He, cfg)                                                 # mol_atom_bond.py edge_finalize
        _mp_save(ctx, lay, cfg, p, V, E, (Wi_, Wh_, Wvo_, Weo_), saved, Hv)
        ctx.kind = kind
        ctx.edge = (Xe, None if He is None else He.detach())
        empty = torch.empty((0, h), dtype=torch.float32, device=dev)
        return (Hv if Hv is not None else empty), (He if He is not None else empty)

    @staticmethod
    def backward(ctx, gHv, gHe):
        V, E = ctx.VE
        Wi, Wh, Wvo, Weo = ctx.W
        Xe, He = ctx.edge
        lay, cfg, kind = ctx.lay, ctx.cfg, ctx.kind
        dev, T = V.device, cfg.hidden_dtype
        h = Wh.shape[0]
        hp, hc = pad_hidden(h), (h + 15) // 16 * 16
        d_e = E.shape[1]
        nE, nV = lay.E, lay.V
        a, ap = cfg.act, cfg.act_param
        f32 = dict(dtype=torch.float32, device=dev)
        entry = None
        dWeo = dbeo = None
        if Weo is not None:
            dWeo = torch.zeros_like(Weo)
            dbeo = torch.zeros(h, **f32) if ctx.has_bias[3] else None
            if nE > 0:
                if gHe.stride(1) != 1:
                    gHe = gHe.contiguous()
                dYe = _hidden(nE, hp, T, dev)          # zero padding: the out-edge segment sum reads 16-column vectors
                act_bwd(gHe, He, nE, h, act=a, act_param=ap, dZ=dYe)                  # dY_e = g_e * tau'(H_e), caller order
                wgrad_tc(dYe, Xe, nE, h, d_e + h, dWeo)
                if dbeo is not None:
                    column_sum(dYe, nE, h, dbeo)
                WeoT = pack_weight_tc(Weo[:, d_e:], transpose=True)
                if kind == "bond":
                    # dZ^{T-1}[inv_perm[e]] = ((dY_e . W_eo[:, d_e:])[e] + dM_v[dst(e)]) * tau'(H^{T-1}[inv_perm[e]])
                    dst_e = mab_tables(lay)[0]

                    def entry(dMv, Y, from_preact, out):
                        linear_tc_rows(dYe, h, WeoT, h, out, R=nE, act=a, act_param=ap, Y=Y, from_preact=from_preact,
                                       out_row=lay.inv_perm, res=dMv, res_row=dst_e if dMv is not None else None)
                else:
                    # atom v receives sum_{src(e)=v} dY_e[e] . W_eo[:, d_e:] = (sum_{src(e)=v} dY_e[e]) . W_eo[:, d_e:]: the
                    # sum over v's out-edges first (segment sum over the in-edges r of v, read through perm[rev[r]]), then a
                    # V-row GEMM whose epilogue adds the read-out's term and applies tau'
                    Se = _empty_hidden(nV, hp, T, dev)
                    segment_sum(dYe, lay.rowptr, nV, h, Se, idx=mab_tables(lay)[2], pad_to=hc)

                    def entry(dHa, Y, from_preact, out):
                        linear_tc_rows(Se, h, WeoT, h, out, R=nV, act=a, act_param=ap, Y=Y, from_preact=from_preact, res=dHa)
        gv = gHv if Wvo is not None else None
        nb = ctx.has_bias[:3]
        if gv is None and entry is None:
            # nothing reaches the depth loop (edge-only module on a batch without edges)
            z = lambda w, b: (torch.zeros_like(w), torch.zeros(w.shape[0], **f32) if b else None)  # noqa: E731
            (dWi, dbi), (dWh, dbh) = z(Wi, nb[0]), z(Wh, nb[1])
            dWvo = dbvo = None
        else:
            dWi, dbi, dWh, dbh, dWvo, dbvo = ctx.plan.mirror(lay, V, E, Wi, Wh, Wvo, cfg, ctx.plan, ctx.saved, gv, nb,
                                                             entry=entry)
        return _mp_grads(ctx, (dWi, dbi, dWh, dbh, dWvo, dbvo, dWeo, dbeo), 3)


# ----------------------------------------------------------------------------------------------
# aggregation
# ----------------------------------------------------------------------------------------------
class SegmentAggFunction(torch.autograd.Function):
    """Mean / Sum / Norm aggregation over molecules (chemprop/nn/agg.py:73-78, 90-95, 112-113)."""

    @staticmethod
    def forward(ctx, H, mol_atom_ptr, atom_mol, n_mols, scale_mode, scale):
        _require_cuda(H)
        Hc = H if H.stride(1) == 1 else H.contiguous()
        # molecule-level output is always f32 (b x d is tiny): whatever follows -- the reference's BatchNorm / FFN heads
        # (models/model.py:126-161) -- holds f32 parameters, so a bf16-tier encoder drops in without a cast by the caller
        out = torch.empty((n_mols, H.shape[1]), dtype=torch.float32, device=H.device)
        segment_sum(Hc, mol_atom_ptr, n_mols, H.shape[1], out, scale_mode=scale_mode, scale=scale,
                    pad_to=H.shape[1])
        ctx.ptr, ctx.atom_mol, ctx.mode, ctx.scale = mol_atom_ptr, atom_mol, scale_mode, scale
        ctx.nV, ctx.in_dtype = H.shape[0], H.dtype
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        if g.dtype not in (torch.float32, torch.bfloat16):
            g = g.float()
        dH = torch.empty((ctx.nV, g.shape[1]), dtype=ctx.in_dtype, device=g.device)
        segment_bcast(g, ctx.atom_mol, ctx.ptr, ctx.nV, g.shape[1], dH, scale_mode=ctx.mode, scale=ctx.scale,
                      n_seg=g.shape[0])
        return dH, None, None, None, None, None


class SegmentAggColumnsFunction(torch.autograd.Function):
    """Mean / Sum / Norm aggregation of several batches of the same molecule count into the column blocks of ONE b x sum(d_c)
    f32 buffer: `torch.cat([agg(H_0, batch_0), agg(H_1, batch_1), ...], 1)` of models/multi.py:51-52 without the cat.  One
    dmpnn_segment_sum per batch writes its block through the row stride `ldy`; the backward is one dmpnn_segment_bcast per
    batch reading its block through `ldg`.  `segs`: the (ptr, seg_of_row, b) of each batch (`segments_of`)."""

    @staticmethod
    def forward(ctx, segs, scale_mode, scale, *Hs):
        _require_cuda(*Hs)
        b = segs[0][2]
        widths = [int(H.shape[1]) for H in Hs]
        out = torch.empty((b, sum(widths)), dtype=torch.float32, device=Hs[0].device)
        c0 = 0
        for H, (ptr, _, _), d in zip(Hs, segs, widths):
            segment_sum(H if H.stride(1) == 1 else H.contiguous(), ptr, b, d, out[:, c0:c0 + d], scale_mode=scale_mode,
                        scale=scale, pad_to=d)
            c0 += d
        ctx.segs, ctx.mode, ctx.scale, ctx.widths = segs, scale_mode, scale, widths
        ctx.rows = [(int(H.shape[0]), H.dtype) for H in Hs]
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        if g.dtype not in (torch.float32, torch.bfloat16):
            g = g.float()
        dHs, c0 = [], 0
        for (ptr, seg_of_row, b), d, (nV, dt) in zip(ctx.segs, ctx.widths, ctx.rows):
            dH = torch.empty((nV, d), dtype=dt, device=g.device)
            segment_bcast(g[:, c0:c0 + d], seg_of_row, ptr, nV, d, dH, scale_mode=ctx.mode, scale=ctx.scale, n_seg=b)
            dHs.append(dH)
            c0 += d
        return (None, None, None, *dHs)


class SegmentBcastFunction(torch.autograd.Function):
    """rows <- their segment's row (`Z[batch]` of chemprop/nn/agg.py:127, nn/ffn.py:127): dmpnn_segment_bcast; the mirror
    is the segment sum."""

    @staticmethod
    def forward(ctx, G, mol_atom_ptr, atom_mol, n_rows):
        _require_cuda(G)
        Gc = G if G.stride(1) == 1 else G.contiguous()
        out = torch.empty((n_rows, G.shape[1]), dtype=G.dtype, device=G.device)
        segment_bcast(Gc, atom_mol, mol_atom_ptr, n_rows, G.shape[1], out, n_seg=G.shape[0])
        ctx.ptr, ctx.n_seg = mol_atom_ptr, G.shape[0]
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dG = torch.empty((ctx.n_seg, g.shape[1]), dtype=g.dtype, device=g.device)
        segment_sum(g, ctx.ptr, ctx.n_seg, g.shape[1], dG, pad_to=g.shape[1])
        return dG, None, None, None
