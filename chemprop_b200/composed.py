"""Composed tier: the reference's own op sequence (chemprop/nn/message_passing/base.py:196-212) with every
tensor op on the path executed by a kernel of libdmpnn_sm90.so, glued together by torch autograd.

It serves the configurations the monolithic tiers (engine.BondMPFunction / AtomMPFunction, which fuse tau into
their kernels) do not cover:

  * activation modules the kernels have no code for -- PReLU (learnable slope: chemprop/nn/utils.py:48), SELU
    (utils.py:35-41), or any user `nn.Module` (utils.py:37-42 returns it as is);
  * dropout > 0 in training mode (base.py:139, :182, :188);
  * AtomMessagePassing(undirected=True) (base.py:202-203 on mixins.py:25-30, which is no longer atom-granular).

`tau` and `dropout` are the caller's own torch modules applied between our kernels -- exactly where the reference
applies them -- so the gradient of a learnable activation and the dropout RNG stream are torch's.  Everything else
(gathers, the three linear layers and their weight gradients, message, reverse averaging, atom scatter-sum) is a
libdmpnn kernel with a hand-written autograd mirror.  Hidden states are f32 `[rows, h]` (unpadded) in the
engine's internal edge order (stable sort by destination atom), so this tier satisfies the tolerance of both
precision settings.  There is no CPU path here either: the wrappers in engine.py refuse CPU tensors.
"""
from __future__ import annotations

import torch
from torch import Tensor

from . import engine as K


def _buf(rows: int, cols: int, like: Tensor) -> Tensor:
    """Uninitialised f32 [rows, cols]; an empty one still has a non-null data pointer (it is a slice of one row)."""
    if rows > 0 and cols > 0:
        return torch.empty((rows, cols), dtype=torch.float32, device=like.device)
    return torch.empty((max(rows, 1), max(cols, 1)), dtype=torch.float32, device=like.device)[:rows, :cols]


def _c(t: Tensor | None) -> Tensor | None:
    if t is None:
        return None
    t = t.detach()
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


# First use of the 3xTF32 kernels from this tier in a process: the same product is also run on the f32 FMA kernel and
# compared (one device sync, once).  This composition was written after the round's last hardware run; until it has been seen
# to agree on the device at hand it does not get to decide a result.  A mismatch disables it (loudly) for the process.
_X3_STATE = {"ok": None}        # None: not checked yet; True / False: verdict


def _x3_first_use_check(out_x3: Tensor, X1c: Tensor, K1: int, Wc: Tensor, N: int, bc, resc, R: int) -> Tensor:
    ref = _buf(R, N, Wc)
    K.linear_fwd(X1c, K1, Wc, ref, N, bias=bc, res=resc, R=R, pad_to=N)
    err = (out_x3 - ref).abs().max()
    scale = ref.abs().max().clamp_min(1e-6)
    ok = bool((torch.isfinite(err) & (err <= 1e-4 * scale)).item())
    _X3_STATE["ok"] = ok
    if not ok:
        import warnings

        warnings.warn("chemprop_b200: the composed tier's 3xTF32 GEMM disagrees with the f32 FMA kernel on this device "
                      f"(max |diff| = {float(err):.3e} at scale {float(scale):.3e}); it stays disabled for this process and "
                      "the f32 FMA result is used -- please report this", RuntimeWarning, stacklevel=3)
        return ref
    return out_x3


class GatherLinear(torch.autograd.Function):
    """Y[r] = [X1[i1(r)] || X2[i2(r)]] . W^T + b + res[r]   (r < R)  -- dmpnn_linear_fwd.
    Covers W_i (mixins.py:8-9, :22-23), W_h with the H_0 residual (base.py:136-138) and W_o (base.py:180).
    Gradients: W, b (dmpnn_linear_wgrad), res (identity), and X1 / X2 when they are not gathered."""

    @staticmethod
    def forward(ctx, X1, idx1, X2, idx2, W, b, res, R):
        X1c, X2c, Wc, bc, resc = _c(X1), _c(X2), _c(W), _c(b), _c(res)
        K1 = X1c.shape[1]
        K2 = 0 if X2c is None else X2c.shape[1]
        N = Wc.shape[0]
        out = _buf(R, N, Wc)
        # a plain (ungathered, single-source) product -- the W_h GEMM of every depth step, 2 E h^2 flop -- runs f32-accurate on
        # the tensor cores (3xTF32, csrc/gemm_x3.cu) when its dimensions allow 16-byte rows; gathered / two-source operands
        # (W_i, W_o) stay on the f32 FMA kernel, which reads them in place
        x3 = (idx1 is None and X2c is None and R > 0 and K1 % 4 == 0 and N % 4 == 0 and 0 < K1 <= 4096 and 0 < N <= 4096
              and X1c.data_ptr() % 16 == 0 and (resc is None or resc.data_ptr() % 16 == 0)
              and K.X3_ENABLED and K._fused_available() and _X3_STATE["ok"] is not False)
        if x3 and _X3_STATE["ok"] is None and X1c.is_cuda and torch.cuda.is_current_stream_capturing():
            x3 = False                                  # the first-use check synchronises: not inside a graph capture
        if x3:
            K.linear_x3(X1c, K1, K.pack_weight_x3(Wc), N, out, bias=bc, res=resc, R=R, pad_to=N)
            if _X3_STATE["ok"] is None:
                out = _x3_first_use_check(out, X1c, K1, Wc, N, bc, resc, R)
                x3 = bool(_X3_STATE["ok"])
        elif R > 0:
            K.linear_fwd(X1c, K1, Wc, out, N, idx1=idx1, X2=X2c, K2=K2, idx2=idx2, bias=bc, res=resc, R=R, pad_to=N)
        ctx.x3 = x3
        ctx.args = (X1c, idx1, X2c, idx2, Wc, K1, K2, N, R)
        ctx.wdtype = W.dtype
        ctx.bdtype = None if b is None else b.dtype
        return out

    @staticmethod
    def backward(ctx, dY):
        X1c, idx1, X2c, idx2, Wc, K1, K2, N, R = ctx.args
        need_x1, _, need_x2, _, need_w, need_b, need_res, _ = ctx.needs_input_grad
        dY = _c(dY)
        x3 = ctx.x3 and dY.data_ptr() % 16 == 0 and _X3_STATE["ok"] is True
        dX1 = dX2 = dW = db = None
        if need_w or need_b:
            dW = torch.zeros_like(Wc)
            db = torch.zeros(N, dtype=torch.float32, device=Wc.device) if need_b else None
            if x3:
                K.wgrad_x3(dY, X1c, R, N, K1, dW)
                if db is not None:
                    K.column_sum(dY, R, N, db)
            elif R > 0:
                K.linear_wgrad(dY, X1c, K1, dW, N, idx1=idx1, X2=X2c, K2=K2, idx2=idx2, dbias=db, R=R)
            dW = dW.to(ctx.wdtype)
            db = None if db is None else db.to(ctx.bdtype)
        if need_x1:
            if idx1 is not None:
                raise K.DmpnnError("GatherLinear: no gradient through a gathered operand")
            dX1 = _buf(R, K1, Wc)
            if x3:
                K.linear_x3(dY, N, K.pack_weight_x3(Wc, transpose=True), K1, dX1, R=R, pad_to=K1)
            elif R > 0:
                K.linear_fwd(dY, N, Wc[:, :K1].t().contiguous(), dX1, K1, R=R, pad_to=K1)
        if need_x2:
            if idx2 is not None:
                raise K.DmpnnError("GatherLinear: no gradient through a gathered operand")
            dX2 = _buf(R, K2, Wc)
            if R > 0:
                K.linear_fwd(dY, N, Wc[:, K1:].t().contiguous(), dX2, K2, R=R, pad_to=K2)
        return dX1, None, dX2, None, dW, db, (dY if need_res else None), None


class BondMessage(torch.autograd.Function):
    """M[e] = sum_{dst(e') = src(e)} H[e'] - H[rev(e)]   (mixins.py:11-18) -- dmpnn_bond_message; the mirror is the
    same kernel reading through `rev` instead of writing through it."""

    @staticmethod
    def forward(ctx, H, lay):
        Hc = _c(H)
        M = _buf(lay.E, Hc.shape[1], Hc)
        K.bond_message(Hc, lay, Hc.shape[1], M)
        ctx.lay = lay
        return M

    @staticmethod
    def backward(ctx, dM):
        dM = _c(dM)
        dH = _buf(ctx.lay.E, dM.shape[1], dM)
        K.bond_message(dM, ctx.lay, dM.shape[1], dH, permute_on_read=True)
        return dH, None


class RevAverage(torch.autograd.Function):
    """H[e] <- (H[e] + H[rev(e)]) / 2   (base.py:202-203) -- dmpnn_rev_average; self-adjoint (rev is an involution)."""

    @staticmethod
    def forward(ctx, H, lay):
        Hc = _c(H)
        out = _buf(lay.E, Hc.shape[1], Hc)
        K.rev_average(Hc, lay, Hc.shape[1], out)
        ctx.lay = lay
        return out

    @staticmethod
    def backward(ctx, g):
        g = _c(g)
        out = _buf(ctx.lay.E, g.shape[1], g)
        K.rev_average(g, ctx.lay, g.shape[1], out)
        return out, None


class SumByDst(torch.autograd.Function):
    """A[v] = sum_{dst(e) = v} H[e]   (base.py:208-211, first half of mixins.py:26-29) -- dmpnn_segment_sum over the
    dst-sorted rows; mirror: dH[e] = dA[dst(e)] (dmpnn_segment_bcast)."""

    @staticmethod
    def forward(ctx, H, lay):
        Hc = _c(H)
        if lay.E == 0:     # no edges: every atom's sum is empty (the kernel is not launched on a 0-row operand)
            A = torch.zeros((lay.V, Hc.shape[1]), dtype=torch.float32, device=Hc.device)
        else:
            A = _buf(lay.V, Hc.shape[1], Hc)
            K.segment_sum(Hc, lay.rowptr, lay.V, Hc.shape[1], A, pad_to=Hc.shape[1])
        ctx.lay = lay
        return A

    @staticmethod
    def backward(ctx, dA):
        lay = ctx.lay
        dA = _c(dA)
        dH = _buf(lay.E, dA.shape[1], dA)
        if lay.E > 0:
            K.segment_bcast(dA, lay.dst_row, None, lay.E, dA.shape[1], dH)
        return dH, None


class GatherBySrc(torch.autograd.Function):
    """M[e] = A[src(e)]   (the `[bmg.edge_index[0]]` of mixins.py:29) -- dmpnn_segment_bcast; mirror:
    dA[v] = sum_{src(e) = v} dM[e] = sum_{e' in in(v)} dM[rev(e')] (dmpnn_segment_sum gathering through rev)."""

    @staticmethod
    def forward(ctx, A, lay):
        Ac = _c(A)
        M = _buf(lay.E, Ac.shape[1], Ac)
        if lay.E > 0:
            K.segment_bcast(Ac, lay.src_row, None, lay.E, Ac.shape[1], M)
        ctx.lay = lay
        return M

    @staticmethod
    def backward(ctx, dM):
        lay = ctx.lay
        dM = _c(dM)
        if lay.E == 0:
            return torch.zeros((lay.V, dM.shape[1]), dtype=torch.float32, device=dM.device), None
        dA = _buf(lay.V, dM.shape[1], dM)
        K.segment_sum(dM, lay.rowptr, lay.V, dM.shape[1], dA, idx=lay.rev_row, pad_to=dM.shape[1])
        return dA, None


class PermuteRows(torch.autograd.Function):
    """out[r] = X[idx[r]] for a permutation `idx` with inverse `inv_idx` -- dmpnn_segment_bcast both ways.  Used to
    hand per-edge results back in the caller's edge order (the engine's internal rows are sorted by destination)."""

    @staticmethod
    def forward(ctx, X, idx, inv_idx):
        Xc = _c(X)
        out = _buf(Xc.shape[0], Xc.shape[1], Xc)
        if Xc.shape[0] > 0:
            K.segment_bcast(Xc, idx, None, Xc.shape[0], Xc.shape[1], out)
        ctx.inv_idx = inv_idx
        return out

    @staticmethod
    def backward(ctx, g):
        g = _c(g)
        out = _buf(g.shape[0], g.shape[1], g)
        if g.shape[0] > 0:
            K.segment_bcast(g, ctx.inv_idx, None, g.shape[0], g.shape[1], out)
        return out, None, None


def _inputs(bmg):
    K._require_cuda(bmg.V, bmg.E)
    return bmg.V.contiguous().float(), bmg.E.contiguous().float()


def bond_edge_states(mp, V, E, lay) -> Tensor:
    """The depth loop of BondMessagePassing (base.py:198-206): final directed-edge hidden states H^{T-1}, internal row
    order.  A batch without edges (tests/integration/test_export.py:15-46) flows through as 0-row tensors, as in the
    reference."""
    tau, drop = mp.tau, mp.dropout
    H0 = GatherLinear.apply(V, lay.src_row, E, lay.perm, mp.W_i.weight, mp.W_i.bias, None, lay.E)      # mixins.py:8-9
    H = tau(H0)                                                                                       # base.py:200
    for _ in range(1, int(mp.depth)):
        if mp.undirected:
            H = RevAverage.apply(H, lay)                                                              # base.py:202-203
        M = BondMessage.apply(H, lay)                                                                 # mixins.py:11-18
        Z = GatherLinear.apply(M, None, None, None, mp.W_h.weight, mp.W_h.bias, H0, lay.E)            # base.py:137-138
        H = drop(tau(Z))                                                                              # base.py:138-139
    return H


def atom_edge_states(mp, V, E, lay) -> Tensor:
    """The depth loop of AtomMessagePassing, edge-granular as in the reference (mixins.py:22-30) so that `undirected`
    (base.py:202-203) keeps its meaning."""
    tau, drop = mp.tau, mp.dropout
    d_e = E.shape[1]
    H0 = GatherLinear.apply(V, lay.src_row, None, None, mp.W_i.weight, mp.W_i.bias, None, lay.E)       # mixins.py:22-23
    AE = None
    if d_e > 0:   # sum of the in-edge bond features of every atom: the loop-invariant half of mixins.py:26-29
        if lay.E > 0:
            AE = _buf(lay.V, d_e, V)
            K.segment_sum(E, lay.rowptr, lay.V, d_e, AE, idx=lay.perm, pad_to=d_e)
        else:
            AE = torch.zeros((lay.V, d_e), dtype=torch.float32, device=V.device)
    H = tau(H0)
    for _ in range(1, int(mp.depth)):
        if mp.undirected:
            H = RevAverage.apply(H, lay)
        M = GatherBySrc.apply(SumByDst.apply(H, lay), lay)                                            # mixins.py:26-29
        Z = GatherLinear.apply(M, None, AE, lay.src_row if AE is not None else None, mp.W_h.weight, mp.W_h.bias,
                               H0, lay.E)                                                             # W_h([M_H || M_E]) + H_0
        H = drop(tau(Z))
    return H


def vertex_readout(mp, W_o, V, H, lay) -> Tensor:
    """M_v = sum_{dst(e)=v} H[e] (base.py:208-211), then dropout(tau(W_o([V || M_v]))) (base.py:180-182)."""
    Mv = SumByDst.apply(H, lay)
    Y = GatherLinear.apply(V, None, Mv, None, W_o.weight, W_o.bias, None, lay.V)
    return mp.dropout(mp.tau(Y))


def edge_readout(mp, W_eo, E, H, lay) -> Tensor:
    """dropout(tau(W_eo([E || H]))) per directed edge, in the CALLER's edge order
    (chemprop/nn/message_passing/mol_atom_bond.py `edge_finalize`)."""
    Hc = PermuteRows.apply(H, lay.inv_perm, lay.perm)          # internal row of caller edge e is inv_perm[e]
    Y = GatherLinear.apply(E, None, Hc, None, W_eo.weight, W_eo.bias, None, lay.E)
    return mp.dropout(mp.tau(Y))


def bond_forward(mp, bmg, lay) -> Tensor:
    """BondMessagePassing.forward up to and including dropout(tau(W_o(.))) (base.py:196-212, :180-182)."""
    V, E = _inputs(bmg)
    return vertex_readout(mp, mp.W_o, V, bond_edge_states(mp, V, E, lay), lay)


def atom_forward(mp, bmg, lay) -> Tensor:
    V, E = _inputs(bmg)
    return vertex_readout(mp, mp.W_o, V, atom_edge_states(mp, V, E, lay), lay)


def mab_forward(mp, bmg, lay, kind: str):
    """_MABMessagePassingBase.forward (mol_atom_bond.py): the same loop, then the vertex and / or the edge read-out."""
    V, E = _inputs(bmg)
    H = (bond_edge_states if kind == "bond" else atom_edge_states)(mp, V, E, lay)
    H_v = vertex_readout(mp, mp.W_vo, V, H, lay) if mp.return_vertex_embeddings else None
    H_e = edge_readout(mp, mp.W_eo, E, H, lay) if mp.return_edge_embeddings else None
    return H_v, H_e
