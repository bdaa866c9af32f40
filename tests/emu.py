"""TEST INFRASTRUCTURE ONLY.  torch-CPU emulations of the libdmpnn kernels behind engine.py's op wrappers, written
from the contracts in include/dmpnn.h, so that the HOST logic (the hand-written autograd mirrors in engine.py and the
composed tier in composed.py: which op, which operand, which index table, in which order) can be checked against the
golden vectors without a GPU.  `patch_engine(monkeypatch)` swaps the wrappers for these; nothing in the product
imports this file, and a GPU run never touches it (the `-m gpu` tests call the real kernels through the C ABI).

The emulation itself is validated by the fact that the GPU-verified monolithic tiers, run through it, reproduce every
golden (tests/test_host_logic.py::test_monolithic_f32_tier_through_emulation, ::test_monolithic_bf16_tier_through_emulation:
the bf16 emulations round where the kernels store bf16, so the tier's 1e-2 bound is checked for real)."""
from __future__ import annotations

import numpy as np
import torch

from chemprop_b200 import _lib, engine
from oracle import layout_np

ACT_NONE, ACT_RELU, ACT_LEAKYRELU, ACT_TANH, ACT_ELU = (_lib.ACT_NONE, _lib.ACT_RELU, _lib.ACT_LEAKYRELU,
                                                         _lib.ACT_TANH, _lib.ACT_ELU)


def _act(x, act, p):
    if act == ACT_NONE:
        return x
    if act == ACT_RELU:
        return torch.relu(x)
    if act == ACT_LEAKYRELU:
        return torch.where(x > 0, x, x * p)
    if act == ACT_TANH:
        return torch.tanh(x)
    if act == ACT_ELU:
        return torch.where(x > 0, x, p * torch.expm1(x))
    raise ValueError(act)


def _dact(y, act, p, from_preact):
    """tau' evaluated from the output y = tau(z) (from_preact False) or from z itself (dmpnn_act_bwd)."""
    one = torch.ones_like(y)
    if act == ACT_NONE:
        return one
    if act == ACT_RELU:
        return (y > 0).to(y.dtype)
    if act == ACT_LEAKYRELU:
        return torch.where(y > 0, one, one * p)
    if act == ACT_TANH:
        t = torch.tanh(y) if from_preact else y
        return 1 - t * t
    if act == ACT_ELU:
        return torch.where(y > 0, one, (p * torch.exp(y)) if from_preact else (y + p))
    raise ValueError(act)


def _rows(X, idx, R, K):
    X = X.float()
    return (X[:R, :K] if idx is None else X[idx[:R].long(), :K])


def _cat(X1, K1, idx1, X2, K2, idx2, R):
    A = _rows(X1, idx1, R, K1)
    if K2:
        A = torch.cat([A, _rows(X2, idx2, R, K2)], dim=1)
    return A


def linear_fwd(X1, K1, W, out, N, *, idx1=None, X2=None, K2=0, idx2=None, bias=None, res=None, act=ACT_NONE,
               act_param=0.0, R=None, pad_to=None):
    R = out.shape[0] if R is None else R
    assert K1 > 0 and W.shape == (N, K1 + K2) and (K2 == 0 or X2 is not None) and out.shape[1] >= N   # "bad sizes"
    Y = _cat(X1, K1, idx1, X2, K2, idx2, R) @ W.float().t()
    if bias is not None:
        Y = Y + bias.float()
    if res is not None:
        Y = Y + res[:R, :N].float()
    out[:R, :N] = _act(Y, act, act_param).to(out.dtype)
    pad_to = min(out.stride(0), out.shape[1]) if pad_to is None else pad_to
    if pad_to > N:
        out[:R, N:pad_to] = 0


def linear_wgrad(dY, X1, K1, dW, N, *, idx1=None, X2=None, K2=0, idx2=None, dbias=None, accumulate=False, R=None):
    R = dY.shape[0] if R is None else R
    assert K1 > 0                                                    # "bad sizes"
    g = dY[:R, :N].float()
    upd = g.t() @ _cat(X1, K1, idx1, X2, K2, idx2, R)
    if accumulate:
        dW += upd
    else:
        dW.copy_(upd)
    if dbias is not None:
        if accumulate:
            dbias += g.sum(0)
        else:
            dbias.copy_(g.sum(0))


def _scale(ptr, s, mode, scale):
    if mode == _lib.SCALE_INV_COUNT:
        return float(ptr[s + 1] - ptr[s])
    if mode == _lib.SCALE_DIV_CONST:
        return float(scale)
    return 1.0


def segment_sum(X, ptr, n_seg, Ccols, out, *, idx=None, act=ACT_NONE, act_param=0.0, scale_mode=_lib.SCALE_NONE,
                scale=1.0, pad_to=None):
    p = ptr.tolist()
    Xf = X.float()
    for s in range(n_seg):
        rows = torch.arange(p[s], p[s + 1])
        if idx is not None:
            rows = idx[rows].long()
        acc = _act(Xf[rows, :Ccols], act, act_param).sum(0)
        if p[s + 1] > p[s]:
            acc = acc / _scale(p, s, scale_mode, scale)
        out[s, :Ccols] = acc.to(out.dtype)     # empty segment -> zero row
    pad_to = min(out.stride(0), out.shape[1]) if pad_to is None else pad_to
    if pad_to > Ccols:
        out[:n_seg, Ccols:pad_to] = 0


def segment_bcast(G, seg_of_row, ptr, R, Ccols, out, *, scale_mode=_lib.SCALE_NONE, scale=1.0, n_seg=0):
    if R == 0:
        return
    seg = seg_of_row[:R].long()
    if ptr is not None and n_seg > 0:     # rows of segment s are [ptr[s], ptr[s+1])
        cnt = (ptr[1:n_seg + 1] - ptr[:n_seg]).long()
        assert int(cnt.sum()) == R
        assert torch.equal(seg, torch.repeat_interleave(torch.arange(n_seg), cnt)), "ptr / seg_of_row disagree"
    Y = G.float()[seg, :Ccols]
    if scale_mode == _lib.SCALE_INV_COUNT:
        Y = Y / (ptr[seg + 1] - ptr[seg]).float().unsqueeze(1)
    elif scale_mode == _lib.SCALE_DIV_CONST:
        Y = Y / scale
    out[:R, :Ccols] = Y.to(out.dtype)


def bond_message(X, lay, Ccols, out, *, act=ACT_NONE, act_param=0.0, permute_on_read=False):
    if lay.E == 0:
        return
    rev = lay.rev_row.long()
    dst = lay.dst_row.long()
    f = _act(X.float()[: lay.E, :Ccols], act, act_param)
    rd = f[rev] if permute_on_read else f                       # value read for in-edge row e'
    s = torch.zeros((lay.V, Ccols)).index_add_(0, dst, rd)      # per destination atom
    val = s[dst] - rd
    if permute_on_read:
        out[: lay.E, :Ccols] = val.to(out.dtype)
    else:
        out[rev, :Ccols] = val.to(out.dtype)


def rev_average(X, lay, Ccols, out, *, act=ACT_NONE, act_param=0.0):
    if lay.E == 0:
        return
    f = _act(X.float()[: lay.E, :Ccols], act, act_param)
    out[: lay.E, :Ccols] = ((f + f[lay.rev_row.long()]) / 2).to(out.dtype)


def act_bwd(G, Yact, R, Ccols, *, act, act_param=0.0, gidx=None, from_preact=False, dZ=None, acc=None):
    if R == 0:
        return
    g = _rows(G, gidx, R, Ccols)
    d = g * _dact(Yact.float()[:R, :Ccols], act, act_param, from_preact)
    if dZ is not None:
        dZ[:R, :Ccols] = d.to(dZ.dtype)
        d = dZ[:R, :Ccols].float()          # the accumulator sees the rounded value, as in the kernel? (f32: identical)
    if acc is not None:
        acc[:R, :Ccols] += d.to(acc.dtype)


def build_layout(edge_index, rev_edge_index, batch, n_mols, meta_host=None):
    L = layout_np.build_layout(edge_index.numpy(), rev_edge_index.numpy(), batch.numpy(), int(n_mols))
    B = int(n_mols)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).astype(np.int32))
    pad = lambda a: t(np.concatenate([a, np.zeros(B + 2 - len(a), np.int32)]))
    meta = [0] * _lib.META_WORDS
    meta[_lib.META_N_TILES], meta[_lib.META_FLAGS] = L["n_tiles"], L["flags"]
    meta[_lib.META_MAX_INDEG], meta[_lib.META_MAX_TILE_ROWS] = L["max_indeg"], L["max_tile_rows"]
    meta[_lib.META_MAX_TILE_ATOMS] = L["max_tile_atoms"]
    assert meta_host is None or list(meta_host) == meta, (meta_host, meta)
    return engine.Layout(int(batch.shape[0]), int(edge_index.shape[1]), B, t(L["perm"]), t(L["inv_perm"]), t(L["rowptr"]),
                         t(L["src_row"]), t(L["dst_row"]), t(L["rev_row"]), t(L["mol_atom_ptr"]), t(L["mol_row_ptr"]),
                         pad(L["tile_mol_ptr"]), pad(L["tile_row_ptr"]), pad(L["tile_atom_ptr"]),
                         torch.tensor(meta, dtype=torch.int32), list(meta))


# ---- bf16 / tensor-core tier ------------------------------------------------------------------------------------
def _bf(x):
    """round to bf16, continue in f32 (what a bf16 store followed by a load does)"""
    return x.to(torch.bfloat16).float()


def pack_weight_tc(W, transpose=False):
    """the 'packed' weight of the emulation is just B[n][k] (bf16-rounded) of C = A . B^T"""
    return _bf(W.detach().float().t() if transpose else W.detach().float()).contiguous()


def pack_weight_bf16(W):
    return _bf(W.detach().float()).contiguous()


def concat_bf16(X1, K1, out, R, *, idx1=None, X2=None, K2=0, idx2=None, width=None):
    width = out.shape[1] if width is None else width
    out[:R, :K1 + K2] = _cat(X1, K1, idx1, X2, K2, idx2, R).to(out.dtype)
    if width > K1 + K2:
        out[:R, K1 + K2:width] = 0


def dropout_keep_bits(rows, h, cfg, like):
    """engine.dropout_keep_bits without the device generator: keep bits from torch's CPU RNG (or the test's mask_fn)."""
    nj = (h + 15) // 16
    if cfg.mask_fn is not None:
        M = cfg.mask_fn(like)[:rows, : nj * 16].to(torch.int32)
    else:
        M = (torch.rand(rows, nj * 16) >= cfg.dropout_p).to(torch.int32)
    w = (M.reshape(rows, nj, 16) << torch.arange(16, dtype=torch.int32)).sum(-1)
    return w.to(torch.uint16).contiguous()


def concat_f32(X1, K1, out, R, *, idx1=None, X2=None, K2=0, idx2=None, width=None):
    width = out.shape[1] if width is None else width
    out[:R, :K1 + K2] = _cat(X1, K1, idx1, X2, K2, idx2, R)
    if width > K1 + K2:
        out[:R, K1 + K2:width] = 0


def linear_tc(A, K, Wpk, N, out, *, bias=None, res=None, act=ACT_NONE, act_param=0.0, R=None):
    R = out.shape[0] if R is None else R
    assert A.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and Wpk.shape == (N, K)
    Y = A[:R, :K].float() @ Wpk.t()
    if bias is not None:
        Y = Y + bias.float()
    if res is not None:
        Y = Y + res[:R, :N].float()
    out[:R, :N] = _act(Y, act, act_param).to(out.dtype)
    n16 = (N + 15) // 16 * 16
    if n16 > N:
        out[:R, N:n16] = 0


def wgrad_tc(dY, X, R, N, K, dW, *, accumulate=False):
    assert dY.dtype == torch.bfloat16 and X.dtype == torch.bfloat16 and dW.dtype == torch.float32
    upd = dY[:R, :N].float().t() @ X[:R, :K].float()
    if accumulate:
        dW[:N, :K] += upd
    else:
        dW[:N, :K] = upd


def wgrad_tc_multi(dYs, X, R, N, K, dW, *, accumulate=False):
    for i, dY in enumerate(dYs):
        wgrad_tc(dY, X, R, N, K, dW, accumulate=accumulate or i > 0)


def pack_weight_x3(W, transpose=False):
    """fp32-accurate tier: the 'packed' weight of the emulation is B[n][k] in f32 (the hi / lo split is exact to 2^-22)"""
    W = W.detach().float()
    return (W.t() if transpose else W).contiguous()


def linear_x3(A, K, Wpk, N, out, *, idx=None, bias=None, res=None, act=ACT_NONE, act_param=0.0, R=None, pad_to=None):
    R = out.shape[0] if R is None else R
    Kw = Wpk.shape[1]                  # the packed weight's own K; A may carry up to 3 zero padding columns beyond it
    assert A.dtype == torch.float32 and out.dtype == torch.float32 and Wpk.shape[0] == N and K % 4 == 0 and 0 <= K - Kw < 4
    assert K == Kw or float(_rows(A, idx, R, K)[:, Kw:].abs().max()) == 0.0
    Y = _rows(A, idx, R, Kw) @ Wpk.t()
    if bias is not None:
        Y = Y + bias.float()
    if res is not None:
        Y = Y + res[:R, :N].float()
    out[:R, :N] = _act(Y, act, act_param)
    pad_to = min(out.stride(0), out.shape[1]) if pad_to is None else pad_to
    pad_to = max(N, min(pad_to, (N + 15) // 16 * 16))
    if pad_to > N:
        out[:R, N:pad_to] = 0


def wgrad_x3(dY, X, R, N, K, dW, *, accumulate=False):
    assert dY.dtype == torch.float32 and X.dtype == torch.float32 and N % 4 == 0 and K % 4 == 0
    upd = dY[:R, :N].t() @ X[:R, :K]
    if accumulate:
        dW[:N, :K] += upd
    else:
        dW[:N, :K] = upd


def bn_train_fwd(X, gamma, beta, running_mean, running_var, eps, momentum, Y, Xhat, mean, invstd):
    B = X.shape[0]
    mu, var = X.mean(0), X.var(0, unbiased=False)
    mean.copy_(mu)
    invstd.copy_(torch.rsqrt(var + eps))
    Xhat.copy_((X - mu) * invstd)
    Y.copy_(Xhat * (gamma if gamma is not None else 1.0) + (beta if beta is not None else 0.0))
    if running_mean is not None:
        running_mean.mul_(1 - momentum).add_(momentum * mu)
    if running_var is not None:
        running_var.mul_(1 - momentum).add_(momentum * (X.var(0, unbiased=True) if B > 1 else var))


def bn_bwd(dY, Xhat, gamma, invstd, dX, dgamma, dbeta):
    B = dY.shape[0]
    sdy, sdyx = dY.sum(0), (dY * Xhat).sum(0)
    if dbeta is not None:
        dbeta.copy_(sdy)
    if dgamma is not None:
        dgamma.copy_(sdyx)
    g = gamma if gamma is not None else 1.0
    dX.copy_(g * invstd / B * (B * dY - sdy - Xhat * sdyx))


def mse_loss(P, Y, w, tw, loss, dP):
    m = torch.isfinite(Y)
    e = torch.where(m, P - torch.nan_to_num(Y), torch.zeros_like(P))
    ww = (w.view(-1, 1) if w is not None else 1.0) * (tw.view(1, -1) if tw is not None else 1.0) * m
    n = m.sum().clamp(min=1)
    loss.copy_(((ww * e * e).sum() / n).reshape(1))
    dP.copy_(2 * ww * e / n)


def column_sum(Y, R, N, out, *, accumulate=False):
    v = Y[:R, :N].float().sum(0)
    if accumulate:
        out += v
    else:
        out.copy_(v)


def scale_mask_(X, M, scale):
    assert X.is_contiguous() and M.is_contiguous() and X.shape == M.shape and X.dtype == M.dtype
    X.copy_((X.float() * M.float() * scale).to(X.dtype))


def _sibling_sum_packed(f, lay, through_rev):
    """The fused kernel's message warps, rounding for rounding (csrc/step_fused.cu, message role): A row r = sum over the
    OTHER in-edge rows x of r's destination atom of f[x] (f[rev x] in the mirror), added in slot order as packed bf16
    (`__hadd2(__hadd2(a0, a1), a2)`, an absent sibling is +0) for in-degree <= 4 and in f32 with one rounding otherwise.
    `f` is bf16-valued f32 [E, C]; returns bf16-valued f32 [E, C] indexed by the A row r."""
    E = lay.E
    rowptr, dst = lay.rowptr.long(), lay.dst_row.long()
    rev = lay.rev_row.long()
    r = torch.arange(E)
    g0 = rowptr[dst]
    d = rowptr[dst + 1] - g0
    rd = f[rev] if through_rev else f
    vals = []
    for k in range(3):
        x = g0 + k
        x = x + (x >= r).long()
        ok = (k < d - 1) & (d <= 4)
        x = torch.where(ok, x, r)
        vals.append(torch.where(ok.unsqueeze(1), rd[x], 0.0))      # an absent slot is +0, its row is not read
    small = _bf(_bf(vals[0] + vals[1]) + vals[2])
    big = d > 4
    if bool(big.any()):
        s = torch.zeros((lay.V, f.shape[1])).index_add_(0, dst, rd)
        small = torch.where(big.unsqueeze(1), _bf(s[dst] - rd), small)   # kernel: f32 sum of the others; same up to f32 order
    return small


def _pad16(h):
    return (h + 15) // 16 * 16


def _mma(A, Wpk, h):
    """A[:, :pad16(h)] . B^T with B = Wpk [h x h] zero-padded to pad16(h) x pad16(h) (k_pack_weight), as the kernel's MMA sees
    it: columns [0, h) are A[:, :h] . Wpk^T and columns [h, pad16(h)) zero, except that a NaN or Inf anywhere in a row of A
    makes the whole result row NaN (0 * NaN = 0 * Inf = NaN)."""
    out = torch.zeros((A.shape[0], _pad16(h)))
    out[:, :h] = A[:, :h] @ Wpk.t()
    out[~torch.isfinite(A).all(1)] = float("nan")
    return out


# The fused-step emulations below read the columns the kernel reads: input rows [0, pad16(h)) (its TMA boxes span pad16(h)
# columns; the FAR windows' global gathers read the same 16-column blocks) and the epilogue's H_0 / Y / addend words in
# [h, pad16(h)), and they produce the output's padding columns the way each mode does: FWD tau(H_0 + 0), MASK 0 * tau'(Y),
# LAST 0 * tau'(H_0) + addends, COPY 0 -- all zero when the inputs' padding is, NaN rows when it is not.
def bond_step_fused(H_prev, H0, H_next, h, Wpk, bias, lay, act, act_param, first_step, M_out=None, drop_bits=None,
                    drop_scale=1.0):
    """H_next[e] = tau(H_0[e] + b + W_h . M[e]),  M = message of g(H_prev), g = tau on the first step (include/dmpnn.h)."""
    hp = _pad16(h)
    f = _act(H_prev.float()[: lay.E, :hp], act if first_step else ACT_NONE, act_param)
    if first_step:
        f = _bf(f)                                    # act_word: tau applied to the bf16 word, result a bf16 word
    A = _sibling_sum_packed(f, lay, through_rev=False)     # A row r is the message of edge rev(r)
    M = torch.zeros((lay.E, hp))
    M[lay.rev_row.long()] = A
    Z = _mma(M, Wpk, h) + H0[: lay.E, :hp].float()
    if bias is not None:
        Z[:, :h] = Z[:, :h] + bias.float()          # the kernel's bias is zero past h
    Y = _act(Z, act, act_param)
    if drop_bits is not None:           # keep ? tau(z) * scale : 0 in f32, one rounding (the kernel's epilogue)
        nj = hp // 16
        keep = ((drop_bits[: lay.E].to(torch.int32).unsqueeze(-1) >> torch.arange(16, dtype=torch.int32)) & 1).reshape(lay.E, nj * 16)
        Y = Y * keep.float() * drop_scale
    H_next[: lay.E, :hp] = Y.to(H_next.dtype)
    if M_out is not None:
        M_out[: lay.E, :hp] = M.to(M_out.dtype)


def bond_step_bwd_fused(dZ, Yact, dOut, h, WpkT, lay, act, act_param, G_out=None, y_is_preact=False, addends=()):
    """dOut = ((S.P) dZ) . W_h [* tau'(Yact)] [+ addends];  G_out = (S.P) dZ   (WpkT holds B = W_h^T of A . B^T)."""
    hp = _pad16(h)
    G = _sibling_sum_packed(dZ.float()[: lay.E, :hp], lay, through_rev=True)
    D = _mma(G, WpkT, h)
    if Yact is not None:
        D = D * _dact(Yact[: lay.E, :hp].float(), act, act_param, y_is_preact)
    for a in addends:
        D = D + a[: lay.E, :hp].float()
    dOut[: lay.E, :hp] = D.to(dOut.dtype)
    if G_out is not None:
        G_out[: lay.E, :hp] = G.to(G_out.dtype)


def atom_tables(lay):
    """engine.atom_tables: the emulated atom step needs no tile tables"""
    return None


def _neighbour_sum_packed(f, lay):
    """The ATOM gather of the fused kernel, rounding for rounding: A row v = sum over the in-edges e of v of f[src(e)], added in
    slot order as packed bf16 (`__hadd2(__hadd2(__hadd2(a0, a1), a2), a3)`, an absent neighbour is +0) for in-degree <= 4 and in f32
    with one rounding otherwise.  `f` is bf16-valued f32 [V, C]."""
    V = lay.V
    rowptr, src = lay.rowptr.long(), lay.src_row.long()
    g0 = rowptr[:V]
    d = rowptr[1:V + 1] - g0
    r = torch.arange(V)
    vals = []
    for k in range(4):
        ok = (k < d) & (d <= 4)
        x = torch.where(ok, src[torch.clamp(g0 + k, max=max(lay.E - 1, 0))], r)
        vals.append(torch.where(ok.unsqueeze(1), f[x], 0.0))
    small = _bf(_bf(_bf(vals[0] + vals[1]) + vals[2]) + vals[3])
    big = d > 4
    if bool(big.any()):
        s = torch.zeros((V, f.shape[1])).index_add_(0, lay.dst_row.long(), f[src])
        small = torch.where(big.unsqueeze(1), _bf(s), small)
    return small


def atom_step_fused(H_prev, H0, H_next, h, Wpk, bias, lay, act, act_param, first_step, N_out=None):
    """H_next[v] = tau(H0[v] + b + W . N[v]),  N = neighbour sum of g(H_prev), g = tau on the first step (include/dmpnn.h)."""
    V, hp = lay.V, _pad16(h)
    f = _act(H_prev.float()[:V, :hp], act if first_step else ACT_NONE, act_param)
    if first_step:
        f = _bf(f)
    N = _neighbour_sum_packed(f, lay)
    Z = _mma(N, Wpk, h) + H0[:V, :hp].float()
    if bias is not None:
        Z[:, :h] = Z[:, :h] + bias.float()
    H_next[:V, :hp] = _act(Z, act, act_param).to(H_next.dtype)
    if N_out is not None:
        N_out[:V, :hp] = N.to(N_out.dtype)


def atom_step_bwd_fused(dZ, Yact, dOut, h, WpkT, lay, act, act_param, G_out=None, y_is_preact=False, addends=()):
    """dOut = (A dZ) . W [* tau'(Yact)] [+ addends];  G_out = A dZ   (WpkT holds B = W^T of A . B^T)."""
    V, hp = lay.V, _pad16(h)
    G = _neighbour_sum_packed(dZ.float()[:V, :hp], lay)
    D = _mma(G, WpkT, h)
    if Yact is not None:
        D = D * _dact(Yact[:V, :hp].float(), act, act_param, y_is_preact)
    for a in addends:
        D = D + a[:V, :hp].float()
    dOut[:V, :hp] = D.to(dOut.dtype)
    if G_out is not None:
        G_out[:V, :hp] = G.to(G_out.dtype)


def bond_message_bwd_masked(dM, Yact, lay, Ccols, out, *, act, act_param=0.0):
    if lay.E == 0:
        return
    G = torch.zeros((lay.E, Ccols))
    bond_message(dM, lay, Ccols, G, permute_on_read=True)
    out[: lay.E, :Ccols] = (G * _dact(Yact[: lay.E, :Ccols].float(), act, act_param, False)).to(out.dtype)


def sum_act_bwd(Zs, G, Ypre, out, R, Ccols, *, act, act_param=0.0):
    if R == 0:
        return
    acc = torch.zeros((R, Ccols))
    for z in Zs:
        acc = acc + z[:R, :Ccols].float()
    if G is not None:
        acc = acc + G[:R, :Ccols].float() * _dact(Ypre[:R, :Ccols].float(), act, act_param, True)
    out[:R, :Ccols] = acc.to(out.dtype)


def segments_of(batch, n_seg=None):
    """engine.segments_of for a bare sorted `batch` (dmpnn_sorted_index_to_ptr): (ptr int32 [B + 1], seg_of_row int32, B)."""
    seg = getattr(batch, "_dmpnn_seg", None)
    if seg is not None and getattr(batch, "_dmpnn_seg_v", None) == batch._version and (n_seg is None or seg[2] == n_seg):
        return seg
    b = batch.numpy()
    assert np.all(np.diff(b) >= 0)
    B = (int(b.max()) + 1 if b.size else 0) if n_seg is None else int(n_seg)
    if b.size and int(b.max()) >= B:
        raise engine.DmpnnError(f"`batch` holds a molecule index outside [0, {B})")
    ptr = np.searchsorted(b, np.arange(B + 1), side="left").astype(np.int32)
    return torch.from_numpy(ptr), batch.to(torch.int32), B


def patch_engine(monkeypatch):
    """Route engine.py's kernel wrappers to the emulations above (host-logic tests only)."""
    for name in ("linear_fwd", "linear_wgrad", "segment_sum", "segment_bcast", "bond_message", "rev_average", "act_bwd",
                 "build_layout", "pack_weight_tc", "pack_weight_bf16", "concat_bf16", "linear_tc", "wgrad_tc", "wgrad_tc_multi", "column_sum",
                 "pack_weight_x3", "linear_x3", "wgrad_x3", "bn_train_fwd", "bn_bwd", "mse_loss", "concat_f32", "dropout_keep_bits",
                 "bond_step_fused", "bond_step_bwd_fused", "bond_message_bwd_masked", "sum_act_bwd", "scale_mask_",
                 "atom_step_fused", "atom_step_bwd_fused", "atom_tables"):
        monkeypatch.setattr(engine, name, globals()[name])
    monkeypatch.setattr(engine, "_require_cuda", lambda *ts: None)
    monkeypatch.setattr(engine, "_fused_available", lambda: True)
    import chemprop_b200.nn.agg as agg_mod
    import chemprop_b200.nn.constrainer as con_mod

    monkeypatch.setattr(engine, "segments_of", segments_of)
    monkeypatch.setattr(agg_mod, "segments_of", segments_of)
    monkeypatch.setattr(con_mod, "segments_of", segments_of)
