"""GPU tier: the column permutation of the packed weight images and the epilogues that store whole column runs through it.

Both weight packers (k_pack_weight of the fused depth step, k_pack_weight_tc of k_linear_tc) put W row acc_out_col(j, nc) at
row j of every chunk / work item (csrc/tc_common.cuh), so that each thread's wgmma accumulator fragment covers contiguous
output columns: the epilogues then load their operands and store their results as 16-byte runs (8-byte in a 16-column tail).
Checked here: the images row by row against a restatement of the permutation, and every epilogue at every chunk / item width
it can meet -- columns [0, h) against a torch reference, [h, pad16(h)) exactly zero, [pad16(h), ld) untouched (NaN)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def acc_out_col(j, nc):
    """Output column held by accumulator column j of an nc-column chunk (tc::acc_out_col)."""
    base = j & ~31
    rem = nc - base
    if rem >= 32:      # 32 g + 8 b + 2 q + e  ->  32 g + 8 q + 2 b + e
        return base + ((j >> 1) & 3) * 8 + ((j >> 3) & 3) * 2 + (j & 1)
    if rem >= 16 and j - base < 16:      # 16-column tail: 8 b + 2 q + e  ->  4 q + 2 b + e
        return base + ((j >> 1) & 3) * 4 + ((j >> 3) & 1) * 2 + (j & 1)
    return j


def test_permutation_is_a_bijection_of_each_chunk():
    for nc in list(range(8, 153, 8)):
        assert sorted(acc_out_col(j, nc) for j in range(nc)) == list(range(nc)), nc
    # thread q's runs: 8 contiguous columns per 32-column group, 4 in a 16-column tail
    for q in range(4):
        assert [acc_out_col(8 * b + 2 * q + e, 32) for b in range(4) for e in range(2)] == list(range(8 * q, 8 * q + 8))
        assert [acc_out_col(8 * b + 2 * q + e, 16) for b in range(2) for e in range(2)] == list(range(4 * q, 4 * q + 4))


def _unswizzle(block_u16, rows):
    """rows x 128-byte K-major SWIZZLE_128B block (16-byte chunk c of row r stored at chunk c ^ (r & 7)) -> [rows, 64]."""
    blk = block_u16.reshape(rows, 8, 8)
    r = np.arange(rows)[:, None]
    return blk[r, np.arange(8)[None, :] ^ (r & 7)].reshape(rows, 64)


def _bf16_bits(W, rows, cols):
    """W rounded to bf16, zero-padded to [rows, cols], as uint16 bit patterns."""
    out = torch.zeros(rows, cols, dtype=torch.bfloat16)
    out[: W.shape[0], : W.shape[1]] = W.detach().float().cpu().bfloat16()
    return out.view(torch.int16).numpy().view(np.uint16)


@pytest.mark.parametrize("N,K", [(300, 200), (200, 300), (256, 256), (12, 44), (236, 300)])
def test_fused_step_weight_image_rows(N, K):
    from chemprop_b200.engine import pack_weight_bf16

    W = torch.randn(N, K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N + K))
    for B in (W, W.t().contiguous()):           # W_h for the forward step, W_h^T for the mirror
        n_, k_ = B.shape
        hpN, hpK = (n_ + 15) // 16 * 16, (k_ + 15) // 16 * 16
        nslab = (hpK + 63) // 64
        img = pack_weight_bf16(B).cpu().numpy().view(np.uint16)
        assert img.size == nslab * hpN * 64
        ref = _bf16_bits(B, hpN, nslab * 64)
        for c in range((hpN + 79) // 80):
            rows = min(80, hpN - 80 * c)
            for s in range(nslab):
                off = (80 * c * nslab + s * rows) * 64
                got = _unswizzle(img[off: off + rows * 64], rows)
                want = ref[[80 * c + acc_out_col(j, rows) for j in range(rows)], 64 * s: 64 * s + 64]
                assert np.array_equal(got, want), (N, K, B.shape, c, s)


@pytest.mark.parametrize("N,K", [(300, 200), (200, 136), (152, 300), (8, 64), (56, 448)])
def test_linear_tc_weight_image_rows(N, K):
    from chemprop_b200.engine import pack_weight_tc

    W = torch.randn(N, K, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N * K))
    for transpose in (False, True):
        Wm = W.t().contiguous() if transpose else W          # packed B[n][k] = W[k][n] when transposed
        B = Wm.t() if transpose else Wm
        n_, k_ = B.shape
        Npad, Kpad = (n_ + 15) // 16 * 16, (k_ + 15) // 16 * 16
        nslab = (Kpad + 63) // 64
        img = pack_weight_tc(Wm, transpose=transpose).cpu().numpy().view(np.uint16)
        assert img.size == nslab * Npad * 64
        ref = _bf16_bits(B, Npad, nslab * 64)
        perm = [r // 152 * 152 + acc_out_col(r % 152, min(152, Npad - r // 152 * 152)) for r in range(Npad)]
        for s in range(nslab):
            got = _unswizzle(img[s * Npad * 64: (s + 1) * Npad * 64], Npad)
            assert np.array_equal(got, ref[perm, 64 * s: 64 * s + 64]), (N, K, transpose, s)


# ---- fused depth step: every last-chunk width (hp - 80 * (nchunks - 1) = 16, 32, 48, 64, 80) ------------------------------
def _check_columns(out, ref, h, what, atol=2e-2):
    hp = (h + 15) // 16 * 16
    o = out.float()
    assert torch.isfinite(o[:, :hp]).all(), f"{what}: columns below pad16(h) left unwritten"
    torch.testing.assert_close(o[:, :h], ref.float(), rtol=2 ** -6, atol=atol, msg=lambda m: f"{what}: {m}")
    assert hp == h or not bool(o[:, h:hp].ne(0).any()), f"{what}: columns [h, pad16(h)) not zero"
    assert bool(torch.isnan(o[:, hp:]).all()), f"{what}: stray writes in [pad16(h), ld)"


def _hidden(rows, h, ld, g, scale=0.7):
    t = torch.zeros(rows, ld, dtype=torch.bfloat16, device="cuda")
    t[:, :h] = (torch.randn(rows, h, device="cuda", generator=g) * scale).bfloat16()
    return t


def _nan_like(t):
    return torch.full_like(t, float("nan"))


WIDTHS = [256, 268, 284, 300, 236, 12, 44]      # last chunk 16, 32, 48, 64, 80 columns; one-chunk 16 and 48


@pytest.mark.parametrize("h", WIDTHS)
def test_bond_step_epilogue_columns(h):
    from chemprop_b200 import _lib
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import bond_step_bwd_fused, bond_step_fused, get_layout, pack_weight_bf16

    bmg = BatchMolGraph(make_molecules(300, seed=h, shuffle_edges=True))
    bmg.to("cuda")
    lay = get_layout(bmg)
    hp = (h + 15) // 16 * 16
    ld = hp + 32                                  # room past pad16(h) that no launch may write
    g = torch.Generator(device="cuda").manual_seed(h)
    H0, dZ, a1 = (_hidden(lay.E, h, ld, g) for _ in range(3))
    Hp = _hidden(lay.E, h, ld, g, 1.0).relu_()
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    Wb = W.bfloat16().float()
    rev, dst = lay.rev_row.long(), lay.dst_row.long()
    R, T = _lib.ACT_RELU, _lib.ACT_TANH

    def message(X):                               # row e' holds M[rev(e')] (bf16), forward
        return (torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)[dst] - X).bfloat16().float()

    # forward, ReLU + bias + dropout keep bits
    nj = hp // 16
    bits = torch.randint(-32768, 32768, (lay.E, nj), device="cuda", dtype=torch.int32, generator=g)
    drop = bits.to(torch.int16).contiguous()
    keep = (((bits & 0xFFFF).unsqueeze(-1) >> torch.arange(16, device="cuda")) & 1).reshape(lay.E, hp)[:, :h].float()
    Hn = _nan_like(H0)
    bond_step_fused(Hp, H0, Hn, h, pack_weight_bf16(W), b, lay, R, 0.0, False, drop_bits=drop, drop_scale=1.25)
    torch.cuda.synchronize()
    ref = torch.zeros(lay.E, h, device="cuda")
    ref[rev] = torch.relu(message(Hp[:, :h].float()) @ Wb.t() + H0[rev, :h].float() + b)
    _check_columns(Hn, (ref * keep * 1.25).bfloat16(), h, "forward relu + bias + dropout")

    # forward, first step, tanh + bias
    Hn = _nan_like(H0)
    bond_step_fused(H0, H0, Hn, h, pack_weight_bf16(W), b, lay, T, 0.0, True)
    torch.cuda.synchronize()
    ref = torch.zeros(lay.E, h, device="cuda")
    ref[rev] = torch.tanh(message(torch.tanh(H0[:, :h].float()).bfloat16().float()) @ Wb.t() + H0[rev, :h].float() + b)
    _check_columns(Hn, ref.bfloat16(), h, "forward tanh first step")

    # mirror: G = (S.P) dZ, D = G . W_h
    WpkT = pack_weight_bf16(W.t().contiguous())
    X = dZ[:, :h].float()[rev]
    D = (torch.zeros(lay.V, h, device="cuda").index_add_(0, dst, X)[dst] - X).bfloat16().float() @ Wb
    for Y, what in ((Hp, "MODE 1"), (None, "MODE 2")):
        dO = _nan_like(H0)
        bond_step_bwd_fused(dZ, Y, dO, h, WpkT, lay, R, 0.0)
        torch.cuda.synchronize()
        ref = D * (Y[:, :h].float() > 0).float() if Y is not None else D
        _check_columns(dO, ref.bfloat16(), h, what)
    for n_add in (0, 1, 2):
        adds = (dZ, a1)[:n_add]
        dO = _nan_like(H0)
        bond_step_bwd_fused(dZ, H0, dO, h, WpkT, lay, R, 0.0, y_is_preact=True, addends=adds)
        torch.cuda.synchronize()
        ref = (D * (H0[:, :h].float() > 0).float()).bfloat16().float()
        for a in adds:
            ref = ref + a[:, :h].float()
        _check_columns(dO, ref.bfloat16(), h, f"MODE 3, {n_add} addends", atol=6.5e-2)


@pytest.mark.parametrize("h", WIDTHS)
def test_atom_step_epilogue_columns(h):
    from chemprop_b200 import _lib
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import atom_step_bwd_fused, atom_step_fused, get_layout, pack_weight_bf16
    from tests.test_gpu_fused_step import _neighbour_sum

    bmg = BatchMolGraph(make_molecules(300, seed=h + 1, shuffle_edges=True, min_atoms=1))
    bmg.to("cuda")
    lay = get_layout(bmg)
    hp = (h + 15) // 16 * 16
    ld = hp + 32
    g = torch.Generator(device="cuda").manual_seed(h + 1)
    H0, dZ = (_hidden(lay.V, h, ld, g) for _ in range(2))
    Hp = _hidden(lay.V, h, ld, g, 1.0).relu_()
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    Wb = W.bfloat16().float()

    Hn = _nan_like(H0)
    atom_step_fused(Hp, H0, Hn, h, pack_weight_bf16(W), b, lay, _lib.ACT_RELU, 0.0, False)
    torch.cuda.synchronize()
    ref = torch.relu(_neighbour_sum(lay, Hp[:, :h].float()) @ Wb.t() + H0[:, :h].float() + b)
    _check_columns(Hn, ref.bfloat16(), h, "atom forward")

    dO = _nan_like(H0)
    atom_step_bwd_fused(dZ, Hp, dO, h, pack_weight_bf16(W.t().contiguous()), lay, _lib.ACT_RELU, 0.0)
    torch.cuda.synchronize()
    ref = (_neighbour_sum(lay, dZ[:, :h].float()) @ Wb) * (Hp[:, :h].float() > 0).float()
    _check_columns(dO, ref.bfloat16(), h, "atom mirror", atol=3e-2)


# ---- k_linear_tc: items of 152 columns (4 groups + 16-column tail + 8-column tail), a 56-column second item at N = 200 ----
@pytest.mark.parametrize("N", [300, 200, 152, 8])
def test_linear_tc_epilogue_columns(N):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import linear_tc, linear_tc_rows, pack_weight_tc

    R, K = 1000, 136
    g = torch.Generator(device="cuda").manual_seed(N)
    A = torch.zeros(R, 144, dtype=torch.bfloat16, device="cuda")
    A[:, :K] = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    Wpk = pack_weight_tc(W)
    Z = A[:, :K].float() @ W.bfloat16().float().t()
    Np = (N + 15) // 16 * 16
    ldc = Np + 32

    def check(out, ref, what, pad_zero=True, atol=2e-3):
        o = out.float()
        torch.testing.assert_close(o[:, :N], ref.float(), rtol=2 ** -7, atol=atol, msg=lambda m: f"{what}: {m}")
        if pad_zero:
            assert not bool(o[:, N:Np].ne(0).any()), f"{what}: columns [N, pad16(N)) not zero"
            assert bool(torch.isnan(o[:, Np:]).all()), f"{what}: stray writes past pad16(N)"
        else:
            assert bool(torch.isnan(o[:, N:]).all()), f"{what}: stray writes past N"

    # bf16 epilogue: act(acc + bias + residual)
    res = torch.zeros(R, ldc, dtype=torch.bfloat16, device="cuda")
    res[:, :N] = torch.randn(R, N, device="cuda", generator=g).bfloat16()
    out = torch.full((R, ldc), float("nan"), dtype=torch.bfloat16, device="cuda")
    linear_tc(A, K, Wpk, N, out, bias=b, res=res, act=_lib.ACT_RELU)
    torch.cuda.synchronize()
    check(out, torch.relu(Z + b + res[:, :N].float()).bfloat16(), "bf16 epilogue", atol=4e-3)

    # f32 epilogue: columns [0, N) only; a row stride of 4k floats takes the 16-byte stores, 4k + 2 the 8-byte ones
    for ldf in (Np + 16, Np + 18):
        outf = torch.full((R, ldf), float("nan"), device="cuda")
        linear_tc_rows(A, K, Wpk, N, outf, bias=b, act=_lib.ACT_TANH)
        torch.cuda.synchronize()
        check(outf, torch.tanh(Z + b), f"f32 epilogue, ldc {ldf}", pad_zero=False, atol=1e-5)

    # mirror epilogue: out[out_row[r]] = (acc + res[res_row[r]]) * tau'(Y[out_row[r]])
    out_row = torch.randperm(R, device="cuda", generator=g).to(torch.int32)
    res_row = torch.randint(0, R, (R,), device="cuda", generator=g).to(torch.int32)
    Y = torch.zeros(R, ldc, dtype=torch.bfloat16, device="cuda")
    Y[:, :N] = torch.randn(R, N, device="cuda", generator=g).relu().bfloat16()
    outm = torch.full((R, ldc), float("nan"), dtype=torch.bfloat16, device="cuda")
    linear_tc_rows(A, K, Wpk, N, outm, act=_lib.ACT_RELU, Y=Y, out_row=out_row, res=res, res_row=res_row)
    torch.cuda.synchronize()
    q = out_row.long()
    ref = torch.empty(R, N, device="cuda")
    ref[q] = (Z + res[res_row.long(), :N].float()) * (Y[q, :N].float() > 0).float()
    check(outm, ref.bfloat16(), "mirror epilogue", atol=4e-3)
