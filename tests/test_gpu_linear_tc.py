"""GPU tier: the bf16 tier's tensor-core GEMMs outside the fused depth step, against float64.

k_linear_tc (dmpnn_linear_tc_bf16 / dmpnn_linear_tc_rows_bf16) runs W_i, W_o, every dX = dY . W of the mirror and the
mol-atom-bond read-outs in three epilogues: bf16 act(acc + bias + res), f32 act(acc + bias), and the mirror's
(acc + res) * tau'(Y).  With ACT x HAS_BIAS that is 25 instantiations.  k_wgrad_tc (dmpnn_wgrad_tc(_multi)_bf16) computes
every weight gradient of the tier.

(a) Exact: integer-valued operands, so that every partial sum is an integer below 2^24 and the f32 accumulator is exact in
    any order.  A dropped, doubled or misaddressed row block, k slab, term, tail or stride shows whatever the tolerance, and a
    bf16 store must equal torch's round-to-nearest-even of the f64 value.
(b) Float64 bounds with the kernel's rounding points on random data, one case per instantiation
    (`test_cases_cover_every_instantiation`): half a bf16 ulp + Lip(tau) 2K u sum|a w| + the f32 rounding of tau / tau' per
    element, and a mean error <= 0.6 of the mean bound, which round-to-nearest meets and truncation does not.  Pre-activations
    reach |z| < 1e-3 and z <= -8, Y holds exact +0 and -0.  k_wgrad_tc, whose products of bf16 operands are exact in f32, is
    held to the fp32 tier's GEMM bound at the tier's row counts: worst <= 1e-5, mean <= 1e-6 of sum |terms|, with the slot count
    and accumulator chain length each case runs asserted.
(c) Edges: R from 0 to 1.25 M, N and K on both sides of every tile, slab and work-item boundary, NaN in every operand column past
    K / N, in operand rows past R, in the mirror residual's and Y's padding, and in every output row or column no launch may
    write; the host-side argument checks; determinism.  dmpnn_linear_tc_bf16 requires zeros in its residual's columns
    [N, pad16(N)) (include/dmpnn.h): its tests put zeros there and NaN past pad16(N)."""
import ctypes
import gc

import pytest
import torch

from tests.test_gpu_fused_activations import MEAN_BAR, U, _check_bound, _code, _dtau64, _lip, _tau64

pytestmark = pytest.mark.gpu

NAN = float("nan")
ACTS = ("none", "relu", "leakyrelu", "tanh", "elu")
CHUNK = 1 << 17                  # rows per f64 reference chunk: peak device memory stays a few GB


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _p16(n):
    return (n + 15) // 16 * 16


def _ld(n):
    """A row stride with spare columns past pad16(n) (NaN: nothing may read or write them)."""
    return _p16(n) + 16


def _buf(rows, ld, dtype=torch.bfloat16):
    return torch.full((rows, ld), NAN, dtype=dtype, device="cuda")


def _fill_(dst, make):
    """dst[r0:r1] = make(r1 - r0), chunk by chunk (million-row operands without million-row temporaries)."""
    for r0 in range(0, dst.shape[0], CHUNK):
        r1 = min(dst.shape[0], r0 + CHUNK)
        dst[r0:r1] = make(r1 - r0).to(dst.dtype)


def _ints(g, lo, hi):
    return lambda n, c: torch.randint(lo, hi + 1, (n, c), device="cuda", generator=g, dtype=torch.int32)


def _report(group, case, worst, mean):
    print(f"[gemm-tc] {group} {case}: worst err / bound {worst:.3f}, mean {mean:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# (a) k_linear_tc, exact
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,K,N,act", [
    (1000, 448, 304, "none"), (1000, 448, 304, "relu"), (1000, 448, 304, "leakyrelu"),     # seven k slabs, two items
    (300, 14, 153, "none"), (300, 14, 153, "leakyrelu"),        # one k16 step; a 1-column 8-column tail
    (129, 193, 8, "relu"), (65, 406, 300, "leakyrelu"), (127, 8, 1, "none"), (64, 384, 129, "relu"),
    (1_250_000, 86, 300, "leakyrelu"),                          # ~10 k tiles: the mbarrier phases wrap thousands of times
])
def test_linear_tc_exact(R, K, N, act):
    """Integer A and W in [-2, 2], a bias on a 2^-4 grid, an integer residual and a slope of 1/4: the accumulator is exact,
    so every epilogue must give torch's round-to-nearest-even of the f64 value, bit for bit.  bf16, f32 (16-byte aligned
    rows and rows that are not) and mirror epilogues; NaN in A past K and past R, in the mirror residual's and Y's columns
    [N, pad16(N)), and in every output element no launch may write."""
    from chemprop_b200.engine import linear_tc, linear_tc_rows, pack_weight_tc

    g = torch.Generator(device="cuda").manual_seed(R + K + N)
    p = 0.25
    Np, ld, extra = _p16(N), _ld(N), 8
    A = _buf(R + extra, (K + 7) // 8 * 8 + 8)
    _fill_(A[:R, :K], lambda n: _ints(g, -2, 2)(n, K))
    W = _ints(g, -2, 2)(N, K).float()
    b = torch.randint(-64, 65, (N,), device="cuda", generator=g).float() / 16
    res = _buf(R, ld)
    _fill_(res[:, :N], lambda n: _ints(g, -8, 8)(n, N))
    res[:, N:Np] = 0                     # dmpnn_linear_tc_bf16's precondition; the mirror's residual keeps NaN there
    res_m = _buf(R, ld)
    res_m[:, :N] = res[:, :N]
    Wpk = pack_weight_tc(W)
    code = _code(act)

    out = _buf(R + extra, ld)
    linear_tc(A, K, Wpk, N, out, bias=b, res=res, act=code, act_param=p, R=R)
    outs = {}
    for ldf in (_p16(N + 4), _p16(N + 4) + 2):           # f32_v4 rows, then rows 8 bytes off 16-byte alignment
        outs[ldf] = _buf(R + extra, ldf, torch.float32)
        linear_tc_rows(A, K, Wpk, N, outs[ldf], R=R, bias=b, act=code, act_param=p)
    Rc = R + 40
    out_row = torch.randperm(Rc, device="cuda", generator=g)[:R].to(torch.int32)
    res_row = torch.randint(0, R, (R,), device="cuda", generator=g, dtype=torch.int32)
    Y = _buf(Rc, ld)
    _fill_(Y[:, :N], lambda n: _ints(g, -2, 2)(n, N))
    Y[3::7, 1:N:3] = -0.0
    outm = _buf(Rc, ld)
    linear_tc_rows(A, K, Wpk, N, outm, R=R, act=code, act_param=p, Y=Y, out_row=out_row, res=res_m, res_row=res_row)
    torch.cuda.synchronize()

    Wd, bd = W.double(), b.double()
    q, s = out_row.long(), res_row.long()
    for r0 in range(0, R, CHUNK):
        r1 = min(R, r0 + CHUNK)
        Z = A[r0:r1, :K].double() @ Wd.t()
        want = _tau64(act, p, Z + bd + res[r0:r1, :N].double()).bfloat16()
        assert torch.equal(out[r0:r1, :N], want), ("bf16 epilogue", r0)
        for ldf, o in outs.items():
            assert torch.equal(o[r0:r1, :N].double(), _tau64(act, p, Z + bd)), ("f32 epilogue", ldf, r0)
        d = _dtau64(act, p, Y[q[r0:r1], :N].double(), False)
        want = ((Z + res[s[r0:r1], :N].double()) * d).bfloat16()
        assert torch.equal(outm[q[r0:r1], :N], want), ("mirror epilogue", r0)
    assert not bool(out[:R, N:Np].float().ne(0).any()), "bf16: columns [N, pad16(N)) not zero (residual padding leaked)"
    assert not bool(outm[q, N:Np].float().ne(0).any()), "mirror: columns [N, pad16(N)) not zero"
    assert bool(torch.isnan(out[:R, Np:].float()).all()) and bool(torch.isnan(out[R:].float()).all())
    for o in outs.values():
        assert bool(torch.isnan(o[:R, N:]).all()) and bool(torch.isnan(o[R:]).all())
    assert bool(torch.isnan(outm[q, Np:].float()).all())
    untouched = torch.ones(Rc, dtype=torch.bool, device="cuda")
    untouched[q] = False
    assert bool(torch.isnan(outm[untouched].float()).all())


def test_linear_tc_transposed_column_slice_exact():
    """dX = dY . W_o[:, d_v:] as the mirror packs it: B[n][k] = W_o[k][d_v + n], a transposed column slice (ldw = d_v + h)."""
    from chemprop_b200.engine import linear_tc, pack_weight_tc

    g = torch.Generator(device="cuda").manual_seed(0)
    h, d_v, R = 300, 72, 4000
    Wo = _ints(g, -2, 2)(h, d_v + h).float()
    dY = _buf(R + 5, _ld(h))
    dY[:R, :h] = _ints(g, -2, 2)(R, h).bfloat16()
    out = _buf(R + 5, _ld(h))
    linear_tc(dY, h, pack_weight_tc(Wo[:, d_v:], transpose=True), h, out, R=R)
    torch.cuda.synchronize()
    assert torch.equal(out[:R, :h], (dY[:R, :h].double() @ Wo[:, d_v:].double()).bfloat16())
    assert not bool(out[:R, h:_p16(h)].float().ne(0).any()) and bool(torch.isnan(out[:R, _p16(h):].float()).all())
    assert bool(torch.isnan(out[R:].float()).all())


# ---------------------------------------------------------------------------------------------------------------------
# (b) k_linear_tc, every instantiation against float64
# ---------------------------------------------------------------------------------------------------------------------
def _instantiations():
    """(ACT, HAS_BIAS, EPI) of every k_linear_tc instantiation the two entry points launch: bf16 and f32 epilogues with and
    without bias for every activation, the mirror epilogue (no bias) for every activation."""
    s = {(a, b, e) for a in ACTS for b in (0, 1) for e in ("bf16", "f32")}
    return s | {(a, 0, "mirror") for a in ACTS}


# (R, K, N): every K slab count 1-7 with K % 16 and K % 64 tails, N over one and two 152-column items with 8- / 16-column tails
SHAPES = [(3000, 300, 300), (1000, 86, 152), (700, 448, 153), (513, 447, 304), (300, 406, 129), (257, 384, 200),
          (129, 193, 256), (128, 192, 64), (127, 134, 16), (65, 14, 8), (64, 16, 1), (63, 372, 300), (1, 8, 300),
          (20000, 328, 300)]


def _cases():
    out = []
    for i, key in enumerate(sorted(_instantiations())):
        p = {"leakyrelu": (0.1, 0.3), "elu": (1.0, 0.5)}.get(key[0], (0.7, 0.7))[i % 2]
        out.append((key, SHAPES[i % len(SHAPES)], p))
    return out


CASES = _cases()


def _case_id(c):
    (act, bias, epi), (R, K, N), p = c
    return "-".join(x for x in (epi, act, "bias" if bias else "", f"p{p}" if act in ("leakyrelu", "elu") else "",
                                f"R{R}-K{K}-N{N}") if x)


def test_cases_cover_every_instantiation():
    want = _instantiations()
    have = {c[0] for c in CASES}
    assert len(want) == 25
    assert have == want, (sorted(want - have), sorted(have - want))
    for act, p in (("leakyrelu", 0.1), ("leakyrelu", 0.3), ("elu", 1.0), ("elu", 0.5)):
        assert any(c[0] == (act, b, "bf16") and c[2] == p for c in CASES for b in (0, 1)), (act, p)
    print(f"[gemm-tc] k_linear_tc instantiations launched by the cases below: {len(have)} of {len(want)}")


def _operands(R, K, N, g, extra=8):
    """A (R + extra rows, NaN past K and past R) with A[:, 0] = 1, and W whose first N/8 output rows are scaled by 1e-3
    (|z| < ~1e-3 there) and whose next N/8 rows take -10 from that column (z <= -8: ELU's saturated region)."""
    A = _buf(R + extra, (K + 7) // 8 * 8 + 8)
    A[:R, :K] = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    A[:R, 0] = 1.0
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    nz, sat = max(1, N // 8), N // 4
    W[:nz] *= 1e-3
    W[nz:sat, 0] = -10.0
    return A, W, nz


def _banded(rows, N, g):
    """Pre-activations: a near-zero band, ELU's saturated region, N(0, 0.7^2) elsewhere."""
    x = torch.randn(rows, N, device="cuda", generator=g) * 0.7
    nz, sat = max(1, N // 8), N // 4
    x[:, :nz] = (torch.rand(rows, nz, device="cuda", generator=g) * 2 - 1) * 1e-3
    x[:, nz:sat] = -2 - 7 * torch.rand(rows, sat - nz, device="cuda", generator=g)
    return x


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_linear_tc_vs_f64(case):
    from chemprop_b200.engine import linear_tc, linear_tc_rows, pack_weight_tc

    (act, bias, epi), (R, K, N), p = case
    what = _case_id(case)
    g = torch.Generator(device="cuda").manual_seed(R + K + N + len(what))
    A, W, nz = _operands(R, K, N, g)
    Np, ld = _p16(N), _ld(N)
    Wpk = pack_weight_tc(W)
    Wb = W.bfloat16().double()                        # the packed image's rounding
    Ad = A[:R, :K].double()
    Z, Ua = Ad @ Wb.t(), Ad.abs() @ Wb.abs().t()
    code, lip = _code(act), _lip(act, p)

    if epi in ("bf16", "f32"):
        b = torch.randn(N, device="cuda", generator=g) * 0.1
        b[:nz] *= 1e-3
        bd = b.double() if bias else torch.zeros(N, dtype=torch.float64, device="cuda")
        rd = torch.zeros_like(Z)
        if epi == "bf16":
            res = _buf(R, ld)
            x = torch.randn(R, N, device="cuda", generator=g) * 0.5
            x[:, :nz] *= 1e-3
            res[:, :N] = x.bfloat16()
            res[:, N:Np] = 0             # the precondition of dmpnn_linear_tc_bf16 (include/dmpnn.h)
            out = _buf(R + 8, ld)
            linear_tc(A, K, Wpk, N, out, bias=b if bias else None, res=res, act=code, act_param=p, R=R)
            rd = res[:, :N].double()
        else:
            out = _buf(R + 8, _p16(N + 4) + 2 * (R % 2), torch.float32)      # odd R: rows not 16-byte aligned
            linear_tc_rows(A, K, Wpk, N, out, R=R, bias=b if bias else None, act=code, act_param=p)
        torch.cuda.synchronize()
        z = Z + bd + rd
        y = _tau64(act, p, z)
        delta = lip * (2 * K * U * Ua + 3 * U * (Z.abs() + bd.abs() + rd.abs())) + 8 * U * y.abs()
        worst, mean = _check_bound(out[:R, :N], y, delta, what, bf16_out=(epi == "bf16"))
        if epi == "bf16":
            assert not bool(out[:R, N:Np].float().ne(0).any()), f"{what}: columns [N, pad16(N)) not zero"
            assert bool(torch.isnan(out[:R, Np:].float()).all()), f"{what}: stray writes past pad16(N)"
        else:
            assert bool(torch.isnan(out[:R, N:]).all()), f"{what}: stray writes past N"
        assert bool(torch.isnan(out[R:].float()).all()), f"{what}: stray writes past row R"
        if act == "elu" and N >= 16 and R >= 64:
            assert z.min().item() < -8.0 and bool((z.abs() < 1e-3).any()), (what, "pre-activation bands not reached")
    else:
        Rc, Rres = R + 40, R // 2 + 3
        out_row = torch.randperm(Rc, device="cuda", generator=g)[:R].to(torch.int32)
        res_row = torch.randint(0, Rres, (R,), device="cuda", generator=g, dtype=torch.int32)
        res = _buf(Rres, ld)
        res[:, :N] = (torch.randn(Rres, N, device="cuda", generator=g) * 0.5).bfloat16()
        q, s = out_row.long(), res_row.long()
        D, r = Z, res[s, :N].double()
        worst, mean = 0.0, 0.0
        for pre in (False, True):
            zy = _banded(Rc, N, g)
            Y = _buf(Rc, ld)
            Y[:, :N] = (zy if pre else _tau64(act, p, zy.double())).bfloat16()
            Y[0::7, 0:N:5] = 0.0
            Y[3::7, 2:N:5] = -0.0
            out = _buf(Rc, ld)
            linear_tc_rows(A, K, Wpk, N, out, R=R, act=code, act_param=p, Y=Y, from_preact=pre, out_row=out_row, res=res,
                           res_row=res_row)
            torch.cuda.synchronize()
            d = _dtau64(act, p, Y[q, :N].double(), pre)
            ref = (D + r) * d
            delta = d.abs() * (2 * K * U * Ua + 2 * U * (D.abs() + r.abs())) + 8 * U * (1 + d.abs()) * (D + r).abs()
            w, m = _check_bound(out[q, :N], ref, delta, f"{what}, from_preact={pre}")
            worst, mean = max(worst, w), max(mean, m)
            assert not bool(out[q, N:Np].float().ne(0).any()), f"{what}: columns [N, pad16(N)) not zero"
            assert bool(torch.isnan(out[q, Np:].float()).all()), f"{what}: stray writes past pad16(N)"
            untouched = torch.ones(Rc, dtype=torch.bool, device="cuda")
            untouched[q] = False
            assert bool(torch.isnan(out[untouched].float()).all()), f"{what}: rows outside out_row written"
    _report("linear_tc", what, worst, mean)


def test_linear_tc_residual_padding_and_aliasing():
    """With the residual's columns [N, pad16(N)) zero (the precondition of dmpnn_linear_tc_bf16) and NaN past pad16(N), C's
    padding is exactly zero (the fused depth step reads it as zeros), also for ELU with a non-default alpha.  A residual that
    aliases C is refused."""
    from chemprop_b200 import DmpnnError
    from chemprop_b200.engine import ACT_ELU, linear_tc, pack_weight_tc

    g = torch.Generator(device="cuda").manual_seed(5)
    for N in (153, 300, 1):
        R, K = 300, 134
        A, W, _ = _operands(R, K, N, g)
        Wpk = pack_weight_tc(W)
        res = _buf(R, _ld(N))
        res[:, :N] = torch.randn(R, N, device="cuda", generator=g).bfloat16()
        res[:, N:_p16(N)] = 0
        out = _buf(R, _ld(N))
        linear_tc(A, K, Wpk, N, out, res=res, act=ACT_ELU, act_param=0.5, R=R)
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out[:, :N].float()).all())
        assert not bool(out[:, N:_p16(N)].float().ne(0).any()), (N, "columns [N, pad16(N)) not zero")
        assert bool(torch.isnan(out[:, _p16(N):].float()).all()), (N, "stray writes past pad16(N)")
    with pytest.raises(DmpnnError):
        linear_tc(A, K, Wpk, N, out, res=out, R=R)


# ---------------------------------------------------------------------------------------------------------------------
# k_wgrad_tc
# ---------------------------------------------------------------------------------------------------------------------
def _wgrad(dYs, X, R, N, K, dW, accumulate=False):
    from chemprop_b200.engine import wgrad_tc, wgrad_tc_multi

    if len(dYs) == 1:
        wgrad_tc(dYs[0], X, R, N, K, dW, accumulate=accumulate)
    else:
        wgrad_tc_multi(dYs, X, R, N, K, dW, accumulate=accumulate)


def _operand_rows(R, C, make, extra=5):
    """(R + extra) x (pad8(C) + 8) bf16: make(n, C) in [0:R, 0:C], NaN in every other column and row."""
    t = _buf(R + extra, (C + 7) // 8 * 8 + 8)
    if R:
        _fill_(t[:R, :C], lambda n: make(n, C))
    return t


def _wgrad64(dYs, X, R, N, K, absolute=False):
    """sum_t dY_t^T X (and sum_t |dY_t|^T |X|) in f64, chunk by chunk of rows."""
    ref = torch.zeros(N, K, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref) if absolute else None
    for r0 in range(0, R, CHUNK):
        r1 = min(R, r0 + CHUNK)
        x = X[r0:r1, :K].double()
        for dY in dYs:
            y = dY[r0:r1, :N].double()
            ref += y.t() @ x
            if absolute:
                mag += y.abs().t() @ x.abs()
            del y
        del x
    return ref, mag


@pytest.mark.parametrize("R,N,K,n_terms,accumulate,strided", [
    (0, 300, 300, 1, False, False), (0, 64, 86, 2, True, True),              # no row: dW = 0 (or unchanged)
    (1, 1, 8, 1, False, False), (63, 8, 14, 1, True, True), (64, 16, 16, 3, False, False),
    (65, 64, 86, 2, False, True), (127, 129, 134, 3, True, False), (128, 152, 192, 1, False, True),
    (129, 153, 193, 2, False, False), (3000, 305, 447, 1, True, True), (2000, 384, 448, 1, False, False),
    (2500, 300, 300, 5, True, False),           # two terms per launch at K = 300: launches of 2, 2 and 1 terms
    (1000, 200, 406, 4, False, True),           # seven X boxes: one term per launch
    (1500, 256, 328, 3, False, False),          # six X boxes: one term per launch
    (7000, 304, 86, 7, True, True),             # launches of 3, 3 and 1 terms
    (1_250_000, 300, 300, 1, False, True),      # C5's edge rows
    (1_250_000, 300, 86, 3, True, False),       # C5's W_i gradient: three terms in one launch
])
def test_wgrad_tc_exact(R, N, K, n_terms, accumulate, strided):
    """dY_t and X integer-valued ({-2..2}, or {-1, 0, 1} where a partial sum could pass 2^24): dW must equal the f64 (exact)
    reference bit for bit.  NaN in dY / X past N / K and past R; a strided dW whose neighbouring columns and rows are NaN
    and must stay NaN; accumulate onto integer-valued dW."""
    g = torch.Generator(device="cuda").manual_seed(R + N + K + n_terms)
    a = 2 if 4 * R * n_terms < (1 << 24) else 1
    dYs = [_operand_rows(R, N, _ints(g, -a, a)) for _ in range(n_terms)]
    X = _operand_rows(R, K, _ints(g, -a, a))
    big = torch.full((N + 2, K + 24), NAN, device="cuda") if strided else None
    dW = big[1:N + 1, 8:8 + K] if strided else torch.full((N, K), NAN, device="cuda")
    init = _ints(g, -1000, 1000)(N, K).float() if accumulate else torch.zeros(N, K, device="cuda")
    if accumulate:
        dW.copy_(init)
    _wgrad(dYs, X, R, N, K, dW, accumulate=accumulate)
    torch.cuda.synchronize()
    ref, _ = _wgrad64(dYs, X, R, N, K)
    assert float(ref.abs().max()) < (1 << 24)
    assert torch.equal(dW.double(), ref + init.double()), (R, N, K, n_terms, float((dW.double() - ref - init).abs().max()))
    if strided:
        keep = torch.ones_like(big, dtype=torch.bool)
        keep[1:N + 1, 8:8 + K] = False
        assert bool(torch.isnan(big[keep]).all()), "writes outside the strided dW view"


def _wgrad_geom(R, N, K, n_terms):
    """(row slots per output tile, k16 accumulate steps chained by one output of slot 0) of k_wgrad_tc: geom() in
    csrc/wgrad_tc.cu (128 x 192 output tiles, 64-row blocks, SM count / tiles slots), four k16 steps per block and term."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    tiles = -(-N // 128) * -(-_p16(K) // 192)
    slots = max(1, sms // tiles)
    blocks = -(-R // 64)
    return slots, -(-blocks // slots) * 4 * n_terms


@pytest.mark.parametrize("name,R,N,K,n_terms,slots,chain", [
    ("C2-W_h", 502_100, 300, 300, 1, 22, 1_428),
    ("C5-W_h", 1_250_000, 300, 300, 1, 22, 3_552),
    ("C5-W_i-3terms", 1_250_000, 300, 86, 3, 44, 5_328),
    ("C4-atom-W_h", 800_000, 300, 328, 1, 22, 2_276),       # K = h + d_e
    ("C4-atom-W_i", 800_000, 300, 134, 1, 44, 1_140),       # K = d_v + d_e
])
def test_wgrad_tc_vs_f64(name, R, N, K, n_terms, slots, chain):
    """Normal data at the tier's row counts.  Products of bf16 operands are exact in f32, so the error is the kernel's
    summation alone: worst <= 1e-5 and mean <= 1e-6 of sum |terms| (the fp32 tier's GEMM bound).  The slot count and chain
    length quoted are those of a 132-SM H100; two calls are bitwise equal."""
    got_slots, got_chain = _wgrad_geom(R, N, K, n_terms)
    if torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count == 132:
        assert (got_slots, got_chain) == (slots, chain), (got_slots, got_chain)
    g = torch.Generator(device="cuda").manual_seed(R + N + K)
    randn = lambda n, c: torch.randn(n, c, device="cuda", generator=g)      # noqa: E731
    dYs = [_operand_rows(R, N, randn) for _ in range(n_terms)]
    X = _operand_rows(R, K, randn)
    dW = torch.full((N, K), NAN, device="cuda")
    _wgrad(dYs, X, R, N, K, dW)
    dW2 = torch.full((N, K), NAN, device="cuda")
    _wgrad(dYs, X, R, N, K, dW2)
    torch.cuda.synchronize()
    assert torch.equal(dW, dW2), "not deterministic"
    ref, mag = _wgrad64(dYs, X, R, N, K, absolute=True)
    rel = (dW.double() - ref).abs() / mag
    worst, mean = rel.max().item(), rel.mean().item()
    print(f"[gemm-tc] wgrad_tc {name} (R {R}, N {N}, K {K}, {n_terms} terms, {got_slots} slots, chain {got_chain} k16 "
          f"steps): worst {worst:.2e}, mean {mean:.2e} of sum |terms|")
    assert worst <= 1e-5 and mean <= 1e-6, (name, worst, mean)


def test_host_checks_refuse_without_launch():
    """Arguments outside what the kernels support return an error from the host check, and nothing is written."""
    from chemprop_b200 import DmpnnError, _lib
    from chemprop_b200.engine import linear_tc, pack_weight_tc

    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(3)
    A = _operand_rows(64, 449, lambda n, c: torch.randn(n, c, device="cuda", generator=g))
    Wpk = pack_weight_tc(torch.randn(304, 448, device="cuda"))
    out = _buf(64, 400)
    for K, N in ((449, 300), (300, 305), (0, 300), (300, 0)):
        with pytest.raises(DmpnnError):
            linear_tc(A, K, Wpk, N, out, R=64)
    with pytest.raises(DmpnnError):
        pack_weight_tc(torch.randn(305, 64, device="cuda"))
    # R = 0: nothing to do, nothing written
    linear_tc(A, 300, Wpk, 300, out, R=0)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out.float()).all())

    ws = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
    dY = _operand_rows(64, 384, lambda n, c: torch.randn(n, c, device="cuda", generator=g))
    X = _operand_rows(64, 448, lambda n, c: torch.randn(n, c, device="cuda", generator=g))
    dW = torch.full((400, 456), NAN, device="cuda")

    def call(n_terms, lddy, N, K):
        arr = (ctypes.c_void_p * n_terms)(*([dY.data_ptr()] * n_terms))
        return lib.dmpnn_wgrad_tc_multi_bf16(ctypes.cast(arr, ctypes.c_void_p), n_terms, lddy, X.data_ptr(), X.stride(0), 64,
                                             N, K, dW.data_ptr(), dW.stride(0), 0, ws.data_ptr(), None)

    assert call(1, dY.stride(0), 300, 300) == 0                          # the valid call, for contrast
    torch.cuda.synchronize()
    dW.fill_(NAN)
    for args in ((1, dY.stride(0), 385, 300), (1, dY.stride(0), 300, 449), (4, dY.stride(0), 300, 86),
                 (3, dY.stride(0), 300, 448), (1, 302, 300, 300), (0, dY.stride(0), 300, 300)):
        assert call(*args) != 0, args
    torch.cuda.synchronize()
    assert bool(torch.isnan(dW).all()), "a refused call wrote dW"
    n = ctypes.c_size_t(0)
    assert lib.dmpnn_wgrad_tc_workspace_bytes(385, 300, ctypes.byref(n)) != 0
    assert lib.dmpnn_wgrad_tc_workspace_bytes(300, 449, ctypes.byref(n)) != 0


def test_concat_bf16():
    from chemprop_b200.engine import concat_bf16

    torch.manual_seed(1)
    V = torch.randn(50, 72, device="cuda")
    E = torch.randn(120, 14, device="cuda")
    i1 = torch.randint(0, 50, (120,), device="cuda", dtype=torch.int32)
    i2 = torch.randperm(120, device="cuda").to(torch.int32)
    out = torch.full((120, 96), float("nan"), dtype=torch.bfloat16, device="cuda")
    concat_bf16(V, 72, out, 120, idx1=i1, X2=E, K2=14, idx2=i2)
    ref = torch.cat([V[i1.long()], E[i2.long()], torch.zeros(120, 10, device="cuda")], 1).bfloat16()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("R,C,ld,gather", [(5000, 304, 304, True), (4097, 300, 304, False), (333, 64, 64, True), (7, 300, 320, True),
                                           (100000, 304, 304, True)])
def test_act_bwd_relu_bf16_fast_path(R, C, ld, gather):
    """All-bf16 ReLU instance of dmpnn_act_bwd (packed-pair mask kernel): dZ[r] = G[gidx[r]] where Y[r] > 0, else 0 --
    bit-exact, including y = 0, y = -0 and NaN (no gradient)."""
    from chemprop_b200.engine import ACT_RELU, act_bwd

    g = torch.Generator(device="cuda").manual_seed(R + C)
    nG = R // 2 + 1 if gather else R
    G = torch.randn(nG, ld, device="cuda", generator=g).bfloat16()
    Y = torch.randn(R, ld, device="cuda", generator=g).bfloat16()
    Y[::7, ::3] = 0.0
    Y[1::7, 1::3] = -0.0
    Y[2::11, 2::5] = float("nan")
    gidx = torch.randint(0, nG, (R,), device="cuda", dtype=torch.int32, generator=g) if gather else None
    dZ = torch.full((R, ld), 9.0, dtype=torch.bfloat16, device="cuda")
    act_bwd(G, Y, R, C, act=ACT_RELU, gidx=gidx, dZ=dZ)
    Gr = G[gidx.long()] if gather else G
    ref = torch.where(Y[:, :C] > 0, Gr[:, :C], torch.zeros((), dtype=torch.bfloat16, device="cuda"))
    assert torch.equal(dZ[:, :C], ref)
    assert bool((dZ[:, C:] == 9.0).all())                                 # nothing written beyond C
    dZ2 = torch.empty_like(dZ)
    act_bwd(G, Y, R, C, act=ACT_RELU, gidx=gidx, dZ=dZ2, from_preact=True)
    assert torch.equal(dZ2[:, :C], ref)


def test_column_sum():
    from chemprop_b200.engine import column_sum

    Y = torch.randn(70001, 320, device="cuda").bfloat16()
    out = torch.zeros(300, device="cuda")
    column_sum(Y, 70001, 300, out)
    torch.testing.assert_close(out, Y[:, :300].float().sum(0), rtol=1e-4, atol=1e-2)
