"""GPU tier: the fp32 tier at the hidden widths it accepts (d_h up to 4096 on the 3xTF32 GEMMs; chemprop's range is
300-2400, CheMeleon uses 2048), every result against float64 torch on the GPU.

- `column_sum`, the bias gradient of every x3 layer, on both sides of its 4-wide kernel's shared-memory limit;
- `linear_x3` / `wgrad_x3` at the wide shapes, and at C3's edge-row count (about 1.1 M rows at h = 600); each weight-
  gradient case states which row-slot regime of `k_wgrad_x3` it runs (geometry of `geom()` in csrc/gemm_x3.cu);
- the SIMT glue kernels of the wide step on both sides of the width at which they leave their vector paths, with the
  columns at and beyond the written width poisoned (NaN) and required untouched;
- the modules end to end: BondMessagePassing at C3's width and depth and at d_h = 1024 / 2048 / 2400 / 1998,
  AtomMessagePassing at 2048, and one bf16 case at 2048 (f32 FMA linears with bf16 storage).

Bounds of the summing kernels are worst-case bounds of recursive summation in the kernel's own order (u = 2^-24 per
rounding, n terms in a chain -> (n - 1) u of the sum of |terms|); an order-independent check with integer-valued data
(every partial sum exact in f32) makes dropped, repeated or misplaced rows fail exactly.  Batch sizes keep the peak
device memory of each case under about 10 GB."""
from __future__ import annotations

import gc
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                 # unit roundoff of f32
REL, REL_MEAN = 1e-5, 1e-6     # the x3 GEMMs' bound (tests/test_gpu_x3.py): of sum |terms|, worst element / mean
NAN = float("nan")
WIDTHS = [1024, 1028, 2048, 2056, 2400, 2398]     # both sides of C / 4 <= 256 and pad8(C) <= 2048; 2398: C % 4 != 0


def _free():
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    _free()


def _ld(C: int) -> int:
    """Row stride with at least 8 spare columns (poisoned, must stay untouched), 64-element aligned."""
    return (C + 8 + 63) // 64 * 64


def _poisoned(R: int, C: int, ld: int | None = None, *, scale: float = 1.0, gen=None) -> torch.Tensor:
    """R x ld f32: randn in [0, C), NaN in [C, ld)."""
    X = torch.full((R, ld or _ld(C)), NAN, device="cuda")
    X[:, :C] = torch.randn(R, C, device="cuda", generator=gen) * scale
    return X


def _fill_(dst: torch.Tensor, rows, chunk: int = 1 << 16):
    """dst[r0:r1] = rows(r1 - r0), chunk by chunk (the generators' temporaries of a million-row operand stay small)."""
    for r0 in range(0, dst.shape[0], chunk):
        r1 = min(dst.shape[0], r0 + chunk)
        dst[r0:r1] = rows(r1 - r0)


def _untouched(out: torch.Tensor, c0: int) -> bool:
    return bool(torch.isnan(out[:, c0:]).all())


def _act64(x, act):
    return {"none": x, "relu": torch.relu(x), "tanh": torch.tanh(x)}[act]


def _code(act):
    from chemprop_b200 import _lib

    return {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]


def _report(group: str, case, err: float, bound: float):
    print(f"[fp32-wide] {group} {case}: worst {err:.3e} of bound {bound:.3e} ({err / bound if bound else 0:.3f})")


# ------------------------------------------------------------------------------------------------------------------
# column_sum
# ------------------------------------------------------------------------------------------------------------------
def _splits(R: int):
    """(S, rows per split) of dmpnn_column_sum (wgrad_splits in csrc/linear.cu)."""
    S = min(296, max(1, (R + 1023) // 1024))
    rps = ((R + S - 1) // S + 15) // 16 * 16
    return S, max(rps, 16)


def _colsum64(Y: torch.Tensor, R: int, N: int, chunk: int = 1 << 14):
    s = torch.zeros(N, dtype=torch.float64, device="cuda")
    a = torch.zeros(N, dtype=torch.float64, device="cuda")
    for r0 in range(0, R, chunk):
        y = Y[r0:min(R, r0 + chunk), :N].double()
        s += y.sum(0)
        a += y.abs().sum(0)
    return s, a


COLSUM_NS = [1, 3, 300, 1536, 1540, 2048, 2052, 2400, 4096]
COLSUM_CASES = ([(N, kind, R) for N in COLSUM_NS for kind in ("f32", "bf16", "f32_ld_odd") for R in (0, 1, 70_001)]
                + [(600, "f32", 1_100_017), (1540, "f32", 1_100_017), (2048, "bf16", 1_100_017), (600, "f32_ld_odd", 1_100_017)])


@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("N,kind,R", COLSUM_CASES)
def test_column_sum_vs_f64(N, kind, R, accumulate):
    """kind: f32 / bf16 rows with a 4-aligned stride (4-wide kernel while 8 N floats fit 48 KB of shared memory, the
    column-per-thread kernel above), or f32 with an odd stride (column-per-thread kernel at every N).
    Order: the 4-wide kernel sums every 8th row of a split in one f32 chain (ceil(rps / 8) terms), adds the 8 warps' chains,
    then the splits with Kahan compensation; the column-per-thread kernel is Kahan throughout.  Bound:
    (ceil(rps / 8) + 10) u sum |y| (+ u |result| for the accumulate add)."""
    from chemprop_b200.engine import column_sum

    g = torch.Generator(device="cuda").manual_seed(N * 7 + R)
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    ld = N + 1 if kind == "f32_ld_odd" else (N + 3) // 4 * 4 + 4
    Y = torch.full((max(R, 1), ld), NAN, dtype=dt, device="cuda")
    out0 = torch.randn(N, device="cuda", generator=g) * 10 if accumulate else torch.full((N,), NAN, device="cuda")

    # 1) integer-valued rows: every partial sum is an integer below 2^24, exact in any order -> the result must be exact
    _fill_(Y[:, :N], lambda n: torch.randint(-8, 9, (n, N), device="cuda", generator=g).to(dt))
    base = out0.round() if accumulate else out0
    out = base.clone()
    column_sum(Y, R, N, out, accumulate=accumulate)
    s, _ = _colsum64(Y, R, N)
    ref = s + (base.double() if accumulate else 0)
    assert torch.equal(out.double(), ref), (N, kind, R, (out.double() - ref).abs().max().item())

    # 2) normal rows with a spread of row scales: error within the bound of the kernel's summation order
    _fill_(Y[:, :N], lambda n: (torch.randn(n, N, device="cuda", generator=g)
                                * torch.rand(n, 1, device="cuda", generator=g) * 4).to(dt))
    out = out0.clone()
    column_sum(Y, R, N, out, accumulate=accumulate)
    s, a = _colsum64(Y, R, N)
    ref = s + (out0.double() if accumulate else 0)
    _, rps = _splits(R)
    bound = (math.ceil(rps / 8) + 10) * U * a + (U * ref.abs() if accumulate else 0) + 1e-30
    err = (out.double() - ref).abs()
    assert bool(torch.isfinite(out).all()) and bool((err <= bound).all()), (N, kind, R, (err / bound).max().item())
    if R > 1:
        _report("column_sum", (N, kind, R, accumulate), (err / a.clamp_min(1e-30)).max().item(),
                (math.ceil(rps / 8) + 10) * U)


# ------------------------------------------------------------------------------------------------------------------
# 3xTF32 GEMMs
# ------------------------------------------------------------------------------------------------------------------
def _x3_slots(R: int, N: int, K: int):
    """(slots, row blocks chained by slot 0) of k_wgrad_x3: geom() in csrc/gemm_x3.cu (128 x 128 output tiles, 32-row
    blocks, SM count / tiles row slots per tile, at least 1, at most the block count)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    tiles = -(-N // 128) * -(-K // 128)
    nb = -(-R // 32)
    slots = max(1, sms // tiles)
    slots = min(slots, nb) if nb > 0 else 1
    return slots, -(-nb // slots)


def _chunked_rel_err(R, f_ref, f_got, chunk):
    """max / mean over all outputs of |got - ref| / mag, evaluated chunk by chunk of rows (f64 copies stay small)."""
    worst, tot, cnt = 0.0, 0.0, 0
    for r0 in range(0, R, chunk):
        r1 = min(R, r0 + chunk)
        ref, mag = f_ref(r0, r1)
        rel = (f_got(r0, r1).double() - ref).abs() / mag
        worst = max(worst, rel.max().item())
        tot += rel.sum().item()
        cnt += rel.numel()
        del ref, mag, rel
    return worst, tot / cnt


@pytest.mark.parametrize("R,K,N,bias,res,act,gather", [
    (1_100_017, 600, 600, True, False, "relu", False),      # C3's edge-row count: W_h / dX GEMMs of h = 600
    (70_001, 672, 600, True, True, "tanh", True),           # W_o of h = 600 (K = d_v + h) through a row gather
    (20_000, 1096, 1024, True, True, "relu", False),
    (20_000, 2048, 2048, True, True, "relu", True),
    (12_000, 2120, 2048, False, True, "none", False),       # CheMeleon's W_o
    (12_000, 2472, 2400, True, False, "tanh", False),
    (8_000, 4096, 4096, True, True, "relu", False),
])
def test_linear_x3_wide_vs_f64(R, K, N, bias, res, act, gather):
    from chemprop_b200 import engine

    g = torch.Generator(device="cuda").manual_seed(R + K + N)
    src = R + 77 if gather else R
    lda, ldc = (K + 63) // 64 * 64, _ld(N)
    A = torch.zeros(src, lda, device="cuda")
    _fill_(A[:, :K], lambda n: torch.randn(n, K, device="cuda", generator=g) * torch.rand(n, 1, device="cuda", generator=g) * 3)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    Rres = None
    if res:
        Rres = torch.zeros(R, ldc, device="cuda")
        Rres[:, :N] = torch.randn(R, N, device="cuda", generator=g)
    idx = torch.randint(0, src, (R,), device="cuda", dtype=torch.int32, generator=g) if gather else None
    out = torch.full((R, ldc), NAN, device="cuda")
    engine.linear_x3(A, K, engine.pack_weight_x3(W), N, out, idx=idx, bias=b, res=Rres, act=_code(act), R=R, pad_to=ldc)
    torch.cuda.synchronize()
    Wd, Wa = W.double().t(), W.double().abs().t()

    def f_ref(r0, r1):
        Ad = (A[idx[r0:r1].long()] if gather else A[r0:r1])[:, :K].double()
        Z = Ad @ Wd
        mag = Ad.abs() @ Wa + 1e-3
        if bias:                 # |b| is a term of the sum too: rows scaled near zero leave Z ~ b, rounded once
            Z += b.double()
            mag += b.double().abs()
        if res:
            Z += Rres[r0:r1, :N].double()
            mag += Rres[r0:r1, :N].double().abs()
        return _act64(Z, act), mag

    worst, mean = _chunked_rel_err(R, f_ref, lambda r0, r1: out[r0:r1, :N], 1 << 15)
    _report("linear_x3", (R, K, N), worst, REL)
    assert worst <= REL and mean <= REL_MEAN, (worst, mean)
    n16 = (N + 15) // 16 * 16
    assert float(out[:, N:n16].abs().max()) == 0.0 if n16 > N else True     # padding columns written as zeros
    assert _untouched(out, n16)                                              # ... nothing beyond pad16(N)


@pytest.mark.parametrize("R,N,K,accumulate,regime", [
    (1_100_017, 600, 600, False, "slotted"),   # C3: the W_h gradient over ~1.1 M edge rows
    (1_100_017, 600, 672, True, "slotted"),    # C3: W_o / W_i-sized operand over as many rows
    (70_001, 600, 672, False, "slotted"),
    (330_017, 1024, 1096, False, "single"),    # from here on one CTA per output tile chains every row block
    (330_017, 2048, 2048, True, "single"),
    (330_017, 2048, 2120, False, "single"),
    (330_017, 2400, 2472, False, "single"),
    (330_017, 4096, 4096, False, "single"),
    (777, 2400, 2472, True, "single"),
])
def test_wgrad_x3_wide_vs_f64(R, N, K, accumulate, regime):
    """dW = dY^T X.  dY and X are row-shifted views of one buffer (X[r] = dY-buffer row r + 1, rows i.i.d.), which halves
    the memory of the 4096-wide case; every product still pairs independent values."""
    from chemprop_b200 import engine

    slots, chain = _x3_slots(R, N, K)
    assert (slots == 1) == (regime == "single"), (slots, regime)
    if regime == "single" and R > 300_000:
        assert chain > 10_000, chain                   # one f32 register chain over more than 10 k row blocks
    g = torch.Generator(device="cuda").manual_seed(R + N + K)
    ld = (max(N, K) + 4 + 3) // 4 * 4
    buf = torch.randn(R + 1, ld, device="cuda", generator=g)
    buf *= torch.rand(R + 1, 1, device="cuda", generator=g) * 2
    dY, X = buf[:R, :N], buf[1:, :K]
    dW0 = torch.randn(N, K, device="cuda", generator=g)
    dW = dW0.clone()
    engine.wgrad_x3(dY, X, R, N, K, dW, accumulate=accumulate)
    torch.cuda.synchronize()
    ref = dW0.double() if accumulate else torch.zeros(N, K, dtype=torch.float64, device="cuda")
    mag = torch.ones(N, K, dtype=torch.float64, device="cuda")
    chunk = max(1024, (1 << 26) // ld)
    for r0 in range(0, R, chunk):
        r1 = min(R, r0 + chunk)
        y, x = buf[r0:r1, :N].double(), buf[r0 + 1:r1 + 1, :K].double()
        ref += y.t() @ x
        mag += y.abs().t() @ x.abs()
        del y, x
    rel = (dW.double() - ref).abs() / mag
    worst, mean = rel.max().item(), rel.mean().item()
    _report("wgrad_x3", (R, N, K, f"slots={slots}", f"chain={chain}"), worst, REL)
    assert worst <= REL and mean <= REL_MEAN, (worst, mean, slots, chain)


# ------------------------------------------------------------------------------------------------------------------
# SIMT glue kernels of the wide step
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def layout():
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules

    bmg = BatchMolGraph(make_molecules(160, seed=11, shuffle_edges=True))
    bmg.to("cuda")
    lay = engine.get_layout(bmg)
    counts = (lay.rowptr[1:] - lay.rowptr[:-1]).long()
    seg = torch.repeat_interleave(torch.arange(lay.V, device="cuda"), counts)     # atom (segment) of every edge row
    return lay, seg, counts


def _segments(n_seg: int, lo: int, hi: int, seed: int):
    g = torch.Generator(device="cuda").manual_seed(seed)
    cnt = torch.randint(lo, hi + 1, (n_seg,), device="cuda", generator=g)
    cnt[::17] = 0                                                                  # empty segments
    ptr = torch.zeros(n_seg + 1, dtype=torch.int32, device="cuda")
    ptr[1:] = cnt.cumsum(0).to(torch.int32)
    seg = torch.repeat_interleave(torch.arange(n_seg, device="cuda"), cnt)
    return ptr, seg, cnt


def _sum_rows64(X64, seg, n_seg):
    return torch.zeros(n_seg, X64.shape[1], dtype=torch.float64, device="cuda").index_add_(0, seg, X64)


@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("mode", ["sum", "mean"])
def test_segment_sum_wide(C, mode):
    """sum: the atom sums M_v over in-edge rows (short segments, no activation); mean: molecule-long segments with ReLU,
    divided by the row count (0 for an empty segment).  Columns [C, pad8(C)) are written as zeros."""
    from chemprop_b200 import _lib, engine

    n_seg = 3000 if mode == "sum" else 300
    ptr, seg, cnt = _segments(n_seg, 1, 6, C) if mode == "sum" else _segments(n_seg, 2, 60, C)
    R = int(ptr[-1])
    X = _poisoned(R, C)
    pad = (C + 7) // 8 * 8
    out = torch.full((n_seg, _ld(C)), NAN, device="cuda")
    act = "none" if mode == "sum" else "relu"
    engine.segment_sum(X, ptr, n_seg, C, out, act=_code(act),
                       scale_mode=_lib.SCALE_NONE if mode == "sum" else _lib.SCALE_INV_COUNT, pad_to=pad)
    x = _act64(X[:, :C].double(), act)
    ref, mag = _sum_rows64(x, seg, n_seg), _sum_rows64(x.abs(), seg, n_seg)
    div = cnt.clamp_min(1).double()[:, None] if mode == "mean" else 1.0
    ref, mag = ref / div, mag / div
    bound = (cnt.double()[:, None] + 1) * U * mag + U * ref.abs()
    err = (out[:, :C].double() - ref).abs()
    assert bool((err <= bound).all()), (err / bound.clamp_min(1e-30)).max().item()
    assert bool((out[:, C:pad] == 0).all()) and _untouched(out, pad)


@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("with_ptr", [False, True])
def test_segment_bcast_wide(C, with_ptr):
    """with ptr: the mean aggregate's backward (segment walk, divided by the count); without: a plain row broadcast."""
    from chemprop_b200 import _lib, engine

    n_seg = 400
    ptr, seg, cnt = _segments(n_seg, 2, 40, C + 1)
    R = int(ptr[-1])
    G = _poisoned(n_seg, C)
    out = torch.full((R, _ld(C)), NAN, device="cuda")
    seg32 = seg.to(torch.int32)
    if with_ptr:
        engine.segment_bcast(G, seg32, ptr, R, C, out, scale_mode=_lib.SCALE_INV_COUNT, n_seg=n_seg)
        ref = G[seg, :C].double() / cnt[seg].double()[:, None]
    else:
        engine.segment_bcast(G, seg32, None, R, C, out)
        ref = G[seg, :C].double()
    err = (out[:, :C].double() - ref).abs()
    assert bool((err <= U * ref.abs()).all()), err.max().item()
    assert _untouched(out, C)


@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("act,from_preact", [("relu", False), ("tanh", False), ("tanh", True)])
def test_act_bwd_wide(C, act, from_preact):
    """dZ = G[gidx] * tau'(Y) with an f32 accumulator: ACC += dZ (the readout's and every depth step's backward)."""
    from chemprop_b200 import engine

    R, RG = 9000, 2500
    g = torch.Generator(device="cuda").manual_seed(C)
    G = _poisoned(RG, C, gen=g)
    Y = _poisoned(R, C, gen=g)
    gidx = torch.randint(0, RG, (R,), device="cuda", dtype=torch.int32, generator=g)
    acc = _poisoned(R, C, gen=g)
    acc0 = acc[:, :C].double()
    dZ = torch.full((R, _ld(C)), NAN, device="cuda")
    engine.act_bwd(G, Y, R, C, act=_code(act), gidx=gidx, from_preact=from_preact, dZ=dZ, acc=acc)
    gd, y = G[gidx.long(), :C].double(), Y[:, :C].double()
    if act == "relu":
        d, dtol = (y > 0).double(), 0.0
    elif from_preact:
        t = torch.tanh(y)
        d, dtol = 1 - t * t, 8 * U          # tanhf is within 2 ulp: 1 - t^2 off by <= ~5 u
    else:
        d, dtol = 1 - y * y, U * (y * y) + U    # 1 - y y: the product's rounding, then the difference's
    ref = gd * d
    tol = gd.abs() * (dtol + U * d.abs())
    err = (dZ[:, :C].double() - ref).abs()
    assert bool((err <= tol).all()), (err / tol.clamp_min(1e-30)).max().item()
    err_acc = (acc[:, :C].double() - (acc0 + ref)).abs()
    assert bool((err_acc <= tol + U * (acc0 + ref).abs()).all())
    assert _untouched(dZ, C) and _untouched(acc, C)


@pytest.mark.parametrize("C", WIDTHS)
@pytest.mark.parametrize("permute_on_read", [False, True])
def test_bond_message_wide(layout, C, permute_on_read):
    """forward (mixins.py:11-18): M[rev r] = sum_{r' -> dst r} H[r'] - H[r]; backward direction (permute on read):
    OUT[r] = sum_{r' -> dst r} X[rev r'] - X[rev r]."""
    from chemprop_b200 import engine

    lay, seg, counts = layout
    X = _poisoned(lay.E, C)
    out = torch.full((lay.E, _ld(C)), NAN, device="cuda")
    engine.bond_message(X, lay, C, out, permute_on_read=permute_on_read)
    rev = lay.rev_row.long()
    x = X[:, :C].double()
    if permute_on_read:
        x = x[rev]
    S, A = _sum_rows64(x, seg, lay.V)[seg], _sum_rows64(x.abs(), seg, lay.V)[seg]
    ref = S - x
    bound = (counts[seg].double()[:, None] + 1) * U * A
    if not permute_on_read:
        ref_w, bound_w = torch.empty_like(ref), torch.empty_like(bound)
        ref_w[rev], bound_w[rev] = ref, bound
        ref, bound = ref_w, bound_w
    err = (out[:, :C].double() - ref).abs()
    assert bool((err <= bound).all()), (err / bound.clamp_min(1e-30)).max().item()
    assert _untouched(out, C)


@pytest.mark.parametrize("C", WIDTHS)
def test_rev_average_wide(layout, C):
    """undirected H~ = (tau(H) + tau(H[rev])) / 2 (base.py:202-203), here with the first step's ReLU applied on load."""
    from chemprop_b200 import engine

    lay, _, _ = layout
    X = _poisoned(lay.E, C)
    out = torch.full((lay.E, _ld(C)), NAN, device="cuda")
    engine.rev_average(X, lay, C, out, act=_code("relu"))
    x = torch.relu(X[:, :C].double())
    ref = (x + x[lay.rev_row.long()]) / 2
    err = (out[:, :C].double() - ref).abs()
    assert bool((err <= U * ref.abs()).all()), err.max().item()
    assert _untouched(out, C)


@pytest.mark.parametrize("C", WIDTHS)
def test_concat_f32_wide(C):
    """[X1[idx1, :K1] || X2[idx2, :K2] || 0] over `width` = C columns: an exact copy, zeros up to the width."""
    from chemprop_b200 import engine

    R, K2 = 5000, 14
    K1 = C - K2 - 6
    g = torch.Generator(device="cuda").manual_seed(C)
    X1 = _poisoned(700, K1, gen=g)
    X2 = _poisoned(R + 9, K2, 16, gen=g)
    i1 = torch.randint(0, 700, (R,), device="cuda", dtype=torch.int32, generator=g)
    i2 = torch.randperm(R + 9, device="cuda", generator=g)[:R].to(torch.int32)
    out = torch.full((R, _ld(C)), NAN, device="cuda")
    engine.concat_f32(X1, K1, out, R, idx1=i1, X2=X2, K2=K2, idx2=i2, width=C)
    assert torch.equal(out[:, :K1], X1[i1.long(), :K1])
    assert torch.equal(out[:, K1:K1 + K2], X2[i2.long(), :K2])
    assert bool((out[:, K1 + K2:C] == 0).all()) and _untouched(out, C)


@pytest.mark.parametrize("C", [c for c in WIDTHS if c % 4 == 0])
@pytest.mark.parametrize("act", ["relu", "tanh"])
def test_sum_act_bwd_wide(C, act):
    """dH_0 total of the mirror: OUT = Z_1 + Z_2 + Z_3 + G * tau'(Ypre) in one pass."""
    from chemprop_b200 import engine

    R = 7000
    g = torch.Generator(device="cuda").manual_seed(C + 5)
    Zs = [_poisoned(R, C, gen=g) for _ in range(3)]
    G, Yp = _poisoned(R, C, gen=g), _poisoned(R, C, gen=g)
    out = torch.full((R, _ld(C)), NAN, device="cuda")
    engine.sum_act_bwd(Zs, G, Yp, out, R, C, act=_code(act))
    y = Yp[:, :C].double()
    d = (y > 0).double() if act == "relu" else 1 - torch.tanh(y) ** 2
    gd = G[:, :C].double() * d
    ref = gd + sum(z[:, :C].double() for z in Zs)
    mag = gd.abs() + sum(z[:, :C].double().abs() for z in Zs)
    tol = 5 * U * mag + (8 * U * G[:, :C].double().abs() if act == "tanh" else 0)
    err = (out[:, :C].double() - ref).abs()
    assert bool((err <= tol).all()), (err / tol.clamp_min(1e-30)).max().item()
    assert _untouched(out, C)


# ------------------------------------------------------------------------------------------------------------------
# modules against the restatement in float64
# ------------------------------------------------------------------------------------------------------------------
# gtol: bar on each weight / bias gradient, of its max-abs (test_medium_batch_vs_oracle's 2e-4 for the fp32 tier).  At
# d_h = 2400 the worst W_i.weight element on the 3xTF32 GEMMs measures 2.1e-4 on an H100 (plain f32 torch, TF32 off: 7.2e-5;
# the SIMT linears: 1.1e-4): each split operand keeps 22 of f32's 24 bits, so a product carries up to ~12 u against an f32
# FMA's u, and that case is held to 3e-4.  At 2048 the three agree (7.6e-5 / 8.0e-5 / 8.0e-5).
@pytest.mark.parametrize("kind,precision,d_h,depth,n_mols,act,gtol", [
    ("bond", "fp32", 600, 6, 1600, "relu", 2e-4),        # C3's width and depth
    ("bond", "fp32", 1024, 3, 500, "relu", 2e-4),
    ("bond", "fp32", 2048, 3, 500, "relu", 2e-4),        # CheMeleon's width
    ("bond", "fp32", 2400, 3, 500, "relu", 3e-4),
    ("bond", "fp32", 1998, 3, 400, "relu", 2e-4),        # d_h % 4 != 0: the SIMT linears
    ("atom", "fp32", 2048, 3, 400, "relu", 2e-4),
    ("bond", "bf16", 2048, 3, 400, "tanh", 6e-2),        # above the bf16 tensor-core limit: f32 FMA linears, bf16 storage
])
def test_module_wide_vs_f64_oracle(kind, precision, d_h, depth, n_mols, act, gtol):
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    torch.manual_seed(0)
    torch.cuda.reset_peak_memory_stats()
    bmg = BatchMolGraph(make_molecules(n_mols, seed=5, shuffle_edges=(kind == "bond")))
    bmg.to("cuda")
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_h=d_h, depth=depth, bias=True, activation=act, precision=precision).cuda()

    # f64 reference on the same weights: forward, mean aggregate, autograd; its graph is freed before the module runs
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward(kind, bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], P["W_i.bias"], P["W_h.weight"], P["W_h.bias"],
                                      P["W_o.weight"], P["W_o.bias"], depth, act=act)
    a_ref = R.aggregate(H_ref, bmg.batch, "mean")
    a_ref.square().sum().backward()
    H_ref, a_ref = H_ref.detach(), a_ref.detach()
    grads_ref = {k: p.grad for k, p in P.items()}
    del P
    _free()

    H = mp(bmg)
    a = MeanAggregation()(H, bmg.batch)
    a.float().square().sum().backward()
    torch.cuda.synchronize()

    hmax = max(1.0, H_ref.abs().max().item())
    if precision == "fp32":
        tol, ftol = (5e-5 if depth >= 6 else 1e-5) * hmax, 2e-5
    else:
        tol, ftol = 1e-2 * hmax, 2e-2
    errH = (H.detach().double() - H_ref).abs().max().item()
    erra = (a.detach().double() - a_ref).abs().max().item()
    _report("module H_v", (kind, precision, d_h, depth), errH, tol)
    _report("module agg", (kind, precision, d_h, depth), erra, tol)
    assert errH <= tol and erra <= tol, (errH, erra, tol)
    names = set()
    for k, p in mp.named_parameters():
        ref = grads_ref[k]
        scale = max(1e-6, ref.abs().max().item())
        err = (p.grad.double() - ref).abs().max().item()
        frob = ((p.grad.double() - ref).norm() / ref.norm().clamp_min(1e-30)).item()
        _report(f"module grad {k} max", (kind, precision, d_h), err / scale, gtol)
        _report(f"module grad {k} frob", (kind, precision, d_h), frob, ftol)
        assert err <= gtol * scale and frob <= ftol, (k, err, scale, frob)
        names.add(k)
    assert names == {"W_i.weight", "W_i.bias", "W_h.weight", "W_h.bias", "W_o.weight", "W_o.bias"}
    print(f"[fp32-wide] peak device memory {(kind, precision, d_h, depth, n_mols)}: "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
