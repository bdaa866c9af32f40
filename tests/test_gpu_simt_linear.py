"""GPU tier: the SIMT f32 GEMMs of csrc/linear.cu -- `dmpnn_linear_fwd` (k_linear_fwd) and `dmpnn_linear_wgrad`
(k_wgrad_partial, k_colsum_partial, k_reduce_splits) -- against float64 torch on the device.

These kernels run the FFN head of every training step, the atom fp32 tier, the bf16 tier past the tensor-core limits
(d_h > 304) and the bond fp32 tier when a width is not a multiple of 4 (d_v = 133).  `FWD_CASES` / `WGRAD_CASES` hold one
case per operand-type instantiation the engine launches (tests/test_simt_linear_host.py takes that census on the CPU and
fails when an entry has no case here) plus geometry cases: row counts on both sides of the 128-row tile and of the
wgrad's 16-row blocks and 1024-row splits (296 splits from R = 302 081), N and K on both sides of the 64-wide tiles, K = 1,
N = 1, a second source whose first 8-wide chunk straddles K1, repeated and out-of-order gathers, 16-byte-aligned and odd
row strides.  Operand columns past K1 / K2 and W's columns past K are NaN, so a read past K fails; output columns in
[N, ldc_pad) must come out 0 and those past ldc_pad, like the row past R, must keep their NaN.

Bounds (u = 2^-24):

- linear_fwd: a thread's fmaf chain over the K products (K roundings), then + bias and + residual:
  |err| <= (K + 3) u (sum_k |a w| + |b| + |res|) * Lip(tau) + tau's own rounding; a bf16 output adds half a bf16 ulp of
  the f64 value.  A wrong k chunk, a gather through the wrong index or a misplaced second source moves an element by the
  size of a term, far past this bound.
- linear_wgrad: an element sum_r dy[r, n] x[r, k] is summed in 16-row blocks (an fmaf chain from zero: <= 16 u of the
  block's sum |terms|), the blocks of a split with Kahan compensation (<= 2 u of the sum of |block sums| plus
  O(blocks * u^2)), and the splits again with Kahan (<= 2 u), so |err| <= 20 u sum_r |dy x| up to terms of order
  blocks * u^2 (below 10^-4 of it at 1.1 M rows); accumulation adds one rounding of the result.  The bias gradient is a
  Kahan sum over the rows of a split and one over the splits: <= 4 u sum |dy|, held to 6 u.  A plain chain in place of
  either Kahan sum fails the "same" cases: every row holds the same positive terms, so every 16-row block adds the same
  value to its split's running sum and the rounding errors of an uncompensated chain all point the same way.  An f32
  emulation of the kernels' order at R = 1 100 017 (296 splits of 3 728 rows) over 40 random (d_n, x_k) gives up to 100 u
  of the sum with plain chains against 3.3 u with Kahan, and for k_colsum_partial's chain 840 u against 0.8 u.
- Integer-exact variants: integer operands whose every partial sum stays below 2^24, so the f32 result must equal the f64
  one exactly (a dropped or doubled chunk, row or split is an integer off), and a bf16 output must equal torch's
  round-to-nearest-even of it bit for bit (a truncating store fails on the first odd integer above 256).

Every case prints its worst error over bound and its mean error over mean bound (held to 0.6).  Device memory stays
under about 10 GB per case: the f64 references are formed in row chunks."""
from __future__ import annotations

import ctypes
import gc
import zlib
from collections import namedtuple

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NAN = float("nan")
MEAN_BAR = 0.6
CHUNK = 1 << 15
DT = {"f32": torch.float32, "bf16": torch.bfloat16}


def fwd_key(x1, x2, res, out, gather, bias, N, K):
    """Census key of a linear_fwd launch: operand types (X1, X2, residual, output; None = absent), a gather, a bias, N == 1,
    K == 1."""
    return ("fwd", x1, x2 or "-", res or "-", out, "gather" if gather else "-", "bias" if bias else "-",
            "N=1" if N == 1 else "N>1", "K=1" if K == 1 else "K>1")


def wgrad_key(dy, x1, x2, gather, bias, accumulate, N, K):
    """Census key of a linear_wgrad launch: operand types (dY, X1, X2; None = absent), a gather, dbias, accumulate, N == 1,
    K == 1."""
    return ("wgrad", dy, x1, x2 or "-", "gather" if gather else "-", "dbias" if bias else "-",
            "acc" if accumulate else "-", "N=1" if N == 1 else "N>1", "K=1" if K == 1 else "K>1")


class FwdCase(namedtuple("FwdCase", "R N K1 K2 x1 x2 res out gather bias act odd exact pad")):
    """gather: "" / "1" / "2" / "12" (which sources are read through an index); pad: ldc_pad - N."""

    @property
    def key(self):
        return fwd_key(self.x1, self.x2 if self.K2 else None, self.res, self.out, bool(self.gather), self.bias, self.N,
                       self.K1 + self.K2)

    @property
    def id(self):
        parts = [f"R{self.R}", f"N{self.N}", f"K{self.K1}+{self.K2}" if self.K2 else f"K{self.K1}", self.x1,
                 self.x2 if self.K2 else "", f"res-{self.res}" if self.res else "", f"out-{self.out}",
                 f"idx{self.gather}" if self.gather else "", "bias" if self.bias else "", self.act,
                 "odd" if self.odd else "", "int" if self.exact else "", f"pad{self.pad}" if self.pad else ""]
        return "-".join(p for p in parts if p)


def F(R, N, K1, K2=0, x1="f32", x2="f32", res=None, out="f32", gather="", bias=False, act="none", odd=False, exact=False,
      pad=0):
    return FwdCase(R, N, K1, K2, x1, x2, res, out, gather, bias, act, odd, exact, pad)


FWD_CASES = [
    # one per census entry (tests/test_simt_linear_host.py), at the shapes the engine gives them
    F(10000, 300, 300, bias=True, act="relu"),                                   # head: hidden layer
    F(50, 1, 300, bias=True),                                                    # head: last layer, n_tasks 1
    F(129, 300, 1, odd=True),                                                    # head: dX of the last layer, n_tasks 1
    F(5000, 300, 300, pad=4),                                                    # dM = dZ . W_h (fp32 bond mirror)
    F(7000, 300, 133, 14, gather="12", pad=4),                                   # bond fp32 W_i on V[src] || E[perm]
    F(7000, 300, 300, res="f32", act="relu", pad=4),                             # bond fp32 W_h + H_0
    F(3000, 300, 133, 300, bias=True, act="leakyrelu"),                          # W_o on [V || M_v]
    F(4000, 2048, 72, 14, out="bf16", gather="12"),                              # bf16 past the tc limits: W_i
    F(3000, 2048, 2048, x1="bf16", res="bf16", out="bf16", act="relu"),          # ... W_h with a bf16 residual
    F(1000, 2048, 72, 2048, x2="bf16", out="bf16", bias=True, act="elu"),        # ... W_o on [V || M_v (bf16)]
    F(1000, 2048, 2048, x1="bf16", out="bf16"),                                  # ... dM_v = dY . W_o^T
    F(3000, 300, 300, 14, res="f32", act="tanh", pad=4),                         # atom fp32 W_h on [N_b || SE] + H_0
    F(2000, 302, 72, out="bf16", pad=2),                                         # atom bf16 W_i (d_h 302)
    F(2000, 302, 302, 14, x1="bf16", res="bf16", out="bf16", act="relu", pad=2), # atom bf16 W_h on [N_b || SE]
    # integer-exact: f32 results equal to f64, bf16 results round to nearest even bit for bit
    F(3000, 300, 300, 14, res="f32", gather="12", exact=True, pad=4),
    F(3000, 2048, 2048, x1="bf16", res="bf16", out="bf16", exact=True),
    F(1000, 300, 72, 300, x2="bf16", out="bf16", bias=True, act="relu", exact=True, odd=True),
    F(129, 1, 2400, exact=True),
    # geometry: R, N, K1, K2 on both sides of the tiles; aligned and odd strides; gathers on either source
    F(1, 1, 1),
    F(127, 12, 7, 14, odd=True, gather="2"),
    F(128, 63, 8, 28, x1="bf16", x2="bf16", out="bf16"),
    F(129, 64, 86, 14, gather="1", odd=True, pad=16),
    F(129, 65, 300, 14, x1="bf16", gather="12", bias=True, act="relu", pad=15),
    F(128, 2048, 2400, act="leakyrelu"),
    F(127, 1, 2400, 28, x2="bf16", odd=True),
    F(1, 300, 300, 300, x1="bf16", x2="bf16", res="bf16", out="bf16", gather="12"),
    F(70001, 300, 300, 28, gather="12", out="bf16", res="f32", act="relu", pad=4),
    F(70001, 2048, 2048, x1="bf16", res="bf16", out="bf16", odd=True),
    F(70001, 12, 1, bias=True),
    F(70001, 65, 7, 300, x2="bf16", odd=True, exact=True, pad=3),
    F(129, 12, 2048, 14, x1="bf16", x2="bf16", odd=True, exact=True, out="bf16"),
]


class WgradCase(namedtuple("WgradCase", "R N K1 K2 dy x1 x2 gather dbias acc odd kind")):
    """kind: "rand" (randn), "int" (integer-exact), "same" (every row the same positive terms: the drift a plain chain
    would show)."""

    @property
    def key(self):
        return wgrad_key(self.dy, self.x1, self.x2 if self.K2 else None, bool(self.gather), self.dbias, self.acc, self.N,
                         self.K1 + self.K2)

    @property
    def id(self):
        parts = [f"R{self.R}", f"N{self.N}", f"K{self.K1}+{self.K2}" if self.K2 else f"K{self.K1}", f"dy-{self.dy}",
                 self.x1, self.x2 if self.K2 else "", f"idx{self.gather}" if self.gather else "",
                 "dbias" if self.dbias else "", "acc" if self.acc else "", "odd" if self.odd else "", self.kind]
        return "-".join(p for p in parts if p)


def W_(R, N, K1, K2=0, dy="f32", x1="f32", x2="f32", gather="", dbias=False, acc=False, odd=False, kind="rand"):
    return WgradCase(R, N, K1, K2, dy, x1, x2, gather, dbias, acc, odd, kind)


WGRAD_CASES = [
    # one per census entry
    W_(50, 1, 300, dbias=True),                                                  # head: last layer, n_tasks 1
    W_(10000, 300, 300, dbias=True),                                             # head: hidden layer
    W_(3000, 300, 133, 300, dbias=True),                                         # fp32 W_o on [V || M_v]
    W_(7000, 300, 300, acc=True),                                                # fp32 bond dW_h
    W_(7000, 300, 133, 14, gather="12"),                                         # fp32 bond dW_i on V[src] || E[perm]
    W_(3000, 2048, 72, 2048, dy="bf16", x2="bf16", dbias=True),                  # bf16 storage: W_o
    W_(3000, 2048, 2048, dy="bf16", x1="bf16", acc=True),                        # ... dW_h
    W_(3000, 300, 300, 14, acc=True),                                            # atom fp32 dW_h on [N_b || SE]
    W_(3000, 300, 72),                                                           # atom fp32 dW_i
    W_(2000, 302, 302, 14, dy="bf16", x1="bf16", acc=True, odd=True),            # atom bf16 dW_h
    # rows: empty, inside one block, both sides of the 16-row block and of the 1024-row split, the first R with 296 splits,
    # C3-like edge-row counts
    W_(0, 300, 300, 14, dbias=True, acc=True),
    W_(0, 1, 300, dbias=True),
    W_(1, 300, 300, 28, gather="12", dbias=True),
    W_(15, 1, 7, dbias=True, odd=True),
    W_(16, 2048, 2048, 14, dy="bf16", x1="bf16", x2="bf16", dbias=True),
    W_(17, 300, 300, 14, dy="bf16", x1="bf16", acc=True, odd=True, gather="2"),
    W_(1023, 65, 86, 14, gather="1", dbias=True),
    W_(1024, 300, 300, 28, kind="int", dbias=True, acc=True),
    W_(1025, 1, 300, 14, kind="int", dbias=True, odd=True),
    W_(302081, 2048, 2048, 14, dy="bf16", x1="bf16", x2="bf16", dbias=True),
    W_(302081, 2048, 2048, 14, dy="bf16", x1="bf16", x2="bf16", kind="int", acc=True),
    W_(302081, 300, 300, 28, gather="12", kind="int", dbias=True),
    W_(1100017, 300, 300, 28, kind="same", dbias=True, acc=True),
    W_(1100017, 12, 300, 14, gather="12", dbias=True),
    W_(1100017, 1, 300, 28, dy="bf16", x1="bf16", kind="int", dbias=True),
    W_(1100017, 64, 1, kind="same", dbias=True),
]


# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _code(act):
    from chemprop_b200 import _lib

    return {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "leakyrelu": _lib.ACT_LEAKYRELU, "tanh": _lib.ACT_TANH,
            "elu": _lib.ACT_ELU}[act]


ACT_P = {"none": 0.0, "relu": 0.0, "leakyrelu": 0.3, "tanh": 0.0, "elu": 0.5}


def _p32(p):
    return float(torch.tensor(p, dtype=torch.float32))


def _tau64(act, z):
    p = _p32(ACT_P[act])
    if act == "relu":
        return torch.relu(z)
    if act == "leakyrelu":
        return torch.where(z > 0, z, p * z)
    if act == "tanh":
        return torch.tanh(z)
    if act == "elu":
        return torch.where(z > 0, z, p * torch.expm1(z))
    return z


def _half_ulp_bf16(x):
    _, e = torch.frexp(x.abs())
    return torch.where(x != 0, torch.pow(2.0, (e - 9).double()), torch.zeros_like(x))


class _Stats:
    """Worst |err| / bound and sum |err| / sum bound over the chunks of one result."""

    def __init__(self, what):
        self.what, self.worst, self.err, self.bound = what, 0.0, 0.0, 0.0

    def add(self, got, ref, bound):
        g = got.double()
        assert bool(torch.isfinite(g).all()), f"{self.what}: non-finite output"
        err = (g - ref).abs()
        assert bool((err[bound == 0] == 0).all()), f"{self.what}: inexact where the bound is 0"
        ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.zeros_like(err))
        if ratio.numel():
            self.worst = max(self.worst, ratio.max().item())
        self.err += err.sum().item()
        self.bound += bound.sum().item()

    def check(self):
        mean = self.err / self.bound if self.bound > 0 else 0.0
        assert self.worst <= 1.0, (self.what, "worst err / bound", self.worst)
        assert mean <= MEAN_BAR, (self.what, "mean err / mean bound", mean)
        return self.worst, mean


def _values(rows, cols, g, kind, lo=-8, hi=8):
    if kind == "int":
        return torch.randint(lo, hi + 1, (rows, cols), device="cuda", generator=g).float()
    return torch.randn(rows, cols, device="cuda", generator=g)


def _operand(rows, K, dt, odd, fill):
    """rows x K view of a NaN-filled buffer: ld a multiple of 8 elements (16-byte rows for f32 and bf16), or with `odd` an odd
    ld and a base one element in (no row 16-byte aligned).  `fill(r0, r1)` gives rows [r0, r1) in f32."""
    ld = (K + 1 + 7) // 8 * 8 + (1 if odd else 0)
    off = 1 if odd else 0
    buf = torch.full((rows, ld), NAN, dtype=DT[dt], device="cuda")
    X = buf[:, off:off + K]
    for r0 in range(0, rows, CHUNK):
        r1 = min(rows, r0 + CHUNK)
        X[r0:r1] = fill(r0, r1).to(X.dtype)
    return X


def _index(R, rows, g):
    """Int32 row index of R entries into `rows` source rows: repeats and out of order."""
    return torch.randint(0, rows, (R,), device="cuda", generator=g, dtype=torch.int64).to(torch.int32)


def _rows64(X, idx, r0, r1):
    return (X[r0:r1] if idx is None else X[idx[r0:r1].long()]).double()


def _report(kind, case, worst, mean):
    print(f"[simt-linear] {kind} {case}: worst err / bound {worst:.3f}, mean err / mean bound {mean:.3f}")


@pytest.mark.parametrize("c", FWD_CASES, ids=[c.id for c in FWD_CASES])
def test_linear_fwd_vs_f64(c):
    from chemprop_b200 import engine

    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.id.encode()))
    kind = "int" if c.exact else "rand"
    K = c.K1 + c.K2
    rows1 = c.R // 2 + 5 if "1" in c.gather else c.R
    rows2 = c.R // 3 + 7 if "2" in c.gather else c.R
    X1 = _operand(rows1, c.K1, c.x1, c.odd, lambda r0, r1: _values(r1 - r0, c.K1, g, kind))
    X2 = _operand(rows2, c.K2, c.x2, not c.odd, lambda r0, r1: _values(r1 - r0, c.K2, g, kind)) if c.K2 else None
    idx1 = _index(c.R, rows1, g) if "1" in c.gather else None
    idx2 = _index(c.R, rows2, g) if "2" in c.gather else None
    Wb = torch.full((c.N, K + 5), NAN, device="cuda")
    Wb[:, :K] = _values(c.N, K, g, kind) if c.exact else _values(c.N, K, g, kind) / K ** 0.5
    W = Wb[:, :K]
    b = None
    if c.bias:
        b = torch.randint(-64, 65, (c.N,), device="cuda", generator=g).float() if c.exact else \
            torch.randn(c.N, device="cuda", generator=g) * 0.1
    res = None
    if c.res:
        res = _operand(c.R, c.N, c.res, c.odd, lambda r0, r1: (16 * _values(r1 - r0, c.N, g, "int", -256, 256)) if c.exact
                       else _values(r1 - r0, c.N, g, kind))
    pad_to = c.N + c.pad
    ldc = pad_to + 3
    out = torch.full((c.R + 1, ldc), NAN, dtype=DT[c.out], device="cuda")
    engine.linear_fwd(X1, c.K1, W, out, c.N, idx1=idx1, X2=X2, K2=c.K2, idx2=idx2, bias=b, res=res, act=_code(c.act),
                      act_param=ACT_P[c.act], R=c.R, pad_to=pad_to)
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[c.R]).all()), "row past R written"
    assert bool((out[:c.R, c.N:pad_to] == 0).all()), "[N, ldc_pad) not zeroed"
    assert bool(torch.isnan(out[:c.R, pad_to:].float()).all()), "columns past ldc_pad written"
    Wd = W.double()
    lip = max(1.0, ACT_P[c.act]) if c.act in ("leakyrelu", "elu") else 1.0
    st = _Stats(c.id)
    for r0 in range(0, c.R, CHUNK // 4):
        r1 = min(c.R, r0 + CHUNK // 4)
        A = _rows64(X1, idx1, r0, r1)
        if c.K2:
            A = torch.cat([A, _rows64(X2, idx2, r0, r1)], 1)
        z = A @ Wd.t()
        mag = A.abs() @ Wd.abs().t()
        if b is not None:
            z, mag = z + b.double(), mag + b.double().abs()
        if res is not None:
            rr = res[r0:r1].double()
            z, mag = z + rr, mag + rr.abs()
        y = _tau64(c.act, z)
        got = out[r0:r1, :c.N]
        if c.exact:
            assert float(mag.max()) < 2 ** 24
            if c.out == "f32":
                assert torch.equal(got.double(), y), f"{c.id}: not exact"
            else:                            # equal values: bit for bit up to the sign of a zero
                assert torch.equal(got.double(), y.to(torch.bfloat16).double()), \
                    f"{c.id}: bf16 store is not round-to-nearest-even"
            continue
        delta = lip * (K + 3) * U * mag + 4 * U * y.abs() + 1e-30
        if c.out == "bf16":
            delta = delta + _half_ulp_bf16(y.abs() + delta)
        st.add(got, y, delta)
    if c.exact:
        print(f"[simt-linear] fwd {c.id}: exact")
        return
    _report("fwd", c.id, *st.check())


def _workspace_bytes(R, N, K):
    from chemprop_b200 import _lib

    n = ctypes.c_size_t(0)
    _lib.check(_lib.load().dmpnn_linear_wgrad_workspace_bytes(R, N, K, ctypes.byref(n)), "wgrad_workspace_bytes")
    return n.value


@pytest.mark.parametrize("c", WGRAD_CASES, ids=[c.id for c in WGRAD_CASES])
def test_linear_wgrad_vs_f64(c):
    from chemprop_b200 import engine

    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.id.encode()))
    K = c.K1 + c.K2
    lo, hi = (-1, 1) if c.R > 400000 else (-3, 3)          # integer partial sums below 2^24
    if c.kind == "same":       # every row [d_n] x [x_k], positive, full mantissas
        dyrow = torch.rand(1, c.N, device="cuda", generator=g) + 0.5
        xrow = torch.rand(1, K, device="cuda", generator=g) + 1.0
        fill_dy = lambda r0, r1: dyrow.expand(r1 - r0, c.N)
        fill_x1 = lambda r0, r1: xrow[:, :c.K1].expand(r1 - r0, c.K1)
        fill_x2 = lambda r0, r1: xrow[:, c.K1:].expand(r1 - r0, c.K2)
    else:
        fill_dy = lambda r0, r1: _values(r1 - r0, c.N, g, c.kind, lo, hi)
        fill_x1 = lambda r0, r1: _values(r1 - r0, c.K1, g, c.kind, lo, hi)
        fill_x2 = lambda r0, r1: _values(r1 - r0, c.K2, g, c.kind, lo, hi)
    rows1 = c.R // 2 + 5 if "1" in c.gather else c.R
    rows2 = c.R // 3 + 7 if "2" in c.gather else c.R
    dY = _operand(c.R, c.N, c.dy, c.odd, fill_dy)
    X1 = _operand(rows1, c.K1, c.x1, not c.odd, fill_x1)
    X2 = _operand(rows2, c.K2, c.x2, c.odd, fill_x2) if c.K2 else None
    idx1 = _index(c.R, rows1, g) if "1" in c.gather else None
    idx2 = _index(c.R, rows2, g) if "2" in c.gather else None
    if c.kind == "same":
        assert idx1 is None and idx2 is None
    dWb = torch.full((c.N, K + 5), NAN, device="cuda")
    old = _values(c.N, K, g, "int" if c.kind == "int" else "rand") if c.acc else None
    if c.acc:
        dWb[:, :K] = old
    dW = dWb[:, :K]
    db = None
    if c.dbias:
        db = _values(1, c.N, g, "int" if c.kind == "int" else "rand")[0] if c.acc else torch.full((c.N,), NAN, device="cuda")
    db_old = None if db is None else db.clone()
    if c.R >= 302081:
        print(f"[simt-linear] wgrad {c.id}: dmpnn_linear_wgrad_workspace_bytes = {_workspace_bytes(c.R, c.N, K)}")
    engine.linear_wgrad(dY, X1, c.K1, dW, c.N, idx1=idx1, X2=X2, K2=c.K2, idx2=idx2, dbias=db, accumulate=c.acc, R=c.R)
    torch.cuda.synchronize()
    gc.collect()
    torch.cuda.empty_cache()                  # the workspace (S N K floats) goes before the reference is formed
    assert bool(torch.isnan(dWb[:, K:]).all()), "dW padding written"
    ref = torch.zeros(c.N, K, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref)
    bref = torch.zeros(c.N, dtype=torch.float64, device="cuda")
    bmag = torch.zeros_like(bref)
    step = max(1, min(CHUNK, (1 << 28) // (8 * max(c.N, K))))
    for r0 in range(0, c.R, step):
        r1 = min(c.R, r0 + step)
        y = dY[r0:r1].double()
        A = _rows64(X1, idx1, r0, r1)
        if c.K2:
            A = torch.cat([A, _rows64(X2, idx2, r0, r1)], 1)
        ref += y.t() @ A
        mag += y.abs().t() @ A.abs()
        bref += y.sum(0)
        bmag += y.abs().sum(0)
        del y, A
    got = dW.double()
    if c.acc:
        ref = ref + old.double()
    if c.kind == "int":
        assert float(mag.max()) < 2 ** 24 and float(bmag.max()) < 2 ** 24
        assert torch.equal(got, ref), f"{c.id}: dW not exact"
        if db is not None:
            assert torch.equal(db.double(), bref + (db_old.double() if c.acc else 0)), f"{c.id}: dbias not exact"
        print(f"[simt-linear] wgrad {c.id}: exact")
        return
    bound = 20 * U * (1 + 1e-3) * mag + (2 * U * (ref.abs() + old.double().abs()) if c.acc and c.R > 0 else 0)
    st = _Stats(c.id + " dW")
    st.add(got, ref, bound)
    w, m = st.check()
    if db is not None:
        bb = bref + (db_old.double() if c.acc else 0)
        bbound = 6 * U * bmag + (2 * U * (bb.abs() + db_old.double().abs()) if c.acc and c.R > 0 else 0)
        sb = _Stats(c.id + " dbias")
        sb.add(db, bb, bbound)
        wb, mb = sb.check()
        w, m = max(w, wb), max(m, mb)
    _report("wgrad", c.id, w, m)
