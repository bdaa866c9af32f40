"""GPU tier: every fused activation -- identity, ReLU, LeakyReLU(slope), tanh, ELU(alpha) -- at non-default parameters, in
every kernel that applies tau or tau'.

(a) The fused depth step: one launch of each of the 101 instantiations that the dispatch of csrc/step_fused_kernel.cuh can
    reach (dispatch_fwd / dispatch_bwd), keyed by the template arguments (ACT, FIRST, BIAS, MODE, FAR, DROP, ATOM) it
    launches; `test_cases_cover_every_instantiation` fails when an instantiation has no case.
(b) Reference: float64 on the GPU with the kernel's rounding points.  The A operand (message / neighbour sum, packed bf16) is
    checked against its restatement first; the output is then computed from the kernel's own operand (M_out / N_out / G_out,
    or an identity first-step launch for steps that do not store it), so a one-ulp tie in the operand does not blur the
    bound on the GEMM and epilogue.  Bound per element: half a bf16 ulp of the reference plus Lip(tau) x an f32
    accumulation term in sum |a w| (Lip = max(1, slope, alpha)); the mean error is held to 0.6 of the mean bound.  The
    inputs put pre-activations in the band |z| < 1e-3, in ELU's saturated region (z to -8 and below), and Y at exactly +0
    and -0 for the masks.  Every output starts NaN: all data columns must be written, [h, pad16(h)) must hold zeros and
    the columns past pad16(h) must keep their NaN.
(c) act_bwd, sum_act_bwd, segment_sum / bond_message / rev_average with tau applied on load, and the epilogues of
    linear_x3 and the SIMT linear_fwd, against float64 with worst-case f32 bounds.
(d) BondMessagePassing / AtomMessagePassing with LeakyReLU(0.3), ELU(alpha=0.5) and Identity against the f64 restatement
    at test_gpu_parity.py::test_medium_batch_vs_oracle's bars (scaled by max|H| once it exceeds 1)."""
import functools
import gc
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu

NAN = float("nan")
U = 2.0 ** -24                                   # unit roundoff of f32
ACTS = ("none", "relu", "leakyrelu", "tanh", "elu")
FWD, MASK, COPY, LAST = 0, 1, 2, 3               # MODE_FWD, MODE_BWD_MASK, MODE_BWD_COPY, MODE_BWD_LAST
MEAN_BAR = 0.6                                   # mean |err| / mean bound (rounding to nearest alone gives <= 0.5)


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _code(act):
    from chemprop_b200 import _lib

    return {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "leakyrelu": _lib.ACT_LEAKYRELU, "tanh": _lib.ACT_TANH,
            "elu": _lib.ACT_ELU}[act]


def _p32(p):
    """The parameter as the kernels see it (a float argument)."""
    return float(np.float32(p))


def _tau64(act, p, z):
    if act == "none":
        return z
    if act == "relu":
        return torch.relu(z)
    if act == "leakyrelu":
        return torch.where(z > 0, z, _p32(p) * z)
    if act == "tanh":
        return torch.tanh(z)
    return torch.where(z > 0, z, _p32(p) * torch.expm1(z))


def _dtau64(act, p, y, from_pre):
    """tau' from the output y = tau(z) (the mirrors' act_grad_from_out) or from the pre-activation (act_grad_from_pre)."""
    one = torch.ones_like(y)
    if act == "none":
        return one
    if act == "relu":
        return (y > 0).to(y.dtype)
    if act == "leakyrelu":
        return torch.where(y > 0, one, _p32(p) * one)
    if act == "tanh":
        t = torch.tanh(y) if from_pre else y
        return 1 - t * t
    return torch.where(y > 0, one, _p32(p) * torch.exp(y) if from_pre else y + _p32(p))


def _lip(act, p):
    return max(1.0, p) if act in ("leakyrelu", "elu") else 1.0


def _half_ulp_bf16(x):
    """Half a bf16 ulp of |x| (f64; 0 at 0): x in [2^(e-1), 2^e) has ulp 2^(e-8)."""
    _, e = torch.frexp(x.abs())
    return torch.where(x != 0, torch.pow(2.0, (e - 9).double()), torch.zeros_like(x))


def _report(group, case, worst, mean):
    print(f"[fused-acts] {group} {case}: worst err / bound {worst:.3f}, mean err / mean bound {mean:.3f}")


def _check_bound(got, ref, delta, what, bf16_out=True):
    """|got - ref| <= (half a bf16 ulp of |ref| + delta, if the output is bf16) + delta everywhere; mean error <= MEAN_BAR of
    the mean bound.  Returns (worst ratio, mean ratio)."""
    g = got.double()
    assert bool(torch.isfinite(g).all()), f"{what}: non-finite output"
    bound = delta + (_half_ulp_bf16(ref.abs() + delta) if bf16_out else 0.0)
    err = (g - ref).abs()
    assert bool((err[bound == 0] == 0).all()), f"{what}: inexact where the bound is 0"
    ratio = torch.where(bound > 0, err / bound.clamp_min(1e-300), torch.zeros_like(err))
    worst, mean = ratio.max().item(), (err.sum() / bound.sum().clamp_min(1e-300)).item()
    assert worst <= 1.0, (what, "worst err / bound", worst, err.max().item())
    assert mean <= MEAN_BAR, (what, "mean err / mean bound", mean)
    return worst, mean


# ---------------------------------------------------------------------------------------------------------------------
# (a) the instantiation matrix of the fused depth step
# ---------------------------------------------------------------------------------------------------------------------
def _instantiations():
    """(ACT, FIRST, BIAS, MODE, FAR, DROP, ATOM) of every k_bond_step_fused instantiation dispatch_fwd / dispatch_bwd launch:
    bond forward = every activation x FIRST x BIAS plus ReLU with keep bits (DROP), each with and without FAR; atom forward
    = every activation x FIRST x BIAS; backward = MODE 2 (activation-free) plus every activation x {MODE 1, MODE 3}, bond with
    and without FAR, atom without."""
    s = set()
    for atom, fars in ((0, (0, 1)), (1, (0,))):
        for far in fars:
            for a in ACTS:
                for first in (0, 1):
                    for bias in (0, 1):
                        s.add((a, first, bias, FWD, far, 0, atom))
                        if a == "relu" and not atom:
                            s.add((a, first, bias, FWD, far, 1, atom))
            s.add(("none", 0, 0, COPY, far, 0, atom))
            for a in ACTS:
                for mode in (MASK, LAST):
                    s.add((a, 0, 0, mode, far, 0, atom))
    return s


def _param(act, i):
    """Alternate the non-default and default parameters; ReLU / tanh / identity get a value they must ignore."""
    return {"leakyrelu": (0.3, 0.1), "elu": (0.5, 1.0)}.get(act, (0.7, 0.7))[i % 2]


def _cases():
    out = []
    for i, key in enumerate(sorted(_instantiations(), key=str)):
        act, first, bias, mode, far, drop, atom = key
        batch = ""
        if atom:       # plain molecules, condensed reaction graphs, or in-degree up to 11 (tiles past the staged table)
            batch = (("dense" if first else "cgr") if bias else "plain") if mode == FWD else \
                    {MASK: "dense" if act in ("tanh", "elu") else "plain", COPY: "dense", LAST: "cgr"}[mode]
        out.append((key, 300, _param(act, i), batch))
    # single-chunk epilogues (hp <= 80): one 64-column and one 16-column case
    out.append((("leakyrelu", 1, 1, FWD, 0, 0, 0), 64, 0.3, ""))
    out.append((("elu", 0, 0, MASK, 0, 0, 0), 16, 0.5, ""))
    out.append((("elu", 0, 1, FWD, 0, 0, 1), 16, 0.5, "dense"))
    return out


CASES = _cases()


def _case_id(c):
    (act, first, bias, mode, far, drop, atom), h, p, batch = c
    parts = ["atom" if atom else "bond", ("fwd", "mask", "copy", "last")[mode], act if mode != COPY else "plain",
             "first" if first else "", "bias" if bias else "", "far" if far else "", "drop" if drop else "",
             batch, f"p{p}" if act in ("leakyrelu", "elu") else "", f"h{h}"]
    return "-".join(x for x in parts if x)


def test_cases_cover_every_instantiation():
    want = _instantiations()
    have = {c[0] for c in CASES}
    assert len(want) == 101
    assert have == want, (sorted(want - have, key=str), sorted(have - want, key=str))
    print(f"[fused-acts] fused-step instantiations launched by the cases below: {len(have)} of {len(want)}")


@functools.lru_cache(maxsize=None)
def _batch(atom, far, batch):
    from tests.test_gpu_fused_step import _atom_setup, _setup

    if atom:
        if batch == "dense":
            from tests.test_gpu_high_degree import _atom_batch

            lay = _atom_batch(seed=31)[0]          # asserts tiles of more than 512 edge rows (global neighbour look-ups)
        else:
            lay = _atom_setup(90 if batch == "cgr" else 700, 16, seed=23, cgr=(batch == "cgr"))[0]
        assert lay.max_tile_atoms <= 128
        return lay, None
    lay = _setup(300, 16, seed=41, big=25)[0] if far else _setup(700, 16, seed=5)[0]
    lay_cpu = SimpleNamespace(E=lay.E, V=lay.V, rowptr=lay.rowptr.cpu(), dst_row=lay.dst_row.cpu(), rev_row=lay.rev_row.cpu())
    return lay, lay_cpu


def _buffer(rows, h, ld, x=None):
    """bf16 rows x ld: x in [0, h), zeros in [h, pad16(h)), NaN past pad16(h) (a kernel must not read or write there)."""
    hp = (h + 15) // 16 * 16
    t = torch.full((rows, ld), NAN, dtype=torch.bfloat16, device="cuda")
    t[:, h:hp] = 0
    if x is not None:
        t[:, :h] = x.bfloat16()
    return t


def _banded(rows, h, g):
    """Pre-activation-like values: columns [0, h/8) in |x| < 1e-3, [h/8, h/4) in [-8, -2] (ELU's saturated region), the
    rest N(0, 0.7^2)."""
    x = torch.randn(rows, h, device="cuda", generator=g) * 0.7
    nz, sat = max(1, h // 8), max(2, h // 4)
    x[:, :nz] = (torch.rand(rows, nz, device="cuda", generator=g) * 2 - 1) * 1e-3
    x[:, nz:sat] = -2 - 6 * torch.rand(rows, sat - nz, device="cuda", generator=g)
    return x


def _signed_zeros_(Y, h):
    """Exact +0 and -0 entries in the data columns of a bf16 buffer (the masks' y > 0 / y + alpha at both zeros)."""
    Y[0::7, 0:h:5] = 0.0
    Y[3::7, 2:h:5] = -0.0
    assert bool((Y[3::7, 2:h:5].view(torch.int16) == -32768).all())


def _weights(h, g):
    """W_h with the output rows of the near-zero band scaled by 1e-3 (so that z stays in |z| < ~2e-3 there), and a bias."""
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    nz = max(1, h // 8)
    W[:nz] *= 1e-3
    b[:nz] *= 1e-3
    return W, b


def _operand_ref(lay, lay_cpu, X, h, atom, through_rev):
    """The A operand with the kernel's rounding points: packed-bf16 sibling / neighbour sums.  Bond forward: indexed by the
    edge whose message it is (M[e]); bond mirror and atoms: by the output row."""
    from tests.emu import _sibling_sum_packed
    from tests.test_gpu_fused_step import _neighbour_sum

    if atom:
        return _neighbour_sum(lay, X)
    A = _sibling_sum_packed(X.cpu(), lay_cpu, through_rev=through_rev).cuda()
    if through_rev:
        return A
    M = torch.zeros_like(A)
    M[lay.rev_row.long()] = A
    return M


def _check_operand(got, ref, h, what):
    """The kernel's operand against its restatement: equal but for rare one-ulp ties (f32 sums of in-degree > 4, tau in f32
    vs f64 on the first step)."""
    g = got[:, :h].float()
    assert bool(torch.isfinite(g).all()), f"{what}: operand rows / columns left unwritten"
    diff = (g - ref).abs()
    frac = (diff != 0).float().mean().item()
    assert frac <= 2e-3, (what, "operand entries off their restatement", frac)
    torch.testing.assert_close(g, ref, rtol=2 ** -7, atol=2 ** -10 * ref.abs().max().item(),
                               msg=lambda m: f"{what} operand: {m}")


def _check_padding(out, h, what):
    hp = (h + 15) // 16 * 16
    assert hp == h or not bool(out[:, h:hp].float().ne(0).any()), f"{what}: columns [h, pad16(h)) not zero"
    assert bool(torch.isnan(out[:, hp:].float()).all()), f"{what}: stray writes past pad16(h)"


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_fused_step_instantiation_vs_f64(case):
    from chemprop_b200.engine import (atom_step_bwd_fused, atom_step_fused, bond_step_bwd_fused, bond_step_fused,
                                      pack_weight_bf16)

    (act, first, bias, mode, far, drop, atom), h, p, batch = case
    what = _case_id(case)
    lay, lay_cpu = _batch(atom, far, batch)
    if not atom:
        trp, tap, nt, wf, nw, dr = lay.step_tables()
        if far:
            assert wf is not None and int(wf[: int(nw.item())].sum()) > 0, "no flagged windows: FAR kernels not reached"
        else:
            assert wf is None
    rows = lay.V if atom else lay.E
    hp = (h + 15) // 16 * 16
    ld = hp + 32
    g = torch.Generator(device="cuda").manual_seed(1000 * h + len(what))
    W, b = _weights(h, g)
    Wb = W.bfloat16().double()
    code = _code(act)
    lip = _lip(act, p)

    if mode == FWD:
        H0 = _buffer(rows, h, ld, _banded(rows, h, g))
        Hin = H0 if first else _buffer(rows, h, ld, torch.randn(rows, h, device="cuda", generator=g) * 0.5)
        out = _buffer(rows, h, ld)
        out[:, h:hp] = NAN
        Mk = _buffer(rows, h, ld)
        Mk[:, h:hp] = NAN
        keep, kw = None, {}
        if drop:
            nj = hp // 16
            bits = torch.randint(-32768, 32768, (rows, nj), device="cuda", dtype=torch.int32, generator=g)
            kw = dict(drop_bits=bits.to(torch.int16).contiguous(), drop_scale=1.25)
            keep = (((bits & 0xFFFF).unsqueeze(-1) >> torch.arange(16, device="cuda")) & 1).reshape(rows, hp)[:, :h].double()
        Wpk = pack_weight_bf16(W)
        bb = b if bias else None
        if atom:
            atom_step_fused(Hin, H0, out, h, Wpk, bb, lay, code, p, bool(first), N_out=Mk if first else None)
        else:
            bond_step_fused(Hin, H0, out, h, Wpk, bb, lay, code, p, bool(first), M_out=Mk if first else None, **kw)
        if not first:       # the same gather, stored: an identity first step on the same input
            scratch = _buffer(rows, h, ld)
            if atom:
                atom_step_fused(Hin, H0, scratch, h, Wpk, None, lay, _code("none"), 0.0, True, N_out=Mk)
            else:
                bond_step_fused(Hin, H0, scratch, h, Wpk, None, lay, _code("none"), 0.0, True, M_out=Mk)
        torch.cuda.synchronize()
        X = Hin[:, :h].double()
        if first:
            X = _tau64(act, p, X)
        opr = _operand_ref(lay, lay_cpu, X.bfloat16().float(), h, atom, through_rev=False)
        _check_operand(Mk, opr, h, what)
        A = Mk[:, :h].double()
        Z = A @ Wb.t()
        Ua = A.abs() @ Wb.abs().t()
        h0 = H0[:, :h].double()
        bd = b.double() if bias else torch.zeros(h, dtype=torch.float64, device="cuda")
        z = Z + h0 + bd
        y = _tau64(act, p, z)
        s = 1.0
        if drop:
            y, s = y * keep * 1.25, 1.25
        delta = s * (lip * (h * 2 * U * Ua + 3 * U * (Z.abs() + h0.abs() + bd.abs())) + 8 * U * y.abs() / s)
        worst, mean = _check_bound(out[:, :h], y, delta, what)
        if act == "elu":
            assert z.min().item() < -8.0 and bool(((z.abs() < 1e-3)).any()), (what, "pre-activation bands not reached")
    else:
        dZ = _buffer(rows, h, ld, torch.randn(rows, h, device="cuda", generator=g))
        Y = None
        if mode == MASK:
            Y = _buffer(rows, h, ld, _tau64(act, p, _banded(rows, h, g).double()))
        elif mode == LAST:
            Y = _buffer(rows, h, ld, _banded(rows, h, g))
        if Y is not None:
            _signed_zeros_(Y, h)
        adds_all = [dZ, _buffer(rows, h, ld, torch.randn(rows, h, device="cuda", generator=g))]
        WpkT = pack_weight_bf16(W.t().contiguous())
        worst, mean = 0.0, 0.0
        for n_add in ((0, 1, 2) if mode == LAST else (0,)):
            adds = tuple(adds_all[:n_add])      # the step's own input is one of the addends in the engine
            out = _buffer(rows, h, ld)
            out[:, h:hp] = NAN
            Gk = _buffer(rows, h, ld)
            Gk[:, h:hp] = NAN
            fn = atom_step_bwd_fused if atom else bond_step_bwd_fused
            fn(dZ, Y, out, h, WpkT, lay, code, p, G_out=Gk, y_is_preact=(mode == LAST), addends=adds)
            torch.cuda.synchronize()
            opr = _operand_ref(lay, lay_cpu, dZ[:, :h].float(), h, atom, through_rev=True)
            _check_operand(Gk, opr, h, what)
            A = Gk[:, :h].double()
            D = A @ Wb
            Ua = A.abs() @ Wb.abs()
            d = torch.ones_like(D) if Y is None else _dtau64(act, p, Y[:, :h].double(), mode == LAST)
            ref = D * d
            asum = torch.zeros_like(ref)
            for a in adds:
                ref = ref + a[:, :h].double()
                asum = asum + a[:, :h].double().abs()
            delta = lip * h * 2 * U * Ua + 8 * U * (1 + d.abs()) * D.abs() + 4 * U * ((D * d).abs() + asum)
            w, m = _check_bound(out[:, :h], ref, delta, f"{what}, {n_add} addends")
            worst, mean = max(worst, w), max(mean, m)
            _check_padding(out, h, f"{what}, {n_add} addends")
    if mode == FWD:
        _check_padding(out, h, what)
    _report("step", what, worst, mean)


# ---------------------------------------------------------------------------------------------------------------------
# (c) the elementwise and linear kernels that apply tau or tau'
# ---------------------------------------------------------------------------------------------------------------------
ACT_PARAMS = [("none", 0.7), ("relu", 0.7), ("leakyrelu", 0.3), ("tanh", 0.7), ("elu", 0.5)]
C_EW = 300
LD_EW = 320


def _poisoned(R, C, dt=torch.float32, g=None, x=None):
    X = torch.full((R, LD_EW), NAN, dtype=dt, device="cuda")
    X[:, :C] = (torch.randn(R, C, device="cuda", generator=g) if x is None else x).to(dt)
    return X


def _preact(R, C, g, scale=2.0):
    """Pre-activations with a near-zero band, ELU's saturated region and exact +0 / -0 entries."""
    x = torch.randn(R, C, device="cuda", generator=g) * scale
    x[:, :20] *= 1e-3
    x[:, 20:40] = -2 - 7 * torch.rand(R, 20, device="cuda", generator=g)
    x[0::5, 40:60] = 0.0
    x[2::5, 40:60] = -0.0
    return x


def _gtol(act, d):
    """Error of tau' evaluated in f32 (tanhf / expf within 2 ulp; 1 - y y and y + alpha rounded once)."""
    return 8 * U * (1 + d.abs()) if act in ("tanh", "elu") else U * d.abs()


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("from_preact", [False, True])
@pytest.mark.parametrize("act,p", ACT_PARAMS)
def test_act_bwd_vs_f64(act, p, from_preact, dt):
    """dZ = G[gidx] * tau'(Y) (Y the output, or the pre-activation), and ACC += dZ in f32."""
    from chemprop_b200 import engine

    dtype = torch.bfloat16 if dt == "bf16" else torch.float32
    R, RG, C = 9000, 2500, C_EW
    g = torch.Generator(device="cuda").manual_seed(hash((act, from_preact, dt)) % 1000)
    G = _poisoned(RG, C, dtype, g)
    z = _preact(R, C, g)
    Y = _poisoned(R, C, dtype, x=z if from_preact else _tau64(act, p, z.double()).float())
    gidx = torch.randint(0, RG, (R,), device="cuda", dtype=torch.int32, generator=g)
    acc = _poisoned(R, C, torch.float32, g)
    acc0 = acc[:, :C].double()
    dZ = torch.full((R, LD_EW), NAN, dtype=dtype, device="cuda")
    engine.act_bwd(G, Y, R, C, act=_code(act), act_param=p, gidx=gidx, from_preact=from_preact, dZ=dZ, acc=acc)
    torch.cuda.synchronize()
    gd = G[gidx.long(), :C].double()
    d = _dtau64(act, p, Y[:, :C].double(), from_preact)
    ref = gd * d
    delta = gd.abs() * _gtol(act, d) + U * ref.abs()
    w, m = _check_bound(dZ[:, :C], ref, delta, f"act_bwd {act} {dt}", bf16_out=(dt == "bf16"))
    extra = 2 * _half_ulp_bf16(ref.abs() + delta) if dt == "bf16" else 0.0     # ACC may add the rounded dZ
    _check_bound(acc[:, :C], acc0 + ref, delta + extra + U * (acc0 + ref).abs(), f"act_bwd acc {act} {dt}", bf16_out=False)
    assert bool(torch.isnan(dZ[:, C:].float()).all()) and bool(torch.isnan(acc[:, C:]).all())
    _report("act_bwd", (act, p, from_preact, dt), w, m)


@pytest.mark.parametrize("dt", ["f32", "bf16"])
@pytest.mark.parametrize("act,p", ACT_PARAMS)
def test_sum_act_bwd_vs_f64(act, p, dt):
    """OUT = Z_1 + Z_2 + Z_3 + G * tau'(Ypre) in one pass."""
    from chemprop_b200 import engine

    dtype = torch.bfloat16 if dt == "bf16" else torch.float32
    R, C = 7000, C_EW
    g = torch.Generator(device="cuda").manual_seed(hash((act, dt)) % 1000 + 7)
    Zs = [_poisoned(R, C, dtype, g) for _ in range(3)]
    G = _poisoned(R, C, dtype, g)
    Yp = _poisoned(R, C, dtype, x=_preact(R, C, g))
    out = torch.full((R, LD_EW), NAN, dtype=dtype, device="cuda")
    engine.sum_act_bwd(Zs, G, Yp, out, R, C, act=_code(act), act_param=p)
    torch.cuda.synchronize()
    d = _dtau64(act, p, Yp[:, :C].double(), True)
    gd = G[:, :C].double() * d
    ref = gd + sum(z[:, :C].double() for z in Zs)
    mag = gd.abs() + sum(z[:, :C].double().abs() for z in Zs)
    delta = 5 * U * mag + G[:, :C].double().abs() * _gtol(act, d)
    w, m = _check_bound(out[:, :C], ref, delta, f"sum_act_bwd {act} {dt}", bf16_out=(dt == "bf16"))
    assert bool(torch.isnan(out[:, C:].float()).all())
    _report("sum_act_bwd", (act, p, dt), w, m)


@pytest.fixture(scope="module")
def ew_layout():
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules

    bmg = BatchMolGraph(make_molecules(160, seed=12, shuffle_edges=True))
    bmg.to("cuda")
    lay = engine.get_layout(bmg)
    counts = (lay.rowptr[1:] - lay.rowptr[:-1]).long()
    seg = torch.repeat_interleave(torch.arange(lay.V, device="cuda"), counts)     # atom (segment) of every edge row
    return lay, seg, counts


def _tau_tol(t):
    """Error of tau evaluated in f32 on an f32 input (tanhf 2 ulp, alpha * expm1f two roundings + 1 ulp)."""
    return 4 * U * t.abs()


@pytest.mark.parametrize("act,p", ACT_PARAMS)
def test_segment_kernels_apply_tau_on_load(ew_layout, act, p):
    """The first step's tau inside segment_sum (M_v = sum of tau(H_0) over in-edges), bond_message and rev_average."""
    from chemprop_b200 import engine

    lay, seg, counts = ew_layout
    C = C_EW
    g = torch.Generator(device="cuda").manual_seed(hash(act) % 1000 + 3)
    X = _poisoned(lay.E, C, x=_preact(lay.E, C, g))
    t = _tau64(act, p, X[:, :C].double())
    S = torch.zeros(lay.V, C, dtype=torch.float64, device="cuda").index_add_(0, seg, t)
    A = torch.zeros(lay.V, C, dtype=torch.float64, device="cuda").index_add_(0, seg, t.abs())
    cnt = counts.double()[:, None]

    out = torch.full((lay.V, LD_EW), NAN, device="cuda")
    engine.segment_sum(X, lay.rowptr, lay.V, C, out, act=_code(act), act_param=p, pad_to=C)
    torch.cuda.synchronize()
    w1, m1 = _check_bound(out[:, :C], S, (cnt + 5) * U * A, f"segment_sum {act}", bf16_out=False)
    assert bool(torch.isnan(out[:, C:]).all())

    out = torch.full((lay.E, LD_EW), NAN, device="cuda")
    engine.bond_message(X, lay, C, out, act=_code(act), act_param=p)
    torch.cuda.synchronize()
    rev = lay.rev_row.long()
    ref, bnd = torch.empty_like(t), torch.empty_like(t)
    ref[rev] = S[seg] - t
    bnd[rev] = (counts[seg].double()[:, None] + 5) * U * (A[seg] + t.abs())
    w2, m2 = _check_bound(out[:, :C], ref, bnd, f"bond_message {act}", bf16_out=False)
    assert bool(torch.isnan(out[:, C:]).all())

    out = torch.full((lay.E, LD_EW), NAN, device="cuda")
    engine.rev_average(X, lay, C, out, act=_code(act), act_param=p)
    torch.cuda.synchronize()
    ref = (t + t[rev]) / 2
    w3, m3 = _check_bound(out[:, :C], ref, 5 * U * (t.abs() + t[rev].abs()), f"rev_average {act}", bf16_out=False)
    assert bool(torch.isnan(out[:, C:]).all())
    _report("segment", (act, p), max(w1, w2, w3), max(m1, m2, m3))


@pytest.mark.parametrize("kernel", ["linear_x3", "linear_fwd"])
@pytest.mark.parametrize("act,p", ACT_PARAMS)
def test_linear_epilogues_vs_f64(act, p, kernel):
    """act(A . W^T + bias + res) with the activation in the epilogue: the 3xTF32 tensor-core kernel (the fp32 tier's W_h /
    W_o GEMMs) and the SIMT kernel (W_i / W_o, the FFN head)."""
    from chemprop_b200 import engine

    R, K, N = 6000, 300, 300
    g = torch.Generator(device="cuda").manual_seed(hash((act, kernel)) % 1000 + 11)
    A = torch.zeros(R, LD_EW, device="cuda")
    A[:, :K] = torch.randn(R, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    res = _poisoned(R, N, x=_preact(R, N, g))
    W[:60] *= 1e-4           # output columns [0, 60): z ~ res, whose bands (near zero, saturated, +-0) then reach tau
    b[:60] *= 1e-4
    out = torch.full((R, LD_EW), NAN, device="cuda")
    if kernel == "linear_x3":
        engine.linear_x3(A, K, engine.pack_weight_x3(W), N, out, bias=b, res=res, act=_code(act), act_param=p, R=R, pad_to=N)
        rel = 1e-5               # tests/test_gpu_x3.py: of sum |terms|
    else:
        engine.linear_fwd(A, K, W.contiguous(), out, N, bias=b, res=res, act=_code(act), act_param=p, R=R, pad_to=N)
        rel = (K + 3) * U
    torch.cuda.synchronize()
    Ad, Wd = A[:, :K].double(), W.double()
    z = Ad @ Wd.t() + b.double() + res[:, :N].double()
    mag = Ad.abs() @ Wd.abs().t() + b.double().abs() + res[:, :N].double().abs()
    y = _tau64(act, p, z)
    delta = _lip(act, p) * rel * mag + _tau_tol(y) + 1e-30
    w, m = _check_bound(out[:, :N], y, delta, f"{kernel} {act}", bf16_out=False)
    assert bool(torch.isnan(out[:, N:]).all())
    if act == "elu":
        assert z.min().item() < -8.0 and bool((z.abs() < 1e-3).any())
    _report(kernel, (act, p), w, m)


# ---------------------------------------------------------------------------------------------------------------------
# (d) the modules against the f64 restatement
# ---------------------------------------------------------------------------------------------------------------------
MODULE_ACTS = [("LeakyReLU(0.3)", lambda: nn.LeakyReLU(0.3)), ("ELU(alpha=0.5)", lambda: nn.ELU(alpha=0.5)),
               ("Identity", nn.Identity)]


def _module_vs_oracle(kind, precision, tau, mgs, monkeypatch):
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation
    from oracle import restatement as R

    calls = {"bond": 0, "atom": 0}
    fb, fa = engine.bond_step_fused, engine.atom_step_fused
    monkeypatch.setattr(engine, "bond_step_fused", lambda *a, **k: (calls.__setitem__("bond", calls["bond"] + 1), fb(*a, **k))[1])
    monkeypatch.setattr(engine, "atom_step_fused", lambda *a, **k: (calls.__setitem__("atom", calls["atom"] + 1), fa(*a, **k))[1])
    torch.manual_seed(0)
    bmg = BatchMolGraph(mgs)
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_h=300, depth=3, bias=True, activation=tau, precision=precision).cuda()
    assert not mp.uses_composed_tier()
    bmg.to("cuda")
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward(kind, bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], P["W_i.bias"], P["W_h.weight"], P["W_h.bias"], P["W_o.weight"],
                                      P["W_o.bias"], 3, tau)
    a_ref = R.aggregate(H_ref, bmg.batch, "mean")
    a_ref.square().sum().backward()
    H = mp(bmg)
    a = MeanAggregation()(H, bmg.batch)
    a.float().square().sum().backward()
    torch.cuda.synchronize()
    # the bars of test_medium_batch_vs_oracle, relative to the hidden-state scale once max|H| exceeds 1 (as there for bf16;
    # Identity leaves H unsquashed)
    tol = (1e-5 if precision == "fp32" else 1e-2) * max(1.0, H_ref.detach().abs().max().item())
    errH = (H.detach().double() - H_ref.detach()).abs().max().item()
    erra = (a.detach().double() - a_ref.detach()).abs().max().item()
    assert errH <= tol and erra <= tol, (errH, erra, tol)
    worst = 0.0
    for k, p in mp.named_parameters():
        ref = P[k].grad
        scale = max(1e-6, ref.abs().max().item())
        bar = (2e-4 if precision == "fp32" else 6e-2) * scale
        err = (p.grad.double() - ref).abs().max().item()
        worst = max(worst, err / bar)
        assert err <= bar, (k, err, scale)
    print(f"[fused-acts] module {kind} {precision} {tau!r}: H {errH / tol:.3f} of bar, worst gradient {worst:.3f} of bar")
    return bmg, calls


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("kind", ["bond", "atom"])
@pytest.mark.parametrize("name,make", MODULE_ACTS, ids=[n for n, _ in MODULE_ACTS])
def test_module_vs_f64_oracle(name, make, kind, precision, monkeypatch):
    from chemprop_b200.data import make_molecules

    mgs = make_molecules(1500, seed=5, shuffle_edges=(kind == "bond"))
    _, calls = _module_vs_oracle(kind, precision, make(), mgs, monkeypatch)
    if precision == "bf16":        # depth 3: two fused steps forward (the first step is stored by the W_i epilogue)
        assert calls[kind] >= 2, calls


@pytest.mark.parametrize("name,make", MODULE_ACTS, ids=[n for n, _ in MODULE_ACTS])
def test_module_windows_of_large_molecules_vs_f64_oracle(name, make, monkeypatch):
    """bf16 BondMessagePassing on a batch with molecules of more than 128 directed edges: the FAR step kernels."""
    from chemprop_b200.data import make_molecules
    from chemprop_b200.engine import get_layout

    mgs = make_molecules(300, seed=9, shuffle_edges=True)
    bigs = make_molecules(20, seed=10, mean_atoms=110.0, std_atoms=40.0, min_atoms=66, max_atoms=200, shuffle_edges=True)
    for i, m in enumerate(bigs):
        mgs.insert(i * 15 + 1, m)
    bmg, calls = _module_vs_oracle("bond", "bf16", make(), mgs, monkeypatch)
    lay = get_layout(bmg)
    wf, nw = lay.step_tables()[3:5]
    assert wf is not None and int(wf[: int(nw.item())].sum()) > 0 and calls["bond"] >= 2, calls
