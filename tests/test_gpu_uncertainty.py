"""GPU tier: target unscaling and the uncertainty predictors on the H100 kernels (csrc/head.cu: dmpnn_pred_transform(_bwd),
dmpnn_mve_loss, dmpnn_evidential_loss, dmpnn_quantile_loss, dmpnn_dirichlet_loss) -- the reference's own training step
(tests/golden/fixture_mpnn_<kind>.npz) eager and as one CUDA graph, the reference's trained checkpoints in eval mode, each
kernel against f64 torch running the reference formulas with autograd down to the raw MLP output, a bf16 encoder with each
head on a packed-loader batch as one graph, and the poisoned-allocation differential.

Bounds.  Each output element is held to  kappa * u * M  with u = 2^-24 and M the f64 sum of the magnitudes of the summands
of the formula the kernel evaluates for that element (products and quotients contribute their magnitude; digamma,
trigamma and lgamma their value's).  kappa = 64 covers the few dozen f32 operations per element.  The loss is held to
u * (kappa * sum_i M_i + depth * sum_i |term_i|) / n, depth = n / 1024 + 12 being the length of the kernel's fixed-order
sum.  Each kernel case also shows that the bound catches a reference computed with the criterion's default v_kl / alpha, a
one-sided amax tie, or unwrapped labels (tests `*_bound_catches_*`)."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch

from tests.test_uncertainty_host import (CKPTS, KINDS, PRED_DIRICHLET, PRED_EVIDENTIAL, PRED_MVE, PRED_QUANTILE,
                                         check_checkpoint, check_uncertainty_head, ref_loss, ref_transform)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
KAPPA = 64.0
ERRS: dict = {}            # kernel -> (worst, mean) error over bound, printed by test_zz_report_margins


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_uncertainty_matches_reference_training_step(kind, graph):
    check_uncertainty_head(kind, "cuda", graph=graph)


@pytest.mark.parametrize("kind", CKPTS)
def test_reference_checkpoint_predicts_as_the_reference(kind):
    check_checkpoint(kind, "cuda")


# ---- the kernels against f64 torch ------------------------------------------------------------------------------------------
LOSS = {"mve": (PRED_MVE, 2), "evidential": (PRED_EVIDENTIAL, 4), "quantile": (PRED_QUANTILE, 2)}
PARAMS = {"mve": {}, "evidential": dict(v_kl=0.35, eps=0.05), "quantile": dict(alpha=0.3), "dirichlet": dict(v_kl=0.35)}
DEFAULTS = {"evidential": dict(v_kl=0.2, eps=0.05), "quantile": dict(alpha=0.1), "dirichlet": dict(v_kl=0.2)}


def _raw(B, T, u, seed, integer=False):
    """Raw MLP outputs from -20 to 1e4 (softplus + 1 and its sums cross the digamma / trigamma switch-over at 6)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn(B, T * u, device="cuda", generator=g) * 3
    pick = torch.rand(B, T * u, device="cuda", generator=g)
    X = torch.where(pick < 0.05, torch.full_like(X, -20.0), X)
    X = torch.where((pick > 0.95) & (pick < 0.97), torch.rand(B, T * u, device="cuda", generator=g) * 1e4, X)
    X = torch.where(pick > 0.99, torch.rand(B, T * u, device="cuda", generator=g) * 20 + 5, X)
    if integer:
        X = X.clamp(-20, 50).round()
    w = torch.rand(B, device="cuda", generator=g) * 1.5 + 0.5
    tw = torch.rand(T, device="cuda", generator=g) * 1.5 + 0.5
    return X, w, tw, g


def _kernel(kind, P, Y, w, tw, u):
    from chemprop_b200 import engine as K

    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    p = PARAMS[kind]
    if kind == "mve":
        K.mve_loss(P, Y, w, tw, loss, dP)
    elif kind == "evidential":
        K.evidential_loss(P, Y, w, tw, p["v_kl"], p["eps"], loss, dP)
    elif kind == "quantile":
        K.quantile_loss(P, Y, w, tw, p["alpha"], loss, dP)
    else:
        K.dirichlet_loss(P, Y, w, tw, u, p["v_kl"], loss, dP)
    return loss, dP


def _digamma_abs(x):
    return torch.digamma(x).abs()


def _magnitudes(kind, P, y, v_kl=0.0, eps=0.0, alpha=0.1):
    """f64 sums of the magnitudes of the summands of each dP entry (b x T x u) and of each loss term (b x T)."""
    if kind == "mve":
        mu, v = P.unbind(-1)
        e = mu.abs() + y.abs()
        return torch.stack((e / v, 0.5 / v + e * e / (2 * v * v)), -1), e * e / (2 * v) + 0.5 * torch.log(2 * math.pi * v).abs() + 1
    if kind == "evidential":
        # r = y - mean is one f32 rounding of exact inputs (relative error u), so |r| is its magnitude; every log of a
        # quantity known to a few u contributes 1 (its absolute error is that quantity's relative error)
        mu, v, a, be = P.unbind(-1)
        r = (y - mu).abs()
        om = 2 * be * (1 + v)
        D = v * r * r + om
        dm = (a + 0.5) * 2 * v * r / D + v_kl * (2 * v + a)
        dv = 0.5 / v + a * 2 * be / om + (a + 0.5) * (r * r + 2 * be) / D + v_kl * 2 * r
        da = om.log().abs() + D.log().abs() + 2 + _digamma_abs(a) + _digamma_abs(a + 0.5) + v_kl * r
        db = a * 2 * (1 + v) / om + (a + 0.5) * 2 * (1 + v) / D
        L = (0.5 * (math.pi / v).log().abs() + a * (om.log().abs() + 1) + (a + 0.5) * (D.log().abs() + 1) + 1
             + torch.lgamma(a).abs() + torch.lgamma(a + 0.5).abs() + v_kl * ((2 * v + a) * r + eps))
        return torch.stack((dm, dv, da, db), -1), L
    if kind == "quantile":
        m, I = P.unbind(-1)
        e = y.abs() + m.abs() + I.abs()
        return torch.ones_like(P), 2 * e
    C = P.shape[-1]
    k = y.trunc()
    k = torch.where(k < 0, k + C, k).clamp(0, C - 1).long()
    t = torch.eye(C, dtype=P.dtype, device=P.device)[k]
    S = P.sum(-1, keepdim=True)
    p = P / S
    at = t + (1 - t) * P
    Sa = at.sum(-1, keepdim=True)
    sp2 = (p * p).sum(-1, keepdim=True)
    pk = (p * t).sum(-1, keepdim=True)
    Bq = (p * (1 - p)).sum(-1, keepdim=True)
    sam1 = (at - 1).sum(-1, keepdim=True)
    dA = 2 / S * (1 + p + pk + sp2)
    dB = (2 + 2 * p + 2 * sp2) / S / (S + 1) + Bq / (S + 1) ** 2
    dK = ((at - 1) * torch.polygamma(1, at)).abs() + torch.polygamma(1, Sa) * sam1
    L = (2 + Bq / (S + 1) + v_kl * (torch.lgamma(Sa).abs() + at.lgamma().abs().sum(-1, keepdim=True) + math.lgamma(C)
                                    + ((at - 1) * (_digamma_abs(at) + _digamma_abs(Sa))).sum(-1, keepdim=True)))
    return dA + dB + v_kl * dK, L[..., 0]


def _bounds(kind, P64, Y, w, tw):
    """Per-entry dP bound (b x T x u) and the loss bound, from the magnitudes at the kernel's own input P."""
    m = torch.isfinite(Y)
    y = torch.where(m, Y, torch.zeros_like(Y)).double()
    Md, ML = _magnitudes(kind, P64, y, **PARAMS[kind])
    ww = (w.double().view(-1, 1) * tw.double().view(1, -1)) * m
    n = max(int(m.sum()), 1)
    dP_bound = KAPPA * U * Md * (ww / n)[..., None]
    depth = m.numel() / 1024 + 12
    loss_bound = U * (KAPPA * float((ML * ww).nan_to_num().sum()) + depth * float((ML * ww).nan_to_num().sum())) / n
    return dP_bound, loss_bound


def _ratio(err, bound):
    r = err / bound.clamp(min=1e-300)
    return float(r.max()), float(r.mean())


def _record(name, worst, mean):
    w0, m0 = ERRS.get(name, (0.0, 0.0))
    ERRS[name] = (max(w0, worst), max(m0, mean))


def _check_loss_kernel(kind, P, Y, w, tw, u, ref_kw=None):
    """The kernel at P against the f64 reference at P; returns the error ratios (loss, dP)."""
    loss, dP = _kernel(kind, P, Y, w, tw, u)
    b, T = Y.shape
    P64 = P.double().view(b, T, u)
    ref_l, ref_g = ref_loss(kind, P64, Y, w.double(), tw.double(), **(ref_kw if ref_kw is not None else PARAMS[kind]))
    dP_bound, loss_bound = _bounds(kind, P64, Y, w, tw)
    rd = _ratio((dP.double().view(b, T, u) - ref_g).abs(), dP_bound)
    err_l = abs(float(loss) - float(ref_l))
    rl = err_l / loss_bound if loss_bound > 0 else (0.0 if err_l == 0 else math.inf)
    return (rl, rd), (loss, dP)


def _targets(kind, P, T, u, g, B):
    if kind == "dirichlet":
        Y = torch.randint(0, u, (B, T), device="cuda", generator=g).float()
        Y = Y + torch.rand(B, T, device="cuda", generator=g) * 0.99               # truncated like .long()
        Y[torch.rand(B, T, device="cuda", generator=g) < 0.1] = -1.0              # wraps to the last class
        return Y
    Pv = P.view(B, T, u)
    Y = torch.randn(B, T, device="cuda", generator=g) * 4
    sel = torch.rand(B, T, device="cuda", generator=g)
    if kind == "evidential":
        Y = torch.where(sel < 0.2, Pv[..., 0], Y)                                 # residual exactly 0
    if kind == "quantile":                                                        # targets exactly on a bound
        lo, hi = Pv[..., 0] - Pv[..., 1] / 2, Pv[..., 0] + Pv[..., 1] / 2
        Y = torch.where(sel < 0.15, lo, torch.where(sel < 0.3, hi, Y))
    return Y


def _loss_case(kind, B, T, u):
    from chemprop_b200 import engine as K

    pk, _ = LOSS.get(kind, (PRED_DIRICHLET, u))
    X, w, tw, g = _raw(B, T, u, seed=B * 41 + T * 7 + u + len(kind), integer=(kind == "quantile"))
    P = torch.empty_like(X)
    K.pred_transform(X, pk, u, None, None, P)
    Y = _targets(kind, P, T, u, g, B)
    Y[torch.rand(B, T, device="cuda", generator=g) < 0.2] = float("nan")
    if T == 12:
        Y[:, 5] = float("nan")                                                    # a fully masked task
    return X, P, Y, w, tw, pk


CASES = [(k, B, T, u) for k in ("mve", "evidential", "quantile") for B in (1, 7, 10000) for T in (1, 12)
         for u in (LOSS[k][1],)] + [("dirichlet", B, T, C) for B in (1, 7, 10000) for T in (1, 12) for C in (2, 3, 10)]


@pytest.mark.parametrize("kind,B,T,u", CASES)
def test_loss_kernel_and_transform_vs_f64_torch(kind, B, T, u):
    from chemprop_b200 import engine as K

    X, P, Y, w, tw, pk = _loss_case(kind, B, T, u)
    # the transform against f64 softplus (+ 1)
    P_ref = ref_transform(X.double(), pk, u).reshape(B, -1)
    out_err = (P.double() - P_ref).abs() / (8 * U * (P_ref.abs() + 1e-30))
    assert float(out_err.max()) <= 1.0, float(out_err.max())
    _record("pred_transform", float(out_err.max()), float(out_err.mean()))
    # the loss kernel at the kernel's own P
    (rl, rd), (loss, dP) = _check_loss_kernel(kind, P, Y, w, tw, u)
    assert rl <= 1.0 and rd[0] <= 1.0, (rl, rd)
    _record(f"{kind}_loss", max(rl, rd[0]), rd[1])
    assert not bool(dP.view(B, T, u)[~torch.isfinite(Y)].ne(0).any())
    # the mirror, taken down to the raw output: f64 autograd through the reference transform and loss
    dX = torch.empty_like(X)
    K.pred_transform_bwd(X, dP, pk, u, None, dX)
    # f64 reference gradient at the kernel's P (the loss check above holds it), chained through f64 autograd of the
    # reference transform at X
    X64 = X.double().requires_grad_(True)
    P64 = ref_transform(X64, pk, u)
    _, g64 = ref_loss(kind, P.double().view(B, T, u), Y, w.double(), tw.double(), **PARAMS[kind])
    (dX_ref,) = torch.autograd.grad(P64, X64, g64)
    Md = _bounds(kind, P.double().view(B, T, u), Y, w, tw)[0] / (KAPPA * U)      # magnitudes x w tw / n
    (dX_mag,) = torch.autograd.grad(ref_transform(X64, pk, u), X64, Md + g64.abs())
    if pk == PRED_QUANTILE:
        v = (Md + g64.abs()).view(B, T, 2)
        dX_mag = torch.cat((0.5 * v[..., 0] + v[..., 1], 0.5 * v[..., 0] + v[..., 1]), 1)
    r = _ratio((dX.double() - dX_ref).abs(), KAPPA * U * dX_mag.abs() + 4 * U * dX_ref.abs())
    assert r[0] <= 1.0, r
    _record("pred_transform_bwd", *r)
    # bit-identical on repeat
    loss2, dP2 = _kernel(kind, P, Y, w, tw, u)
    dX2 = torch.empty_like(X)
    K.pred_transform_bwd(X, dP2, pk, u, None, dX2)
    assert torch.equal(loss, loss2) and torch.equal(dP, dP2) and torch.equal(dX, dX2)


@pytest.mark.parametrize("kind", ["evidential", "quantile", "dirichlet"])
def test_loss_bound_catches_the_default_parameter(kind):
    """A reference computed with the criterion's default v_kl / alpha in place of the configured one is outside the bound."""
    u = {"evidential": 4, "quantile": 2, "dirichlet": 3}[kind]
    X, P, Y, w, tw, _ = _loss_case(kind, 10000, 12, u)
    (rl, rd), _ = _check_loss_kernel(kind, P, Y, w, tw, u, ref_kw=DEFAULTS[kind])
    assert rd[0] > 10 or rl > 10, (rl, rd)


def test_quantile_bound_catches_a_one_sided_tie():
    """Targets exactly on a bound: torch's amax splits the gradient; taking one side is outside the bound."""
    X, P, Y, w, tw, _ = _loss_case("quantile", 7, 12, 2)
    m = torch.isfinite(Y)
    Pv = P.view(7, 12, 2)
    lo = Pv[..., 0] - Pv[..., 1] / 2
    ties = m & (Y == lo)
    assert int(ties.sum()) > 0
    _, dP = _kernel("quantile", P, Y, w, tw, 2)
    _, ref = ref_loss("quantile", Pv.double(), Y, w.double(), tw.double(), **PARAMS["quantile"])
    dP_bound, _ = _bounds("quantile", Pv.double(), Y, w, tw)
    a = PARAMS["quantile"]["alpha"] / 2
    one_sided = ref.clone()
    n = max(int(m.sum()), 1)
    sc = (w.double().view(-1, 1) * tw.double().view(1, -1)) / n
    one_sided[..., 0] = torch.where(ties, ref[..., 0] + 0.5 * (a - (a - 1)) * sc, ref[..., 0])     # tau_0 instead of the mean
    err = (dP.double().view(7, 12, 2) - one_sided).abs()[ties][:, 0]
    assert bool((err > dP_bound[ties][:, 0]).all())
    assert bool(((dP.double().view(7, 12, 2) - ref).abs() <= dP_bound).all())


def test_dirichlet_label_wrap_and_out_of_range_labels():
    """Label -1 is the last class (torch.eye(C)[-1]); label C and -C - 1 give NaN in their row only."""
    C = 3
    X, P, _, w, tw, _ = _loss_case("dirichlet", 6, 2, C)
    Y = torch.tensor([[0.0, -1.0], [2.0, -3.0], [3.0, 1.0], [-4.0, 0.0], [1.5, -0.5], [float("nan"), 2.0]], device="cuda")
    loss, dP = _kernel("dirichlet", P, Y, w, tw, C)
    assert bool(torch.isnan(loss).all())
    bad = torch.zeros(6, 2, dtype=torch.bool, device="cuda")
    bad[2, 0] = bad[3, 0] = True
    rows = dP.view(6, 2, C)
    assert torch.equal(torch.isnan(rows).all(-1), bad) and bool(torch.isfinite(rows[~bad]).all())
    ok = ~bad.any(1)
    (rl, rd), _ = _check_loss_kernel("dirichlet", P[ok], Y[ok], w[ok], tw, C)
    assert rl <= 1.0 and rd[0] <= 1.0
    # without the wrap, -1 would be no class at all: that reference is outside the bound (NaN vs finite)
    Yw = Y[ok].clone()
    Yw[Yw < 0] = float(C)
    l_nowrap, _ = ref_loss("dirichlet", P[ok].double().view(-1, 2, C), Yw, w[ok].double(), tw.double(), v_kl=0.35)
    loss_ok, dP_ok = _kernel("dirichlet", P[ok], Y[ok], w[ok], tw, C)
    assert bool(torch.isnan(l_nowrap)) and bool(torch.isfinite(loss_ok)) and bool(torch.isfinite(dP_ok).all())


def test_losses_with_every_target_masked_and_empty_batches():
    for kind, u in (("mve", 2), ("evidential", 4), ("quantile", 2), ("dirichlet", 3)):
        X, P, Y, w, tw, _ = _loss_case(kind, 9, 4, u)
        Y = torch.full_like(Y, float("nan"))
        loss, dP = _kernel(kind, P, Y, w, tw, u)
        assert float(loss) == 0.0 and not bool(dP.ne(0).any())
        E = torch.empty(0, 4 * u, device="cuda")
        assert float(_kernel(kind, E, torch.empty(0, 4, device="cuda"), None, None, u)[0]) == 0.0


def test_eval_transforms_unscale_like_the_reference():
    from chemprop_b200 import _lib
    from chemprop_b200 import engine as K

    B, T = 1000, 12
    for kind, u in ((_lib.PRED_REGRESSION, 1), (PRED_MVE, 2), (PRED_EVIDENTIAL, 4), (PRED_QUANTILE, 2),
                    (_lib.PRED_DIRICHLET_PROBS, 5), (_lib.PRED_DIRICHLET_BINARY, 2)):
        X, _, _, g = _raw(B, T, u, seed=kind + 3)
        scaled = kind <= PRED_QUANTILE
        mean = torch.randn(T, device="cuda", generator=g) if scaled else None
        scale = torch.rand(T, device="cuda", generator=g) * 3 + 0.1 if scaled else None
        out = torch.empty_like(X)
        K.pred_transform(X, kind, u, mean, scale, out)
        ref = ref_transform(X.double(), kind, u, None if mean is None else mean.double(),
                            None if scale is None else scale.double()).reshape(B, -1)
        mag = ref_transform(X.double().abs(), kind, u, None if mean is None else mean.double().abs(),
                            None if scale is None else scale.double()).reshape(B, -1).abs() + ref.abs()
        if kind == PRED_QUANTILE:            # hi - lo: both unscaled bounds enter each output
            lo, hi = X.double().abs().chunk(2, 1)
            m2 = (lo + hi) * scale.double().view(1, -1) + 2 * mean.double().abs().view(1, -1)
            mag = torch.cat((m2, m2), 1) + ref.abs()
        assert bool(((out.double() - ref).abs() <= 16 * U * mag).all()), kind
        if kind == _lib.PRED_REGRESSION:                                  # X * scale + mean rounded as torch rounds it
            assert torch.equal(out, X * scale.view(1, -1) + mean.view(1, -1))


# ---- a bf16 encoder with each head: one CUDA graph on a packed-loader batch -------------------------------------------------
def _head(kind, d_h):
    import chemprop_b200.nn as N

    tw = torch.linspace(0.5, 2.0, 12)
    if kind == "mve":
        return N.EngineMveFFN(n_tasks=12, input_dim=d_h, task_weights=tw)
    if kind == "evidential":
        return N.EngineEvidentialFFN(n_tasks=12, input_dim=d_h, criterion=N.EngineEvidentialLoss(tw, v_kl=0.35, eps=0.05))
    if kind == "quantile":
        return N.EngineQuantileFFN(n_tasks=12, input_dim=d_h, criterion=N.EngineQuantileLoss(tw, alpha=0.3))
    if kind == "binary_dirichlet":
        return N.EngineBinaryDirichletFFN(n_tasks=12, input_dim=d_h, task_weights=tw)
    return N.EngineMulticlassDirichletFFN(n_classes=10, n_tasks=1, input_dim=d_h)


def _targets_for(kind, rng, n):
    T = 1 if kind == "multiclass_dirichlet" else 12
    if kind == "multiclass_dirichlet":
        Y = rng.integers(0, 10, size=(n, T))
    elif kind == "binary_dirichlet":
        Y = rng.integers(0, 2, size=(n, T))
    else:
        Y = rng.normal(size=(n, T))
    Y = Y.astype(np.float32)
    Y[rng.random(Y.shape) < 0.15] = np.nan
    return Y


@pytest.mark.parametrize("kind", KINDS)
def test_bf16_encoder_with_uncertainty_head_in_a_cuda_graph(kind):
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedBatchLoader, PackedMolGraphDataset, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    mgs = make_molecules(900, seed=41, shuffle_edges=True, min_atoms=1)
    rng = np.random.default_rng(5)
    Y, w = _targets_for(kind, rng, 900), rng.uniform(0.5, 2.0, size=900).astype(np.float32)
    ds = PackedMolGraphDataset.from_molgraphs(mgs).to("cuda")
    loader = PackedBatchLoader(ds, batch_size=512, shuffle=True, seed=3, device="cuda", arrays={"Y": Y, "w": w})
    it = iter(loader)
    batch = next(it)
    it.close()
    torch.manual_seed(0)
    model = N.EngineMPNN(N.BondMessagePassing(d_v=ds.d_v, d_e=ds.d_e, precision="bf16"), N.MeanAggregation(),
                         _head(kind, 300), batch_norm=True).cuda().train()
    Yb, wb = batch.extras["Y"], batch.extras["w"]
    for p in model.parameters():
        p.grad = torch.zeros_like(p)

    def fn(b):
        for p in model.parameters():
            p.grad.zero_()
        loss = model.training_loss(b, Yb, wb)
        loss.backward()
        return loss

    eager = fn(batch.bmg).detach().clone()
    eager_grads = {k: p.grad.clone() for k, p in model.named_parameters()}
    assert bool(torch.isfinite(eager))
    step = CudaGraphStep(fn)
    for _ in range(2):
        out = step(batch.bmg).clone()
        assert torch.equal(out, eager)
        for k, p in model.named_parameters():
            assert torch.equal(p.grad, eager_grads[k]), k
    assert step.captures == 1 and step.replays == 2
    model.eval()
    with torch.no_grad():
        preds = model(batch.bmg)
    assert bool(torch.isfinite(preds).all())


# ---- poisoned allocations: every output and every gradient entry is written ---------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_uncertainty_step_does_not_depend_on_uninitialised_memory(kind, monkeypatch):
    import chemprop_b200.nn as N
    from tests.uninit_matrix import POISONS, assert_bit_identical, install_poison, make_batch

    bmg = make_batch({}, "cuda", n_mols=150)
    Y = torch.from_numpy(_targets_for(kind, np.random.default_rng(9), 150)).cuda()
    w = (torch.rand(150, generator=torch.Generator().manual_seed(9)) + 0.5).cuda()

    def run(fill):
        with monkeypatch.context() as m:
            install_poison(m, fill)
            torch.manual_seed(1234)
            ut = N.UnscaleTransform(torch.linspace(-1, 1, 12), torch.linspace(0.5, 2, 12))
            head = _head(kind, 300)
            if kind in ("mve", "evidential", "quantile"):
                head.output_transform = ut
            model = N.EngineMPNN(N.BondMessagePassing(precision="bf16"), N.MeanAggregation(), head,
                                 batch_norm=True).cuda().train()
            loss = model.training_loss(bmg, Y, w)
            loss.backward()
            out = {"loss": loss.detach().reshape(1)}
            out.update({"grad." + k: p.grad.detach() for k, p in model.named_parameters()})
            model.eval()
            with torch.no_grad():
                out["preds"] = model(bmg)
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in out.items()}

    ref = run(0.0)
    for name in sorted(POISONS):
        assert_bit_identical(ref, run(POISONS[name]), f"{name} fill")


def test_zz_report_margins():
    """Worst and mean error over bound of each kernel across the f64 cases above (recorded in DESIGN.md section 10)."""
    for k, (worst, mean) in sorted(ERRS.items()):
        print(f"MARGIN {k}: worst {worst:.3g} mean {mean:.3g}")
