"""GPU tier: count-data regression on the H100 kernels -- dmpnn_enrichment_loss (NLogProbEnrichment), dmpnn_pinball_loss_rows
(PointQuantileLoss) and dmpnn_pred_transform(_bwd) kind 7 (RegressionFFN's Softplus output) against float64 torch running
the restatements of tests/test_enrichment_host.py with autograd; the reference's own training steps
(tests/golden/fixture_mpnn_{enrichment_*,quantile_point}.npz) on both encoder tiers, eager and as one CUDA graph replayed
across same-signature twins; repeated launches and poisoned outputs.

Bounds.  As in tests/test_gpu_uncertainty.py, each element is held to  kappa * u * M  (u = 2^-24, kappa = 64) with M the
f64 magnitude of what the kernel evaluates for it.  For the enrichment term, with Mz the sum of the magnitudes of z's
summands over |zscale| and c the clamped z / zscale: M_L = |L| + |dL/dc| Mz, and the gradient's
M_g = |dL/dc| / |zscale d| (M_dz + |dz| (1 + (|c| + 1) Mz)), M_dz being the sum of the magnitudes of dz/dRd's two terms
(the second factor is the error z carries into dL/dc, whose log-derivative is at most |c| + 1).  Rows whose |z / zscale|
lies within its own error of zinterval may fall on either side of the clamp and are left out of the gradient check (they
are counted, and must stay under 0.5 %).  The loss is held to u (kappa sum_i w_i M_L,i + depth sum_i |w_i L_i|) / n with depth the
longest summation path of the kernel's fixed-order reduction (tests/test_gpu_mab_model.py's _depth).  The worst and mean
error-to-bound ratios are printed by test_zz_report_margins."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_enrichment_host import (KINDS, METHODS, PRED_SOFTPLUS, build_model, check_head, ref_enrichment_loss,
                                        ref_pinball_loss)
from tests.test_gpu_mab_model import _depth
from tests.util import golden_bmg, load_golden

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = 2.0 ** -24
KAPPA = 64.0
ERRS: dict = {}


def _record(name, worst, mean):
    w0, m0 = ERRS.get(name, (0.0, 0.0))
    ERRS[name] = (max(w0, worst), max(m0, mean))


# ---- the enrichment kernel against float64 -------------------------------------------------------------------------------
def _magnitudes(R, Y, d, method, zscale, zinterval):
    """f64 per-row (L, dL/dR unweighted, M_L, M_g, ambiguous-at-the-clamp) at the kernel's own input."""
    R = R.double().reshape(-1)
    k = torch.nan_to_num(Y.double(), nan=0.0)
    k1, k2 = k[:, 0], k[:, 1]
    Rd = R / d
    if method == "score":
        D = torch.sqrt((k1 + k2) * Rd)
        z = (k1 - k2 * Rd) / D
        Mz = (k1.abs() + (k2 * Rd).abs()) / D
        t1, t2 = -k2 / D, -z / (2 * Rd)
    elif method == "wald":
        D = torch.sqrt(k1 + k2 * Rd ** 2)
        z = (k1 - k2 * Rd) / D
        Mz = (k1.abs() + (k2 * Rd).abs()) / D
        t1, t2 = -k2 / D, -z * k2 * Rd / D ** 2
    else:
        A, Bq, S = torch.sqrt(k1 + 0.375), torch.sqrt((k2 + 0.375) * Rd), torch.sqrt(1 + Rd)
        z = 2 * (A - Bq) / S
        Mz = 2 * (A + Bq) / S
        t1, t2 = -(k2 + 0.375) / (Bq * S), -z / (2 * (1 + Rd))
    c = z / zscale
    Mz = Mz / abs(zscale)
    cl = c.clamp(-zinterval, zinterval)
    x = cl.abs() / math.sqrt(2)
    L = -torch.log(torch.special.erfc(x))
    dLdc = torch.sign(cl) * math.sqrt(2 / math.pi) * torch.exp(-x * x) / torch.special.erfc(x)
    dz = t1 + t2
    M_L = L.abs() + dLdc.abs() * Mz
    M_g = dLdc.abs() / abs(zscale * d) * ((t1.abs() + t2.abs()) + dz.abs() * (1 + (cl.abs() + 1) * Mz))
    ambiguous = (c.abs() - zinterval).abs() <= KAPPA * U * Mz
    return L, M_L, M_g, ambiguous


def _enrich_inputs(B, method, seed, zero_rows=False):
    g = torch.Generator().manual_seed(seed)
    R = torch.exp(torch.empty(B).uniform_(math.log(1e-6), math.log(1e3), generator=g)).float().view(B, 1)
    lam = torch.exp(torch.empty(B, 2).uniform_(math.log(0.1), math.log(1e4), generator=g))
    Y = torch.poisson(lam, generator=g).float()
    Y[torch.rand(B, 2, generator=g) < 0.08] = float("nan")
    if B > 3:
        Y[1] = float("nan")                                                  # a fully masked row
    if method != "sqrt" and not zero_rows:                                   # keep z finite everywhere
        k = torch.nan_to_num(Y)
        Y[(k == 0).all(1), 0] = 1.0
    w = torch.rand(B, generator=g) + 0.5
    tw = torch.tensor([1.0, 0.5])
    d = float(np.float32(float(torch.nansum(Y[:, 1])) / max(float(torch.nansum(Y[:, 0])), 1.0)))
    return R, Y, w, tw, d


def _enrich_call(R, Y, w, tw, d, method, zscale, zinterval, dR=None):
    from chemprop_b200 import _lib, engine

    loss = torch.empty(1, device=DEV)
    dR = torch.empty_like(R) if dR is None else dR
    engine.enrichment_loss(R, Y, w, tw, d, _lib.ENRICH_METHODS[method], zscale, zinterval, loss, dR)
    return loss, dR


def _check_enrichment(R, Y, w, tw, d, method, zscale, zinterval, name="enrichment"):
    Rc, Yc, wc, twc = (t.to(DEV) for t in (R, Y, w, tw))
    loss, dR = _enrich_call(Rc, Yc, wc, twc, d, method, zscale, zinterval)
    ref_l, ref_g = ref_enrichment_loss(R.double(), Y.double(), w.double(), tw.double(), d, method, zscale, zinterval)
    L, M_L, M_g, amb = _magnitudes(R, Y, d, method, zscale, zinterval)
    m = torch.isfinite(Y.double())
    ww = w.double() * (m.double() * tw.double().view(1, 2)).sum(1)
    n = max(int(m.sum()), 1)
    g_bound = KAPPA * U * M_g * ww / n
    err = (dR.double().cpu().view(-1) - ref_g.view(-1)).abs()
    keep = ~amb
    assert int(amb.sum()) <= max(2, Y.shape[0] // 200), int(amb.sum())
    r = err[keep] / g_bound[keep].clamp(min=1e-300)
    assert bool((err[keep] <= g_bound[keep]).all()), float(r.max())
    l_bound = U * (KAPPA * float((M_L * ww).sum()) + _depth(Y.shape[0], single_block=True) * float((L * ww).abs().sum())) / n
    err_l = abs(float(loss) - float(ref_l))
    assert err_l <= l_bound, (err_l, l_bound)
    _record(name, max(float(r.max()) if r.numel() else 0.0, err_l / l_bound if l_bound else 0.0),
            float(r.mean()) if r.numel() else 0.0)
    return loss, dR


@pytest.mark.parametrize("method", list(METHODS))
@pytest.mark.parametrize("B", [1, 7, 10_000, 1_000_003])
def test_enrichment_kernel_against_float64(B, method):
    R, Y, w, tw, d = _enrich_inputs(B, method, seed=B + len(method))
    zscale, zinterval = (1.0, 5.0) if method != "score" else (1.7, 3.0)
    _check_enrichment(R, Y, w, tw, d, method, zscale, zinterval, f"enrichment_{method}")


def test_enrichment_at_the_clamp_bounds_and_at_zero():
    """Rd = 1 exactly (R = d): score with (k1, k2) = (4, 0) and (0, 4) gives z = +-2 exactly, which with zinterval 2 sits on
    the clamp's bounds, where the gradient passes; (9, 0) gives z = 3, beyond them; k1 = k2 gives z = 0 exactly (every
    method), where d|c|/dc = 0."""
    d = 2.0
    R = torch.full((5, 1), d)
    Y = torch.tensor([[4.0, 0.0], [0.0, 4.0], [3.0, 3.0], [7.0, 7.0], [9.0, 0.0]])
    w, tw = torch.ones(5), torch.ones(2)
    for method in METHODS:
        loss, dR = _check_enrichment(R, Y, w, tw, d, method, 1.0, 2.0, f"enrichment_{method}")
        assert dR[2, 0] == 0 and dR[3, 0] == 0
    _, dR = _enrich_call(R.to(DEV), Y.to(DEV), w.to(DEV), tw.to(DEV), d, "score", 1.0, 2.0)
    assert dR[0, 0] != 0 and dR[1, 0] != 0                                       # at +-zinterval: passes
    assert dR[4, 0] == 0                                                         # z = 3 beyond it: zero
    _, dR = _enrich_call(R.to(DEV), Y.to(DEV), w.to(DEV), tw.to(DEV), d, "score", 1.0, 1.999)
    assert dR[0, 0] == 0 and dR[1, 0] == 0


def test_enrichment_nan_from_masked_rows_and_fully_masked_batches():
    """score with a row of zero counts: NaN loss even when that row is fully masked (the reference raises for it); a NaN
    prediction likewise; every count masked gives loss 0 and dR 0."""
    R, Y, w, tw, d = _enrich_inputs(64, "score", seed=5)
    Y[10] = float("nan")                                                          # masked: counts enter z as 0 -> 0 / 0
    loss, dR = _enrich_call(R.to(DEV), Y.to(DEV), w.to(DEV), tw.to(DEV), d, "score", 1.0, 5.0)
    assert torch.isnan(loss).all() and torch.isnan(dR[10]).all()
    R2 = R.clone()
    R2[3] = float("nan")
    Yk = torch.nan_to_num(Y, nan=1.0)
    loss, _ = _enrich_call(R2.to(DEV), Yk.to(DEV), w.to(DEV), tw.to(DEV), d, "sqrt", 1.0, 5.0)
    assert torch.isnan(loss).all()
    Yn = torch.full_like(Y, float("nan"))
    loss, dR = _enrich_call(R.to(DEV), Yn.to(DEV), w.to(DEV), tw.to(DEV), d, "sqrt", 1.0, 5.0)
    assert float(loss) == 0.0 and bool((dR == 0).all())


# ---- the pinball kernel against float64 ----------------------------------------------------------------------------------
@pytest.mark.parametrize("R,T", [(1, 1), (14, 3), (1025, 2), (249_000, 1), (1_100_000, 2)])
def test_pinball_loss_rows_against_float64(R, T):
    from chemprop_b200 import engine

    g = torch.Generator().manual_seed(R + T)
    P = torch.randn(R, T, generator=g)
    Y = torch.randn(R, T, generator=g)
    Y[torch.rand(R, T, generator=g) < 0.1] = float("nan")
    tie = torch.rand(R, T, generator=g) < 0.05
    Y = torch.where(tie, P, Y)                                                   # diff == 0 exactly
    w, tw, alpha = torch.rand(R, generator=g) + 0.5, torch.linspace(0.5, 1.5, T), 0.3
    loss, dP = torch.empty(1, device=DEV), torch.empty(R, T, device=DEV)
    engine.pinball_loss_rows(P.to(DEV), Y.to(DEV), w.to(DEV), tw.to(DEV), alpha, loss, dP)
    ref_l, ref_g = ref_pinball_loss(P.double(), Y.double(), w.double(), tw.double(), alpha)
    m = torch.isfinite(Y)
    n = max(int(m.sum()), 1)
    ww = w.double().view(-1, 1) * tw.double().view(1, -1)
    g_bound = KAPPA * U * ref_g.abs() + 1e-300
    err = (dP.double().cpu() - ref_g).abs()
    assert bool((err <= g_bound).all()), float((err / g_bound).max())
    assert bool((dP.cpu()[tie & m] != 0).all())
    exp_tie = (1 - alpha) * (ww / n)[tie & m]
    np.testing.assert_allclose(dP.double().cpu()[tie & m].numpy(), exp_tie.numpy(), rtol=1e-6)
    terms = torch.where(m, (torch.nan_to_num(Y.double()) - P.double()).abs() * ww, torch.zeros_like(ww))
    l_bound = U * (KAPPA + _depth(R * T)) * float(terms.sum()) / n
    assert abs(float(loss) - float(ref_l)) <= l_bound
    _record("pinball_loss_rows", float((err / g_bound).max()), float((err / g_bound).mean()))


# ---- the Softplus output transform ----------------------------------------------------------------------------------------
def test_softplus_transform_forward_and_backward():
    from chemprop_b200 import engine

    X = torch.cat((torch.tensor([-120.0, -80.0, -30.0, -10.0, -1.0, 0.0, 1.0, 19.0, 19.999, 20.0, 20.001, 21.0, 60.0]),
                   torch.randn(4096, generator=torch.Generator().manual_seed(3)) * 8)).view(-1, 1)
    Xc = X.to(DEV)
    out, dX = torch.empty_like(Xc), torch.empty_like(Xc)
    engine.pred_transform(Xc, PRED_SOFTPLUS, 1, None, None, out)
    G = torch.rand_like(X) + 0.5
    engine.pred_transform_bwd(Xc, G.to(DEV), PRED_SOFTPLUS, 1, None, dX)
    x64 = X.double().requires_grad_(True)
    y64 = F.softplus(x64)
    (g64,) = torch.autograd.grad(y64, x64, G.double())
    for ours, ref, name in ((out, y64.detach(), "softplus"), (dX, g64, "softplus_bwd")):
        err = (ours.double().cpu() - ref).abs()
        bound = 8 * U * ref.abs() + 1e-44
        assert bool((err <= bound).all()), (name, float((err / bound).max()))
        _record(name, float((err / bound).max()), float((err / bound).mean()))


# ---- the reference's training steps -------------------------------------------------------------------------------------
@pytest.mark.parametrize("graph", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_matches_reference_training_step(kind, graph):
    check_head(kind, DEV, graph=graph)


@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_bf16_tier_matches_reference_training_step(kind):
    check_head(kind, DEV, graph=True, precision="bf16")


def _mgs(g):
    from chemprop_b200.data import MolGraph

    batch, ei, rev = g["batch"], g["edge_index"], g["rev_edge_index"]
    out = []
    for i in range(int(g["n_mols"])):
        a = np.nonzero(batch == i)[0]
        e = np.nonzero(np.isin(ei[0], a))[0]
        a0, e0 = (a[0] if a.size else 0), (e[0] if e.size else 0)
        out.append(MolGraph(g["V"][a], g["E"][e], ei[:, e] - a0, rev[e] - e0))
    return out


@pytest.mark.parametrize("kind", ["enrichment_sqrt", "enrichment_wald", "quantile_point"])
def test_graph_replays_across_same_signature_twins_are_the_eager_steps(kind):
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.graph import CudaGraphStep
    from tests import graph_twins as TW

    g = load_golden(f"fixture_mpnn_{kind}")
    Y, w = torch.from_numpy(g["Y"]).to(DEV), torch.from_numpy(g["w"]).to(DEV)
    mgs = _mgs(g)
    batches = [golden_bmg(g, DEV)] + [BatchMolGraph(TW.twin(mgs, s)) for s in (1, 2)]
    for b in batches[1:]:
        b.to(DEV)

    def fresh():
        m = build_model(kind, g).to(DEV).train()
        for p in m.parameters():
            p.grad = torch.zeros_like(p)
        return m

    def step_of(model):
        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            out = model.training_loss(b, Y, w)
            out.backward()
            return out
        return fn

    eager = []
    for b in batches:
        m = fresh()
        loss = step_of(m)(b).detach().clone()
        eager.append((loss, {k: p.grad.clone() for k, p in m.named_parameters()}))
    model = fresh()
    state = {k: v.clone() for k, v in model.state_dict().items()}
    step = CudaGraphStep(step_of(model))
    for b, (loss, grads) in zip(batches, eager):
        model.load_state_dict(state)
        out = step(b).clone()
        assert torch.equal(out, loss)
        for k, p in model.named_parameters():
            assert torch.equal(p.grad, grads[k]), k
    assert step.captures == 1


# ---- outputs --------------------------------------------------------------------------------------------------------------
def test_repeated_launches_are_bit_identical_and_poisoned_outputs_are_written():
    from chemprop_b200 import engine

    R, Y, w, tw, d = _enrich_inputs(10_000, "wald", seed=11)
    Rc, Yc, wc, twc = (t.to(DEV) for t in (R, Y, w, tw))
    first = _enrich_call(Rc, Yc, wc, twc, d, "wald", 1.0, 5.0)
    for fill in (float("nan"), 7.0):
        loss, dR = torch.full((1,), fill, device=DEV), torch.full((10_000, 3), fill, device=DEV)
        engine.enrichment_loss(Rc, Yc, wc, twc, d, 2, 1.0, 5.0, loss, dR[:, :1])
        assert torch.equal(loss, first[0]) and torch.equal(dR[:, :1], first[1])
        assert bool((dR[:, 1:] == fill).all() if fill == fill else dR[:, 1:].isnan().all())   # padding left untouched
    P = torch.randn(50_000, 2, device=DEV)
    Yp = torch.randn(50_000, 2, device=DEV)
    ref = None
    for fill in (None, float("nan"), -3.0):
        loss = torch.empty(1, device=DEV) if fill is None else torch.full((1,), fill, device=DEV)
        dP = torch.empty(50_000, 2, device=DEV) if fill is None else torch.full((50_000, 2), fill, device=DEV)
        engine.pinball_loss_rows(P, Yp, None, None, 0.3, loss, dP)
        if ref is None:
            ref = (loss.clone(), dP.clone())
        assert torch.equal(loss, ref[0]) and torch.equal(dP, ref[1])
    X = torch.randn(3000, 1, device=DEV)
    outs = []
    for fill in (float("nan"), 1.0):
        o = torch.full_like(X, fill)
        engine.pred_transform(X, PRED_SOFTPLUS, 1, None, None, o)
        outs.append(o)
    assert torch.equal(outs[0], outs[1])


def test_del_notebook_model_trains_evaluates_and_predicts_as_a_cuda_graph():
    """examples/training_NLogProbEnrichment.ipynb's model from Engine* classes: a few optimizer steps as one captured
    graph, evaluate with the criterion as the metric, predict."""
    import chemprop_b200.nn as N
    from chemprop_b200.graph import CudaGraphStep

    g = load_golden("fixture_mpnn_enrichment_sqrt")
    n1, n2 = int(g["n1"]), int(g["n2"])
    torch.manual_seed(0)
    model = N.EngineMPNN(N.BondMessagePassing(d_h=40), N.MeanAggregation(),
                         N.EngineRegressionFFN(input_dim=40, criterion=N.EngineNLogProbEnrichment(n1=n1, n2=n2),
                                               output_transform=torch.nn.Softplus()), batch_norm=True).to(DEV).train()
    bmg = golden_bmg(g, DEV)
    Y, w = torch.from_numpy(g["Y"]).to(DEV), torch.from_numpy(g["w"]).to(DEV)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, capturable=True)

    def fn(b):
        opt.zero_grad(set_to_none=False)
        loss = model.training_loss(b, Y, w)
        loss.backward()
        opt.step()
        return loss

    for p in model.parameters():
        p.grad = torch.zeros_like(p)
    step = CudaGraphStep(fn)
    losses = [float(step(bmg)) for _ in range(30)]
    assert step.captures == 1 and all(map(math.isfinite, losses)) and losses[-1] < losses[0]
    out = model.evaluate([(bmg, None, None, Y, w, None, None)],
                         metrics=[N.EngineCriterionMetric(N.EngineNLogProbEnrichment(n1=n1, n2=n2).to(DEV))])
    assert math.isfinite(out["val_loss"]) and math.isfinite(out["val/EngineNLogProbEnrichment"])
    preds = model.predict([(bmg, None, None, Y, w, None, None)])
    assert preds.shape == (14, 1) and bool((preds > 0).all())


def test_zz_report_margins():
    for k, (worst, mean) in sorted(ERRS.items()):
        print(f"{k}: worst error / bound {worst:.3g}, mean {mean:.3g}")
