"""CPU tier: count-data regression -- EngineNLogProbEnrichment on EngineRegressionFFN's Softplus output, and
EnginePointQuantileLoss at every level (csrc/head.cu's dmpnn_enrichment_loss and dmpnn_pred_transform kind 7,
csrc/row_head.cu's dmpnn_pinball_loss_rows) through torch emulations of their kernel wrappers, against the reference's own
`MPNN.training_step` (tests/golden/fixture_mpnn_{enrichment_*,quantile_point}.npz, written by
tools/make_golden_enrichment.py): shape rules and refusals, task weights, masks, the output transforms, the validation
loss and its error, and which kernels a step launches.  The float64 restatements below are also the oracle of
tests/test_gpu_enrichment.py; they are pinned to the reference's own float64 step here."""
from __future__ import annotations

import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from tests.test_spectral_host import patch_spectral
from tests.test_uncertainty_host import pred_transform as _uq_pred_transform
from tests.test_uncertainty_host import pred_transform_bwd as _uq_pred_transform_bwd
from tests.util import golden_bmg, load_golden

PRED_SOFTPLUS = 7
METHODS = {"sqrt": 0, "score": 1, "wald": 2}
KINDS = ("enrichment_sqrt", "enrichment_score", "enrichment_wald", "quantile_point")


# ---- float64 restatements of the criteria (chemprop/nn/metrics.py:264-288, 616-692), dtype-generic ------------------------
def ref_zstats(R, k1, k2, d, method):
    """NLogProbEnrichment.get_zstats with d = n2 / n1 (no NaN check: the caller sees the NaN)."""
    Rd = R / d
    if method == "score":
        return (k1 - k2 * Rd) / torch.sqrt((k1 + k2) * Rd)
    if method == "wald":
        return (k1 - k2 * Rd) / torch.sqrt(k1 + k2 * Rd ** 2)
    return 2 * (torch.sqrt(k1 + 3 / 8.0) - torch.sqrt((k2 + 3 / 8.0) * Rd)) / torch.sqrt(1 + Rd)


def ref_enrichment_unreduced(R, Y, d, method, zscale, zinterval, exact=True):
    """b-vector of terms; Y's NaN counts enter z as 0 (training_step's nan_to_num).  exact: -log(erfc) (the value the
    kernel is held to); otherwise the reference's -log(1 - erf)."""
    k = torch.nan_to_num(Y, nan=0.0).to(R.dtype)
    z = ref_zstats(R.reshape(-1), k[:, 0], k[:, 1], d, method)
    a = torch.clamp(z / zscale, -zinterval, zinterval).abs() / math.sqrt(2)
    return -torch.log(torch.special.erfc(a)) if exact else -torch.log(1 - torch.erf(a))


def _weights(w, tw, b, T, dtype):
    ww = torch.ones(b, T, dtype=dtype) if w is None else w.reshape(-1, 1).to(dtype).expand(b, T)
    return ww * (1.0 if tw is None else tw.reshape(1, -1).to(dtype))


def ref_enrichment_loss(R, Y, w, tw, d, method, zscale, zinterval):
    """The kernel's contract (include/dmpnn.h) on the reference formula, gradient by autograd: sum L w tw m / sum m with the
    b x 1 loss broadcast over the b x 2 mask; every term enters (masked ones times 0), so a NaN z gives a NaN loss; loss 0
    when every count is masked."""
    m = torch.isfinite(Y)
    with torch.enable_grad():
        Rl = R.detach().clone().requires_grad_(True)
        L = ref_enrichment_unreduced(Rl, Y, d, method, zscale, zinterval)
        loss = (L.view(-1, 1) * _weights(w, tw, *Y.shape, R.dtype) * m).sum() / m.sum().clamp(min=1)
        (g,) = torch.autograd.grad(loss, Rl) if Rl.numel() else (torch.zeros_like(Rl),)
    return loss.detach(), g


def ref_pinball_loss(P, Y, w, tw, alpha):
    """PointQuantileLoss under the kernels' reduction: NaN targets masked, loss 0 and dP 0 when every target is masked;
    dL/dp at y == p is torch.where's second branch, 1 - alpha."""
    m = torch.isfinite(Y)
    with torch.enable_grad():
        Pl = P.detach().clone().requires_grad_(True)
        diff = torch.where(m, Y, torch.zeros_like(Y)).to(P.dtype) - Pl
        L = torch.where(diff > 0, alpha * diff, (1 - alpha) * (-diff))
        loss = torch.where(m, L * _weights(w, tw, *Y.shape, P.dtype), torch.zeros_like(L)).sum() / m.sum().clamp(min=1)
        (g,) = torch.autograd.grad(loss, Pl) if Pl.numel() else (torch.zeros_like(Pl),)
    return loss.detach(), torch.where(m, g, torch.zeros_like(g))


# ---- torch emulations of the engine wrappers (the kernels' contract, include/dmpnn.h) -------------------------------------
CALLS: list = []


def enrichment_loss(P, Y, w, tw, d, method, zscale, zinterval, loss, dP):
    CALLS.append("enrichment_loss")
    assert P.shape == (Y.shape[0], 1) and Y.shape[1] == 2 and (tw is None or tw.numel() == 2)
    assert w is None or w.numel() == Y.shape[0]
    name = {v: k for k, v in METHODS.items()}[method]
    f32 = lambda t: None if t is None else t.double()  # noqa: E731 -- the kernel is held to float64
    l, g = ref_enrichment_loss(P.double(), Y.double(), f32(w), f32(tw), float(np.float32(d)), name, zscale, zinterval)
    loss.copy_(l.reshape(1))
    if dP is not None:
        dP.copy_(g)


def pinball_loss_rows(P, Y, w, tw, alpha, loss, dP):
    CALLS.append("pinball_loss_rows")
    assert P.shape == Y.shape and (tw is None or tw.numel() == Y.shape[1]) and (w is None or w.numel() == Y.shape[0])
    l, g = ref_pinball_loss(P.double(), Y.double(), None if w is None else w.double(), None if tw is None else tw.double(),
                            alpha)
    loss.copy_(l.reshape(1))
    if dP is not None:
        dP.copy_(g)


def pred_transform(X, kind, u, mean, scale, out):
    if kind != PRED_SOFTPLUS:
        return _uq_pred_transform(X, kind, u, mean, scale, out)
    CALLS.append("pred_transform_softplus")
    assert u == 1 and mean is None and scale is None
    out.copy_(F.softplus(X))


def pred_transform_bwd(X, dOut, kind, u, scale, dX):
    if kind != PRED_SOFTPLUS:
        return _uq_pred_transform_bwd(X, dOut, kind, u, scale, dX)
    CALLS.append("pred_transform_bwd_softplus")
    with torch.enable_grad():
        x = X.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(F.softplus(x), x, dOut.reshape(x.shape))
    dX.copy_(g)


def patch_enrichment(monkeypatch):
    """patch_spectral plus the new wrappers; CALLS records their launches."""
    from chemprop_b200 import engine

    patch_spectral(monkeypatch)
    CALLS.clear()
    for name in ("enrichment_loss", "pinball_loss_rows", "pred_transform", "pred_transform_bwd"):
        monkeypatch.setattr(engine, name, globals()[name])


# ---- the training-step fixtures -----------------------------------------------------------------------------------------
def build_model(kind: str, g: dict, precision: str = "fp32"):
    """EngineMPNN of the fixture's configuration holding its initial state (strict load of the reference's state dict minus
    the criterion's torchmetrics states)."""
    import chemprop_b200.nn as N

    kw = dict(input_dim=40, hidden_dim=24, n_layers=2)
    if kind.startswith("enrichment"):
        crit = N.EngineNLogProbEnrichment(torch.ones(2), n1=int(g["n1"]), n2=int(g["n2"]), method=str(g["method"]),
                                          zscale=float(g["zscale"]), zinterval=float(g["zinterval"]))
        pred = N.EngineRegressionFFN(n_tasks=1, **kw, criterion=crit, output_transform=nn.Softplus())
    else:
        pred = N.EngineRegressionFFN(n_tasks=3, **kw, criterion=N.EnginePointQuantileLoss(torch.ones(3),
                                                                                          alpha=float(g["alpha"])))
    model = N.EngineMPNN(N.BondMessagePassing(d_h=40, depth=3, precision=precision), N.MeanAggregation(), pred,
                         batch_norm=True)
    state = {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")}
    res = model.load_state_dict({k: v for k, v in state.items() if not k.endswith(("total_loss", "num_samples"))},
                                strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model


def assert_within_reference_gap(ours, g: dict, key: str, rtol: float = 2e-4, atol: float = 2e-6):
    """|ours - ref32| <= 2 |ref32 - ref64| + rtol |ref32| + atol elementwise: the reference's own f32-vs-f64 gap, widened
    by the tolerance of the other fp32 fixtures."""
    ref32, ref64 = np.asarray(g[key], np.float64), np.asarray(g["f64." + key], np.float64)
    ours = np.asarray(ours, np.float64)
    bar = 2 * np.abs(ref32 - ref64) + rtol * np.abs(ref32) + atol
    err = np.abs(ours - ref32)
    assert ours.shape == ref32.shape and (err <= bar).all(), (key, float((err / bar).max()))


def check_head(kind: str, device: str, graph: bool = False, precision: str = "fp32"):
    """EngineMPNN.training_loss with the fixture's head and criterion against the reference's `MPNN.training_step`: loss,
    every gradient and the batch-norm running statistics within the reference's own f32-vs-f64 gap, eval-mode
    predictions.  `graph`: the step runs as one captured CUDA graph, and its replay must be bit-identical to the eager
    step."""
    g = load_golden(f"fixture_mpnn_{kind}")
    model = build_model(kind, g, precision).to(device).train()
    bmg = golden_bmg(g, device)
    Y, w = torch.from_numpy(g["Y"]).to(device), torch.from_numpy(g["w"]).to(device)
    loss = model.training_loss(bmg, Y, w)
    loss.backward()
    if graph:
        from chemprop_b200.graph import CudaGraphStep

        eager = loss.detach().clone()
        eager_grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        model = build_model(kind, g, precision).to(device).train()
        for p in model.parameters():
            p.grad = torch.zeros_like(p)
        rm0, rv0, nb0 = model.bn.running_mean.clone(), model.bn.running_var.clone(), model.bn.num_batches_tracked.clone()

        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            out = model.training_loss(b, Y, w)
            out.backward()
            return out

        step = CudaGraphStep(fn)
        step(bmg)
        model.bn.running_mean.copy_(rm0); model.bn.running_var.copy_(rv0); model.bn.num_batches_tracked.copy_(nb0)
        loss = step(bmg).clone()
        assert step.captures == 1 and step.replays == 2
        assert torch.equal(loss, eager)
        for k, p in model.named_parameters():
            assert torch.equal(p.grad, eager_grads[k]), k
    # the bf16 encoder tier: its own rounding, far above the reference's gap
    tol, bn_tol = ((dict(rtol=2e-4, atol=2e-6), dict(rtol=1e-5, atol=1e-6)) if precision == "fp32"
                   else (dict(rtol=5e-2, atol=1e-2), dict(rtol=1e-3, atol=1e-4)))
    assert_within_reference_gap(loss.detach().cpu().numpy(), g, "loss", **tol)
    for k, p in model.named_parameters():
        assert_within_reference_gap(p.grad.cpu().numpy(), g, "grad." + k, **tol)
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        assert_within_reference_gap(getattr(model.bn, k).cpu().numpy(), g, "after.bn." + k, **bn_tol)
    model.eval()
    with torch.no_grad():
        preds = model(bmg)
    assert preds.shape == g["preds_eval"].shape
    np.testing.assert_allclose(preds.cpu().numpy(), g["preds_eval"], rtol=tol["rtol"], atol=tol["atol"])
    return model


@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_matches_reference_training_step(kind, monkeypatch):
    patch_enrichment(monkeypatch)
    check_head(kind, "cpu")


def _z(g, preds):
    R = torch.from_numpy(np.asarray(preds, np.float64))
    k = torch.nan_to_num(torch.from_numpy(g["Y"]).double())
    return ref_zstats(R.reshape(-1), k[:, 0], k[:, 1], int(g["n2"]) / int(g["n1"]), str(g["method"])) / float(g["zscale"])


def test_fixtures_cover_the_cases_the_heads_must_handle():
    at_clamp = 0
    for kind in KINDS[:3]:
        g = load_golden(f"fixture_mpnn_{kind}")
        Y = g["Y"]
        assert Y.shape == (14, 2) and np.isnan(Y).sum() == 1 and (Y == 0).any() and g["w"].std() > 0
        assert int(g["n1"]) == np.nansum(Y[:, 0]) and int(g["n2"]) == np.nansum(Y[:, 1])
        assert (g["preds_train"] > 0).all()                                   # the Softplus output
        z = _z(g, g["f64.preds_train"])
        assert torch.isfinite(z).all()
        at_clamp += int((z.abs() >= float(g["zinterval"])).sum())
    assert at_clamp >= 2
    assert {float(load_golden(f"fixture_mpnn_{k}")["zscale"]) for k in KINDS[:3]} != {1.0}
    g = load_golden("fixture_mpnn_enrichment_score_raises")
    assert (np.nan_to_num(g["Y"]) == 0).all(1).any() and "Got nan loss" in str(g["error"])
    g = load_golden("fixture_mpnn_quantile_point")
    assert g["Y"].shape == (14, 3) and np.isnan(g["Y"]).sum() == 3 and float(g["alpha"]) == 0.3


@pytest.mark.parametrize("kind", KINDS)
def test_restatements_reproduce_the_reference_float64_step(kind):
    """The float64 restatements, on the reference's own float64 predictions, give its float64 loss."""
    g = load_golden(f"fixture_mpnn_{kind}")
    P = torch.from_numpy(g["f64.preds_train"])
    Y, w = torch.from_numpy(g["Y"]).double(), torch.from_numpy(g["w"]).double()
    tw = torch.from_numpy(g["param.predictor.criterion.task_weights"]).double()
    if kind.startswith("enrichment"):
        l, _ = ref_enrichment_loss(P, Y, w, tw, int(g["n2"]) / int(g["n1"]), str(g["method"]), float(g["zscale"]),
                                   float(g["zinterval"]))
        # the reference's f32 1 - erf, on its f32 predictions, gives its f32 loss
        P32 = torch.from_numpy(g["preds_train"])
        L32 = ref_enrichment_unreduced(P32, torch.from_numpy(g["Y"]), int(g["n2"]) / int(g["n1"]), str(g["method"]),
                                       float(g["zscale"]), float(g["zinterval"]), exact=False)
        m = torch.isfinite(torch.from_numpy(g["Y"]))
        l32 = (L32.view(-1, 1) * torch.from_numpy(g["w"]).view(-1, 1) * tw.float() * m).sum() / m.sum()
        np.testing.assert_allclose(float(l32), float(g["loss"]), rtol=1e-5)
    else:
        l, _ = ref_pinball_loss(P, Y, w, tw, float(g["alpha"]))
    # 1e-9: the reference's float64 1 - erf keeps about 10 digits of erfc near |z| = 5
    np.testing.assert_allclose(float(l), float(g["f64.loss"]), rtol=1e-9)


def test_erfc_holds_the_terms_the_reference_rounds_away():
    """At |z| = 5 the reference's f32 1 - erf gives 14.3329; the exact term is 14.3719."""
    z = torch.tensor([5.0, 4.0])
    exact = -torch.log(torch.special.erfc(z.double() / math.sqrt(2)))
    ref32 = -torch.log(1 - torch.erf(z / math.sqrt(2)))
    assert abs(float(exact[0]) - 14.3719) < 1e-3 and abs(float(ref32[0]) - 14.3329) < 1e-3


# ---- the criteria's host rules ----------------------------------------------------------------------------------------------
def _enrich_case(b=6, seed=0):
    import chemprop_b200.nn as N

    gen = torch.Generator().manual_seed(seed)
    R = torch.rand(b, 1, generator=gen) + 0.2
    Y = torch.poisson(torch.full((b, 2), 3.0), generator=gen)
    Y[0, 0] = 0.0
    Y[2, 1] = float("nan")
    crit = N.EngineNLogProbEnrichment(n1=int(np.nansum(Y[:, 0])), n2=int(np.nansum(Y[:, 1])))
    return crit, R, Y, torch.rand(b, generator=gen) + 0.5


def test_shape_rules_and_refusals(monkeypatch):
    """b x 1 predictions and b x 2 counts only; an unknown method, and bound masks, are refused on the host before any
    launch; the other criteria keep their own b x T rule."""
    import chemprop_b200.nn as N

    patch_enrichment(monkeypatch)
    crit, R, Y, w = _enrich_case()
    crit(R, Y, None, w)
    assert CALLS == ["enrichment_loss"]
    CALLS.clear()
    for P, T in ((R.expand(6, 2), Y), (R, Y[:, :1]), (R[:, 0], Y), (R, torch.cat((Y, Y), 1)), (R[:5], Y)):
        with pytest.raises(ValueError, match="b x 1 predictions and b x 2"):
            crit(P, T, None, w)
    crit.method = "exact"
    with pytest.raises(ValueError, match="Unsupported method: exact"):
        crit(R, Y, None, w)
    crit.method = "sqrt"
    lt = torch.zeros(6, 2, dtype=torch.bool)
    with pytest.raises(NotImplementedError, match="takes no lt_mask"):
        crit(R, Y, None, w, lt, None)
    pin = N.EnginePointQuantileLoss(alpha=0.2)
    with pytest.raises(NotImplementedError, match="takes no lt_mask"):
        pin(R, Y[:, :1], None, w, lt[:, :1], None)
    with pytest.raises(ValueError, match="b x T predictions and b x T targets"):
        pin(R, Y, None, w)
    assert CALLS == []
    with pytest.raises(ValueError, match="b x T predictions and b x T targets"):     # the others' rule is unchanged
        N.EngineMAE()(R, Y, None, w)


def test_task_weights_of_one_or_two_entries(monkeypatch):
    patch_enrichment(monkeypatch)
    crit, R, Y, w = _enrich_case()
    crit.task_weights = torch.full((1, 1), 0.7)
    one = crit(R, Y, None, w)
    crit.task_weights = torch.full((1, 2), 0.7)
    assert torch.equal(one, crit(R, Y, None, w))
    crit.task_weights = torch.tensor([[1.0, 0.25]])
    l, _ = ref_enrichment_loss(R.double(), Y.double(), w.double(), crit.task_weights.double(), crit.n2 / crit.n1, "sqrt",
                               1.0, 5.0)
    np.testing.assert_allclose(float(crit(R, Y, None, w)), float(l), rtol=1e-6)
    crit.task_weights = torch.ones(1, 3)
    with pytest.raises(ValueError, match="weights must have"):
        crit(R, Y, None, w)


def test_a_mask_is_nan_targets(monkeypatch):
    patch_enrichment(monkeypatch)
    crit, R, Y, w = _enrich_case()
    mask = torch.ones_like(Y, dtype=torch.bool)
    mask[4, 0] = mask[5] = False
    Rg = R.clone().requires_grad_(True)
    a = crit(Rg, Y, mask, w)
    (ga,) = torch.autograd.grad(a, Rg)
    b = crit(Rg, torch.where(mask, Y, torch.full_like(Y, float("nan"))), None, w)
    (gb,) = torch.autograd.grad(b, Rg)
    assert torch.equal(a, b) and torch.equal(ga, gb) and ga[5] == 0


def test_softplus_output_in_both_modes_and_other_transforms_refused(monkeypatch):
    import chemprop_b200.nn as N

    patch_enrichment(monkeypatch)
    torch.manual_seed(0)
    Z = torch.randn(5, 16)
    pred = N.EngineRegressionFFN(input_dim=16, hidden_dim=8, output_transform=nn.Softplus())
    raw = pred._mlp(Z).detach()
    for train in (True, False):
        pred.train(train)
        np.testing.assert_allclose(pred(Z).detach().numpy(), F.softplus(raw).numpy(), rtol=1e-6)
        assert torch.equal(pred.train_step(Z), pred(Z))
    assert CALLS.count("pred_transform_softplus") == 6
    Zg = Z.clone().requires_grad_(True)
    pred.train()
    pred(Zg).sum().backward()
    assert "pred_transform_bwd_softplus" in CALLS
    for t in (nn.Softplus(beta=2), nn.Softplus(threshold=10), nn.ReLU(), nn.Sigmoid(), N.ScaleTransform([0.0], [1.0])):
        pred.output_transform = t
        for train in (True, False):
            pred.train(train)
            with pytest.raises(ValueError, match="output transforms"):
                pred(Z)
    mve = N.EngineMveFFN(input_dim=16, hidden_dim=8, output_transform=nn.Softplus())
    with pytest.raises(ValueError, match="output transforms nn.Identity, UnscaleTransform \\("):
        mve(Z)


def test_the_kernel_contract_refuses_bad_launch_arguments():
    """The new entry points check their arguments on the host, before any CUDA call; kind 7 takes only u = 1."""
    from chemprop_b200 import _lib

    lib = _lib.load()
    buf = np.zeros(64, dtype=np.float32)
    L = buf.ctypes.data
    assert lib.dmpnn_enrichment_loss(L, 1, L, 2, None, None, 4, 1.0, 3, 1.0, 5.0, L, L, 1, None) != 0
    assert b"enrichment_loss: unknown method" in lib.dmpnn_last_error()
    for d, zs, zi in ((0.0, 1.0, 5.0), (float("inf"), 1.0, 5.0), (1.0, 0.0, 5.0), (1.0, 1.0, -1.0), (1.0, 1.0, float("nan"))):
        assert lib.dmpnn_enrichment_loss(L, 1, L, 2, None, None, 4, d, 0, zs, zi, L, L, 1, None) != 0
    assert lib.dmpnn_enrichment_loss(L, 1, L, 1, None, None, 4, 1.0, 0, 1.0, 5.0, L, L, 1, None) != 0
    assert b"enrichment_loss: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_pinball_loss_rows(L, 2, L, 2, None, None, 4, 2, float("nan"), L, L, 2, L, None) != 0
    assert lib.dmpnn_pinball_loss_rows(L, 1, L, 2, None, None, 4, 2, 0.1, L, L, 2, L, None) != 0
    assert b"pinball_loss_rows: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, PRED_SOFTPLUS, 2, None, None, L, 4, None) != 0
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, PRED_SOFTPLUS, 1, L, L, L, 4, None) != 0
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, 8, 1, None, None, L, 4, None) != 0
    assert lib.dmpnn_pred_transform_bwd(L, 4, L, 4, 2, 2, PRED_SOFTPLUS, 1, L, L, 4, None) != 0


# ---- metrics and evaluate ---------------------------------------------------------------------------------------------------
def test_criterion_metric_accumulates_across_batches(monkeypatch):
    from chemprop_b200.nn import EngineCriterionMetric

    patch_enrichment(monkeypatch)
    crit, R, Y, w = _enrich_case(b=10, seed=3)
    m = EngineCriterionMetric(crit)
    m.update(R[:4], Y[:4], Y[:4].isfinite(), w[:4])
    m.update(R[4:], Y[4:], Y[4:].isfinite(), w[4:])
    np.testing.assert_allclose(float(m.compute()), float(crit(R, Y, None, w)), rtol=1e-6)
    assert int(m._status) == 0


def _batches(g):
    bmg = golden_bmg(g, "cpu")
    return [(bmg, None, None, torch.from_numpy(g["Y"]), torch.from_numpy(g["w"]), None, None)]


def test_evaluate_gives_val_loss_and_the_criterion_metric(monkeypatch):
    import chemprop_b200.nn as N

    patch_enrichment(monkeypatch)
    g = load_golden("fixture_mpnn_enrichment_sqrt")
    model = build_model("enrichment_sqrt", g)
    crit = N.EngineNLogProbEnrichment(n1=int(g["n1"]), n2=int(g["n2"]))
    out = model.evaluate(_batches(g), metrics=[N.EngineCriterionMetric(crit)])
    assert set(out) == {"val_loss", "val/EngineNLogProbEnrichment"}
    model.eval()
    with torch.no_grad():
        R = model(golden_bmg(g, "cpu"))
    Y, w = torch.from_numpy(g["Y"]), torch.from_numpy(g["w"])
    tw = model.predictor.criterion.task_weights
    d = int(g["n2"]) / int(g["n1"])
    np.testing.assert_allclose(out["val_loss"], float(ref_enrichment_loss(R.double(), Y.double(), w.double(), tw.double(),
                                                                          d, "sqrt", 1.0, 1.5)[0]), rtol=1e-5)
    np.testing.assert_allclose(out["val/EngineNLogProbEnrichment"],
                               float(ref_enrichment_loss(R.double(), Y.double(), None, None, d, "sqrt", 1.0, 5.0)[0]),
                               rtol=1e-5)


def test_zero_counts_under_score_give_a_nan_step_and_evaluate_raises_the_references_error(monkeypatch):
    """Where the reference's training step raises, the engine's step returns NaN (it never synchronises); evaluate raises
    the reference's ValueError at its one host sync, from the validation loss and from the metric alike."""
    import chemprop_b200.nn as N

    patch_enrichment(monkeypatch)
    g = load_golden("fixture_mpnn_enrichment_score_raises")
    g = {**g, "zscale": 1.0, "zinterval": 5.0, "method": "score"}
    model = build_model("enrichment_score", g).train()
    (bmg, _, _, Y, w, _, _), = _batches(g)
    assert torch.isnan(model.training_loss(bmg, Y, w))
    with pytest.raises(ValueError, match=str(g["error"]).replace("(", r"\(").replace(")", r"\)")):
        model.evaluate(_batches(g), metrics=[])
    with pytest.raises(ValueError, match="Got nan loss with method 'score'"):
        model.evaluate(_batches(g), metrics=[N.EngineCriterionMetric(model.predictor.criterion)], stage="test")
    model.predictor.criterion.method = "sqrt"                          # sqrt has no NaN on zero counts
    assert math.isfinite(model.evaluate(_batches(g), metrics=[])["val_loss"])


# ---- which kernels a step launches --------------------------------------------------------------------------------------------
def test_a_del_step_launches_the_new_kernels(monkeypatch):
    patch_enrichment(monkeypatch)
    g = load_golden("fixture_mpnn_enrichment_wald")
    model = build_model("enrichment_wald", g).train()
    (bmg, _, _, Y, w, _, _), = _batches(g)
    model.training_loss(bmg, Y, w).backward()
    assert CALLS == ["pred_transform_softplus", "enrichment_loss", "pred_transform_bwd_softplus"]


def test_mol_atom_bond_pinball_runs_the_row_kernel_at_every_level(monkeypatch):
    import chemprop_b200.nn as N
    from tests.test_mab_model_host import build_training_model, patch_mab_model

    census = []
    patch_mab_model(monkeypatch, census)
    patch_enrichment(monkeypatch)
    from chemprop_b200 import engine

    fn = engine.pinball_loss_rows
    monkeypatch.setattr(engine, "pinball_loss_rows",
                        lambda P, *a: (census.append(("pinball_loss_rows", int(P.shape[0]), int(P.shape[1]), False)),
                                       fn(P, *a))[1])
    g = load_golden("fixture_mab_model_reg")
    model = build_training_model("reg", g).train()
    for lv, T in (("mol", 2), ("atom", 2), ("bond", 1)):
        getattr(model, f"{lv}_predictor").criterion = N.EnginePointQuantileLoss(torch.linspace(0.5, 1.5, T), alpha=0.3)
    bmg = golden_bmg(g, "cpu")
    targetss = [torch.from_numpy(g[f"Y.{lv}"]) for lv in ("mol", "atom", "bond")]
    weightss = [torch.from_numpy(g[k]) if k in g else None for k in ("w.mol", "w.atom", "w.bond")]
    X_d = torch.from_numpy(g["X_d"]) if "X_d" in g else None
    loss = model.training_loss(bmg, targetss, weightss, None, None, X_d)
    loss.backward()
    rows = [r for r in census if r[0] == "pinball_loss_rows"]
    assert [r[1:3] for r in rows] == [(t.shape[0], t.shape[1]) for t in targetss]
    assert not [r for r in census if r[0] in ("regression_loss_rows", "mse_loss", "regression_loss")]
    assert torch.isfinite(loss)
