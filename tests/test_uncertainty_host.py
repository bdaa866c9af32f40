"""CPU tier: target unscaling and the uncertainty predictors (EngineMveFFN, EngineEvidentialFFN, EngineQuantileFFN,
EngineBinaryDirichletFFN, EngineMulticlassDirichletFFN; csrc/head.cu's dmpnn_pred_transform(_bwd), dmpnn_mve_loss,
dmpnn_evidential_loss, dmpnn_quantile_loss, dmpnn_dirichlet_loss) through torch emulations of their kernel wrappers,
against the reference's own `MPNN.training_step` (tests/golden/fixture_mpnn_<kind>.npz) and the reference's trained
checkpoints (tests/golden/fixture_ckpt_<kind>.npz), both written by tools/make_golden_uncertainty.py; and the host-side
argument checks of the new entry points.  The reference formulas below, in any dtype, are also the f64 oracle of
tests/test_gpu_uncertainty.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_classification_host import patch_classification
from tests.util import golden_bmg, load_golden

PRED_REGRESSION, PRED_MVE, PRED_EVIDENTIAL, PRED_QUANTILE, PRED_DIRICHLET, PRED_DIRICHLET_PROBS, PRED_DIRICHLET_BINARY = \
    range(7)


# ---- the reference formulas (chemprop/nn/predictors.py, nn/transforms.py, nn/metrics.py), dtype-generic -----------------
def ref_transform(X, kind, u, mean=None, scale=None):
    """Raw MLP output X (b x T*u) -> b x T x u, as the reference predictors compute it."""
    b = X.shape[0]
    unscale = (lambda v: v) if scale is None else (lambda v: v * scale.view(1, -1).to(v.dtype) + mean.view(1, -1).to(v.dtype))
    unvar = (lambda v: v) if scale is None else (lambda v: v * (scale.view(1, -1).to(v.dtype) ** 2))
    if kind == PRED_REGRESSION:
        return unscale(X).unsqueeze(2)
    if kind == PRED_MVE:
        m, v = torch.chunk(X, 2, 1)
        return torch.stack((unscale(m), unvar(F.softplus(v))), 2)
    if kind == PRED_EVIDENTIAL:
        m, v, a, be = torch.chunk(X, 4, 1)
        return torch.stack((unscale(m), F.softplus(v), F.softplus(a) + 1, unvar(F.softplus(be))), 2)
    if kind == PRED_QUANTILE:
        lo, hi = torch.chunk(X, 2, 1)
        lo, hi = unscale(lo), unscale(hi)
        return torch.stack(((lo + hi) / 2, hi - lo), 2)
    a = F.softplus(X.reshape(b, -1, u)) + 1
    if kind == PRED_DIRICHLET:
        return a
    S = a.sum(-1, keepdim=True)
    if kind == PRED_DIRICHLET_PROBS:
        return a / S
    return torch.stack(((a / S)[..., 1], 2 / S[..., 0]), 2)


def ref_unreduced(kind, P, y, v_kl=0.2, eps=1e-8, alpha=0.1):
    """b x T unreduced loss of the reference criterion; y holds finite values (masked targets replaced)."""
    if kind == "mve":
        mean, var = torch.unbind(P, -1)
        return (mean - y) ** 2 / (2 * var) + (2 * torch.pi * var).log() / 2
    if kind == "evidential":
        mean, v, a, be = torch.unbind(P, -1)
        r = y - mean
        tb = 2 * be * (1 + v)
        nll = (0.5 * (torch.pi / v).log() - a * tb.log() + (a + 0.5) * torch.log(v * r ** 2 + tb) + torch.lgamma(a)
               - torch.lgamma(a + 0.5))
        return nll + v_kl * ((2 * v + a) * r.abs() - eps)
    if kind == "quantile":
        mean, interval = torch.unbind(P, -1)
        bounds = torch.tensor([-1 / 2, 1 / 2], dtype=P.dtype, device=P.device).view(-1, 1, 1)
        tau = torch.tensor([[alpha / 2, 1 - alpha / 2], [alpha / 2 - 1, -alpha / 2]], dtype=P.dtype,
                           device=P.device).view(2, 2, 1, 1)
        return (tau * (y - (mean + bounds * interval))).amax(0).sum(0)
    # Dirichlet: torch.eye(C)[targets.long()], with the rows the reference would raise on made NaN
    C = P.shape[2]
    k = y.trunc()
    bad = (k < -C) | (k >= C)
    k = torch.where(k < 0, k + C, k).clamp(0, C - 1).long()
    t = torch.eye(C, dtype=P.dtype, device=P.device)[k]
    S = P.sum(-1, keepdim=True)
    p = P / S
    A = (t - p).square().sum(-1, keepdim=True)
    B = ((p * (1 - p)) / (S + 1)).sum(-1, keepdim=True)
    al = t + (1 - t) * P
    Sa = al.sum(-1, keepdim=True)
    ln_a = Sa.lgamma() - al.lgamma().sum(-1, keepdim=True)
    ln_b = -torch.lgamma(torch.tensor(float(C), dtype=P.dtype, device=P.device))
    kl = ln_a + ln_b + torch.sum((al - 1) * (torch.digamma(al) - torch.digamma(Sa)), -1, keepdim=True)
    L = (A + B + v_kl * kl).mean(-1)
    return torch.where(bad, torch.full_like(L, float("nan")), L)


def ref_loss(kind, P, Y, w, tw, **kw):
    """The kernels' reduction of the reference criterion: sum w tw m L / sum m (0 when every target is masked), with its
    gradient in P by autograd (masked rows exactly 0, as the kernels write them)."""
    m = torch.isfinite(Y)
    with torch.enable_grad():
        Pl = P.detach().clone().requires_grad_(True)
        y = torch.where(m, Y, torch.zeros_like(Y)).to(P.dtype)
        L = ref_unreduced(kind, Pl, y, **kw)
        ww = ((w.view(-1, 1).to(P.dtype) if w is not None else 1.0)
              * (tw.reshape(1, -1).to(P.dtype) if tw is not None else 1.0))
        loss = torch.where(m, L * ww, torch.zeros_like(L)).sum() / m.sum().clamp(min=1)
        (g,) = torch.autograd.grad(loss, Pl) if Pl.numel() else (torch.zeros_like(Pl),)
    g = torch.where(m[..., None], g, torch.zeros_like(g))
    return loss.detach(), g


# ---- torch emulations of the engine wrappers (the kernels' contract, include/dmpnn.h) -------------------------------------
def pred_transform(X, kind, u, mean, scale, out):
    out.copy_(ref_transform(X, kind, u, mean, scale).reshape(out.shape))


def pred_transform_bwd(X, dOut, kind, u, scale, dX):
    mean = None if scale is None else torch.zeros_like(scale)
    with torch.enable_grad():
        x = X.detach().clone().requires_grad_(True)
        y = ref_transform(x, kind, u, mean, scale)
        (g,) = torch.autograd.grad(y, x, dOut.reshape(y.shape))
    dX.copy_(g)


def _emu_loss(kind, P, Y, w, tw, u, loss, dP, **kw):
    b, T = Y.shape
    l, g = ref_loss(kind, P.reshape(b, T, u), Y, w, tw, **kw)
    loss.copy_(l.reshape(1))
    if dP is not None:
        dP.copy_(g.reshape(dP.shape))


def mve_loss(P, Y, w, tw, loss, dP):
    _emu_loss("mve", P, Y, w, tw, 2, loss, dP)


def evidential_loss(P, Y, w, tw, v_kl, eps, loss, dP):
    _emu_loss("evidential", P, Y, w, tw, 4, loss, dP, v_kl=v_kl, eps=eps)


def quantile_loss(P, Y, w, tw, alpha, loss, dP):
    _emu_loss("quantile", P, Y, w, tw, 2, loss, dP, alpha=alpha)


def dirichlet_loss(P, Y, w, tw, C, v_kl, loss, dP):
    _emu_loss("dirichlet", P, Y, w, tw, C, loss, dP, v_kl=v_kl)


def patch_uncertainty(monkeypatch):
    """emu.patch_engine, the classification wrappers and the six uncertainty wrappers."""
    from chemprop_b200 import engine

    patch_classification(monkeypatch)
    for name in ("pred_transform", "pred_transform_bwd", "mve_loss", "evidential_loss", "quantile_loss", "dirichlet_loss"):
        monkeypatch.setattr(engine, name, globals()[name])


# ---- the training-step fixtures -----------------------------------------------------------------------------------------
KINDS = ("mve", "evidential", "quantile", "binary_dirichlet", "multiclass_dirichlet")
V_KL, EPS, ALPHA, N_CLASSES = 0.35, 0.05, 0.3, 4          # tools/make_golden_uncertainty.py


def build_model(kind: str, g: dict, precision: str = "fp32"):
    """EngineMPNN of the fixture's configuration holding its initial state (strict load of the reference's state dict minus
    the criterion's torchmetrics states)."""
    import chemprop_b200.nn as N

    tw = torch.ones(3)
    kw = dict(n_tasks=3, input_dim=40, hidden_dim=24, n_layers=2)
    ut = N.UnscaleTransform([0.0] * 3, [1.0] * 3)            # values come from the state dict
    if kind == "mve":
        pred = N.EngineMveFFN(**kw, output_transform=ut)
    elif kind == "evidential":
        pred = N.EngineEvidentialFFN(**kw, criterion=N.EngineEvidentialLoss(tw, v_kl=V_KL, eps=EPS), output_transform=ut)
    elif kind == "quantile":
        pred = N.EngineQuantileFFN(**kw, criterion=N.EngineQuantileLoss(tw, alpha=ALPHA), output_transform=ut)
    elif kind == "binary_dirichlet":
        pred = N.EngineBinaryDirichletFFN(**kw, criterion=N.EngineDirichletLoss(tw, v_kl=V_KL))
    else:
        pred = N.EngineMulticlassDirichletFFN(n_classes=N_CLASSES, **kw, criterion=N.EngineDirichletLoss(tw, v_kl=V_KL))
    model = N.EngineMPNN(N.BondMessagePassing(d_h=40, depth=3, precision=precision), N.MeanAggregation(), pred,
                         batch_norm=True)
    state = {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")}
    res = model.load_state_dict({k: v for k, v in state.items() if not k.endswith(("total_loss", "num_samples"))},
                                strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model


def check_uncertainty_head(kind: str, device: str, rtol: float = 2e-4, atol: float = 2e-6, graph: bool = False):
    """EngineMPNN.training_loss with an uncertainty head against the reference's `MPNN.training_step`: loss, every gradient,
    the batch-norm running statistics after the step, eval-mode predictions (unscaled for the regression kinds).  `graph`:
    the step runs as one captured CUDA graph (the recipe of tests/util.py::check_mpnn_head)."""
    g = load_golden(f"fixture_mpnn_{kind}")
    model = build_model(kind, g).to(device)
    model.train()
    bmg = golden_bmg(g, device)
    Y, w = torch.from_numpy(g["Y"]).to(device), torch.from_numpy(g["w"]).to(device)
    if graph:
        from chemprop_b200.graph import CudaGraphStep

        for p in model.parameters():
            p.grad = torch.zeros_like(p)
        rm0, rv0, nb0 = model.bn.running_mean.clone(), model.bn.running_var.clone(), model.bn.num_batches_tracked.clone()

        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            loss = model.training_loss(b, Y, w)
            loss.backward()
            return loss

        step = CudaGraphStep(fn)
        step(bmg)
        model.bn.running_mean.copy_(rm0); model.bn.running_var.copy_(rv0); model.bn.num_batches_tracked.copy_(nb0)
        loss = step(bmg).clone()
        assert step.captures == 1 and step.replays == 2
    else:
        loss = model.training_loss(bmg, Y, w)
        loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy(), g["loss"], rtol=rtol, atol=atol)
    for k, p in model.named_parameters():
        np.testing.assert_allclose(p.grad.cpu().numpy(), g["grad." + k], rtol=rtol, atol=atol, err_msg=k)
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        np.testing.assert_allclose(getattr(model.bn, k).cpu().numpy(), g["after.bn." + k], rtol=1e-5, atol=1e-6, err_msg=k)
    model.eval()
    with torch.no_grad():
        preds = model(bmg)
    assert preds.shape == g["preds_eval"].shape
    np.testing.assert_allclose(preds.cpu().numpy(), g["preds_eval"], rtol=rtol, atol=1e-5)


@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_uncertainty_matches_reference_training_step(kind, monkeypatch):
    patch_uncertainty(monkeypatch)
    check_uncertainty_head(kind, "cpu")


def test_fixtures_cover_the_cases_the_heads_must_handle():
    for kind in KINDS:
        g = load_golden(f"fixture_mpnn_{kind}")
        assert g["Y"].shape == (14, 3) and np.isnan(g["Y"]).any() and g["w"].std() > 0
        tw = g["param.predictor.criterion.task_weights"]
        assert tw.shape == (1, 3) and np.ptp(tw) > 0
        if kind.endswith("dirichlet"):
            assert (g["Y"] == -1).any()                               # a label that wraps to the last class
        else:                                                         # a non-trivial UnscaleTransform
            assert not np.allclose(g["param.predictor.output_transform.scale"], 1.0)
            assert not np.allclose(g["param.predictor.output_transform.mean"], 0.0)
    q = load_golden("fixture_mpnn_quantile")
    np.testing.assert_allclose(q["param.predictor.criterion.tau"].reshape(2, 2),
                               [[ALPHA / 2, 1 - ALPHA / 2], [ALPHA / 2 - 1, -ALPHA / 2]], rtol=1e-6)


# ---- the reference's trained checkpoints ----------------------------------------------------------------------------------
CKPTS = ("regression", "regression_mve", "regression_evidential", "regression_quantile", "classification_dirichlet",
         "multiclass_dirichlet")


def build_checkpoint_model(g: dict, kind: str):
    """The engine model of a reference checkpoint from its recorded hparams, loaded with strict=True.  The fixture holds every
    tensor after the encoder; the encoder's tensors are recorded as shapes only, and take the regression checkpoint's trained
    weights (the `bond_d3_trained` golden) for that checkpoint and zeros for the others."""
    import chemprop_b200.nn as N

    cls = {"RegressionFFN": N.EngineRegressionFFN, "MveFFN": N.EngineMveFFN, "EvidentialFFN": N.EngineEvidentialFFN,
           "QuantileFFN": N.EngineQuantileFFN, "BinaryDirichletFFN": N.EngineBinaryDirichletFFN,
           "MulticlassDirichletFFN": N.EngineMulticlassDirichletFFN}[str(g["hp.predictor"])]
    T, d_h = int(g["hp.n_tasks"]), int(g["hp.d_h"])
    kw = dict(n_tasks=T, input_dim=d_h, hidden_dim=int(g["hp.hidden_dim"]), n_layers=int(g["hp.n_layers"]))
    if int(g["hp.n_classes"]):
        kw["n_classes"] = int(g["hp.n_classes"])
    if "param.predictor.output_transform.mean" in g:
        kw["output_transform"] = N.UnscaleTransform([0.0] * T, [1.0] * T)
    agg = N.NormAggregation(norm=float(g["hp.norm"])) if float(g["hp.norm"]) else N.MeanAggregation()
    model = N.EngineMPNN(N.BondMessagePassing(d_h=d_h, depth=int(g["hp.depth"])), agg, cls(**kw),
                         batch_norm=bool(g["hp.batch_norm"]))
    state = {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")}
    enc = load_golden("bond_d3_trained") if kind == "regression" else {}
    for k, v in g.items():
        if k.startswith("shape."):
            name = k[len("shape."):]
            w = enc.get("param." + name[len("message_passing."):])
            state[name] = torch.from_numpy(w) if w is not None else torch.zeros(tuple(int(n) for n in v))
            assert tuple(state[name].shape) == tuple(int(n) for n in v), name
    res = model.load_state_dict(state, strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model


def check_checkpoint(kind: str, device: str, rtol: float = 1e-4, atol: float = 1e-5):
    """Eval-mode predictions of the checkpoint's head (batch norm, predictor, unscaling) on the reference's aggregated
    encoder output, and, for the regression checkpoint, of the whole model on the fixture's molecules."""
    g = load_golden(f"fixture_ckpt_{kind}")
    model = build_checkpoint_model(g, kind).to(device).eval()
    with torch.no_grad():
        preds = model.predictor(model.bn(torch.from_numpy(g["H"]).to(device)))
        assert preds.shape == g["preds_eval"].shape
        np.testing.assert_allclose(preds.cpu().numpy(), g["preds_eval"], rtol=rtol, atol=atol)
        if kind == "regression":
            np.testing.assert_allclose(model(golden_bmg(g, device)).cpu().numpy(), g["preds_eval"], rtol=rtol, atol=atol)


@pytest.mark.parametrize("kind", CKPTS)
def test_reference_checkpoint_loads_strictly_and_predicts_as_the_reference(kind, monkeypatch):
    patch_uncertainty(monkeypatch)
    check_checkpoint(kind, "cpu")


# ---- module surface ---------------------------------------------------------------------------------------------------------
def test_predictors_rebuild_from_their_hparams_with_the_reference_shapes():
    import chemprop_b200.nn as N

    ut = N.UnscaleTransform([1.0, 2.0], [3.0, 4.0])
    mods = [N.EngineMveFFN(n_tasks=2, input_dim=16, hidden_dim=8, output_transform=ut),
            N.EngineEvidentialFFN(n_tasks=2, input_dim=16, hidden_dim=8, criterion=N.EngineEvidentialLoss(v_kl=0.3)),
            N.EngineQuantileFFN(n_tasks=2, input_dim=16, hidden_dim=8),
            N.EngineBinaryDirichletFFN(n_tasks=2, input_dim=16, hidden_dim=8),
            N.EngineMulticlassDirichletFFN(n_classes=5, n_tasks=2, input_dim=16, hidden_dim=8),
            N.EngineRegressionFFN(n_tasks=2, input_dim=16, hidden_dim=8, output_transform=ut)]
    outs = [4, 8, 4, 4, 10, 2]
    crits = [N.EngineMVELoss, N.EngineEvidentialLoss, N.EngineQuantileLoss, N.EngineDirichletLoss, N.EngineDirichletLoss]
    for i, mod in enumerate(mods):
        assert mod.n_tasks == 2 and mod.output_dim == outs[i]
        if i < len(crits):
            assert type(mod.criterion) is crits[i]
        back = mod.hparams["cls"](**{k: v for k, v in mod.hparams.items() if k != "cls"})
        assert type(back) is type(mod) and back.n_tasks == mod.n_tasks and back.output_dim == mod.output_dim
        assert set(back.state_dict()) == set(mod.state_dict())
    assert mods[0].hparams["output_transform"] is ut and mods[1].hparams["criterion"].v_kl == 0.3
    assert mods[1].criterion.eps == 1e-8 and mods[2].criterion.alpha == 0.1 and mods[3].criterion.v_kl == 0.2
    q = N.EngineQuantileLoss(torch.ones(3), alpha=0.2)
    assert q.bounds.shape == (2, 1, 1) and q.tau.shape == (2, 2, 1, 1)
    assert set(q.state_dict()) == {"task_weights", "bounds", "tau"}


def test_unscale_transform_is_the_references():
    from chemprop_b200.nn import UnscaleTransform

    class _Scaler:
        mean_, scale_ = np.array([1.5, -2.0]), np.array([2.0, 0.5])

    t = UnscaleTransform.from_standard_scaler(_Scaler(), pad=1)
    assert t.mean.shape == (1, 3) and t.scale.shape == (1, 3)
    X = torch.randn(4, 3)
    assert torch.equal(t.train()(X), X) and torch.equal(t.transform_variance(X), X)
    t.eval()
    torch.testing.assert_close(t(X), X * t.scale + t.mean)
    torch.testing.assert_close(t.transform_variance(X), X * t.scale ** 2)


def test_x_d_transform_scales_descriptors_in_eval_mode(monkeypatch):
    import chemprop_b200.nn as N

    patch_uncertainty(monkeypatch)
    g = load_golden("fixture_mpnn_mve")
    bmg = golden_bmg(g, "cpu")
    X_d = torch.randn(14, 3)
    xt = N.ScaleTransform([1.0, 2.0, 3.0], [2.0, 4.0, 8.0])
    model = N.EngineMPNN(N.BondMessagePassing(d_h=40, depth=3), N.MeanAggregation(),
                         N.EngineRegressionFFN(input_dim=43), X_d_transform=xt).eval()
    with torch.no_grad():
        fp = model.fingerprint(bmg, X_d=X_d)
    torch.testing.assert_close(fp[:, 40:], (X_d - xt.mean) / xt.scale)
    assert set(model.state_dict()) >= {"X_d_transform.mean", "X_d_transform.scale"}


def test_entry_points_validate_their_arguments_before_touching_the_device():
    """The six new entry points check their arguments on the host, before any CUDA call: callable (and failing cleanly,
    naming the entry point) without a GPU."""
    from chemprop_b200 import _lib

    lib = _lib.load()
    buf = np.zeros(64, dtype=np.float32)
    L = buf.ctypes.data
    nan = float("nan")
    # transform: unknown kind, u not matching the kind, mean without scale, scale with a Dirichlet kind, short strides
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, 7, 2, None, None, L, 4, None) != 0
    assert b"pred_transform" in lib.dmpnn_last_error()
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, 1, 3, None, None, L, 6, None) != 0
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, 1, 2, L, None, L, 4, None) != 0
    assert lib.dmpnn_pred_transform(L, 4, 2, 2, 4, 2, L, L, L, 4, None) != 0
    assert lib.dmpnn_pred_transform(L, 3, 2, 2, 1, 2, None, None, L, 4, None) != 0
    assert b"pred_transform: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_pred_transform(L, 4, 2, 0, 0, 1, None, None, L, 4, None) != 0
    assert lib.dmpnn_pred_transform(None, 4, 0, 2, 1, 2, None, None, None, 4, None) == 0      # B = 0: no launch
    # mirror: the eval-only kinds have no kernel mirror; scale only with the regression kinds; short dX stride
    assert lib.dmpnn_pred_transform_bwd(L, 4, L, 4, 2, 2, 5, 2, None, L, 4, None) != 0
    assert b"pred_transform_bwd" in lib.dmpnn_last_error()
    assert lib.dmpnn_pred_transform_bwd(L, 4, L, 4, 2, 2, 4, 2, L, L, 4, None) != 0
    assert lib.dmpnn_pred_transform_bwd(L, 4, L, 4, 2, 2, 1, 2, None, L, 3, None) != 0
    assert lib.dmpnn_pred_transform_bwd(L, 8, L, 8, 2, 2, 2, 3, None, L, 8, None) != 0
    # losses: T = 0, short P / dP strides, non-finite parameters, C = 0, missing loss
    assert lib.dmpnn_mve_loss(L, 4, L, 2, None, None, 3, 0, L, None, 4, None) != 0
    assert b"mve_loss" in lib.dmpnn_last_error()
    assert lib.dmpnn_mve_loss(L, 3, L, 2, None, None, 3, 2, L, None, 4, None) != 0
    assert lib.dmpnn_mve_loss(L, 4, L, 2, None, None, 3, 2, L, L, 3, None) != 0
    assert lib.dmpnn_mve_loss(L, 4, L, 2, None, None, 3, 2, None, None, 4, None) != 0
    assert lib.dmpnn_evidential_loss(L, 8, L, 2, None, None, 3, 2, nan, 1e-8, L, None, 8, None) != 0
    assert b"evidential_loss" in lib.dmpnn_last_error()
    assert lib.dmpnn_evidential_loss(L, 7, L, 2, None, None, 3, 2, 0.2, 1e-8, L, None, 8, None) != 0
    assert lib.dmpnn_quantile_loss(L, 4, L, 2, None, None, 3, 2, float("inf"), L, None, 4, None) != 0
    assert b"quantile_loss" in lib.dmpnn_last_error()
    assert lib.dmpnn_quantile_loss(L, 4, L, 1, None, None, 3, 2, 0.1, L, None, 4, None) != 0
    assert lib.dmpnn_dirichlet_loss(L, 6, L, 2, None, None, 3, 2, 0, 0.2, L, None, 6, None) != 0
    assert b"dirichlet_loss" in lib.dmpnn_last_error()
    assert lib.dmpnn_dirichlet_loss(L, 5, L, 2, None, None, 3, 2, 3, 0.2, L, None, 6, None) != 0
    assert lib.dmpnn_dirichlet_loss(L, 6, L, 2, None, None, 3, 2, 3, nan, L, None, 6, None) != 0
    assert lib.dmpnn_dirichlet_loss(L, 2 ** 40, L, 2 ** 20, None, None, 3, 2 ** 20, 2 ** 20, 0.2, L, None, 2 ** 40,
                                    None) != 0
