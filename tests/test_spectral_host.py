"""CPU tier: the spectral predictor (EngineSpectralFFN with EngineSID / EngineWasserstein) and the regression-loss family
(EngineMAE, EngineRMSE, EngineBoundedMSE, EngineBoundedMAE, EngineBoundedRMSE; csrc/head.cu's dmpnn_spectral_transform(_bwd),
dmpnn_sid_loss, dmpnn_wasserstein_loss, dmpnn_regression_loss) through torch emulations of their kernel wrappers, against
the reference's own `MPNN.training_step` (tests/golden/fixture_mpnn_<kind>.npz, written by tools/make_golden_spectral.py);
strict state-dict loads, hparams rebuilds, masks through the packed loader and the host-side argument checks of the new
entry points.  The reference formulas below, in any dtype, are also the f64 oracle of tests/test_gpu_spectral.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_uncertainty_host import patch_uncertainty
from tests.util import golden_bmg, load_golden

LOSS_MSE, LOSS_MAE, LOSS_RMSE = range(3)
SPEC_SOFTPLUS, SPEC_EXP = range(2)


# ---- the reference formulas (chemprop/nn/predictors.py:342-376, nn/metrics.py:59-183, 547-585), dtype-generic ----------
def ref_spectral(X, act):
    """SpectralFFN: the activation twice, then normalised over every bin."""
    a = torch.exp if act == SPEC_EXP else F.softplus
    Y = a(a(X))
    return Y / Y.sum(1, keepdim=True)


def ref_spectral_unreduced(kind, P, Y, threshold):
    """b x T unreduced SID / Wasserstein with the reference's masking: Y NaN where masked."""
    m = torch.isfinite(Y)
    t = torch.where(m, Y, torch.zeros_like(Y)).to(P.dtype)          # training_step's nan_to_num
    p = P if threshold is None else P.clamp(min=threshold)
    pn = p / (p * m).sum(1, keepdim=True)
    if kind == "wasserstein":
        return (t.cumsum(1) - pn.cumsum(1)).abs()
    t = t.masked_fill(~m, 1)
    pn = pn.masked_fill(~m, 1)
    return (pn / t).log() * pn + (t / pn).log() * t


def ref_spectral_loss(kind, P, Y, w, tw, threshold):
    """The kernels' reduction and conventions (include/dmpnn.h) on the reference formula, gradient by autograd: rows with
    every bin masked add 0 and get dP = 0; loss 0 when every target is masked."""
    m = torch.isfinite(Y)
    live = m.any(1, keepdim=True)
    with torch.enable_grad():
        Pl = P.detach().clone().requires_grad_(True)
        Pu = torch.where(live, Pl, torch.ones_like(Pl))               # a dead row: any finite stand-in, no gradient
        L = ref_spectral_unreduced(kind, Pu, Y, threshold)
        ww = ((w.view(-1, 1).to(P.dtype) if w is not None else 1.0)
              * (tw.reshape(1, -1).to(P.dtype) if tw is not None else 1.0))
        loss = torch.where(m & live, L * ww, torch.zeros_like(L)).sum() / m.sum().clamp(min=1)
        (g,) = torch.autograd.grad(loss, Pl) if Pl.numel() else (torch.zeros_like(Pl),)
    g = torch.where(live, g, torch.zeros_like(g))
    if kind == "sid":
        g = torch.where(m, g, torch.zeros_like(g))
    return loss.detach(), g


def ref_regression_loss(kind, P, Y, w, tw, lt=None, gt=None):
    """MSE / MAE / RMSE (bounded with lt / gt) under the kernels' reduction: loss 0 and dP 0 when every target is masked,
    dP 0 where RMSE's loss is 0."""
    m = torch.isfinite(Y)
    with torch.enable_grad():
        Pl = P.detach().clone().requires_grad_(True)
        y = torch.where(m, Y, torch.zeros_like(Y)).to(P.dtype)
        p = Pl
        if lt is not None:
            p = torch.where((p < y) & lt, y, p)
        if gt is not None:
            p = torch.where((p > y) & gt, y, p)
        L = (p - y).abs() if kind == LOSS_MAE else (p - y) ** 2
        ww = ((w.view(-1, 1).to(P.dtype) if w is not None else 1.0)
              * (tw.reshape(1, -1).to(P.dtype) if tw is not None else 1.0))
        loss = torch.where(m, L * ww, torch.zeros_like(L)).sum() / m.sum().clamp(min=1)
        if kind == LOSS_RMSE:
            if float(loss.detach()) == 0.0:
                return loss.detach(), torch.zeros_like(P)
            loss = loss.sqrt()
        (g,) = torch.autograd.grad(loss, Pl) if Pl.numel() else (torch.zeros_like(Pl),)
    return loss.detach(), torch.where(m, g, torch.zeros_like(g))


# ---- torch emulations of the engine wrappers (the kernels' contract, include/dmpnn.h) -------------------------------------
def spectral_transform(X, act, out):
    out.copy_(ref_spectral(X, act))


def spectral_transform_bwd(X, dOut, act, dX):
    with torch.enable_grad():
        x = X.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(ref_spectral(x, act), x, dOut)
    dX.copy_(g)


def _check_weights(P, w, tw):
    """The kernels read exactly b weights and T task weights."""
    b, T = P.shape
    assert w is None or w.numel() == b, (None if w is None else w.numel(), b)
    assert tw is None or tw.numel() == T, (None if tw is None else tw.numel(), T)


def _emu(kind, P, Y, w, tw, threshold, loss, dP):
    _check_weights(P, w, tw)
    l, g = ref_spectral_loss(kind, P, Y, w, tw, threshold)
    loss.copy_(l.reshape(1))
    if dP is not None:
        dP.copy_(g)


def sid_loss(P, Y, w, tw, threshold, loss, dP):
    _emu("sid", P, Y, w, tw, threshold, loss, dP)


def wasserstein_loss(P, Y, w, tw, threshold, loss, dP):
    _emu("wasserstein", P, Y, w, tw, threshold, loss, dP)


def regression_loss(P, Y, w, tw, lt_mask, gt_mask, kind, loss, dP):
    _check_weights(P, w, tw)
    lt = None if lt_mask is None else lt_mask.bool()
    gt = None if gt_mask is None else gt_mask.bool()
    l, g = ref_regression_loss(kind, P, Y, w, tw, lt, gt)
    loss.copy_(l.reshape(1))
    if dP is not None:
        dP.copy_(g)


def patch_spectral(monkeypatch):
    """patch_uncertainty plus the five new wrappers."""
    from chemprop_b200 import engine

    patch_uncertainty(monkeypatch)
    for name in ("spectral_transform", "spectral_transform_bwd", "sid_loss", "wasserstein_loss", "regression_loss"):
        monkeypatch.setattr(engine, name, globals()[name])


# ---- the training-step fixtures -----------------------------------------------------------------------------------------
KINDS = ("spectral_sid", "spectral_wasserstein", "mae", "rmse", "bounded_mse", "bounded_mae", "bounded_rmse")
N_BINS, THRESHOLD = 40, 0.025                                   # tools/make_golden_spectral.py


def build_model(kind: str, g: dict, precision: str = "fp32"):
    """EngineMPNN of the fixture's configuration holding its initial state (strict load of the reference's state dict minus
    the criterion's torchmetrics states)."""
    import chemprop_b200.nn as N

    if kind.startswith("spectral"):
        kw = dict(n_tasks=N_BINS, input_dim=40, hidden_dim=24, n_layers=2)
        if kind == "spectral_sid":
            pred = N.EngineSpectralFFN(**kw, threshold=THRESHOLD)
        else:
            pred = N.EngineSpectralFFN(**kw, criterion=N.EngineWasserstein(torch.ones(N_BINS), threshold=THRESHOLD),
                                       spectral_activation="exp")
    else:
        crit = {"mae": N.EngineMAE, "rmse": N.EngineRMSE, "bounded_mse": N.EngineBoundedMSE,
                "bounded_mae": N.EngineBoundedMAE, "bounded_rmse": N.EngineBoundedRMSE}[kind](torch.ones(3))
        pred = N.EngineRegressionFFN(n_tasks=3, input_dim=40, hidden_dim=24, n_layers=2, criterion=crit)
    model = N.EngineMPNN(N.BondMessagePassing(d_h=40, depth=3, precision=precision), N.MeanAggregation(), pred,
                         batch_norm=True)
    state = {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")}
    res = model.load_state_dict({k: v for k, v in state.items() if not k.endswith(("total_loss", "num_samples"))},
                                strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model


def check_spectral_head(kind: str, device: str, rtol: float = 2e-4, atol: float = 2e-6, graph: bool = False):
    """EngineMPNN.training_loss with the fixture's head and criterion against the reference's `MPNN.training_step`: loss,
    every gradient, the batch-norm running statistics after the step, eval-mode predictions.  `graph`: the step runs as one
    captured CUDA graph, and its replay must be bit-identical to the eager step."""
    g = load_golden(f"fixture_mpnn_{kind}")
    model = build_model(kind, g).to(device)
    model.train()
    bmg = golden_bmg(g, device)
    Y, w = torch.from_numpy(g["Y"]).to(device), torch.from_numpy(g["w"]).to(device)
    masks = {}
    if "lt_mask" in g:
        masks = {"lt_mask": torch.from_numpy(g["lt_mask"]).to(device), "gt_mask": torch.from_numpy(g["gt_mask"]).to(device)}
    loss = model.training_loss(bmg, Y, w, **masks)
    loss.backward()
    if graph:
        from chemprop_b200.graph import CudaGraphStep

        eager = loss.detach().clone()
        eager_grads = {k: p.grad.clone() for k, p in model.named_parameters()}
        model = build_model(kind, g).to(device).train()
        for p in model.parameters():
            p.grad = torch.zeros_like(p)
        rm0, rv0, nb0 = model.bn.running_mean.clone(), model.bn.running_var.clone(), model.bn.num_batches_tracked.clone()

        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            out = model.training_loss(b, Y, w, **masks)
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
    np.testing.assert_allclose(loss.detach().cpu().numpy(), g["loss"], rtol=rtol, atol=atol)
    for k, p in model.named_parameters():
        np.testing.assert_allclose(p.grad.cpu().numpy(), g["grad." + k], rtol=rtol, atol=atol, err_msg=k)
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        np.testing.assert_allclose(getattr(model.bn, k).cpu().numpy(), g["after.bn." + k], rtol=1e-5, atol=1e-6, err_msg=k)
    model.eval()
    with torch.no_grad():
        preds = model(bmg)
    assert preds.shape == g["preds_eval"].shape
    np.testing.assert_allclose(preds.cpu().numpy(), g["preds_eval"], rtol=rtol, atol=1e-6)


@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_matches_reference_training_step(kind, monkeypatch):
    patch_spectral(monkeypatch)
    check_spectral_head(kind, "cpu")


def test_fixtures_cover_the_cases_the_heads_must_handle():
    for kind in KINDS:
        g = load_golden(f"fixture_mpnn_{kind}")
        Y, p = g["Y"], g["preds_train"]
        m = np.isfinite(Y)
        assert (~m).any() and g["w"].std() > 0 and np.ptp(g["param.predictor.criterion.task_weights"]) > 0
        if kind.startswith("spectral"):
            assert Y.shape == (14, N_BINS) and (~m[:, 0]).any() and (Y[m] > 0).all()
            np.testing.assert_allclose(np.nansum(Y, 1)[m.all(1)], 1.0, rtol=1e-5)
            assert 0.2 < (p < THRESHOLD).mean() < 0.8                      # the clamp is active on both sides
            assert "ffn.2.2.weight" in {k[len("param.predictor."):] for k in g if k.startswith("param.predictor.")}
        if kind.startswith("bounded"):
            lt, gt = g["lt_mask"], g["gt_mask"]
            for mk in (lt, gt):
                assert (mk & m & (p < Y)).any() and (mk & m & (p > Y)).any() and (mk & ~m).any()


@pytest.mark.parametrize("kind", KINDS)
def test_reference_state_dict_loads_strictly_and_hparams_cover_the_references(kind):
    g = load_golden(f"fixture_mpnn_{kind}")
    model = build_model(kind, g)
    ref_keys = {k[len("param."):] for k in g if k.startswith("param.") and not k.endswith(("total_loss", "num_samples"))}
    assert set(model.state_dict()) == ref_keys
    hp = dict(model.predictor.hparams)
    if kind.startswith("spectral"):
        assert set(hp) >= {str(k) for k in g["hp_keys"]}
    back = hp.pop("cls")(**hp)
    assert type(back) is type(model.predictor) and set(back.state_dict()) == set(model.predictor.state_dict())


def test_spectral_predictor_surface():
    import chemprop_b200.nn as N

    m = N.EngineSpectralFFN(n_tasks=40, input_dim=16, hidden_dim=8, n_layers=2, task_weights=torch.linspace(1, 2, 40),
                            threshold=1e-3, spectral_activation="exp")
    assert m.n_tasks == 40 and m.output_dim == 40 and m.input_dim == 16
    assert type(m.criterion) is N.EngineSID and m.criterion.threshold == 1e-3
    assert type(m.ffn.spectral_activation).__name__ == "_Exp" and "spectral_activation" in dict(m.ffn.named_children())
    assert m.train_step == m.forward or m.train_step.__func__ is m.forward.__func__
    hp = dict(m.hparams)
    back = hp.pop("cls")(**hp)
    assert type(back.criterion) is N.EngineSID and back.criterion.threshold == 1e-3
    torch.testing.assert_close(back.criterion.task_weights, m.criterion.task_weights)
    assert type(back.ffn.spectral_activation).__name__ == "_Exp"
    for act in ("softplus", None):
        assert isinstance(N.EngineSpectralFFN(n_tasks=4, input_dim=8, spectral_activation=act).ffn.spectral_activation,
                          torch.nn.Softplus)
    with pytest.raises(ValueError):
        N.EngineSpectralFFN(n_tasks=4, input_dim=8, spectral_activation="relu")
    w = N.EngineWasserstein(torch.ones(3), threshold=0.1)
    assert w.threshold == 0.1 and set(w.state_dict()) == {"task_weights"}
    r = N.EngineRegressionFFN(n_tasks=2, input_dim=16, hidden_dim=8)     # the other predictors' hparams do not change
    assert set(r.hparams) == {"n_tasks", "input_dim", "hidden_dim", "n_layers", "dropout", "activation", "cls"}


def test_only_the_bounded_criteria_take_lt_and_gt_masks(monkeypatch):
    import chemprop_b200.nn as N

    patch_spectral(monkeypatch)
    torch.manual_seed(0)
    preds, Y = torch.randn(6, 3), torch.randn(6, 3)
    mask = torch.rand(6, 3) > 0.3
    for cls in (N.EngineMAE, N.EngineRMSE, N.EngineSID, N.EngineWasserstein):
        with pytest.raises(NotImplementedError):
            cls(torch.ones(3))(preds.abs(), Y.abs(), lt_mask=mask)
    lt, gt = torch.rand(6, 3) > 0.5, torch.rand(6, 3) > 0.5
    for cls, kind in ((N.EngineBoundedMSE, LOSS_MSE), (N.EngineBoundedMAE, LOSS_MAE), (N.EngineBoundedRMSE, LOSS_RMSE)):
        c = cls(torch.ones(3))
        a = c(preds, Y, mask, None, lt, gt)
        b = c(preds, torch.where(mask, Y, torch.full_like(Y, float("nan"))), None, None, lt, gt)
        assert torch.equal(a, b)
        ref, _ = ref_regression_loss(kind, preds, torch.where(mask, Y, torch.full_like(Y, float("nan"))), None, None, lt, gt)
        torch.testing.assert_close(a, ref)
        assert not torch.equal(c(preds, Y), a)                            # the bounds change the value


def test_boolean_masks_travel_through_the_packed_loader_to_the_criterion(monkeypatch):
    """b x T boolean lt / gt masks ride PackedBatchLoader(arrays=...) next to the targets, row for row, and
    EngineMPNN.training_loss hands them to the bounded criterion."""
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedBatchLoader, PackedMolGraphDataset, make_molecules

    patch_spectral(monkeypatch)
    n = 60
    mgs = make_molecules(n, seed=3, min_atoms=1)
    rng = np.random.default_rng(2)
    Y = rng.normal(size=(n, 3)).astype(np.float32)
    lt, gt = rng.random((n, 3)) < 0.4, rng.random((n, 3)) > 0.6
    ds = PackedMolGraphDataset.from_molgraphs(mgs)
    loader = PackedBatchLoader(ds, batch_size=25, shuffle=True, seed=1, arrays={"Y": Y, "lt": lt, "gt": gt})
    batch = next(iter(loader))
    ids = batch.ids
    assert batch.extras["lt"].dtype == torch.bool and torch.equal(batch.extras["lt"], torch.from_numpy(lt[ids]))
    assert torch.equal(batch.extras["gt"], torch.from_numpy(gt[ids]))
    torch.manual_seed(0)
    model = N.EngineMPNN(N.BondMessagePassing(d_v=ds.d_v, d_e=ds.d_e, d_h=32), N.MeanAggregation(),
                         N.EngineRegressionFFN(n_tasks=3, input_dim=32, criterion=N.EngineBoundedMSE(torch.ones(3))))
    seen = {}
    import chemprop_b200.engine as K
    inner = K.regression_loss

    def spy(P, Yb, w, tw, ltm, gtm, kind, loss, dP):
        seen.update(lt=ltm, gt=gtm)
        inner(P, Yb, w, tw, ltm, gtm, kind, loss, dP)

    monkeypatch.setattr(K, "regression_loss", spy)
    model.training_loss(batch.bmg, batch.extras["Y"], lt_mask=batch.extras["lt"], gt_mask=batch.extras["gt"])
    assert torch.equal(seen["lt"].bool(), batch.extras["lt"]) and torch.equal(seen["gt"].bool(), batch.extras["gt"])
    model.training_loss(batch.bmg, batch.extras["Y"])
    assert seen["lt"] is None and seen["gt"] is None


def test_entry_points_validate_their_arguments_before_touching_the_device():
    """The new entry points check their arguments on the host, before any CUDA call: callable (and failing cleanly,
    naming the entry point) without a GPU."""
    import ctypes as C

    from chemprop_b200 import _lib

    lib = _lib.load()
    buf = np.zeros(64, dtype=np.float32)
    L = buf.ctypes.data
    nan, inf = float("nan"), float("inf")
    # regression family: unknown kind, T = 0, short mask stride, short P stride, missing loss
    assert lib.dmpnn_regression_loss(L, 4, L, 4, None, None, None, None, 0, 2, 4, 3, L, L, 4, None) != 0
    assert b"regression_loss: unknown kind" in lib.dmpnn_last_error()
    assert lib.dmpnn_regression_loss(L, 4, L, 4, None, None, None, None, 0, 2, 0, 1, L, L, 4, None) != 0
    assert lib.dmpnn_regression_loss(L, 4, L, 4, None, None, L, None, 3, 2, 4, 1, L, L, 4, None) != 0
    assert b"regression_loss: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_regression_loss(L, 3, L, 4, None, None, None, None, 0, 2, 4, 1, L, L, 4, None) != 0
    assert lib.dmpnn_regression_loss(L, 4, L, 4, None, None, None, None, 0, 2, 4, 1, None, L, 4, None) != 0
    # transform: unknown activation, short strides, T = 0; B = 0 launches nothing
    assert lib.dmpnn_spectral_transform(L, 4, 2, 4, 2, L, 4, None) != 0
    assert b"spectral_transform: unknown activation" in lib.dmpnn_last_error()
    assert lib.dmpnn_spectral_transform(L, 3, 2, 4, 0, L, 4, None) != 0
    assert lib.dmpnn_spectral_transform(L, 4, 2, 0, 0, L, 4, None) != 0
    assert lib.dmpnn_spectral_transform(None, 4, 0, 4, 1, None, 4, None) == 0
    assert lib.dmpnn_spectral_transform_bwd(L, 4, L, 4, 2, 4, -1, L, 4, None) != 0
    assert b"spectral_transform_bwd" in lib.dmpnn_last_error()
    assert lib.dmpnn_spectral_transform_bwd(L, 4, L, 4, 2, 4, 0, L, 3, None) != 0
    assert lib.dmpnn_spectral_transform_bwd(L, 4, None, 4, 2, 4, 0, L, 4, None) != 0
    # workspace query: B rows of partial losses plus the count partials
    n = C.c_size_t(0)
    assert lib.dmpnn_spectral_loss_workspace_bytes(10000, C.byref(n)) == 0 and n.value >= 10000 * 4
    assert lib.dmpnn_spectral_loss_workspace_bytes(-1, C.byref(n)) != 0
    # losses: missing workspace, short strides, infinite threshold, T = 0
    for fn, name in ((lib.dmpnn_sid_loss, b"sid_loss"), (lib.dmpnn_wasserstein_loss, b"wasserstein_loss")):
        assert fn(L, 4, L, 4, None, None, 2, 4, nan, L, L, 4, None, None) != 0
        assert name + b": bad args" in lib.dmpnn_last_error()
        assert fn(L, 4, L, 3, None, None, 2, 4, nan, L, L, 4, L, None) != 0
        assert name + b": row strides" in lib.dmpnn_last_error()
        assert fn(L, 4, L, 4, None, None, 2, 4, nan, L, L, 3, L, None) != 0
        assert fn(L, 4, L, 4, None, None, 2, 4, inf, L, L, 4, L, None) != 0
        assert name + b": threshold" in lib.dmpnn_last_error()
        assert fn(L, 4, L, 4, None, None, 2, 0, nan, L, L, 4, L, None) != 0


def test_default_task_weight_broadcasts_and_other_sizes_are_refused(monkeypatch):
    """Every new criterion defaults to `task_weights=1.0` (a 1 x 1 buffer), as the reference's do: it reaches the kernel
    as T ones.  Task weights of another size, or weights that are not one per molecule, are refused on the host."""
    import chemprop_b200.nn as N

    patch_spectral(monkeypatch)
    torch.manual_seed(3)
    b, T = 5, 3
    preds, Y = torch.randn(b, T), torch.randn(b, T)
    Y[1, 2] = float("nan")
    spec = torch.rand(b, T) + 0.1
    w = torch.rand(b) + 0.5
    for cls, kind in ((N.EngineMAE, LOSS_MAE), (N.EngineRMSE, LOSS_RMSE), (N.EngineBoundedMSE, LOSS_MSE),
                      (N.EngineBoundedMAE, LOSS_MAE), (N.EngineBoundedRMSE, LOSS_RMSE)):
        for tw, ref_tw in ((None, torch.ones(T)), (2.0, torch.full((T,), 2.0))):
            c = cls() if tw is None else cls(tw)
            assert c.task_weights.shape == (1, 1)
            torch.testing.assert_close(c(preds, Y, None, w), ref_regression_loss(kind, preds, Y, w, ref_tw)[0])
        with pytest.raises(ValueError):
            cls(torch.ones(2))(preds, Y)
        with pytest.raises(ValueError):
            cls()(preds, Y, None, torch.ones(b + 1))
    for cls, kind in ((N.EngineSID, "sid"), (N.EngineWasserstein, "wasserstein")):
        torch.testing.assert_close(cls()(spec, Y.abs(), None, w),
                                   ref_spectral_loss(kind, spec, Y.abs(), w, torch.ones(T), None)[0])
        with pytest.raises(ValueError):
            cls(torch.ones(T + 1))(spec, Y.abs())


def test_regression_criteria_are_leaves_of_one_private_base():
    import chemprop_b200.nn as N
    from chemprop_b200.nn.head import _RegressionCriterion

    classes = (N.EngineMAE, N.EngineRMSE, N.EngineBoundedMSE, N.EngineBoundedMAE, N.EngineBoundedRMSE)
    for a in classes:
        assert issubclass(a, _RegressionCriterion)
        assert not any(issubclass(a, o) for o in classes if o is not a)


def test_wasserstein_with_an_explicit_mask_ignores_the_masked_targets(monkeypatch):
    """`mask` drops a bin as a NaN target does: it adds 0 to the target cumsum (the reference's training_step, which hands
    its criterion `targets.nan_to_num(0)`), whatever finite value the caller left there."""
    import chemprop_b200.nn as N

    patch_spectral(monkeypatch)
    torch.manual_seed(4)
    P, Y = torch.rand(4, 9) + 0.1, torch.rand(4, 9) + 0.1
    mask = torch.rand(4, 9) > 0.3
    c = N.EngineWasserstein(torch.ones(9))
    a = c(P, Y, mask)
    assert torch.equal(a, c(P, torch.where(mask, Y, torch.full_like(Y, float("nan")))))
    assert torch.equal(a, c(P, torch.where(mask, Y, torch.full_like(Y, 5.0)), mask))
    L = ref_spectral_unreduced("wasserstein", P, torch.where(mask, Y, torch.full_like(Y, float("nan"))), None)
    torch.testing.assert_close(a, (L * mask).sum() / mask.sum())
