"""GPU tier: the device metrics (csrc/metrics.cu, chemprop_b200/nn/metrics.py) against the float64 restatement
oracle/metrics_np.py -- every kind at B in {1, 7, 4097, 1 000 003} and T in {1, 12}, the multiclass MCC at C = 3 and 10,
masked / single-class / logit inputs, AUROC and AUPRC on over 10 M kept, heavily tied pairs, accumulation over uneven batches,
bitwise repeatability, NaN-filled workspaces, no host sync in `update`, and `EngineMPNN.evaluate` on regression (with
target unscaling), binary, multiclass, spectral and multicomponent models against the oracle applied to the model's own
predictions."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from oracle import metrics_np as O

pytestmark = pytest.mark.gpu

REG = ("mse", "mae", "rmse", "bounded-mse", "bounded-mae", "bounded-rmse", "r2")
CLF = ("binary-mcc", "accuracy", "f1", "roc", "prc")


def _metric(name, tw=None):
    from chemprop_b200.nn.metrics import EngineMetricRegistry

    return EngineMetricRegistry[name](1.0 if tw is None else tw)


def _updates(B, T, seed, *, clf, logits=False, mask_p=0.2, levels=None):
    g = np.random.default_rng(seed)
    if clf:
        P = g.normal(size=(B, T)) * 3 if logits else g.random((B, T))
        Y = (g.random((B, T)) < 0.35).astype(np.float32)
    else:
        P = g.normal(size=(B, T))
        Y = g.normal(size=(B, T))
    if levels:
        P = np.floor(P * levels) / levels
    P = P.astype(np.float32)
    m = g.random((B, T)) >= mask_p
    return dict(preds=P, targets=Y, mask=m, weights=(g.random(B) * 1.5 + 0.5).astype(np.float32),
                lt_mask=g.random((B, T)) < 0.2, gt_mask=g.random((B, T)) < 0.2)


def _cuda(u):
    return {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in u.items()}


def _run(name, updates, tw=None):
    m = _metric(name, tw)
    for u in updates:
        m.update(**_cuda(u))
    return m, float(m.compute())


def _check(name, got, want, rtol=1e-9):
    if np.isnan(want):
        assert np.isnan(got), (name, got)
    else:
        assert abs(got - want) <= rtol * max(1.0, abs(want)), (name, got, want, abs(got - want))


@pytest.mark.parametrize("T", [1, 12])
@pytest.mark.parametrize("B", [1, 7, 4097, 1_000_003])
def test_every_kind_against_the_oracle(B, T):
    tw = (np.arange(T) % 3 + 0.5).astype(np.float32)
    regs = [_updates(B, T, 10 + B + T, clf=False), _updates(max(1, B // 3), T, 11 + B, clf=False)]
    for name in REG:
        _, got = _run(name, regs, tw)
        want = O.METRICS[name](regs, tw)
        _check(name, got, want, 1e-9 if name != "r2" else 1e-8)
    clfs = [_updates(B, T, 20 + B + T, clf=True), _updates(max(1, B // 3), T, 21 + B, clf=True, logits=True)]
    for name in CLF:
        _, got = _run(name, clfs, tw)
        want = O.METRICS[name](clfs, tw)
        # logit updates go through a float32 sigmoid; the device's expf and numpy's exp may differ by an ulp
        _check(name, got, want, 1e-6)


@pytest.mark.parametrize("C", [3, 10])
@pytest.mark.parametrize("B", [1, 7, 4097, 100_003])
def test_multiclass_mcc_against_the_oracle(B, C):
    g = np.random.default_rng(B + C)
    T = 4
    tw = np.array([0.5, 1.0, 2.0, 1.5], np.float32)
    ups = []
    for k, b in enumerate((B, max(1, B // 2))):
        logits = g.normal(size=(b, T, C)).astype(np.float32) * 2
        P = logits if k else O.softmax32(logits)                 # one probability update, one logit update
        ups.append(dict(preds=P, targets=g.integers(0, C, (b, T)).astype(np.float32), mask=g.random((b, T)) > 0.2,
                        weights=(g.random(b) + 0.5).astype(np.float32)))
    _, got = _run("multiclass-mcc", ups, tw)
    _check("multiclass-mcc", got, O.multiclass_mcc(ups, tw), 1e-6)


def test_edge_cases_all_masked_single_class_logits():
    B, T = 513, 3
    u = _updates(B, T, 5, clf=True)
    # all masked: MSE 0/0 = NaN as the reference; AUROC 0, AUPRC NaN (no pair), accuracy / F1 0 (torchmetrics' safe divide)
    allm = dict(u, mask=np.zeros((B, T), bool))
    assert np.isnan(_run("mse", [allm])[1])
    assert _run("roc", [allm])[1] == 0.0 and np.isnan(_run("prc", [allm])[1])
    assert _run("accuracy", [allm])[1] == 0.0 and _run("f1", [allm])[1] == 0.0
    # single class: AUROC 0 either way (torchmetrics zeroes fpr or tpr); AUPRC NaN without positives, 1 without negatives
    pos = dict(u, targets=np.ones((B, T), np.float32))
    neg = dict(u, targets=np.zeros((B, T), np.float32))
    assert _run("roc", [pos])[1] == 0.0 and _run("roc", [neg])[1] == 0.0
    assert np.isnan(_run("prc", [neg])[1]) and np.isnan(O.auprc([neg]))
    _check("prc", _run("prc", [pos])[1], O.auprc([pos]))
    assert abs(_run("prc", [pos])[1] - 1.0) < 1e-12
    # logits: one value outside [0, 1] in the masked-in entries switches the whole update to sigmoid
    lg = dict(u, preds=u["preds"].copy())
    lg["preds"][0, 0], lg["mask"][0, 0] = 1.5, True
    # the sigmoid of these unquantised scores creates f32 ties, and the device's expf and numpy's exp can round a score to
    # either side of one: the ranking metrics differ from the oracle by ~1e-6 here
    for name in CLF:
        _check(name, _run(name, [lg])[1], O.METRICS[name]([lg]), 1e-5)
    # ... but not when it is masked out (ClassificationMixin formats preds[mask]); the MCCs test every prediction
    lg["mask"][0, 0] = False
    for name in ("roc", "accuracy", "binary-mcc"):
        _check(name, _run(name, [lg])[1], O.METRICS[name]([lg]), 1e-6)
    # a masked-in target outside {0, 1}: compute() is NaN and evaluate() raises
    bad = dict(u, targets=u["targets"].copy())
    bad["targets"][3, 1], bad["mask"][3, 1] = 2.0, True
    for name in CLF:
        assert np.isnan(_run(name, [bad])[1]), name


def test_ranking_on_ten_million_tied_pairs():
    n_b, T = 1_060_000, 10
    u = _updates(n_b, T, 77, clf=True, mask_p=0.05, levels=256)
    u["preds"] = np.clip(u["preds"], 0, 1)
    s, y = O.binary_formatted([u])
    assert s.size >= 10_000_000 and np.unique(s).size <= 257
    roc, prc = _run("roc", [u])[1], _run("prc", [u])[1]
    want_roc, want_prc = O.auroc_from(s, y), O.auprc_from(s, y)
    print(f"[metrics] 10M tied pairs: AUROC {roc!r} vs {want_roc!r}, AUPRC {prc!r} vs {want_prc!r}")
    assert abs(roc - want_roc) <= 1e-12 * abs(want_roc)
    assert abs(prc - want_prc) <= 1e-9 * abs(want_prc)


def test_uneven_batches_accumulate_to_the_concatenated_batch_and_repeat_bitwise():
    T = 12
    parts = [_updates(b, T, 300 + b, clf=True) for b in (1, 4096, 17, 100_000, 333)]
    cat = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
    for name in REG + CLF + ("multiclass-mcc",):
        if name == "multiclass-mcc":
            ps = [dict(p, preds=np.stack([1 - p["preds"], p["preds"]], -1)) for p in parts]
            c = dict(cat, preds=np.stack([1 - cat["preds"], cat["preds"]], -1))
        else:
            ps, c = parts, cat
        m1, v1 = _run(name, ps)
        _, v2 = _run(name, ps)
        _, vc = _run(name, [c])
        assert np.float64(v1).tobytes() == np.float64(v2).tobytes(), name            # bitwise repeatable
        _check(name, v1, vc, 1e-12)                                                  # one batch, within rounding


def _lib_ws(nbytes, fill):
    return torch.full((max(nbytes, 1),), fill, dtype=torch.uint8, device="cuda")


def test_workspace_contents_do_not_matter():
    """Every entry point with a workspace of 0x00 bytes and one of 0xFF bytes (NaN in every f32 / f64 slot): identical bits."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import _stream

    lib = _lib.load()
    B, T, C = 70_001, 5, 4
    g = torch.Generator(device="cuda").manual_seed(3)
    P = torch.rand(B, T * C, device="cuda", generator=g)
    Y = (torch.rand(B, T, device="cuda", generator=g) * C).floor()
    Yb = (Y > 1).float()
    M = (torch.rand(B, T, device="cuda", generator=g) > 0.3).to(torch.uint8)
    w = torch.rand(B, device="cuda", generator=g)
    n = ctypes.c_size_t(0)
    _lib.check(lib.dmpnn_metric_workspace_bytes(B, T, C, ctypes.byref(n)), "ws")
    outs = []
    for fill in (0, 255):
        ws = _lib_ws(n.value, fill)
        f = torch.zeros(T * (2 * C + 2) + 8 * T, dtype=torch.float64, device="cuda")
        i = torch.zeros(8, dtype=torch.int64, device="cuda")
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        for kind in range(5):
            _lib.check(lib.dmpnn_metric_accumulate(kind, P.data_ptr(), T * C, (Yb if kind >= 2 else Y).data_ptr(), T,
                                                   M.data_ptr(), w.data_ptr(), None, None, None, T, B, T,
                                                   f[T * (2 * C + 2):].data_ptr(), i.data_ptr(), st.data_ptr(),
                                                   ws.data_ptr(), _stream()), "acc")
        _lib.check(lib.dmpnn_metric_multiclass_mcc(P.data_ptr(), T * C, Y.data_ptr(), T, M.data_ptr(), T, w.data_ptr(), B, T,
                                                   C, f.data_ptr(), st.data_ptr(), ws.data_ptr(), _stream()), "mcc")
        sc = torch.empty(B * T, device="cuda")
        lb = torch.empty(B * T, dtype=torch.uint8, device="cuda")
        kp = torch.empty_like(lb)
        _lib.check(lib.dmpnn_metric_rank_format(P.data_ptr(), T * C, Yb.data_ptr(), T, M.data_ptr(), T, B, T, sc.data_ptr(),
                                                lb.data_ptr(), kp.data_ptr(), st.data_ptr(), ws.data_ptr(), _stream()), "fmt")
        nc = ctypes.c_size_t(0)
        _lib.check(lib.dmpnn_rank_curve_workspace_bytes(B * T, ctypes.byref(nc)), "curve ws")
        wc = _lib_ws(nc.value, fill)
        out = torch.empty(2, dtype=torch.float64, device="cuda")
        _lib.check(lib.dmpnn_rank_curve(sc.data_ptr(), lb.data_ptr(), kp.data_ptr(), B * T, out.data_ptr(), wc.data_ptr(),
                                        nc.value, _stream()), "curve")
        outs.append([x.cpu().numpy().tobytes() for x in (f, i, st, out)])
    assert outs[0] == outs[1]
    assert int(torch.from_numpy(np.frombuffer(outs[0][2], np.int32).copy())[0]) == 0


def test_update_does_not_synchronise():
    from chemprop_b200.nn.head import _BCECriterion
    from chemprop_b200.nn.metrics import EngineCriterionMetric

    T = 12
    u = _cuda(_updates(5000, T, 9, clf=True))
    mc = dict(u, preds=torch.stack([1 - u["preds"], u["preds"]], -1))
    metrics = [(_metric(n), u) for n in REG + CLF] + [(_metric("multiclass-mcc"), mc),
                                                      (EngineCriterionMetric(_BCECriterion(torch.ones(T)).cuda()), u)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for m, args in metrics:
            kw = dict(args) if m.alias.startswith("bounded") else {k: v for k, v in args.items() if k not in ("lt_mask", "gt_mask")}
            m.update(**kw)
            m.update(**kw)
            m.compute()
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---- EngineMPNN.evaluate ---------------------------------------------------------------------------------------------------
N_MOL, BS, D_H = 3000, 1000, 64


def _mol_batches(T, targets_fn, seed=0, mc=False):
    from chemprop_b200.data import BatchMolGraph, MulticomponentTrainingBatch, TrainingBatch, make_molecules

    g = np.random.default_rng(seed)
    comps = [make_molecules(N_MOL, seed=seed + c, mean_atoms=12, std_atoms=4, min_atoms=1) for c in range(2 if mc else 1)]
    out = []
    for lo in range(0, N_MOL, BS):
        hi = min(N_MOL, lo + BS)
        b = hi - lo
        Y = targets_fn(g, b, T).astype(np.float32)
        Y[g.random((b, T)) < 0.15] = np.nan
        Y = torch.from_numpy(Y).cuda()
        w = torch.from_numpy((g.random((b, 1)) + 0.5).astype(np.float32)).cuda()
        if mc:
            bmg = BatchMolGraph([comps[c][m] for m in range(lo, hi) for c in range(2)])
            bmg.to("cuda")
            out.append(MulticomponentTrainingBatch(bmg, None, None, Y, w, None, None))
        else:
            bmg = BatchMolGraph(comps[0][lo:hi])
            bmg.to("cuda")
            out.append(TrainingBatch(bmg, None, None, Y, w, None, None))
    return out


def _np_updates(model, batches, train_modules=(), weights_one=True, train_step=False):
    """The oracle's updates from the model's own predictions, in the mode the reference's hook sets."""
    flags = [(m, m.training) for m in model.modules()]
    model.eval()
    for m in train_modules:
        m.train()
    ups = []
    with torch.no_grad():
        for bt in batches:
            Z = model.fingerprint(bt[0], bt[1], bt[2])
            P = model.predictor.train_step(Z) if train_step else model.predictor(Z)
            if not train_step and model.predictor.n_targets > 1:
                P = P[..., 0]
            Y = bt[3].cpu().numpy()
            ups.append(dict(preds=P.float().cpu().numpy(), targets=np.nan_to_num(Y, nan=0.0), mask=np.isfinite(Y),
                            weights=np.ones(len(Y)) if weights_one else bt[4].cpu().numpy().reshape(-1)))
    for m, f in flags:
        m.training = f
    return ups


def _val_modules(model):
    return model._eval_modules()


def test_evaluate_regression_bf16_val_stays_scaled_test_unscales():
    import chemprop_b200.nn as N

    T = 3
    torch.manual_seed(0)
    mean, scale = np.array([1.0, -2.0, 0.5]), np.array([2.0, 0.5, 3.0])
    model = N.EngineMPNN(N.BondMessagePassing(d_h=D_H, precision="bf16"),
                         predictor=N.EngineRegressionFFN(n_tasks=T, input_dim=D_H,
                                                         output_transform=N.UnscaleTransform(mean, scale))).cuda()
    batches = _mol_batches(T, lambda g, b, T: g.normal(size=(b, T)))
    model.train()
    metrics = [_metric("mse"), _metric("r2"), _metric("mae")]
    val = model.evaluate(batches, metrics, stage="val")
    assert all(m.training for m in model.modules())                     # every flag restored
    val_ups = _np_updates(model, batches, [model.predictor.output_transform])
    for name in ("mse", "r2", "mae"):
        _check(name, val[f"val/{name}"], O.METRICS[name](val_ups), 1e-9)
    loss_ups = _np_updates(model, batches, [model.predictor.output_transform], weights_one=False, train_step=True)
    _check("val_loss", val["val_loss"], O.mse(loss_ups), 1e-6)
    test = model.evaluate(batches, metrics, stage="test")
    assert set(test) == {"test/mse", "test/r2", "test/mae"}
    test_ups = _np_updates(model, batches)
    for name in ("mse", "r2", "mae"):
        _check(name, test[f"test/{name}"], O.METRICS[name](test_ups), 1e-9)
    # the unscaling is on in test mode only: the scaled predictions differ from the unscaled ones by the transform
    p_val, p_test = val_ups[0]["preds"], test_ups[0]["preds"]
    np.testing.assert_allclose(p_val * scale + mean, p_test, rtol=1e-5, atol=1e-5)
    assert not np.allclose(p_val, p_test)
    # default metric: MSE
    assert set(model.evaluate(batches, stage="test")) == {"test/mse"}


def _bce64(ups, tw):
    s = n = 0.0
    for u in ups:
        x, y, m, w = (np.asarray(u[k], np.float64) for k in ("preds", "targets", "mask", "weights"))
        L = np.maximum(x, 0) - x * y + np.log1p(np.exp(-np.abs(x)))
        s += (L * w[:, None] * tw[None, :] * m).sum()
        n += m.sum()
    return s / n


def test_evaluate_binary_head():
    import chemprop_b200.nn as N

    T = 4
    torch.manual_seed(1)
    tw = torch.tensor([1.0, 0.5, 2.0, 1.0])
    model = N.EngineMPNN(N.BondMessagePassing(d_h=D_H),
                         predictor=N.EngineBinaryClassificationFFN(n_tasks=T, input_dim=D_H, task_weights=tw)).cuda()
    batches = _mol_batches(T, lambda g, b, T: (g.random((b, T)) < 0.4).astype(float), seed=3)
    names = ("roc", "prc", "accuracy", "f1", "binary-mcc")
    val = model.evaluate(batches, [_metric(n) for n in names])
    ups = _np_updates(model, batches, _val_modules(model))
    for name in names:
        _check(name, val[f"val/{name}"], O.METRICS[name](ups), 1e-6)
    _check("val_loss", val["val_loss"], _bce64(_np_updates(model, batches, _val_modules(model), False, True), tw.numpy()), 1e-5)
    assert set(model.evaluate(batches, stage="test")) == {"test/roc"}                       # default metric
    bad = [batches[0]._replace(Y=torch.where(batches[0].Y.isfinite(), batches[0].Y * 2, batches[0].Y))]
    with pytest.raises(ValueError, match="roc"):
        model.evaluate(bad)


def test_evaluate_multiclass_and_spectral_heads():
    import chemprop_b200.nn as N

    T, C = 2, 3
    torch.manual_seed(2)
    model = N.EngineMPNN(N.BondMessagePassing(d_h=D_H),
                         predictor=N.EngineMulticlassClassificationFFN(n_classes=C, n_tasks=T, input_dim=D_H)).cuda()
    batches = _mol_batches(T, lambda g, b, T: g.integers(0, C, (b, T)).astype(float), seed=4)
    res = model.evaluate(batches, stage="test")
    _check("multiclass-mcc", res["test/multiclass-mcc"], O.multiclass_mcc(_np_updates(model, batches)), 1e-6)

    T = 16
    spec = N.EngineMPNN(N.BondMessagePassing(d_h=D_H), predictor=N.EngineSpectralFFN(n_tasks=T, input_dim=D_H)).cuda()

    def spectra(g, b, T):
        y = g.random((b, T)) + 0.05
        return y / y.sum(1, keepdims=True)

    batches = _mol_batches(T, spectra, seed=5)
    res = spec.evaluate(batches)
    assert set(res) == {"val_loss", "val/EngineSID"}
    ups = _np_updates(spec, batches, _val_modules(spec))

    def sid(ups, use_w):
        s = n = 0.0
        for u in ups:
            p, y, m = (np.asarray(u[k], np.float64) for k in ("preds", "targets", "mask"))
            w = np.asarray(u["weights"], np.float64) if use_w else np.ones(len(p))
            pn = p / (p * m).sum(1, keepdims=True)
            y, pn = np.where(m, y, 1.0), np.where(m, pn, 1.0)
            L = np.log(pn / y) * pn + np.log(y / pn) * y
            s += (L * m * w[:, None]).sum()
            n += m.sum()
        return s / n

    _check("val/EngineSID", res["val/EngineSID"], sid(ups, False), 1e-5)
    _check("val_loss", res["val_loss"], sid(_np_updates(spec, batches, _val_modules(spec), False, True), True), 1e-5)


def test_evaluate_multicomponent_union_batch():
    import chemprop_b200.nn as N

    T = 2
    torch.manual_seed(4)
    block = N.BondMessagePassing(d_h=D_H)
    mp = N.EngineMulticomponentMessagePassing([block], n_components=2, shared=True)
    model = N.EngineMulticomponentMPNN(mp, predictor=N.EngineRegressionFFN(n_tasks=T, input_dim=2 * D_H)).cuda()
    batches = _mol_batches(T, lambda g, b, T: g.normal(size=(b, T)), seed=6, mc=True)
    res = model.evaluate(batches, [_metric("rmse"), _metric("r2")])
    ups = _np_updates(model, batches, _val_modules(model))
    _check("rmse", res["val/rmse"], O.rmse(ups), 1e-9)
    _check("r2", res["val/r2"], O.r2(ups), 1e-9)
    _check("val_loss", res["val_loss"], O.mse(_np_updates(model, batches, _val_modules(model), False, True)), 1e-6)


def test_criterion_metric_reproduces_the_reference_validation_loss():
    """EngineCriterionMetric over the golden batches (tests/golden/fixture_metrics.npz, the reference's own criteria):
    every engine criterion reduces a batch to sum L w tw m / sum m, so value x count accumulates the reference's epoch
    value; each batch's value is checked too."""
    import chemprop_b200.nn as N
    from chemprop_b200.nn.head import _BCECriterion, _Criterion
    from chemprop_b200.nn.metrics import EngineCriterionMetric
    from tests.util import load_golden

    g = load_golden("fixture_metrics")
    make = {"mse": _Criterion, "mae": N.EngineMAE, "rmse": N.EngineRMSE, "bounded-mse": N.EngineBoundedMSE,
            "bounded-mae": N.EngineBoundedMAE, "bounded-rmse": N.EngineBoundedRMSE, "bce": _BCECriterion,
            "sid": N.EngineSID}
    for name in [str(x) for x in g["criteria"]]:
        crit = make[name](torch.from_numpy(g[f"crit.{name}.task_weights"])).cuda()
        m = EngineCriterionMetric(crit)
        for i in range(len(g[f"crit.{name}.batch_values"])):
            u = {k: torch.from_numpy(g[f"crit.{name}.{i}.{k}"]).cuda()
                 for k in ("preds", "targets", "mask", "weights", "lt_mask", "gt_mask")}
            u["weights"] = u["weights"].view(-1, 1)
            m.update(**u)
            bounds = (u["lt_mask"], u["gt_mask"]) if crit._bounded else ()
            v = float(crit(u["preds"], u["targets"], u["mask"], u["weights"], *bounds))
            assert abs(v - float(g[f"crit.{name}.batch_values"][i])) <= 1e-5 * max(1.0, abs(v)), (name, i)
        want = float(g[f"crit.{name}.value"])
        assert abs(float(m.compute()) - want) <= 1e-5 * max(1.0, abs(want)), name
