"""CPU tier for the device metrics (csrc/metrics.cu, chemprop_b200/nn/metrics.py, EngineMPNN.evaluate): the float64
restatement oracle/metrics_np.py against the reference's own metric classes (tests/golden/fixture_metrics.npz, written by
tools/make_golden_metrics.py) and against sklearn where the definitions coincide; the new C entry points refusing bad
arguments before any CUDA call; `evaluate`'s host logic through the kernel emulations of tests/emu_metrics.py; and `sync_`
on gloo with two ranks."""
from __future__ import annotations

import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import metrics_np as O
from tests.util import load_golden

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fixture_metrics.npz")


# ---- the oracle against the reference's classes --------------------------------------------------------------------------
def _golden_updates(g, prefix, n):
    keys = ("preds", "targets", "mask", "weights", "lt_mask", "gt_mask")
    return [{k: g[f"{prefix}.{i}.{k}"] for k in keys if f"{prefix}.{i}.{k}" in g} for i in range(n)]


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="fixture not generated")
def test_oracle_matches_the_reference_metric_classes():
    g = load_golden("fixture_metrics")
    names = [str(x) for x in g["names"]]
    assert {"mse", "mae", "rmse", "bounded-mse", "bounded-mae", "bounded-rmse", "binary-mcc", "multiclass-mcc"} <= set(names)
    for name in names:
        n = int(g[f"{name}.n"])
        for variant in ("prob", "logit") if name.endswith("mcc") else ("plain",):
            ups = _golden_updates(g, f"{name}.{variant}", n)
            tw = g[f"{name}.task_weights"]
            want = float(g[f"{name}.{variant}.value"])
            got = O.METRICS[name](ups, tw)
            # the reference sums in float32
            assert abs(got - want) <= 2e-6 * max(1.0, abs(want)), (name, variant, got, want)


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="fixture not generated")
def test_criterion_as_metric_is_value_times_count():
    """Each reference criterion's epoch value equals sum_k value_k n_k / sum_k n_k of its per-batch values (the sqrt of the
    mean of value_k^2 n_k for RMSE), which is what EngineCriterionMetric accumulates from the engine criteria."""
    g = load_golden("fixture_metrics")
    for name in [str(x) for x in g["criteria"]]:
        vals, counts = g[f"crit.{name}.batch_values"], g[f"crit.{name}.batch_counts"]
        got = O.criterion_metric(list(zip(vals.astype(np.float64), counts)), rmse_type=name in ("rmse", "bounded-rmse"))
        assert abs(got - float(g[f"crit.{name}.value"])) <= 2e-6 * max(1.0, abs(got)), name


def _clf(n, T, seed, logits=False):
    r = np.random.default_rng(seed)
    P = (r.normal(size=(n, T)) * 2 if logits else np.floor(r.random((n, T)) * 64) / 64).astype(np.float32)
    return dict(preds=P, targets=(r.random((n, T)) < 0.4).astype(np.float32), mask=r.random((n, T)) > 0.2)


def test_oracle_against_sklearn():
    skm = pytest.importorskip("sklearn.metrics")
    ups = [_clf(500, 3, 1), _clf(301, 3, 2)]
    s, y = O.binary_formatted(ups)
    assert abs(O.auroc(ups) - skm.roc_auc_score(y, s)) < 1e-12
    assert abs(O.auprc(ups) - skm.auc(*skm.precision_recall_curve(y, s)[1::-1])) < 1e-12
    assert abs(O.accuracy(ups) - skm.accuracy_score(y, s > 0.5)) < 1e-12
    assert abs(O.f1(ups) - skm.f1_score(y, s > 0.5)) < 1e-12
    lg = [_clf(400, 2, 3, logits=True)]
    s2, y2 = O.binary_formatted(lg)
    assert abs(O.auroc(lg) - skm.roc_auc_score(y2, s2)) < 1e-12
    r = np.random.default_rng(4)
    P, Y = r.normal(size=(200, 3)).astype(np.float32), r.normal(size=(200, 3)).astype(np.float32)
    m = r.random((200, 3)) > 0.3
    assert abs(O.r2([dict(preds=P, targets=Y, mask=m)]) - skm.r2_score(Y[m].astype(np.float64), P[m].astype(np.float64))) < 1e-9
    # multiclass MCC with probability inputs: s = sum w over the masked-in rows, so the soft MCC is sklearn's weighted MCC
    C, b = 4, 300
    probs = O.softmax32(r.normal(size=(b, 1, C)).astype(np.float32))
    t = r.integers(0, C, (b, 1)).astype(np.float32)
    w = (r.random(b) + 0.5).astype(np.float32)
    mk = r.random((b, 1)) > 0.2
    got = O.multiclass_mcc([dict(preds=probs, targets=t, mask=mk, weights=w)])
    want = skm.matthews_corrcoef(t[:, 0][mk[:, 0]], probs[:, 0].argmax(-1)[mk[:, 0]], sample_weight=w[mk[:, 0]])
    assert abs(got - want) < 1e-6


def test_ranking_edge_cases_pinned():
    u = _clf(50, 2, 5)
    neg = dict(u, targets=np.zeros_like(u["targets"]))
    pos = dict(u, targets=np.ones_like(u["targets"]))
    assert O.auroc([neg]) == 0.0 and O.auroc([pos]) == 0.0            # torchmetrics zeroes fpr or tpr
    assert np.isnan(O.auprc([neg])) and abs(O.auprc([pos]) - 1.0) < 1e-12


# ---- C entry points refuse bad arguments on the host -----------------------------------------------------------------------
def test_metric_entry_points_validate_before_touching_the_device():
    from chemprop_b200 import _lib

    lib = _lib.load()
    n = ctypes.c_size_t(0)
    st = np.zeros(1, np.int32)
    f = np.zeros(64, np.float64)
    i = np.zeros(8, np.int64)
    buf = np.zeros(16, np.float32)
    ptr = buf.ctypes.data
    assert lib.dmpnn_metric_workspace_bytes(-1, 1, 1, ctypes.byref(n)) != 0
    assert lib.dmpnn_metric_workspace_bytes(5, 0, 1, ctypes.byref(n)) != 0
    assert lib.dmpnn_metric_workspace_bytes(5, 2, 1, ctypes.byref(n)) == 0 and n.value > 0
    assert lib.dmpnn_metric_accumulate(9, ptr, 1, ptr, 1, None, None, None, None, None, 1, 4, 1, f.ctypes.data,
                                       i.ctypes.data, st.ctypes.data, ptr, None) != 0
    assert b"unknown kind" in lib.dmpnn_last_error()
    assert lib.dmpnn_metric_accumulate(0, ptr, 1, ptr, 1, None, None, None, None, None, 1, -1, 1, f.ctypes.data,
                                       i.ctypes.data, None, ptr, None) != 0                        # B < 0
    assert lib.dmpnn_metric_accumulate(0, None, 1, ptr, 1, None, None, None, None, None, 1, 4, 1, f.ctypes.data,
                                       i.ctypes.data, None, ptr, None) != 0                        # null P
    assert lib.dmpnn_metric_accumulate(3, ptr, 1, ptr, 1, None, None, None, None, None, 1, 4, 1, None, i.ctypes.data,
                                       None, ptr, None) != 0                                       # classification: status
    assert lib.dmpnn_metric_accumulate(2, ptr, 1, ptr, 1, None, None, None, ptr, None, 1, 4, 1, f.ctypes.data,
                                       i.ctypes.data, None, ptr, None) != 0                        # bounds only for MSE / MAE
    assert lib.dmpnn_metric_accumulate(0, ptr, 1, ptr, 1, None, None, None, None, None, 1, 0, 1, f.ctypes.data,
                                       i.ctypes.data, None, None, None) == 0                       # B = 0: nothing to do
    assert lib.dmpnn_metric_multiclass_mcc(ptr, 2, ptr, 1, None, 1, None, 4, 1, 1, f.ctypes.data, st.ctypes.data, ptr,
                                           None) != 0                                              # C < 2
    assert b"C >= 2" in lib.dmpnn_last_error()
    assert lib.dmpnn_metric_multiclass_mcc(ptr, 2, ptr, 1, None, 1, None, 4, 1, 3, f.ctypes.data, st.ctypes.data, ptr,
                                           None) != 0                                              # ldp < T C
    assert lib.dmpnn_metric_rank_format(ptr, 1, ptr, 1, None, 1, 4, 1, None, ptr, ptr, st.ctypes.data, ptr, None) != 0
    assert lib.dmpnn_rank_curve_workspace_bytes(-1, ctypes.byref(n)) != 0
    assert lib.dmpnn_rank_curve_workspace_bytes(0, ctypes.byref(n)) == 0 and n.value == 0
    assert lib.dmpnn_rank_curve(None, None, None, 10, f.ctypes.data, None, 0, None) != 0           # null inputs
    assert lib.dmpnn_rank_curve(ptr, ptr, ptr, 10, None, ptr, 0, None) != 0                        # null out


# ---- evaluate's host logic through the emulations ------------------------------------------------------------------------
@pytest.fixture
def emulated(monkeypatch):
    from tests import emu_metrics
    from tests.test_spectral_host import patch_spectral
    from tests.test_uncertainty_host import patch_uncertainty

    patch_uncertainty(monkeypatch)
    patch_spectral(monkeypatch)
    emu_metrics.patch_metrics(monkeypatch)


def _batches(T, kind="reg", n=40, bs=16, seed=0):
    from chemprop_b200.data import BatchMolGraph, TrainingBatch, make_molecules

    r = np.random.default_rng(seed)
    mgs = make_molecules(n, seed=seed, mean_atoms=6, std_atoms=2, min_atoms=1)
    out = []
    for lo in range(0, n, bs):
        b = min(bs, n - lo)
        Y = (r.random((b, T)) < 0.4).astype(np.float32) if kind == "clf" else r.normal(size=(b, T)).astype(np.float32)
        Y[r.random((b, T)) < 0.2] = np.nan
        w = (r.random((b, 1)) + 0.5).astype(np.float32)
        out.append(TrainingBatch(BatchMolGraph(mgs[lo:lo + b]), None, None, torch.from_numpy(Y), torch.from_numpy(w),
                                 None, None))
    return out


class _Recorder:
    """An EngineMetric stand-in recording what evaluate passes and the modes the model is in."""
    alias = "rec"
    _status = None

    def __init__(self, model):
        self.model, self.calls = model, []

    def reset(self):
        self.calls = []

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        mp, pr = self.model.message_passing, self.model.predictor
        self.calls.append(dict(shape=tuple(preds.shape), weights=weights.clone(), finite=bool(targets.isfinite().all()),
                               modes=(self.model.training, mp.training, mp.V_d_transform.training,
                                      mp.graph_transform.training, self.model.X_d_transform.training,
                                      pr.output_transform.training, pr.ffn.training), grad=torch.is_grad_enabled()))

    def compute(self):
        return torch.tensor(float(len(self.calls)))


def _reg_model(T):
    import chemprop_b200.nn as N

    torch.manual_seed(0)
    return N.EngineMPNN(N.BondMessagePassing(d_h=16, depth=2), predictor=N.EngineRegressionFFN(
        n_tasks=T, input_dim=16, output_transform=N.UnscaleTransform(np.arange(T) * 1.0, np.arange(T) + 1.0)))


def test_evaluate_modes_weights_and_restoration(emulated):
    from chemprop_b200.nn.metrics import EngineMSEMetric

    T = 3
    model = _reg_model(T)
    batches = _batches(T)
    model.train()
    model.predictor.ffn.eval()                              # an odd flag, to see that each flag is restored as it was
    before = {n: m.training for n, m in model.named_modules()}
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    seen = []
    crit = model.predictor.criterion
    orig = crit.forward

    def spy(preds, targets, mask=None, weights=None, *a):
        seen.append(weights.clone())
        return orig(preds, targets, mask, weights, *a)

    crit.forward = spy
    rec = _Recorder(model)
    res = model.evaluate(batches, [rec, EngineMSEMetric()], stage="val")
    assert set(res) == {"val_loss", "val/rec", "val/mse"} and res["val/rec"] == len(batches)
    assert {n: m.training for n, m in model.named_modules()} == before
    assert all(torch.equal(v, model.state_dict()[k]) for k, v in sd.items()) and set(sd) == set(model.state_dict())
    for c, bt in zip(rec.calls, batches):
        # eval mode, except the transforms on_validation_model_eval keeps in training mode
        assert c["modes"] == (False, False, True, True, True, True, False) and not c["grad"]
        assert torch.equal(c["weights"], torch.ones_like(bt.w)) and c["finite"]
    assert len(seen) == len(batches) and all(torch.equal(s, bt.w) for s, bt in zip(seen, batches))
    res = model.evaluate(batches, [rec], stage="test")
    assert set(res) == {"test/rec"} and len(seen) == len(batches)           # no criterion in the test stage
    assert all(c["modes"] == (False,) * 7 for c in rec.calls)
    with pytest.raises(ValueError, match="stage"):
        model.evaluate(batches, stage="train")


def test_evaluate_matches_the_oracle_through_the_emulation(emulated):
    from chemprop_b200.nn.metrics import EngineMetricRegistry

    T = 3
    model = _reg_model(T)
    batches = _batches(T)
    names = ("mse", "mae", "rmse", "r2")
    res = model.evaluate(batches, [EngineMetricRegistry[n]() for n in names], stage="test")
    model.eval()
    with torch.no_grad():
        ups = [dict(preds=model(bt.bmg).numpy(), targets=np.nan_to_num(bt.Y.numpy()), mask=np.isfinite(bt.Y.numpy()))
               for bt in batches]
    for n in names:
        assert abs(res[f"test/{n}"] - O.METRICS[n](ups)) < 1e-9 * max(1, abs(res[f"test/{n}"])), n


def test_evaluate_takes_the_first_target_and_the_default_metrics(emulated):
    import chemprop_b200.nn as N
    from chemprop_b200.nn.metrics import (EngineAUROCMetric, EngineCriterionMetric, EngineMSEMetric,
                                          EngineMulticlassMCCMetric, default_metric)

    T = 2
    model = N.EngineMPNN(N.BondMessagePassing(d_h=16, depth=2), predictor=N.EngineMveFFN(n_tasks=T, input_dim=16))
    rec = _Recorder(model)
    model.evaluate(_batches(T), [rec], stage="test")
    assert all(c["shape"][1:] == (T,) for c in rec.calls)                   # preds[..., 0] of b x T x 2
    defaults = {N.EngineRegressionFFN: EngineMSEMetric, N.EngineMveFFN: EngineMSEMetric, N.EngineEvidentialFFN: EngineMSEMetric,
                N.EngineQuantileFFN: EngineMSEMetric, N.EngineBinaryClassificationFFN: EngineAUROCMetric,
                N.EngineBinaryDirichletFFN: EngineAUROCMetric}
    for cls, want in defaults.items():
        assert type(default_metric(cls(n_tasks=2, input_dim=8))) is want, cls
    for cls in (N.EngineMulticlassClassificationFFN, N.EngineMulticlassDirichletFFN):
        assert type(default_metric(cls(n_classes=3, n_tasks=2, input_dim=8))) is EngineMulticlassMCCMetric
    sid = default_metric(N.EngineSpectralFFN(n_tasks=4, input_dim=8))
    assert isinstance(sid, EngineCriterionMetric) and type(sid.criterion) is N.EngineSID and sid.criterion.threshold is None
    # binary head: the default AUROC on the probabilities
    bin_model = N.EngineMPNN(N.BondMessagePassing(d_h=16, depth=2), predictor=N.EngineBinaryClassificationFFN(
        n_tasks=T, input_dim=16))
    bts = _batches(T, "clf")
    res = bin_model.evaluate(bts, stage="test")
    bin_model.eval()
    with torch.no_grad():
        ups = [dict(preds=bin_model(bt.bmg).numpy(), targets=np.nan_to_num(bt.Y.numpy()), mask=np.isfinite(bt.Y.numpy()))
               for bt in bts]
    assert abs(res["test/roc"] - O.auroc(ups)) < 1e-12


def test_metric_state_stays_out_of_the_state_dict(emulated):
    from chemprop_b200.nn.metrics import EngineMetricRegistry

    T = 3
    model = _reg_model(T)
    keys = set(model.state_dict())
    model.evaluate(_batches(T), [EngineMetricRegistry[n]() for n in ("mse", "r2")])
    assert set(model.state_dict()) == keys and not any(k.startswith("metrics") for k in keys)


def test_criterion_metric_accumulates_value_times_count(emulated):
    import chemprop_b200.nn as N
    from chemprop_b200.nn.metrics import EngineCriterionMetric

    r = np.random.default_rng(7)
    for crit, rm in ((N.EngineRMSE(torch.tensor([1.0, 2.0])), True), (N.EngineMAE(torch.tensor([1.0, 0.5])), False)):
        m = EngineCriterionMetric(crit)
        pairs = []
        for b in (5, 11, 3):
            P = torch.from_numpy(r.normal(size=(b, 2)).astype(np.float32))
            Y = torch.from_numpy(r.normal(size=(b, 2)).astype(np.float32))
            mask = torch.from_numpy(r.random((b, 2)) > 0.3)
            m.update(P, Y, mask)
            pairs.append((float(crit(P, Y, mask)), int(mask.sum())))
        assert abs(float(m.compute()) - O.criterion_metric(pairs, rm)) < 1e-9


# ---- sync_ over two ranks --------------------------------------------------------------------------------------------------
def _sync_worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from chemprop_b200.nn.metrics import EngineAUROCMetric, EngineMSEMetric

    mse = EngineMSEMetric()
    mse._alloc(torch.device("cpu"), 2)
    mse._f[0], mse._i[0] = 1.5 * (rank + 1), 3 * (rank + 1)                 # states filled by hand
    mse.sync_()
    roc = EngineAUROCMetric()
    roc._status = torch.zeros(1, dtype=torch.int32)
    n = 3 + 2 * rank                                                        # uneven: padded to the largest rank's size
    roc._lists = ([torch.full((n,), rank + 0.25)], [torch.full((n,), rank, dtype=torch.uint8)],
                  [torch.ones(n, dtype=torch.uint8)])
    roc.sync_()
    q.put((rank, float(mse._f[0]), int(mse._i[0]), [x.tolist() for x in roc._lists[0]],
           [x.tolist() for x in roc._lists[1]]))
    dist.destroy_process_group()


def test_sync_over_gloo_world2():
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() + 977) % 2000
    procs = [ctx.Process(target=_sync_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in res:
        assert r[1] == 4.5 and r[2] == 9
        assert r[3] == [[0.25] * 3, [1.25] * 5] and r[4] == [[0] * 3, [1] * 5]
