"""Validation and test metrics accumulated on the device: chemprop's `MetricRegistry` (chemprop/nn/metrics.py:59-499) on the
engine's kernels (csrc/metrics.cu), without torchmetrics.

Every metric has the reference's `update(preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None)`,
`compute()` and `reset()`, and a `task_weights` attribute.  `update` only enqueues launches: each adds the batch into f64
sums and int64 counts on the device (or, for AUROC / AUPRC, appends the batch's formatted scores to a list, as
torchmetrics' `cat` states do).  `compute()` returns a 0-d f64 device tensor and does not synchronise either; it is NaN
where an update met a target its metric cannot take (a binary label outside {0, 1}, a class outside [-C, C)), which the
reference would have refused with an exception.  `EngineMPNN.evaluate` reads every value with one host sync and raises
there instead.

The metrics are plain objects, not modules: their state never enters a model's `state_dict` (the reference's `metrics.*`
keys are stripped when its checkpoints load into the engine's models), so they are passed to `evaluate` rather than
registered on the model.  `sync_(group)` sums the states over a process group and gathers the ranking lists, as
torchmetrics' `dist_reduce_fx` does for data-parallel evaluation."""
from __future__ import annotations

import torch
import torch.distributed as dist
from torch import Tensor

from .. import _lib
from .. import engine as K
from .head import _loss_weights, _RegressionCriterion

__all__ = ["EngineMetric", "EngineMetricRegistry", "EngineCriterionMetric", "default_metric"]


def _mask_u8(targets: Tensor, mask: Tensor | None) -> Tensor:
    """b x T uint8 mask; None selects every entry, as the reference's `torch.ones_like(targets, dtype=torch.bool)`."""
    if mask is None:
        return torch.ones(targets.shape, dtype=torch.uint8, device=targets.device)
    return mask.to(torch.uint8).expand(targets.shape).contiguous()


class EngineMetric:
    """Base of the engine's metrics: the reference's interface, state allocated on the device of the first update."""
    alias = ""
    higher_is_better = False
    _n_f = 0                       # f64 state entries (a function of T where per task)
    _n_i = 0                       # int64 state entries

    def __init__(self, task_weights=1.0):
        self.task_weights = torch.as_tensor(task_weights, dtype=torch.float).view(1, -1)
        self.reset()

    def reset(self):
        self._f = self._i = self._status = None

    # ---- state ----
    def _alloc(self, dev, T: int):
        if self._status is None:
            self._f = torch.zeros(self._f_size(T), dtype=torch.float64, device=dev)
            self._i = torch.zeros(self._n_i, dtype=torch.int64, device=dev)
            self._status = torch.zeros(1, dtype=torch.int32, device=dev)
            self._T = T

    def _f_size(self, T: int) -> int:
        return self._n_f

    def _tw(self, T: int, dev) -> Tensor:
        tw = self.task_weights.to(dev, non_blocking=True).reshape(-1)
        return (tw.expand(T) if tw.numel() == 1 else tw).contiguous()

    def _states(self) -> list[Tensor]:
        return [self._f, self._i, self._status]

    def _checked(self, v: Tensor) -> Tensor:
        return torch.where(self._status[0] != 0, torch.full_like(v, float("nan")), v)

    @staticmethod
    def _inputs(preds: Tensor, targets: Tensor, *others):
        """preds, targets as contiguous f32; every tensor argument must be on the GPU (the kernels read them there)."""
        K._require_cuda(preds, targets, *others)
        if preds.shape[:2] != targets.shape or targets.dim() != 2:
            raise ValueError(f"expected b x T targets and predictions of the same leading shape, got {tuple(preds.shape)} "
                             f"and {tuple(targets.shape)}")
        return preds.float().contiguous(), targets.float().contiguous()

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        raise NotImplementedError

    def compute(self) -> Tensor:
        raise NotImplementedError

    def sync_(self, group=None):
        """Sum the states over `group` (every rank must have updated at least once, so that the states exist)."""
        for t in self._states():
            if t is not None and t.numel():
                dist.all_reduce(t, group=group)
        return self

    def __repr__(self) -> str:
        return f"{type(self).__name__}(task_weights={self.task_weights.tolist()})"


class _ElementwiseMetric(EngineMetric):
    """MSE / MAE (`ChempropMetric.update`, metrics.py:78-123): f[0] = sum L w tw m, i[0] = sum m; RMSE takes the sqrt."""
    _kind = _lib.METRIC_SQERR
    _sqrt = False
    _bounded = False
    _n_f, _n_i = 1, 1

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        P, Y = self._inputs(preds, targets, mask, weights, lt_mask, gt_mask)
        b, T = Y.shape
        self._alloc(P.device, T)
        w, _ = _loss_weights(weights, None, b, T)
        lt, gt = ((None if m is None else m.to(torch.uint8).expand(b, T).contiguous()) for m in
                  ((lt_mask, gt_mask) if self._bounded else (None, None)))
        K.metric_accumulate(self._kind, P, Y, _mask_u8(Y, mask), w, self._tw(T, P.device), lt, gt, self._f, self._i,
                            self._status)

    def compute(self) -> Tensor:
        v = self._f[0] / self._i[0]
        return v.sqrt() if self._sqrt else v


class EngineMSEMetric(_ElementwiseMetric):
    alias = "mse"


class EngineMAEMetric(_ElementwiseMetric):
    alias = "mae"
    _kind = _lib.METRIC_ABSERR


class EngineRMSEMetric(_ElementwiseMetric):
    alias = "rmse"
    _sqrt = True


class EngineBoundedMSEMetric(EngineMSEMetric):
    alias = "bounded-mse"
    _bounded = True


class EngineBoundedMAEMetric(EngineMAEMetric):
    alias = "bounded-mae"
    _bounded = True


class EngineBoundedRMSEMetric(EngineRMSEMetric):
    alias = "bounded-rmse"
    _bounded = True


class EngineR2Metric(EngineMetric):
    """R2Score (metrics.py:184-199; torchmetrics' R2Score of preds[mask], targets[mask]): one score pooled over every task;
    weights and task weights are ignored, as in the reference.  Near-constant targets follow torchmetrics: 1 when the
    residual sum is also ~0, 0 otherwise (atol 1e-4); fewer than two values give NaN (torchmetrics raises)."""
    alias = "r2"
    higher_is_better = True
    _n_f, _n_i = 3, 1

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        P, Y = self._inputs(preds, targets, mask, weights, lt_mask, gt_mask)
        self._alloc(P.device, Y.shape[1])
        K.metric_accumulate(_lib.METRIC_R2, P, Y, _mask_u8(Y, mask), None, None, None, None, self._f, self._i, self._status)

    def compute(self) -> Tensor:
        s, s2, rss = self._f
        n = self._i[0].double()
        tss = s2 - s * (s / n)
        near0 = lambda x: x.abs() <= 1e-4                                           # noqa: E731 -- torch.isclose(x, 0, atol=1e-4)
        v = torch.where(near0(rss), torch.ones_like(rss), torch.where(near0(tss), torch.zeros_like(rss), 1 - rss / tss))
        return torch.where(n < 2, torch.full_like(v, float("nan")), v)


class _ConfusionMetric(EngineMetric):
    """torchmetrics' BinaryAccuracy / BinaryF1Score on preds[mask] (metrics.py:463-499): pooled counts at p > 0.5."""
    higher_is_better = True
    _n_i = 4

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        P, Y = self._inputs(preds, targets, mask, weights, lt_mask, gt_mask)
        self._alloc(P.device, Y.shape[1])
        K.metric_accumulate(_lib.METRIC_CONFUSION, P, Y, _mask_u8(Y, mask), None, None, None, None, None, self._i,
                            self._status)

    def _states(self) -> list[Tensor]:
        return [self._i, self._status]


def _safe_div(a: Tensor, b: Tensor) -> Tensor:
    """torchmetrics' _safe_divide: 0 where the denominator is 0."""
    return torch.where(b == 0, torch.zeros_like(a), a / torch.where(b == 0, torch.ones_like(b), b))


class EngineAccuracyMetric(_ConfusionMetric):
    alias = "accuracy"

    def compute(self) -> Tensor:
        tp, fp, tn, fn = self._i.double()
        return self._checked(_safe_div(tp + tn, tp + fp + tn + fn))


class EngineF1Metric(_ConfusionMetric):
    alias = "f1"

    def compute(self) -> Tensor:
        tp, fp, tn, fn = self._i.double()
        return self._checked(_safe_div(2 * tp, 2 * tp + fp + fn))


class EngineBinaryMCCMetric(EngineMetric):
    """BinaryMCCMetric (metrics.py:306-371): per-task soft TP / FP / TN / FN weighted by w m, mean of MCC * task weight."""
    alias = "binary-mcc"
    higher_is_better = True

    def _f_size(self, T: int) -> int:
        return 4 * T

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        P, Y = self._inputs(preds, targets, mask, weights, lt_mask, gt_mask)
        b, T = Y.shape
        self._alloc(P.device, T)
        w, _ = _loss_weights(weights, None, b, T)
        K.metric_accumulate(_lib.METRIC_SOFT_MCC, P, Y, _mask_u8(Y, mask), w, None, None, None, self._f, None,
                            self._status)

    def _states(self) -> list[Tensor]:
        return [self._f, self._status]

    def compute(self) -> Tensor:
        tp, fp, tn, fn = self._f.view(4, -1)
        mcc = (tp * tn - fp * fn) / ((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn) + 1e-8).sqrt()
        return self._checked((mcc * self._tw(self._T, mcc.device).double()).mean())


class EngineMulticlassMCCMetric(EngineMetric):
    """MulticlassMCCMetric (metrics.py:374-460) on b x T x C class probabilities (softmax of the update where any value lies
    outside [0, 1]): per task the sums p, t, c, s, weighted by w m; MCC per task, times the task weight, averaged."""
    alias = "multiclass-mcc"
    higher_is_better = True

    def _f_size(self, T: int) -> int:
        return T * (2 * self._C + 2)

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        K._require_cuda(preds, targets, mask, weights)
        if preds.dim() != 3 or preds.shape[:2] != targets.shape:
            raise ValueError(f"expected b x T x C predictions and b x T targets, got {tuple(preds.shape)} and "
                             f"{tuple(targets.shape)}")
        b, T, C_ = preds.shape
        if self._status is None:
            self._C = C_
        elif C_ != self._C:
            raise ValueError(f"{C_} classes after {self._C}")
        P, Y = preds.float().reshape(b, T * C_).contiguous(), targets.float().contiguous()
        self._alloc(P.device, T)
        w, _ = _loss_weights(weights, None, b, T)
        K.metric_multiclass_mcc(P, Y, _mask_u8(Y, mask), w, C_, self._f, self._status)

    def _states(self) -> list[Tensor]:
        return [self._f, self._status]

    def compute(self) -> Tensor:
        C_ = self._C
        st = self._f.view(self._T, 2 * C_ + 2)
        p, t, c, s = st[:, :C_], st[:, C_:2 * C_], st[:, 2 * C_], st[:, 2 * C_ + 1]
        s2 = s.square()
        cov_ytyp = c * s - (p * t).sum(1)
        cov_ypyp = s2 - (p * p).sum(1)
        cov_ytyt = s2 - (t * t).sum(1)
        x = cov_ypyp * cov_ytyt
        mcc = torch.where(x == 0, torch.zeros_like(x), cov_ytyp / x.sqrt())
        return self._checked((mcc * self._tw(self._T, mcc.device).double()).mean())


class _RankingMetric(EngineMetric):
    """torchmetrics' BinaryAUROC / BinaryPrecisionRecallCurve on preds[mask] (metrics.py:480-489): each update appends its
    formatted scores, labels and keep flags (dmpnn_metric_rank_format); `compute` concatenates them and sorts once
    (dmpnn_rank_curve).  One class absent: AUROC 0 (torchmetrics zeroes fpr or tpr); AUPRC as its formula gives it (NaN
    without positives, 1 without negatives)."""
    higher_is_better = True
    _out = 0

    def reset(self):
        super().reset()
        self._lists = ([], [], [])

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        P, Y = self._inputs(preds, targets, mask, weights, lt_mask, gt_mask)
        b, T = Y.shape
        if self._status is None:
            self._status = torch.zeros(1, dtype=torch.int32, device=P.device)
        score = torch.empty(b * T, dtype=torch.float32, device=P.device)
        label = torch.empty(b * T, dtype=torch.uint8, device=P.device)
        keep = torch.empty(b * T, dtype=torch.uint8, device=P.device)
        K.metric_rank_format(P, Y, _mask_u8(Y, mask), score, label, keep, self._status)
        for lst, x in zip(self._lists, (score, label, keep)):
            lst.append(x)

    def _cat(self):
        return [torch.cat(lst) if len(lst) != 1 else lst[0] for lst in self._lists]

    def compute(self) -> Tensor:
        score, label, keep = self._cat()
        out = torch.empty(2, dtype=torch.float64, device=score.device)
        K.rank_curve(score, label, keep, out)
        return self._checked(out[self._out])

    def _states(self) -> list[Tensor]:
        return [self._status]

    def sync_(self, group=None):
        """Sum the status flags and all-gather the formatted entries, each rank's padded to the largest rank's size (the
        padding is not kept)."""
        super().sync_(group)
        mine = self._cat()
        dev = mine[0].device
        n = torch.tensor([mine[0].numel()], dtype=torch.int64, device=dev)
        ns = [torch.zeros_like(n) for _ in range(dist.get_world_size(group))]
        dist.all_gather(ns, n, group=group)
        sizes = [int(x) for x in ns]
        top = max(sizes)
        gathered = []
        for x in mine:
            padded = torch.zeros(top, dtype=x.dtype, device=dev)
            padded[:x.numel()] = x
            parts = [torch.empty_like(padded) for _ in sizes]
            dist.all_gather(parts, padded, group=group)
            gathered.append([p[:k] for p, k in zip(parts, sizes)])
        self._lists = tuple(gathered)
        return self


class EngineAUROCMetric(_RankingMetric):
    alias = "roc"


class EngineAUPRCMetric(_RankingMetric):
    alias = "prc"
    _out = 1


class EngineCriterionMetric(EngineMetric):
    """Any engine criterion as the reference's validation-loss accumulator (`MPNN.metrics[-1]`, models/model.py:99-103,
    181): each update adds the criterion's batch value times the batch's mask count in f64 -- every engine criterion
    reduces a batch to sum L w tw m / sum m, so the sum is the reference's `total_loss` -- and `compute` divides by the
    total count.  For the RMSE criteria the value squared times the count is added, and `compute` takes the sqrt.  A criterion
    whose reference raises where its loss is NaN (`nan_error()` not None: EngineNLogProbEnrichment) sets the status flag on a
    NaN batch value, and `EngineMPNN.evaluate` raises the reference's error."""
    _n_f, _n_i = 1, 1

    def __init__(self, criterion):
        self.criterion = criterion
        self.alias = type(criterion).__name__
        self._rmse = isinstance(criterion, _RegressionCriterion) and criterion._kind == _lib.LOSS_RMSE
        super().__init__(criterion.task_weights)

    def update(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        # the criterion's kernel reads its task weights on the device: refuse a criterion left on the host before any launch
        K._require_cuda(preds, targets, self.criterion.task_weights)
        self._alloc(targets.device, targets.shape[1])
        bounds = (lt_mask, gt_mask) if self.criterion._bounded else ()
        with torch.no_grad():
            v = self.criterion(preds, targets, mask, weights, *bounds).double()
        m = targets.isfinite() if mask is None else mask & targets.isfinite()
        n = m.sum()
        self._f.add_((v * v if self._rmse else v) * n)
        self._i.add_(n)
        if self.criterion.nan_error() is not None:
            self._status.bitwise_or_(v.isnan().to(torch.int32))

    def _states(self) -> list[Tensor]:
        return [self._f, self._i, self._status]

    def compute(self) -> Tensor:
        v = self._f[0] / self._i[0]
        return v.sqrt() if self._rmse else v

    def __repr__(self) -> str:
        return f"EngineCriterionMetric({self.criterion!r})"


# chemprop's MetricRegistry names (metrics.py:133-499)
EngineMetricRegistry = {
    "mse": EngineMSEMetric,
    "mae": EngineMAEMetric,
    "rmse": EngineRMSEMetric,
    "bounded-mse": EngineBoundedMSEMetric,
    "bounded-mae": EngineBoundedMAEMetric,
    "bounded-rmse": EngineBoundedRMSEMetric,
    "r2": EngineR2Metric,
    "binary-mcc": EngineBinaryMCCMetric,
    "multiclass-mcc": EngineMulticlassMCCMetric,
    "roc": EngineAUROCMetric,
    "prc": EngineAUPRCMetric,
    "accuracy": EngineAccuracyMetric,
    "f1": EngineF1Metric,
}


def default_metric(predictor) -> EngineMetric:
    """The predictor's `_T_default_metric()` (chemprop/nn/predictors.py:164-348), built without arguments as the reference
    does: MSE for the regression family, AUROC for the binary predictors, multiclass MCC for the multiclass ones, SID for
    the spectral predictor."""
    from .head import (EngineBinaryClassificationFFN, EngineBinaryDirichletFFN, EngineMulticlassClassificationFFN,
                       EngineSID, EngineSpectralFFN)

    if isinstance(predictor, EngineSpectralFFN):          # its criterion's task weights live on the predictor's device
        return EngineCriterionMetric(EngineSID().to(predictor.criterion.task_weights.device))
    if isinstance(predictor, EngineMulticlassClassificationFFN):      # and its Dirichlet subclass
        return EngineMulticlassMCCMetric()
    if isinstance(predictor, (EngineBinaryClassificationFFN, EngineBinaryDirichletFFN)):
        return EngineAUROCMetric()
    return EngineMSEMetric()
