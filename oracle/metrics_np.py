"""TEST INFRASTRUCTURE ONLY.  A float64 numpy restatement of chemprop's validation / test metrics (chemprop/nn/metrics.py
:59-499) and of the torchmetrics definitions they wrap (R2Score, BinaryAccuracy, BinaryF1Score, BinaryAUROC,
BinaryPrecisionRecallCurve + auc), written out here because torchmetrics is not a dependency.

Each metric is a function of a list of updates, every update a dict with `preds` (b x T, or b x T x C), `targets` (b x T),
and optionally `mask` (b x T bool; default: everything), `weights` (b), `lt_mask` / `gt_mask`; `task_weights` is 1 or T
values.  Classification updates are formatted per update as torchmetrics does: where a considered prediction lies outside
[0, 1] (or is NaN) the update's predictions go through a float32 sigmoid (softmax for the multiclass MCC)."""
from __future__ import annotations

import numpy as np


def _f64(x):
    return np.asarray(x, dtype=np.float64)


def _parts(u, T=None):
    P, Y = np.asarray(u["preds"]), np.asarray(u["targets"], dtype=np.float32)
    b = Y.shape[0]
    m = np.ones(Y.shape, bool) if u.get("mask") is None else np.asarray(u["mask"], bool)
    w = np.ones(b) if u.get("weights") is None else _f64(u["weights"]).reshape(-1)
    return P, Y, m, w


def _tw(task_weights, T):
    tw = _f64(1.0 if task_weights is None else task_weights).reshape(-1)
    return np.broadcast_to(tw, (T,)) if tw.size == 1 else tw


def sigmoid32(x):
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(over="ignore"):
        return (np.float32(1) / (np.float32(1) + np.exp(-x))).astype(np.float32)


def softmax32(x):
    x = np.asarray(x, dtype=np.float32)
    e = np.exp(x - x.max(-1, keepdims=True))
    return (e / e.sum(-1, keepdims=True)).astype(np.float32)


def _out_of_unit(p) -> bool:
    p = np.asarray(p)
    return bool(p.size) and not bool(np.all((p >= 0) & (p <= 1)))


# ---- ChempropMetric family (metrics.py:78-181) ------------------------------------------------------------------------
def elementwise_sums(updates, kind: str, task_weights=None, bounded=False):
    """(sum L w tw m, sum m) over the updates; kind 'se' or 'ae'."""
    s, n = 0.0, 0
    for u in updates:
        P, Y, m, w = _parts(u)
        P, Y = _f64(P), _f64(Y)
        if bounded:
            lt = np.zeros(Y.shape, bool) if u.get("lt_mask") is None else np.asarray(u["lt_mask"], bool)
            gt = np.zeros(Y.shape, bool) if u.get("gt_mask") is None else np.asarray(u["gt_mask"], bool)
            P = np.where((P < Y) & lt, Y, P)
            P = np.where((P > Y) & gt, Y, P)
        e = P - Y
        L = e * e if kind == "se" else np.abs(e)
        L = np.where(m, L, 0.0) * w[:, None] * _tw(task_weights, Y.shape[1])[None, :]
        s += L.sum()
        n += int(m.sum())
    return s, n


def mse(updates, task_weights=None, bounded=False):
    s, n = elementwise_sums(updates, "se", task_weights, bounded)
    return s / n if n else np.nan


def mae(updates, task_weights=None, bounded=False):
    s, n = elementwise_sums(updates, "ae", task_weights, bounded)
    return s / n if n else np.nan


def rmse(updates, task_weights=None, bounded=False):
    return np.sqrt(mse(updates, task_weights, bounded))


def criterion_metric(values_and_counts, rmse_type=False):
    """The validation-loss accumulator from per-batch criterion values v_k and mask counts n_k."""
    s = sum((v * v if rmse_type else v) * n for v, n in values_and_counts)
    n = sum(n for _, n in values_and_counts)
    r = s / n
    return np.sqrt(r) if rmse_type else r


# ---- torchmetrics R2Score on preds[mask], targets[mask] (metrics.py:184-199) ---------------------------------------------
def r2(updates):
    s = s2 = rss = 0.0
    n = 0
    for u in updates:
        P, Y, m, _ = _parts(u)
        p, y = _f64(P)[m], _f64(Y)[m]
        s += y.sum()
        s2 += (y * y).sum()
        rss += ((y - p) ** 2).sum()
        n += y.size
    if n < 2:
        return np.nan
    tss = s2 - s * (s / n)
    if abs(rss) <= 1e-4:
        return 1.0
    if abs(tss) <= 1e-4:
        return 0.0
    return 1 - rss / tss


# ---- binary classification on preds[mask] (ClassificationMixin, metrics.py:463-499) --------------------------------------
def binary_formatted(updates):
    """Concatenated (scores, labels) of the masked-in entries, each update formatted on its own."""
    ss, ls = [], []
    for u in updates:
        P, Y, m, _ = _parts(u)
        p = np.asarray(P, dtype=np.float32)[m]
        y = np.trunc(Y[m]).astype(np.int64)
        if np.any((y != 0) & (y != 1)):
            raise ValueError("binary targets must be 0 or 1")
        ss.append(sigmoid32(p) if _out_of_unit(p) else p)
        ls.append(y)
    return np.concatenate(ss) if ss else np.zeros(0, np.float32), np.concatenate(ls) if ls else np.zeros(0, np.int64)


def confusion(updates):
    s, y = binary_formatted(updates)
    hit = s > np.float32(0.5)
    return int((hit & (y == 1)).sum()), int((hit & (y == 0)).sum()), int((~hit & (y == 0)).sum()), int((~hit & (y == 1)).sum())


def accuracy(updates):
    tp, fp, tn, fn = confusion(updates)
    d = tp + fp + tn + fn
    return (tp + tn) / d if d else 0.0


def f1(updates):
    tp, fp, tn, fn = confusion(updates)
    d = 2 * tp + fp + fn
    return 2 * tp / d if d else 0.0


def clf_curve(scores, labels):
    """torchmetrics' _binary_clf_curve: (fps, tps) at each distinct score, scores descending."""
    s = _f64(scores)
    order = np.argsort(-s, kind="stable")
    s, y = s[order], _f64(labels)[order]
    ends = np.r_[np.nonzero(np.diff(s))[0], s.size - 1]
    tps = np.cumsum(y)[ends]
    fps = 1 + ends - tps
    return fps, tps


def auroc_from(scores, labels):
    if np.size(scores) == 0:          # no pair (torchmetrics raises): 0, as the engine
        return 0.0
    fps, tps = clf_curve(scores, labels)
    fps, tps = np.r_[0.0, fps], np.r_[0.0, tps]
    fpr = np.zeros_like(fps) if fps[-1] <= 0 else fps / fps[-1]
    tpr = np.zeros_like(tps) if tps[-1] <= 0 else tps / tps[-1]
    return float(np.sum(np.diff(fpr) * (tpr[1:] + tpr[:-1]) / 2))


def auprc_from(scores, labels):
    if np.size(scores) == 0:          # no pair: NaN, as without positives
        return float("nan")
    fps, tps = clf_curve(scores, labels)
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = tps / (tps + fps)
        recall = tps / tps[-1]
    precision = np.r_[precision[::-1], 1.0]
    recall = np.r_[recall[::-1], 0.0]
    # torchmetrics.utilities.compute.auc: recall decreases, so the area is -trapz(precision, recall)
    return float(-np.sum(np.diff(recall) * (precision[1:] + precision[:-1]) / 2))


def auroc(updates):
    return auroc_from(*binary_formatted(updates))


def auprc(updates):
    return auprc_from(*binary_formatted(updates))


# ---- soft MCCs (metrics.py:306-460) ------------------------------------------------------------------------------------
def binary_mcc(updates, task_weights=None):
    acc = None
    for u in updates:
        P, Y, m, w = _parts(u)
        p = np.asarray(P, dtype=np.float32)
        p = _f64(sigmoid32(p) if _out_of_unit(p) else p)
        t = np.trunc(_f64(Y))
        wm = w[:, None] * m
        c = np.stack([(t * p * wm).sum(0), ((1 - t) * p * wm).sum(0), ((1 - t) * (1 - p) * wm).sum(0),
                      (t * (1 - p) * wm).sum(0)])
        acc = c if acc is None else acc + c
    tp, fp, tn, fn = acc
    mcc = (tp * tn - fp * fn) / np.sqrt((tp + fp) * (tp + fn) * (tn + fp) * (tn + fn) + 1e-8)
    return float(np.mean(mcc * _tw(task_weights, tp.size)))


def multiclass_mcc_sums(updates):
    acc = None
    for u in updates:
        P, Y, m, w = _parts(u)
        p = np.asarray(P, dtype=np.float32)
        p = softmax32(p) if _out_of_unit(p) else p
        C = p.shape[2]
        t = np.trunc(_f64(Y)).astype(np.int64)
        eye = np.eye(C)
        bin_t = eye[np.where(m, t, 0)]
        bin_p = eye[p.argmax(-1)]
        wm = (w[:, None] * m)[..., None]
        sums = (np.concatenate([(bin_p * wm).sum(0), (bin_t * wm).sum(0)], 1),
                (bin_p * bin_t * wm).sum(2).sum(0), (_f64(p) * wm).sum(2).sum(0))
        acc = sums if acc is None else tuple(a + b for a, b in zip(acc, sums))
    return acc


def multiclass_mcc(updates, task_weights=None):
    pt, c, s = multiclass_mcc_sums(updates)
    C = pt.shape[1] // 2
    p, t = pt[:, :C], pt[:, C:]
    cov_ytyp = c * s - (p * t).sum(1)
    cov_ypyp = s * s - (p * p).sum(1)
    cov_ytyt = s * s - (t * t).sum(1)
    x = cov_ypyp * cov_ytyt
    with np.errstate(invalid="ignore", divide="ignore"):
        mcc = np.where(x == 0, 0.0, cov_ytyp / np.sqrt(x))
    return float(np.mean(mcc * _tw(task_weights, c.size)))


METRICS = {
    "mse": mse, "mae": mae, "rmse": rmse,
    "bounded-mse": lambda us, tw=None: mse(us, tw, True), "bounded-mae": lambda us, tw=None: mae(us, tw, True),
    "bounded-rmse": lambda us, tw=None: rmse(us, tw, True),
    "r2": lambda us, tw=None: r2(us), "binary-mcc": binary_mcc, "multiclass-mcc": multiclass_mcc,
    "roc": lambda us, tw=None: auroc(us), "prc": lambda us, tw=None: auprc(us),
    "accuracy": lambda us, tw=None: accuracy(us), "f1": lambda us, tw=None: f1(us),
}
