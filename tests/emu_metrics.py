"""TEST INFRASTRUCTURE ONLY.  torch-CPU emulations of the metric kernels behind engine.py's wrappers (csrc/metrics.cu),
written from their contracts in include/dmpnn.h, so that the host logic of chemprop_b200/nn/metrics.py and
`EngineMPNN.evaluate` runs without a GPU.  `patch_metrics(monkeypatch)` swaps the wrappers for these; the `-m gpu` tests
call the real kernels."""
from __future__ import annotations

import torch

from chemprop_b200 import _lib, engine


def _m(Y, mask):
    return Y.isfinite() if mask is None else mask.bool()


def _sig(P):
    return 1 / (1 + torch.exp(-P.float()))


def _out_of_unit(p) -> bool:
    return bool(p.numel()) and not bool(((p >= 0) & (p <= 1)).all())


def metric_accumulate(kind, P, Y, mask, w, tw, lt_mask, gt_mask, fstate, istate, status):
    B, T = Y.shape
    m = _m(Y, mask)
    P64, Y64 = P.double(), Y.double()
    if kind in (_lib.METRIC_SQERR, _lib.METRIC_ABSERR):
        e = P64 - Y64
        for bm, cmp in ((lt_mask, P < Y), (gt_mask, P > Y)):
            if bm is not None:
                e = torch.where(bm.bool() & cmp, torch.zeros_like(e), e)
        L = e * e if kind == _lib.METRIC_SQERR else e.abs()
        ww = (w.double().view(-1, 1) if w is not None else 1.0) * (tw.double().view(1, -1) if tw is not None else 1.0)
        fstate[0] += torch.where(m, L * ww, torch.zeros_like(L)).sum()
        istate[0] += m.sum()
        return
    if kind == _lib.METRIC_R2:
        y, p = Y64[m], P64[m]
        fstate[0:3] += torch.stack([y.sum(), (y * y).sum(), ((y - p) ** 2).sum()])
        istate[0] += m.sum()
        return
    lab = torch.trunc(Y64)
    if bool((m & (lab != 0) & (lab != 1)).any()):
        status[0] = 1
    if kind == _lib.METRIC_CONFUSION:
        p = P[m].float()
        p = _sig(p) if _out_of_unit(p) else p
        y = lab[m]
        hit = p > 0.5
        istate += torch.stack([(hit & (y == 1)).sum(), (hit & (y == 0)).sum(), (~hit & (y == 0)).sum(),
                               (~hit & (y == 1)).sum()])
        return
    p = (_sig(P) if _out_of_unit(P) else P.float()).double()
    wm = (w.double().view(-1, 1) if w is not None else 1.0) * m
    t = torch.where(m, lab, torch.zeros_like(lab))
    fstate += torch.stack([(t * p * wm).sum(0), ((1 - t) * p * wm).sum(0), ((1 - t) * (1 - p) * wm).sum(0),
                           (t * (1 - p) * wm).sum(0)]).reshape(-1)


def metric_multiclass_mcc(P, Y, mask, w, C, fstate, status):
    B, T = Y.shape
    p = P.float().view(B, T, C)
    p = torch.softmax(p, 2) if _out_of_unit(p) else p
    m = _m(Y, mask)
    t = torch.trunc(Y.double()).long()
    t = torch.where(t < 0, t + C, t)
    if bool((m & ((t < 0) | (t >= C))).any()):
        status[0] = 1
    t = torch.where(m & (t >= 0) & (t < C), t, torch.zeros_like(t))
    eye = torch.eye(C, dtype=torch.float64)
    wm = ((w.double().view(-1, 1) if w is not None else 1.0) * m)[..., None]
    bp, bt = eye[p.argmax(-1)], eye[t]
    sums = torch.cat([(bp * wm).sum(0), (bt * wm).sum(0), (bp * bt * wm).sum(2).sum(0)[:, None],
                      (p.double() * wm).sum(2).sum(0)[:, None]], 1)
    fstate += sums.reshape(-1)


def metric_rank_format(P, Y, mask, score, label, keep, status):
    m = _m(Y, mask)
    lab = torch.trunc(Y.double())
    if bool((m & (lab != 0) & (lab != 1)).any()):
        status[0] = 1
    sig = _out_of_unit(P[m])
    s = _sig(P) if sig else P.float()
    score.copy_(torch.where(m, s, torch.zeros_like(s)).reshape(-1))
    label.copy_(torch.where(m & (lab == 1), 1, 0).to(torch.uint8).reshape(-1))
    keep.copy_(m.to(torch.uint8).reshape(-1))


def rank_curve(score, label, keep, out):
    import numpy as np

    from oracle import metrics_np as O

    k = keep.bool()
    s, y = score[k].numpy(), label[k].numpy()
    if s.size == 0:
        out.copy_(torch.tensor([0.0, float("nan")], dtype=torch.float64))
        return
    with np.errstate(invalid="ignore", divide="ignore"):
        out.copy_(torch.tensor([O.auroc_from(s, y), O.auprc_from(s, y)], dtype=torch.float64))


def patch_metrics(monkeypatch):
    for name in ("metric_accumulate", "metric_multiclass_mcc", "metric_rank_format", "rank_curve"):
        monkeypatch.setattr(engine, name, globals()[name])
    monkeypatch.setattr(engine, "_require_cuda", lambda *ts: None)
