"""GPU tier: EngineMolAtomBondMPNN and csrc/row_head.cu on the device.

- The training-step fixtures of tools/make_golden_mab_model.py (the reference's own `MolAtomBondMPNN.training_step`) with
  fp32 and bf16 MAB encoders, eagerly and, without constraints, as one CUDA graph whose replay is bit-identical to the
  eager step; the trained checkpoints in eval mode.
- dmpnn_{regression,bce,ce}_loss_rows against float64 torch, within bounds derived from their summation order, at R in
  {0, 1, 1023, 1025, 249 k, 1.1 M} rows; every target masked, bounded masks, repeated launches bit-identical, and
  agreement with the single-block kernels.
- dmpnn_edge_pair_mean exact, NaN rows on shuffled edge pairs.
- Poisoned allocations: NaN or 1e30 in every buffer the new entry points write or use as workspace gives identical bits."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_mab_model_host import (CKPT_CASES, TRAIN_CASES, assert_constraints_met, check_checkpoint, check_training,
                                       patch_mab_model, ref_edge_pair_mean, run_step)
from tests.test_spectral_host import ref_regression_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24
LOSS_MSE, LOSS_MAE, LOSS_RMSE = range(3)


@pytest.mark.parametrize("case", TRAIN_CASES)
def test_training_fixture_eager_and_graph_fp32_encoder(case):
    _, bmg, predss, cons = check_training(case, DEV, "fp32", graph=case != "constrained")
    if cons is not None:
        assert_constraints_met(bmg, predss, cons)


@pytest.mark.parametrize("case", TRAIN_CASES)
def test_training_fixture_eager_and_graph_bf16_encoder(case, monkeypatch):
    """The bf16 encoder keeps 8 mantissa bits through the depth loop and its mirror, which the fixtures' 32-wide layers and
    per-batch normalisation amplify beyond a useful bound against the reference.  So the whole step (loss, every gradient,
    running statistics, eval predictions) is checked against the same step through the rounding-aware emulation of the
    bf16 tier (tests/emu_mab.py) within 2 % of each tensor's scale, as tests/test_gpu_mab_bf16.py does; the head after the
    encoder is f32 either way.  Eager and graph replay stay bit-identical."""
    with monkeypatch.context() as m:
        patch_mab_model(m)
        expect = run_step(case, "cpu", "bf16")
    _, bmg, predss, cons = check_training(case, DEV, "bf16", rtol=2e-2, graph=case != "constrained", scaled=True,
                                          expect=expect)
    if cons is not None:
        assert_constraints_met(bmg, predss, cons)


@pytest.mark.parametrize("name", CKPT_CASES)
def test_checkpoint_predicts_as_the_reference(name):
    _, bmg, predss, cons = check_checkpoint(name, DEV)
    if cons is not None:
        assert_constraints_met(bmg, predss, cons, atol=2e-4)


# ---- the _rows criteria against float64 ------------------------------------------------------------------------------------
def _inputs(R, T, C=1, kind="reg", seed=0, all_masked=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    P = torch.randn(R, T * C, device=DEV, generator=g) * 2
    if kind == "reg":
        Y = torch.randn(R, T, device=DEV, generator=g)
    elif kind == "bce":
        Y = torch.rand(R, T, device=DEV, generator=g)
    else:
        Y = torch.randint(0, C, (R, T), device=DEV, generator=g).float()
    Y = torch.where(torch.rand(R, T, device=DEV, generator=g) < 0.1, torch.full_like(Y, float("nan")), Y)
    if all_masked:
        Y = torch.full_like(Y, float("nan"))
    w = torch.rand(R, device=DEV, generator=g) + 0.5
    tw = torch.rand(T, device=DEV, generator=g) + 0.5
    return P, Y, w, tw


def _ref64(kind, P, Y, w, tw, C=1, loss_kind=LOSS_MSE, lt=None, gt=None):
    """loss, dP and sum |terms| / n (the magnitude the summation bound scales) in float64."""
    P64, Y64, w64, tw64 = P.double(), Y.double(), w.double(), tw.double()
    m = torch.isfinite(Y64)
    n = max(int(m.sum()), 1)
    if kind == "reg":
        loss, g = ref_regression_loss(loss_kind, P64, Y64, w64, tw64, lt, gt)
        y = torch.where(m, Y64, torch.zeros_like(Y64))
        e = P64 - y
        if lt is not None:
            e = torch.where(lt & (P64 < y), torch.zeros_like(e), e)
        if gt is not None:
            e = torch.where(gt & (P64 > y), torch.zeros_like(e), e)
        terms = e.abs() if loss_kind == LOSS_MAE else e * e
    else:
        with torch.enable_grad():
            Pl = P64.clone().requires_grad_(True)
            y = torch.where(m, Y64, torch.zeros_like(Y64))
            if kind == "bce":
                terms = F.binary_cross_entropy_with_logits(Pl, y, reduction="none")
            else:
                X = Pl.view(P.shape[0], P.shape[1] // C, C)
                terms = torch.logsumexp(X, -1) - X.gather(-1, y.long()[..., None])[..., 0]
            ww = w64.view(-1, 1) * tw64.view(1, -1)
            loss = torch.where(m, terms * ww, torch.zeros_like(terms)).sum() / n
            (g,) = torch.autograd.grad(loss, Pl) if P.numel() else (torch.zeros_like(Pl),)
        terms = terms.detach()
    ww = w64.view(-1, 1) * tw64.view(1, -1)
    mag = float(torch.where(m, (terms * ww).abs(), torch.zeros_like(terms)).sum()) / n
    return float(loss), g.detach(), mag


def _depth(n, single_block=False):
    """Summands on the longest path of the reduction (serial per-thread run, shuffle tree, warp partials; for the _rows
    kernels twice, the second pass over the per-CTA partials), plus a few roundings of each term and of the division."""
    if single_block:
        return -(-n // 1024) + 5 + 32 + 8
    G = max(1, min(1024, -(-n // 2048)))
    chunk = max(1, -(-n // G))
    return -(-chunk // 256) + -(-G // 256) + 2 * (5 + 8) + 8


def _call(kind, P, Y, w, tw, C=1, loss_kind=LOSS_MSE, lt=None, gt=None, rows=True, dP=None):
    from chemprop_b200 import engine

    loss = torch.empty(1, device=DEV)
    dP = torch.empty_like(P) if dP is None else dP
    lt8 = None if lt is None else lt.to(torch.uint8).contiguous()
    gt8 = None if gt is None else gt.to(torch.uint8).contiguous()
    if kind == "reg":
        (engine.regression_loss_rows(P, Y, w, tw, lt8, gt8, loss_kind, loss, dP) if rows
         else engine.regression_loss(P, Y, w, tw, lt8, gt8, loss_kind, loss, dP))
    elif kind == "bce":
        (engine.bce_loss_rows if rows else engine.bce_loss)(P, Y, w, tw, loss, dP)
    else:
        (engine.ce_loss_rows if rows else engine.ce_loss)(P, Y, w, tw, C, loss, dP)
    return loss, dP


def _check(kind, R, T, C=1, loss_kind=LOSS_MSE, bounded=False, all_masked=False):
    P, Y, w, tw = _inputs(R, T, C, kind, seed=R + 7 * T + C, all_masked=all_masked)
    lt = gt = None
    if bounded:
        sel = torch.rand(R, T, device=DEV)
        lt, gt = sel < 0.35, sel > 0.65
    loss, dP = _call(kind, P, Y, w, tw, C, loss_kind, lt, gt)
    ref, g, mag = _ref64(kind, P, Y, w, tw, C, loss_kind, lt, gt)
    n = R * T
    rmse = loss_kind == LOSS_RMSE and kind == "reg"
    bound, bound_one = (_depth(n, one) * EPS * mag + 1e-30 for one in (False, True))
    if rmse:
        bound, bound_one = (b / max(2 * ref, 1e-30) + 2 * EPS * ref for b in (bound, bound_one))
    assert abs(float(loss) - ref) <= bound, (kind, R, T, C, float(loss), ref, bound)
    if R == 0:
        assert float(loss) == 0.0
        return
    if all_masked:
        assert float(loss) == 0.0 and not dP.any()
        return
    # dP is elementwise: a few roundings of the term's derivative, 1 / n rounded once, RMSE's 1 / (2 loss) carrying the
    # loss's relative error
    rel = 16 * EPS + (bound / max(ref, 1e-30) if rmse else 0.0)
    tol = rel * g.abs() + 8 * EPS * float(g.abs().max()) + 1e-30
    assert bool(((dP.double() - g).abs() <= tol).all()), (kind, R, T, C, float((dP.double() - g).abs().max()))
    loss2, dP2 = _call(kind, P, Y, w, tw, C, loss_kind, lt, gt)
    assert torch.equal(loss, loss2) and torch.equal(dP, dP2), "repeated launches differ"
    one, dP1 = _call(kind, P, Y, w, tw, C, loss_kind, lt, gt, rows=False)
    assert abs(float(one) - ref) <= bound_one and abs(float(one) - float(loss)) <= bound + bound_one, (float(one), float(loss))
    rel_one = 16 * EPS + (bound_one / max(ref, 1e-30) if rmse else 0.0)
    assert bool(((dP1.double() - dP.double()).abs() <= tol + rel_one * g.abs() + 8 * EPS * float(g.abs().max())).all())


ROWS = (0, 1, 1023, 1025, 249_000, 1_100_000)


@pytest.mark.parametrize("R", ROWS)
@pytest.mark.parametrize("T", (1, 12))
@pytest.mark.parametrize("loss_kind", (LOSS_MSE, LOSS_MAE, LOSS_RMSE))
def test_regression_loss_rows_against_float64(R, T, loss_kind):
    _check("reg", R, T, loss_kind=loss_kind)


@pytest.mark.parametrize("R", (1025, 249_000))
@pytest.mark.parametrize("loss_kind", (LOSS_MSE, LOSS_MAE, LOSS_RMSE))
def test_bounded_regression_loss_rows_against_float64(R, loss_kind):
    _check("reg", R, 12, loss_kind=loss_kind, bounded=True)


@pytest.mark.parametrize("R", ROWS)
@pytest.mark.parametrize("T", (1, 12))
def test_bce_loss_rows_against_float64(R, T):
    _check("bce", R, T)


@pytest.mark.parametrize("R", ROWS)
@pytest.mark.parametrize("T", (1, 12))
@pytest.mark.parametrize("C", (2, 10))
def test_ce_loss_rows_against_float64(R, T, C):
    _check("ce", R, T, C)


@pytest.mark.parametrize("kind", ("reg", "bce", "ce"))
def test_rows_criteria_with_every_target_masked(kind):
    _check(kind, 5000, 3, C=4 if kind == "ce" else 1, all_masked=True)


def test_ce_loss_rows_marks_out_of_range_labels():
    P, Y, w, tw = _inputs(3000, 2, 4, "ce", seed=3)
    Y[1500, 1] = 4.0
    loss, dP = _call("ce", P, Y, w, tw, 4)
    assert torch.isnan(loss).all() and torch.isnan(dP[1500, 4:8]).all() and torch.isfinite(dP[:1500]).all()


# ---- the pair mean ---------------------------------------------------------------------------------------------------------
def test_edge_pair_mean_is_exact_and_nan_on_shuffled_pairs():
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn.mol_atom_bond_model import EdgePairMeanFunction

    bmg = BatchMolGraph(make_molecules(300, seed=3, mean_atoms=12))
    bmg.to(DEV)
    rev = bmg.rev_edge_index.to(torch.int32)
    E = rev.shape[0]
    P = (torch.randn(E, 5, device=DEV) * 1e3).requires_grad_(True)
    out = EdgePairMeanFunction.apply(P, rev)
    assert torch.equal(out, (P[::2] + P[1::2]) / 2)
    G = torch.randn_like(out)
    out.backward(G)
    assert torch.equal(P.grad[::2], G / 2) and torch.equal(P.grad[1::2], G / 2)
    sbmg = BatchMolGraph(make_molecules(300, seed=3, mean_atoms=12, shuffle_edges=True))
    sbmg.to(DEV)
    srev = sbmg.rev_edge_index.to(torch.int32)
    Es = srev.shape[0]
    bad = srev[0::2].long() != torch.arange(1, Es, 2, device=DEV)
    assert bool(bad.any())
    Ps = torch.randn(Es, 5, device=DEV)
    got = EdgePairMeanFunction.apply(Ps, srev)
    want = ref_edge_pair_mean(Ps, srev)
    assert torch.isnan(got[bad]).all() and torch.equal(got[~bad], want[~bad])


# ---- poisoned allocations --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ("reg", "bce", "ce", "pair"))
def test_poisoned_buffers_give_identical_bits(kind, monkeypatch):
    from chemprop_b200 import engine

    results = []
    Pp = torch.randn(4000, 3, device=DEV)
    for poison in (float("nan"), 1e30):
        real = engine._rows_workspace

        def poisoned(fn, B, T, dev, _real=real, _p=poison):
            ws = _real(fn, B, T, dev)
            ws.view(-1)[: ws.numel() // 4 * 4].view(torch.float32).fill_(_p)
            return ws

        monkeypatch.setattr(engine, "_rows_workspace", poisoned)
        if kind == "pair":
            P = Pp
            rev = torch.arange(4000, device=DEV, dtype=torch.int32) ^ 1
            out = torch.full((2000, 3), poison, device=DEV)
            engine.edge_pair_mean(P, rev, out)
            dP = torch.full((4000, 3), poison, device=DEV)
            engine.edge_pair_mean_bwd(out, dP)
            results.append((out.clone(), dP.clone()))
        else:
            C = 3 if kind == "ce" else 1
            P, Y, w, tw = _inputs(70_000, 2, C, kind, seed=11)
            loss, dP = _call(kind, P, Y, w, tw, C, dP=torch.full_like(P, poison))
            results.append((loss.clone(), dP.clone()))
        monkeypatch.setattr(engine, "_rows_workspace", real)
    for a, b in zip(*results):
        assert torch.equal(a, b)
