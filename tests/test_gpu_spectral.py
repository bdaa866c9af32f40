"""GPU tier: the spectral predictor and the regression-loss family on the H100 kernels (csrc/head.cu:
dmpnn_spectral_transform(_bwd), dmpnn_sid_loss, dmpnn_wasserstein_loss, dmpnn_regression_loss) -- the reference's own
training step (tests/golden/fixture_mpnn_<kind>.npz) eager and as one CUDA graph, each kernel against f64 torch running the
reference formulas with autograd, bitwise repeatability of the multi-block reductions at b = 10 000 x T = 1 801, a bf16
encoder with EngineSpectralFFN at T = 1 801, and the poisoned-allocation differential.

Bounds.  u = 2^-24, depth = T / 256 + 16 (the length of a row's fixed-order sum or scan chunk chain plus the 8-warp tree).
Each element is held to (kappa + depth) u M with kappa = 64 and M the f64 sum of the magnitudes of what enters it:
  - transform: M = out (softplus); exp(exp(x)) carries x's relative error times e^x, so M = out (1 + e^x) for exp;
  - SID: a_j = W_j (|log(pn/t)| + 1 + t/pn) / n, M_j = (a_j + m_j sum_i a_i pn_i) / S;
  - Wasserstein: M_k = (Gm_k + m_k sum_i Gm_i pn_i) / S with Gm_k = sum_{j >= k} W_j / n.  The cumsums carry about
    (kappa + depth) u (Ct + Cp); where |D_j| is within that ("near" a tie) f32 does not determine the sign, and both
    choices are allowed: on top of the rounding bound, (Gt_k + m_k sum_i Gt_i pn_i) / S with
    Gt_k = sum_{j >= k} 2 W_j near_j / n (one sign flip moves G_k by 2 W_j / n for every k <= j).
The loss is held to (kappa + depth) u sum_j W_j M_j / n with M_j the magnitudes of the loss term's parts."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from tests.test_spectral_host import (KINDS, LOSS_MAE, LOSS_MSE, LOSS_RMSE, SPEC_EXP, SPEC_SOFTPLUS,
                                      check_spectral_head, ref_regression_loss, ref_spectral, ref_spectral_loss)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
KAPPA = 64.0


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind", KINDS)
def test_engine_mpnn_matches_reference_training_step(kind, graph):
    check_spectral_head(kind, "cuda", graph=graph)


# ---- the kernels against f64 torch ------------------------------------------------------------------------------------------
def _depth(T):
    return T / 256 + 16


def _raw(B, T, act, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if act == SPEC_EXP:
        X = (torch.randn(B, T, device="cuda", generator=g) * 1.2).clamp(-6, 2.5)
    else:
        X = torch.randn(B, T, device="cuda", generator=g) * 3
        pick = torch.rand(B, T, device="cuda", generator=g)
        X = torch.where(pick < 0.03, torch.full_like(X, -30.0), X)                # softplus(softplus(x)) ~ 1e-13
        X = torch.where(pick > 0.97, torch.rand(B, T, device="cuda", generator=g) * 40, X)   # past the threshold of 20
    return X, g


def _spectra(B, T, g):
    """Positive normalised target spectra with about 10 % masked bins."""
    Y = torch.rand(B, T, device="cuda", generator=g) + 0.05
    Y = Y / Y.sum(1, keepdim=True)
    Y[torch.rand(B, T, device="cuda", generator=g) < 0.1] = float("nan")
    return Y


SHAPES = [(1, 1), (7, 2), (64, 37), (10000, 1801), (300, 4001)]


@pytest.mark.parametrize("act", [SPEC_SOFTPLUS, SPEC_EXP], ids=["softplus", "exp"])
@pytest.mark.parametrize("B,T", SHAPES)
def test_spectral_transform_and_mirror_vs_f64(B, T, act):
    from chemprop_b200 import engine as K

    X, g = _raw(B, T, act, seed=B + 3 * T + act)
    out = torch.empty_like(X)
    K.spectral_transform(X, act, out)
    X64 = X.double().requires_grad_(True)
    ref = ref_spectral(X64, act)
    amp = (1 + X.double().exp()) if act == SPEC_EXP else 1.0
    assert bool(((out.double() - ref.detach()).abs() <= (KAPPA + _depth(T)) * U * ref.detach() * amp).all())
    if T == 1:
        assert bool((out == 1).all())
    G = torch.randn(B, T, device="cuda", generator=g)
    dX = torch.empty_like(X)
    K.spectral_transform_bwd(X, G, act, dX)
    (dref,) = torch.autograd.grad(ref, X64, G.double())
    with torch.no_grad():
        sp = torch.nn.functional.softplus
        y = torch.exp(torch.exp(X64)) if act == SPEC_EXP else sp(sp(X64))
        S = y.sum(1, keepdim=True)
        o = y / S
        a2 = (y * X64.exp()) if act == SPEC_EXP else (torch.sigmoid(sp(X64)) * torch.sigmoid(X64))
        mag = (G.double().abs() + (G.double().abs() * o).sum(1, keepdim=True)) / S * a2 * amp
    err = (dX.double() - dref).abs()
    assert bool((err <= (KAPPA + _depth(T)) * U * mag).all()), float((err / mag.clamp(min=1e-300)).max())
    out2, dX2 = torch.empty_like(X), torch.empty_like(X)
    K.spectral_transform(X, act, out2)
    K.spectral_transform_bwd(X, G, act, dX2)
    assert torch.equal(out, out2) and torch.equal(dX, dX2)


def _loss_kernel(kind, P, Y, w, tw, thr):
    from chemprop_b200 import engine as K

    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    (K.sid_loss if kind == "sid" else K.wasserstein_loss)(P, Y, w, tw, thr, loss, dP)
    return loss, dP


def _spectral_bounds(kind, P, Y, w, tw, thr):
    """Per-entry dP bound and loss bound (module docstring) from f64 quantities at the kernel's own P."""
    B, T = P.shape
    m = torch.isfinite(Y)
    live = m.any(1, keepdim=True)
    P64 = P.double()
    c = P64 if thr is None else P64.clamp(min=thr)
    S = torch.where(live, (c * m).sum(1, keepdim=True), torch.ones_like(c[:, :1]))
    pn = c / S
    t = torch.where(m, Y, torch.zeros_like(Y)).double()
    n = max(int(m.sum()), 1)
    W = (w.double().view(-1, 1) * tw.double().view(1, -1)) * m * live / n
    k = KAPPA + _depth(T)
    if kind == "sid":
        ts = torch.where(m, t, torch.ones_like(t))
        lr = (pn / ts).log().abs()
        a = W * (lr + 1 + ts / pn)
        mag = (a + m * (a * pn).sum(1, keepdim=True)) / S
        Lm = W * (pn * lr + ts * lr + pn + ts)
    else:
        Ct, Cp = t.cumsum(1), pn.cumsum(1)
        D = Ct - Cp
        near = D.abs() <= k * U * (Ct + Cp)
        Gm = W.flip(1).cumsum(1).flip(1)
        Gt = (2 * W * near).flip(1).cumsum(1).flip(1)                   # a flipped sign at a near tie, not scaled by u
        mag = (Gm + m * (Gm * pn).sum(1, keepdim=True)) / S
        tie = (Gt + m * (Gt * pn).sum(1, keepdim=True)) / S
        Lm = W * (D.abs() + Ct + Cp)
        return k * U * mag + tie, k * U * float(Lm.nan_to_num().sum())
    return k * U * mag, k * U * float(Lm.nan_to_num().sum())


def _spectral_case(B, T, seed, thr_frac=0.5):
    """Normalised predictions (the transform's output) and targets; threshold at the thr_frac quantile of a row, with
    about 5 % of the predictions set exactly to it."""
    from chemprop_b200 import engine as K

    X, g = _raw(B, T, SPEC_SOFTPLUS, seed)
    P = torch.empty_like(X)
    K.spectral_transform(X, SPEC_SOFTPLUS, P)
    thr = float(P[0].float().quantile(thr_frac)) if T > 1 else float(P[0, 0])
    P = torch.where(torch.rand(B, T, device="cuda", generator=g) < 0.05, torch.full_like(P, thr), P)
    Y = _spectra(B, T, g)
    if B > 3:
        Y[2] = float("nan")                                                       # a fully masked row
    w = torch.rand(B, device="cuda", generator=g) * 1.5 + 0.5
    tw = torch.rand(T, device="cuda", generator=g) * 1.5 + 0.5
    return P, Y, w, tw, thr


@pytest.mark.parametrize("threshold", [True, False], ids=["threshold", "no_threshold"])
@pytest.mark.parametrize("kind", ["sid", "wasserstein"])
@pytest.mark.parametrize("B,T", SHAPES)
def test_spectral_loss_vs_f64(kind, B, T, threshold):
    P, Y, w, tw, thr = _spectral_case(B, T, seed=7 * B + T)
    thr = thr if threshold else None
    loss, dP = _loss_kernel(kind, P, Y, w, tw, thr)
    ref_l, ref_g = ref_spectral_loss(kind, P.double(), Y, w.double(), tw.double(), thr)
    bound, lbound = _spectral_bounds(kind, P, Y, w, tw, thr)
    err = (dP.double() - ref_g).abs()
    assert bool((err <= bound + 1e-300).all()), float((err / bound.clamp(min=1e-300)).max())
    assert abs(float(loss) - float(ref_l)) <= lbound, (float(loss), float(ref_l), lbound)
    if B > 3:
        assert not bool(dP[2].ne(0).any())                                       # the fully masked row
    if kind == "sid":
        assert not bool(dP[~torch.isfinite(Y)].ne(0).any())
    loss2, dP2 = _loss_kernel(kind, P, Y, w, tw, thr)
    assert torch.equal(loss, loss2) and torch.equal(dP, dP2)


def test_clamp_passes_the_gradient_at_the_threshold_as_torch_does():
    """torch.clamp(min=) passes the gradient where the input equals the bound; the kernels do the same."""
    x = torch.tensor([0.5, 1.0, 2.0], dtype=torch.float64, requires_grad=True)
    (gx,) = torch.autograd.grad(x.clamp(min=1.0).sum(), x)
    assert gx.tolist() == [0.0, 1.0, 1.0]
    P = torch.tensor([[0.25, 0.5, 0.25, 0.125]], device="cuda")
    Y = torch.tensor([[0.25, 0.25, 0.25, 0.25]], device="cuda")
    w, tw = torch.ones(1, device="cuda"), torch.ones(4, device="cuda")
    for kind in ("sid", "wasserstein"):
        _, dP = _loss_kernel(kind, P, Y, w, tw, 0.25)
        _, ref = ref_spectral_loss(kind, P.double(), Y, w.double(), tw.double(), 0.25)
        assert float(dP[0, 3]) == 0.0 and float(ref[0, 3]) == 0.0               # clamped: no gradient
        assert float(ref[0, 0]) != 0.0 and abs(float(dP[0, 0]) - float(ref[0, 0])) <= 1e-5 * abs(float(ref[0, 0]))


def test_wasserstein_cumsum_ties_have_zero_subgradient():
    """Exact ties of the two cumsums (dyadic values, exact in f32): d|D|/dD = 0 there, as torch's abs; taking sign +1 at a
    tie instead is caught."""
    P = torch.tensor([[2.0, 1.0, 1.0], [1.0, 1.0, 2.0]], device="cuda")
    Y = torch.tensor([[0.5, 0.125, 0.375], [0.25, 0.25, 0.5]], device="cuda")     # row 0: ties at bins 0, 2; row 1: all
    w, tw = torch.tensor([1.0, 0.5], device="cuda"), torch.tensor([1.0, 2.0, 0.5], device="cuda")
    loss, dP = _loss_kernel("wasserstein", P, Y, w, tw, None)
    ref_l, ref = ref_spectral_loss("wasserstein", P.double(), Y, w.double(), tw.double(), None)
    torch.testing.assert_close(dP.double(), ref, rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(loss.double().reshape(()), ref_l, rtol=1e-6, atol=1e-7)
    assert not bool(dP[1].ne(0).any()) and float(loss) == pytest.approx(0.125 * 2 / 6, rel=1e-6)
    # sign(0) = +1 at row 0's first tie would add -W_0 to G_0 and change dP[0] by more than the bound
    one_sided = ref.clone()
    one_sided[0, 0] -= 1.0 * 1.0 / 6 / 4 * (1 - 0.5)
    assert float((dP.double() - one_sided).abs().max()) > 1e-3


def test_spectral_degenerate_cases_follow_the_stated_conventions():
    w, tw = torch.ones(3, device="cuda"), torch.ones(4, device="cuda")
    P = torch.tensor([[0.1, 0.2, 0.3, 0.4], [0.25, 0.25, 0.25, 0.25], [0.4, 0.3, 0.2, 0.1]], device="cuda")
    nan = float("nan")
    # every bin of every row masked: loss 0, dP 0
    for kind in ("sid", "wasserstein"):
        loss, dP = _loss_kernel(kind, P, torch.full_like(P, nan), w, tw, None)
        assert float(loss) == 0.0 and not bool(dP.ne(0).any())
        E = torch.empty(0, 4, device="cuda")
        assert float(_loss_kernel(kind, E, E, None, None, None)[0]) == 0.0
    # SID with a masked-in target of exactly 0: loss NaN, that row's masked-in dP NaN, its masked bins 0, other rows finite
    Y = torch.tensor([[0.25, 0.25, 0.25, 0.25], [0.0, 0.5, nan, 0.5], [0.1, 0.2, 0.3, 0.4]], device="cuda")
    loss, dP = _loss_kernel("sid", P, Y, w, tw, None)
    assert bool(torch.isnan(loss).all())
    assert bool(torch.isnan(dP[1, [0, 1, 3]]).all()) and float(dP[1, 2]) == 0.0
    assert bool(torch.isfinite(dP[[0, 2]]).all())


@pytest.mark.parametrize("kind", [LOSS_MSE, LOSS_MAE, LOSS_RMSE], ids=["mse", "mae", "rmse"])
@pytest.mark.parametrize("bounded", [False, True], ids=["plain", "bounded"])
@pytest.mark.parametrize("B,T", [(1, 1), (7, 12), (10000, 12)])
def test_regression_loss_vs_f64(kind, bounded, B, T):
    """Residuals of exactly 0 (MAE's subgradient 0) and predictions exactly at a censored bound, NaN targets; MSE without
    bounds is bit for bit dmpnn_mse_loss."""
    from chemprop_b200 import engine as K

    g = torch.Generator(device="cuda").manual_seed(B + T + kind)
    P = torch.randn(B, T, device="cuda", generator=g) * 2
    Y = torch.randn(B, T, device="cuda", generator=g) * 2
    Y = torch.where(torch.rand(B, T, device="cuda", generator=g) < 0.15, P, Y)                 # residual exactly 0
    Y[torch.rand(B, T, device="cuda", generator=g) < 0.15] = float("nan")
    w = torch.rand(B, device="cuda", generator=g) + 0.5
    tw = torch.rand(T, device="cuda", generator=g) + 0.5
    lt = gt = None
    if bounded:
        sel = torch.rand(B, T, device="cuda", generator=g)
        lt, gt = sel < 0.4, sel > 0.6
    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    K.regression_loss(P, Y, w, tw, None if lt is None else lt.to(torch.uint8),
                      None if gt is None else gt.to(torch.uint8), kind, loss, dP)
    ref_l, ref_g = ref_regression_loss(kind, P.double(), Y, w.double(), tw.double(), lt, gt)
    m = torch.isfinite(Y)
    n = max(int(m.sum()), 1)
    depth = m.numel() / 1024 + 12
    e = (P.double() - torch.where(m, Y, torch.zeros_like(Y)).double()).abs()
    Wt = w.double().view(-1, 1) * tw.double().view(1, -1) * m
    kd = KAPPA + depth
    Lm = float((Wt * (e if kind == LOSS_MAE else e * e)).sum()) / n
    rl = float(ref_l)
    # RMSE: sqrt halves the MSE value's relative error, and rounds once more
    lb = kd * U * (Lm / (2 * rl) + rl) if kind == LOSS_RMSE and rl > 0 else kd * U * Lm
    assert abs(float(loss) - rl) <= lb + 1e-30, (float(loss), rl, lb)
    gm = Wt / n * (1 if kind == LOSS_MAE else 2 * e)
    if kind == LOSS_RMSE:                          # the MSE gradient over 2 loss; the loss' own error scales every entry
        gm = gm / (2 * rl) if rl > 0 else gm
    assert bool(((dP.double() - ref_g).abs() <= KAPPA * U * gm + kd * U * ref_g.abs()).all())
    exact = m & (Y == P)
    assert not bool(dP[exact].ne(0).any())                                                   # zero residuals
    if bounded:
        assert not bool(dP[m & ((lt & (P < Y)) | (gt & (P > Y)))].ne(0).any())              # satisfied bounds
    if kind == LOSS_MSE and not bounded:
        l2, d2 = torch.empty(1, device="cuda"), torch.empty_like(P)
        K.mse_loss(P, Y, w, tw, l2, d2)
        assert torch.equal(loss, l2) and torch.equal(dP, d2)


@pytest.mark.parametrize("tw", [None, 2.0], ids=["default", "scalar"])
def test_default_constructed_criteria_at_several_tasks(tw):
    """The criteria's default `task_weights=1.0` (and any scalar) weigh every task alike on the device, T = 12, against
    the reference formulas with T equal task weights; loss and dLoss/dpreds through autograd."""
    import chemprop_b200.nn as N

    B, T = 500, 12
    g = torch.Generator(device="cuda").manual_seed(21)
    preds = torch.randn(B, T, device="cuda", generator=g)
    Y = torch.randn(B, T, device="cuda", generator=g)
    Y[torch.rand(B, T, device="cuda", generator=g) < 0.15] = float("nan")
    w = torch.rand(B, device="cuda", generator=g) + 0.5
    sel = torch.rand(B, T, device="cuda", generator=g)
    lt, gt = sel < 0.3, sel > 0.7
    ref_tw = torch.full((T,), 1.0 if tw is None else tw, dtype=torch.float64, device="cuda")
    cases = [(N.EngineMAE, LOSS_MAE, False), (N.EngineRMSE, LOSS_RMSE, False), (N.EngineBoundedMSE, LOSS_MSE, True),
             (N.EngineBoundedMAE, LOSS_MAE, True), (N.EngineBoundedRMSE, LOSS_RMSE, True)]
    for cls, kind, bounded in cases:
        c = (cls() if tw is None else cls(tw)).cuda()
        P = preds.clone().requires_grad_(True)
        loss = c(P, Y, None, w, lt, gt) if bounded else c(P, Y, None, w)
        loss.backward()
        ref_l, ref_g = ref_regression_loss(kind, preds.double(), Y, w.double(), ref_tw, lt if bounded else None,
                                           gt if bounded else None)
        torch.testing.assert_close(loss.detach().double(), ref_l, rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(P.grad.double(), ref_g, rtol=1e-4, atol=1e-9)
    spec = torch.rand(B, T, device="cuda", generator=g) + 0.05
    spec = spec / spec.sum(1, keepdim=True)
    Ys = torch.rand(B, T, device="cuda", generator=g) + 0.05
    Ys = Ys / Ys.sum(1, keepdim=True)
    Ys[torch.rand(B, T, device="cuda", generator=g) < 0.1] = float("nan")
    for cls, kind in ((N.EngineSID, "sid"), (N.EngineWasserstein, "wasserstein")):
        c = (cls() if tw is None else cls(tw)).cuda()
        P = spec.clone().requires_grad_(True)
        loss = c(P, Ys, None, w)
        loss.backward()
        ref_l, ref_g = ref_spectral_loss(kind, spec.double(), Ys, w.double(), ref_tw, None)
        bound, lbound = _spectral_bounds(kind, spec, Ys, w, ref_tw.float(), None)
        assert abs(float(loss.detach()) - float(ref_l)) <= lbound
        assert bool(((P.grad.double() - ref_g).abs() <= bound + 1e-300).all())


def test_host_masks_are_refused_before_the_device():
    import chemprop_b200.nn as N
    from chemprop_b200._lib import DmpnnError

    P, Y = torch.randn(4, 3, device="cuda"), torch.randn(4, 3, device="cuda")
    with pytest.raises(DmpnnError):
        N.EngineBoundedMSE()(P, Y, lt_mask=torch.zeros(4, 3, dtype=torch.bool))
    with pytest.raises(DmpnnError):
        N.EngineBoundedMAE()(P, Y, gt_mask=torch.zeros(4, 3, dtype=torch.bool))


def test_rmse_with_zero_residuals_and_every_target_masked():
    from chemprop_b200 import engine as K

    P = torch.randn(5, 3, device="cuda")
    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    K.regression_loss(P, P.clone(), None, None, None, None, LOSS_RMSE, loss, dP)
    assert float(loss) == 0.0 and not bool(dP.ne(0).any())
    K.regression_loss(P, torch.full_like(P, float("nan")), None, None, None, None, LOSS_RMSE, loss, dP)
    assert float(loss) == 0.0 and not bool(dP.ne(0).any())


def test_spectral_kernels_are_bitwise_repeatable_at_full_size():
    """b = 10 000, T = 1 801: the multi-block count, row and finish launches give identical bits on every call."""
    from chemprop_b200 import engine as K

    P, Y, w, tw, thr = _spectral_case(10000, 1801, seed=99)
    X, _ = _raw(10000, 1801, SPEC_SOFTPLUS, 98)
    first = None
    for _ in range(3):
        outs = [*_loss_kernel("sid", P, Y, w, tw, thr), *_loss_kernel("wasserstein", P, Y, w, tw, thr)]
        o, dX = torch.empty_like(X), torch.empty_like(X)
        K.spectral_transform(X, SPEC_SOFTPLUS, o)
        K.spectral_transform_bwd(X, P, SPEC_SOFTPLUS, dX)
        outs += [o, dX]
        if first is None:
            first = [t.clone() for t in outs]
        else:
            assert all(torch.equal(a, b) for a, b in zip(first, outs))


# ---- a bf16 encoder with EngineSpectralFFN at T = 1 801 -------------------------------------------------------------------------
def test_bf16_encoder_with_spectral_head_at_1801_bins():
    """One CUDA graph replay equals the eager step bit for bit; the head's gradients (its GEMMs at N = 1 801 through
    dmpnn_linear_fwd / dmpnn_linear_wgrad / dmpnn_column_sum, the transform and SID) match f64 torch on the same
    fingerprint."""
    import chemprop_b200.nn as N
    from chemprop_b200.data import PackedBatchLoader, PackedMolGraphDataset, make_molecules
    from chemprop_b200.graph import CudaGraphStep

    T = 1801
    mgs = make_molecules(900, seed=43, shuffle_edges=True, min_atoms=1)
    rng = np.random.default_rng(7)
    Y = rng.uniform(0.05, 1.0, size=(900, T))
    Y = (Y / Y.sum(1, keepdims=True)).astype(np.float32)
    Y[rng.random(Y.shape) < 0.1] = np.nan
    w = rng.uniform(0.5, 2.0, size=900).astype(np.float32)
    ds = PackedMolGraphDataset.from_molgraphs(mgs).to("cuda")
    loader = PackedBatchLoader(ds, batch_size=512, shuffle=True, seed=3, device="cuda", arrays={"Y": Y, "w": w})
    it = iter(loader)
    batch = next(it)
    it.close()
    torch.manual_seed(0)
    head = N.EngineSpectralFFN(n_tasks=T, input_dim=300, hidden_dim=300, n_layers=2, threshold=1e-4)
    model = N.EngineMPNN(N.BondMessagePassing(d_v=ds.d_v, d_e=ds.d_e, precision="bf16"), N.MeanAggregation(), head,
                         batch_norm=True).cuda().train()
    Yb, wb = batch.extras["Y"], batch.extras["w"]
    for p in model.parameters():
        p.grad = torch.zeros_like(p)

    def fn(b):
        for p in model.parameters():
            p.grad.zero_()
        loss = model.training_loss(b, Yb, wb)
        loss.backward()
        return loss

    state = {k: v.clone() for k, v in model.state_dict().items()}
    eager = fn(batch.bmg).detach().clone()
    eager_grads = {k: p.grad.clone() for k, p in model.named_parameters()}
    assert bool(torch.isfinite(eager))
    model.load_state_dict(state)
    step = CudaGraphStep(fn)
    for _ in range(2):
        model.load_state_dict(state)
        out = step(batch.bmg).clone()
        assert torch.equal(out, eager)
        for k, p in model.named_parameters():
            assert torch.equal(p.grad, eager_grads[k]), k
    assert step.captures == 1 and step.replays == 2
    # the head alone against f64 torch on the engine's own fingerprint
    model.load_state_dict(state)
    with torch.no_grad():
        Z = model.fingerprint(batch.bmg).float()
    head.zero_grad()
    Zl = Z.clone().requires_grad_(True)
    loss = head.criterion(head.train_step(Zl), Yb, None, wb)
    loss.backward()
    lin = [b[-1] for b in head.ffn if isinstance(b, torch.nn.Sequential)]
    Ws = [(l.weight.detach().double().requires_grad_(True), l.bias.detach().double().requires_grad_(True)) for l in lin]
    Z64 = Z.double().requires_grad_(True)
    x = Z64
    for i, (W, b) in enumerate(Ws):
        x = x @ W.t() + b
        if i + 1 < len(Ws):
            x = torch.relu(x)
    P64 = ref_spectral(x, SPEC_SOFTPLUS)
    l64, gP = ref_spectral_loss("sid", P64.detach(), Yb, wb.double(), head.criterion.task_weights.double().view(-1), 1e-4)
    P64.backward(gP)
    assert abs(float(loss.detach()) - float(l64)) <= 1e-4 * abs(float(l64))
    for (W, b), l in zip(Ws, lin):
        for mine, ref in ((l.weight.grad, W.grad), (l.bias.grad, b.grad)):
            rel = float((mine.double() - ref).norm() / ref.norm().clamp(min=1e-300))
            assert rel <= 1e-3, rel
    rel = float((Zl.grad.double() - Z64.grad).norm() / Z64.grad.norm())
    assert rel <= 1e-3, rel
    model.eval()
    with torch.no_grad():
        preds = model(batch.bmg)
    assert preds.shape == (len(batch.ids), T) and bool(torch.isfinite(preds).all())
    torch.testing.assert_close(preds.sum(1), torch.ones(len(batch.ids), device="cuda"), rtol=1e-5, atol=1e-5)


# ---- poisoned allocations: every output and every gradient entry is written ---------------------------------------------------
def _poison_head(kind):
    import chemprop_b200.nn as N

    if kind == "spectral_sid":
        return N.EngineSpectralFFN(n_tasks=37, input_dim=300, task_weights=torch.linspace(0.5, 2, 37), threshold=0.02)
    if kind == "spectral_wasserstein":
        return N.EngineSpectralFFN(n_tasks=37, input_dim=300, spectral_activation="exp",
                                   criterion=N.EngineWasserstein(torch.linspace(0.5, 2, 37), threshold=0.02))
    crit = {"mae": N.EngineMAE, "rmse": N.EngineRMSE, "bounded_mse": N.EngineBoundedMSE, "bounded_mae": N.EngineBoundedMAE,
            "bounded_rmse": N.EngineBoundedRMSE}[kind](torch.linspace(0.5, 2, 12))
    return N.EngineRegressionFFN(n_tasks=12, input_dim=300, criterion=crit)


@pytest.mark.parametrize("kind", KINDS)
def test_new_heads_do_not_depend_on_uninitialised_memory(kind, monkeypatch):
    import chemprop_b200.nn as N
    from tests.uninit_matrix import POISONS, assert_bit_identical, install_poison, make_batch

    bmg = make_batch({}, "cuda", n_mols=150)
    rng = np.random.default_rng(9)
    T = 37 if kind.startswith("spectral") else 12
    Y = rng.uniform(0.05, 1.0, size=(150, T)) if kind.startswith("spectral") else rng.normal(size=(150, T))
    if kind.startswith("spectral"):
        Y = Y / Y.sum(1, keepdims=True)
    Y = Y.astype(np.float32)
    Y[rng.random(Y.shape) < 0.15] = np.nan
    Y[3] = np.nan                                                              # a fully masked row
    Y = torch.from_numpy(Y).cuda()
    masks = {}
    if kind.startswith("bounded"):
        sel = torch.from_numpy(rng.random((150, T))).cuda()
        masks = {"lt_mask": sel < 0.3, "gt_mask": sel > 0.7}
    w = (torch.rand(150, generator=torch.Generator().manual_seed(9)) + 0.5).cuda()

    def run(fill):
        with monkeypatch.context() as m:
            install_poison(m, fill)
            torch.manual_seed(1234)
            model = N.EngineMPNN(N.BondMessagePassing(precision="bf16"), N.MeanAggregation(), _poison_head(kind),
                                 batch_norm=True).cuda().train()
            loss = model.training_loss(bmg, Y, w, **masks)
            loss.backward()
            out = {"loss": loss.detach().reshape(1)}
            out.update({"grad." + k: p.grad.detach() for k, p in model.named_parameters()})
            model.eval()
            with torch.no_grad():
                out["preds"] = model(bmg)
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in out.items()}

    ref = run(0.0)
    assert bool(torch.isfinite(ref["loss"]).all())
    for name in sorted(POISONS):
        assert_bit_identical(ref, run(POISONS[name]), f"{name} fill")
