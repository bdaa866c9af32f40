"""GPU tier: the molecule-level head on the engine's kernels (csrc/head.cu: batch norm, MSE criterion; FFN GEMMs with the
activation in the epilogue) and the whole training step as ONE CUDA graph (chemprop_b200/graph.py) -- SURVEY.md section 8f-2,
against the reference's own `MPNN.training_step` (tests/golden/fixture_mpnn_head.npz, oracle/make_golden.py::mpnn_head_case)."""
import gc
import itertools
import math

import numpy as np
import pytest
import torch
from torch import nn

pytestmark = pytest.mark.gpu


def test_engine_mpnn_head_matches_reference_training_step():
    from tests.util import check_mpnn_head

    check_mpnn_head("cuda")


def test_training_step_as_one_cuda_graph_matches_reference():
    from tests.util import check_mpnn_head

    check_mpnn_head("cuda", graph=True)


@pytest.mark.parametrize("B,d", [(1, 40), (7, 300), (10000, 300), (513, 33)])
def test_batch_norm_kernels_vs_torch(B, d):
    from chemprop_b200.nn import EngineBatchNorm1d

    torch.manual_seed(B + d)
    ours, ref = EngineBatchNorm1d(d).cuda(), torch.nn.BatchNorm1d(d).cuda()
    with torch.no_grad():
        ours.weight.uniform_(0.5, 1.5); ours.bias.normal_()
        ref.load_state_dict(ours.state_dict())
    x = (torch.randn(B, d, device="cuda") * 3 + 1).requires_grad_(True)
    x2 = x.detach().clone().requires_grad_(True)
    G = torch.randn(B, d, device="cuda")
    if B == 1:
        with pytest.raises(ValueError):
            ref(x2)                                  # torch refuses a training batch of one, and so does the module
        with pytest.raises(ValueError):
            ours(x)
        assert int(ours.num_batches_tracked) == 0
        return
    (ours(x) * G).sum().backward()
    (ref(x2) * G).sum().backward()
    torch.testing.assert_close(x.grad, x2.grad, rtol=2e-4, atol=2e-5)
    torch.testing.assert_close(ours.weight.grad, ref.weight.grad, rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(ours.bias.grad, ref.bias.grad, rtol=2e-4, atol=2e-4)
    torch.testing.assert_close(ours.running_mean, ref.running_mean, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ours.running_var, ref.running_var, rtol=1e-5, atol=1e-6)
    assert int(ours.num_batches_tracked) == 1


def test_cuda_graph_step_replays_new_batches_of_the_same_signature():
    """Graph replay with NEW data: same molecules' topology (same signature), different features and targets -> equals eager."""
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.graph import CudaGraphStep
    from chemprop_b200.nn import BondMessagePassing, EngineMPNN

    torch.manual_seed(0)
    mgs = make_molecules(600, seed=3)
    model = EngineMPNN(BondMessagePassing(precision="bf16"), batch_norm=True).cuda().train()
    for p in model.parameters():
        p.grad = torch.zeros_like(p)
    Y = torch.randn(600, 1, device="cuda")

    def fn(b):
        for p in model.parameters():
            p.grad.zero_()
        loss = model.training_loss(b, Y)
        loss.backward()
        return loss

    step = CudaGraphStep(fn)
    a = BatchMolGraph(mgs)
    a.to("cuda")
    step(a)
    b = BatchMolGraph(mgs)
    b.V = b.V * 0.5 + 0.1                           # new features, same topology
    b.to("cuda")
    Y.copy_(torch.randn(600, 1, device="cuda"))
    bn_state = {k: v.clone() for k, v in model.bn.state_dict().items()}
    loss_g = step(b).clone()
    grads_g = {k: p.grad.clone() for k, p in model.named_parameters()}
    assert step.captures == 1 and step.replays == 2
    model.bn.load_state_dict(bn_state)
    loss_e = fn(b)
    torch.testing.assert_close(loss_g, loss_e, rtol=1e-5, atol=1e-6)
    for k, p in model.named_parameters():
        torch.testing.assert_close(grads_g[k], p.grad, rtol=1e-4, atol=1e-6, msg=k)
    c = BatchMolGraph(make_molecules(500, seed=4))   # another signature: captured on first sight
    c.to("cuda")
    Y2 = Y[:500].clone()
    model2_loss = None
    step2 = CudaGraphStep(lambda bb: fn_sized(bb))

    def fn_sized(bb):
        for p in model.parameters():
            p.grad.zero_()
        loss = model.training_loss(bb, Y2 if len(bb) == 500 else Y)
        loss.backward()
        return loss

    l1 = step2(c).clone()
    l2 = step2(b).clone()
    assert step2.captures == 2 and torch.isfinite(l1) and torch.isfinite(l2)


# ---------------------------------------------------------------------------------------------------------------------
# batch norm against float64, each result held to a bound from the kernels' summation order
# ---------------------------------------------------------------------------------------------------------------------
U = 2.0 ** -24
NAN = float("nan")
MEAN_BAR = 0.6
BN_CASES = [(2, 1, True), (2, 2048, False), (7, 31, True), (7, 300, False), (8, 32, False), (8, 33, True), (9, 33, False),
            (9, 2048, True), (10000, 300, True), (10000, 2048, False), (10000, 1, False), (250000, 33, True),
            (250000, 300, False), (250000, 32, True)]


@pytest.fixture()
def _release_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


def _f32(x):
    return float(np.float32(x))


def _strided(B, d, ld, fill=NAN):
    buf = torch.full((B, ld), fill, device="cuda")
    return buf, buf[:, :d]


def _ratio(got, ref, bound, what):
    """(worst |err| / bound, sum |err| / sum bound); exact where the bound is 0."""
    err = (got.double() - ref).abs()
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite"
    assert bool((err[bound == 0] == 0).all()), f"{what}: inexact where the bound is 0"
    worst = (err / bound.clamp_min(1e-300)).max().item()
    mean = err.sum().item() / max(bound.sum().item(), 1e-300)
    assert worst <= 1.0, (what, "worst err / bound", worst)
    assert mean <= MEAN_BAR, (what, "mean err / mean bound", mean)
    return worst, mean


@pytest.mark.parametrize("B,d,affine", BN_CASES, ids=[f"B{b}-d{d}-{'affine' if a else 'plain'}" for b, d, a in BN_CASES])
def test_batch_norm_kernels_vs_f64(B, d, affine, _release_memory):
    """engine.bn_train_fwd / bn_bwd against float64.  Both kernels sum a column in 8 warps, each a plain chain over every
    8th row (n = ceil(B / 8) terms), then add the 8 partials in order; with u = 2^-24:

    - mean: |m^ - m| <= e_m = (n + 9) u sum|x| / B (n - 1 + 7 additions, the division);
    - variance: v^ = (1 + theta) sum (x - m^)^2 / B with |theta| <= (n + 11) u (the rounded x - m^ squared: 2 u; the fmaf
      chain: n; the partials: 7; the division: 1), and sum (x - m^)^2 / B = v + (m - m^)^2 exactly, so
      |v^ - v| <= theta (v + e_m^2) + e_m^2 -- the biased variance: the unbiased one moves v by v / (B - 1), past this
      bound at every B <= 10 000 here;
    - inv-std = rsqrtf(v^ + eps): the interval of rsqrt over v + eps +- (|v^ - v| + u (v + eps)), widened by rsqrtf's
      2 ulp (4 u);
    - x_hat = (x - m^) inv^: e_m inv + |x - m| e_inv + 3 u (|x - m| + e_m) inv;  Y = fmaf(x_hat, g, b): g e_xhat + u |Y|;
    - the running statistics: the update's 4 roundings of its terms plus momentum times the error of m^ / the unbiased v^;
    - backward: sum dy and sum dy x_hat as above ((n + 7) u of the sums of |terms|), and
      dX = (g inv / B) (B dy - sum dy - x_hat sum dy x_hat) with 3 roundings inside the bracket and 3 outside.

    Columns have |mean| / std from 0 to 10^3 and std from 10^-2 to 10^2; one column is constant (3.25: every sum exact),
    where the mean must be exact, x_hat and dgamma zero and inv-std rsqrtf(eps).  Operands and outputs have row strides
    larger than d, with NaN padding that must stay untouched."""
    from chemprop_b200 import engine

    g = torch.Generator(device="cuda").manual_seed(B * 7919 + d * 31 + affine)
    eps, mo = _f32(1e-5), _f32(0.1)
    ratio = torch.tensor([0.0, 1.0, 10.0, 100.0, 1000.0], device="cuda")[torch.arange(d, device="cuda") % 5]
    std = torch.pow(10.0, torch.rand(d, device="cuda", generator=g) * 4 - 2)
    std[0] = 1.0                                     # a centred unit column: the unbiased variance must fail its bound
    mu = ratio * std * torch.where(torch.rand(d, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    _, X = _strided(B, d, d + 3)
    X.copy_(mu + std * torch.randn(B, d, device="cuda", generator=g))
    const = d // 2 if d > 1 else None
    if const is not None:
        X[:, const] = 3.25
    gamma = (torch.rand(d, device="cuda", generator=g) + 0.5) if affine else None
    beta = torch.randn(d, device="cuda", generator=g) if affine else None
    rm0 = torch.randn(d, device="cuda", generator=g)
    rv0 = torch.rand(d, device="cuda", generator=g) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    Yb, Y = _strided(B, d, d + 5)
    Hb, Xhat = _strided(B, d, d + 2)
    mean, invstd = torch.full((d,), NAN, device="cuda"), torch.full((d,), NAN, device="cuda")
    engine.bn_train_fwd(X, gamma, beta, rm, rv, eps, mo, Y, Xhat, mean, invstd)
    dYb, dY = _strided(B, d, d + 1)
    dY.copy_(torch.randn(B, d, device="cuda", generator=g))
    dXb, dX = _strided(B, d, d + 7)
    dgamma = torch.full((d,), NAN, device="cuda") if affine else None
    dbeta = torch.full((d,), NAN, device="cuda") if affine else None
    engine.bn_bwd(dY, Xhat, gamma, invstd, dX, dgamma, dbeta)
    torch.cuda.synchronize()
    for buf, what in ((Yb, "Y"), (Hb, "x_hat"), (dXb, "dX")):
        assert bool(torch.isnan(buf[:, d:]).all()), f"{what}: padding written"

    n = math.ceil(B / 8)
    Xd = X.double()
    m = Xd.mean(0)
    xc = Xd - m
    v = (xc * xc).mean(0)
    e_m = (n + 9) * U * Xd.abs().sum(0) / B
    theta = (n + 11) * U
    e_v = theta * (v + e_m ** 2) + e_m ** 2
    ve = v + eps
    spread = e_v + U * (ve + e_v)
    inv = ve.rsqrt()
    inv_hi = (ve - spread).clamp_min(1e-300).rsqrt() * (1 + 4 * U)
    inv_lo = (ve + spread).rsqrt() * (1 - 4 * U)
    e_inv = torch.maximum(inv_hi - inv, inv - inv_lo)
    xh = xc * inv
    e_x = e_m * inv_hi + xc.abs() * e_inv + 3 * U * (xc.abs() + e_m) * inv_hi
    gd = gamma.double() if affine else torch.ones_like(m)
    bd = beta.double() if affine else torch.zeros_like(m)
    y = xh * gd + bd
    e_y = gd.abs() * e_x + U * (y.abs() + gd.abs() * e_x)
    vu = (xc * xc).sum(0) / (B - 1)
    e_vu = theta * (vu + e_m ** 2 * B / (B - 1)) + e_m ** 2 * B / (B - 1)
    rm_ref = (1 - mo) * rm0.double() + mo * m
    rv_ref = (1 - mo) * rv0.double() + mo * vu
    e_rm = 4 * U * ((1 - mo) * rm0.double().abs() + mo * (m.abs() + e_m)) + mo * e_m
    e_rv = 4 * U * ((1 - mo) * rv0.double().abs() + mo * (vu + e_vu)) + mo * e_vu
    res = [_ratio(mean, m, e_m, "mean"), _ratio(invstd, inv, e_inv, "inv-std"), _ratio(Xhat, xh, e_x, "x_hat"),
           _ratio(Y, y, e_y, "Y"), _ratio(rm, rm_ref, e_rm, "running_mean"), _ratio(rv, rv_ref, e_rv, "running_var")]
    # backward, from the kernel's own x_hat and inv-std
    H, iv, gy = Xhat.double(), invstd.double(), dY.double()
    sdy, sdyx = gy.sum(0), (gy * H).sum(0)
    e_a = (n + 7) * U * gy.abs().sum(0)
    e_b = (n + 7) * U * (gy * H).abs().sum(0)
    k = gd * iv / B
    inner = B * gy - sdy - H * sdyx
    e_in = 3 * U * (B * gy.abs() + sdy.abs() + e_a + H.abs() * (sdyx.abs() + e_b)) + e_a + H.abs() * e_b
    e_dx = k.abs() * e_in * (1 + 3 * U) + 3 * U * k.abs() * (inner.abs() + e_in)
    res.append(_ratio(dX, k * inner, e_dx, "dX"))
    if affine:
        res += [_ratio(dbeta, sdy, e_a, "dbeta"), _ratio(dgamma, sdyx, e_b, "dgamma")]
    if const is not None:
        assert mean[const].item() == 3.25 and bool((Xhat[:, const] == 0).all())
        assert abs(invstd[const].item() - 1 / math.sqrt(eps)) <= 4 * U / math.sqrt(eps)
        if affine:
            assert dgamma[const].item() == 0.0 and bool((Y[:, const] == beta[const]).all())
    if B <= 10000:        # the unbiased variance, had it normalised, would be caught by the inv-std bound
        wrong = (vu + eps).rsqrt()
        assert bool(((wrong - inv).abs() > e_inv).any()), "bound too loose to reject the unbiased variance"
    worst = max(r[0] for r in res)
    meanr = max(r[1] for r in res)
    print(f"[bn] B={B} d={d} affine={affine}: worst err / bound {worst:.3f}, mean err / mean bound {meanr:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# the regression head at chemprop's shapes against float64 autograd
# ---------------------------------------------------------------------------------------------------------------------
_SELU_ALPHA, _SELU_SCALE = 1.6732632423543772848170429916717, 1.0507009873554804934193349852946
HEAD_ACTS = [("ReLU", nn.ReLU), ("LeakyReLU(0.3)", lambda: nn.LeakyReLU(0.3)), ("SELU", nn.SELU)]


def _head_cases():
    out = []
    for i, (inp, hid, nl, nt) in enumerate(itertools.product((300, 2048), (300, 2048), (1, 3), (1, 12))):
        out.append((inp, hid, nl, nt, (1, 50, 10000)[i % 3], HEAD_ACTS[(i + i // 3) % 3][0]))
    return out


HEAD_CASES = _head_cases()


@pytest.mark.parametrize("inp,hid,nl,nt,B,act", HEAD_CASES,
                         ids=[f"in{a}-h{b}-L{c}-T{d}-B{e}-{f}" for a, b, c, d, e, f in HEAD_CASES])
def test_regression_ffn_vs_f64_autograd(inp, hid, nl, nt, B, act, _release_memory):
    """EngineRegressionFFN on the GPU (dmpnn_linear_fwd with the activation in the epilogue for ReLU / LeakyReLU, torch's
    SELU between plain GEMMs; the mirror on dmpnn_act_bwd / dmpnn_linear_wgrad / dmpnn_linear_fwd) against torch autograd
    of the same MLP in float64, at the fp32 tier's module bars: outputs 2e-5 and gradients 2e-4 of max(1, max |ref|).

    The three activations have a kink at 0.  The reference takes each hidden unit's branch from the sign of the module's
    own f32 pre-activation (its GEMM's output, which for a fused activation is tau(z), of the sign of z), so that a unit
    whose z lies within rounding of 0 does not put tau''s jump in slope into the gradient comparison; those units must
    have |z| below 1e-4 of the layer's largest."""
    from chemprop_b200.nn import EngineRegressionFFN

    torch.manual_seed(inp + hid + nl + nt + B)
    tau = dict(HEAD_ACTS)[act]()
    ffn = EngineRegressionFFN(n_tasks=nt, input_dim=inp, hidden_dim=hid, n_layers=nl, activation=tau).cuda()
    g = torch.Generator(device="cuda").manual_seed(B + nt)
    Z = torch.randn(B, inp, device="cuda", generator=g) * 2.0
    P = {k: v.detach().double().requires_grad_(True) for k, v in ffn.state_dict().items() if not k.startswith("criterion")}
    lins = [blk[-1] for blk in ffn.ffn]
    outs = []
    hooks = [m.register_forward_hook(lambda m, a, o: outs.append(o.detach())) for m in lins]
    Zg = Z.clone().requires_grad_(True)
    Y = ffn(Zg)
    for h in hooks:
        h.remove()
    pos, neg = {"ReLU": (lambda x: x, lambda x: 0 * x), "LeakyReLU(0.3)": (lambda x: x, lambda x: _f32(0.3) * x),
                "SELU": (lambda x: _SELU_SCALE * x, lambda x: _SELU_SCALE * _SELU_ALPHA * torch.expm1(x))}[act]
    X = Z.double()
    for i in range(nl + 1):                            # nn/ffn.py:38-61: Linear, then [act, dropout, Linear]
        if i > 0:
            up = outs[i - 1] > 0
            flip = up != (X > 0)
            assert bool((X.detach().abs()[flip] <= 1e-4 * X.detach().abs().max()).all()), "branch differs away from 0"
            X = torch.where(up, pos(X), neg(X))
        j = 0 if i == 0 else 2
        X = torch.nn.functional.linear(X, P[f"ffn.{i}.{j}.weight"], P[f"ffn.{i}.{j}.bias"])
    G = torch.randn(X.shape, dtype=torch.float64, device="cuda", generator=g)
    (X * G).sum().backward()
    (Y.double() * G).sum().backward()
    torch.cuda.synchronize()
    bar = 2e-5 * max(1.0, X.abs().max().item())
    err = (Y.detach().double() - X.detach()).abs().max().item()
    assert err <= bar, ("Y", err, bar)
    worst = err / bar
    for k, prm in ffn.named_parameters():
        ref = P[k].grad
        e = (prm.grad.double() - ref).abs().max().item()
        b = 2e-4 * max(1.0, ref.abs().max().item())
        assert e <= b, (k, e, b)
        worst = max(worst, e / b)
    print(f"[head] in={inp} hidden={hid} layers={nl} tasks={nt} B={B} {act}: worst err / bar {worst:.3f}")
