"""CPU tier: activations whose parameter changes the sign of tau(z) for z < 0 -- nn.LeakyReLU(negative_slope < 0),
nn.ELU(alpha < 0) -- and the non-default parameters the fused kernels do serve.

The monolithic tiers' backward passes take tau' from the stored OUTPUT y = tau(z) (act_grad_from_out in csrc/common.cuh:
y > 0 ? 1 : slope for LeakyReLU, y > 0 ? 1 : y + alpha for ELU, restated by tests/emu.py), which is tau'(z) only while tau
keeps the sign of z.  Modules with a negative (or non-finite) parameter therefore run on the composed tier, where the
caller's own module runs under torch autograd; the rest stay monolithic.  Every case is held to its tier's bar against torch
autograd of the reference op sequence in float64, with the module itself as tau, through the kernel emulation."""
import math
import warnings

import pytest
import torch
from torch import nn

from tests import emu

NEGATIVE = [("LeakyReLU(-0.2)", lambda: nn.LeakyReLU(-0.2)), ("ELU(alpha=-0.5)", lambda: nn.ELU(alpha=-0.5))]
FUSED = [("LeakyReLU(0.3)", lambda: nn.LeakyReLU(0.3)), ("ELU(alpha=0.5)", lambda: nn.ELU(alpha=0.5)),
         ("Identity", nn.Identity)]
ACTS = NEGATIVE + FUSED


def _bars(precision, H_ref):
    """(forward, weight-gradient) bars of each tier against the f64 oracle: fp32 as tests/test_host_logic.py's randomised
    configurations, bf16 as tests/test_gpu_parity.py::test_medium_batch_vs_oracle (1e-2 of the hidden-state scale, 6e-2
    of the largest gradient)."""
    if precision == "fp32":
        return 2e-5, 2e-4
    return 1e-2 * max(1.0, H_ref.abs().max().item()), 6e-2


def test_fused_activation_predicate():
    from chemprop_b200 import _lib
    from chemprop_b200.nn.message_passing import engine_activation, is_fused_activation

    for tau in (nn.ReLU(), nn.Tanh(), nn.Identity(), nn.LeakyReLU(), nn.LeakyReLU(0.0), nn.LeakyReLU(-0.0),
                nn.LeakyReLU(0.3), nn.LeakyReLU(2.0), nn.ELU(), nn.ELU(alpha=0.0), nn.ELU(alpha=0.5), nn.ELU(alpha=3.0)):
        assert is_fused_activation(tau), tau
    for tau in (nn.LeakyReLU(-0.2), nn.LeakyReLU(-1e-30), nn.LeakyReLU(math.nan), nn.LeakyReLU(math.inf),
                nn.ELU(alpha=-0.5), nn.ELU(alpha=math.nan), nn.ELU(alpha=math.inf), nn.ELU(alpha=-math.inf),
                nn.PReLU(), nn.SELU()):
        assert not is_fused_activation(tau), tau
        with pytest.raises(NotImplementedError):
            engine_activation(tau)
    assert engine_activation(nn.LeakyReLU(0.3)) == (_lib.ACT_LEAKYRELU, pytest.approx(0.3))
    assert engine_activation(nn.ELU(alpha=0.5)) == (_lib.ACT_ELU, 0.5)
    assert engine_activation(nn.Identity()) == (_lib.ACT_NONE, 0.0)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("kind", ["bond", "atom"])
@pytest.mark.parametrize("name,make", ACTS, ids=[n for n, _ in ACTS])
def test_message_passing_gradients_vs_f64_autograd(name, make, kind, precision, monkeypatch):
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    monkeypatch.setattr(engine, "_WARNED", set())
    torch.manual_seed(0)
    tau = make()
    negative = any(name == n for n, _ in NEGATIVE)
    bmg = BatchMolGraph(make_molecules(40, seed=3))
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_h=64, depth=3, bias=True, activation=tau, precision=precision)
    P = {k: v.detach().double().requires_grad_(True) for k, v in mp.state_dict().items()}
    H_ref = R.message_passing_forward(kind, bmg.V.double(), bmg.E.double(), bmg.edge_index, bmg.rev_edge_index,
                                      P["W_i.weight"], P["W_i.bias"], P["W_h.weight"], P["W_h.bias"], P["W_o.weight"],
                                      P["W_o.bias"], 3, tau)
    G = torch.randn(H_ref.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    (H_ref * G).sum().backward()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        H = mp(bmg)
    (H.double() * G).sum().backward()
    h_bar, g_bar = _bars(precision, H_ref)
    err = (H.detach().double() - H_ref.detach()).abs().max().item()
    assert err <= h_bar, (name, kind, precision, "H", err, h_bar)
    for k, p in mp.named_parameters():
        ref = P[k].grad
        scale = max(1.0, ref.abs().max().item()) if precision == "fp32" else max(1e-6, ref.abs().max().item())
        err = (p.grad.double() - ref).abs().max().item()
        assert err <= g_bar * scale, (name, kind, precision, k, err, g_bar * scale)
    assert mp.uses_composed_tier() == negative, (name, mp.uses_composed_tier())
    if negative and precision == "bf16":         # the one-time notice that bf16 was asked for and f32 composed runs
        want = f"configuration (activation {tau!r}) runs on the composed tier"
        assert any(want in str(w.message) for w in caught if w.category is RuntimeWarning), [str(w.message) for w in caught]


@pytest.mark.parametrize("name,make", ACTS, ids=[n for n, _ in ACTS])
def test_regression_ffn_gradients_vs_f64_autograd(name, make, monkeypatch):
    """EngineRegressionFFN folds a fused activation into the epilogue of the GEMM before it (linear_fwd act=..., mirror
    dmpnn_act_bwd from the output); any other module runs as tau(lin(X)) under torch autograd."""
    from chemprop_b200 import engine
    from chemprop_b200.nn import EngineRegressionFFN

    emu.patch_engine(monkeypatch)
    acts_seen = []
    lin = engine.linear_fwd

    def spy(*a, **k):
        acts_seen.append((k.get("act", emu.ACT_NONE), k.get("act_param", 0.0)))
        return lin(*a, **k)

    monkeypatch.setattr(engine, "linear_fwd", spy)
    torch.manual_seed(0)
    tau = make()
    negative = any(name == n for n, _ in NEGATIVE)
    ffn = EngineRegressionFFN(n_tasks=3, input_dim=40, hidden_dim=[48, 32], n_layers=2, activation=tau)
    Z = torch.randn(57, 40, generator=torch.Generator().manual_seed(2)) * 2.0
    P = {k: v.detach().double().requires_grad_(True) for k, v in ffn.state_dict().items() if not k.startswith("criterion")}
    X = Z.double()
    for i in range(3):                                 # nn/ffn.py:38-61: Linear, then [act, dropout, Linear]
        if i > 0:
            X = tau(X)
        X = torch.nn.functional.linear(X, P[f"ffn.{i}.{0 if i == 0 else 2}.weight"], P[f"ffn.{i}.{0 if i == 0 else 2}.bias"])
    G = torch.randn(X.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    (X * G).sum().backward()
    Y = ffn(Z)
    (Y.double() * G).sum().backward()
    assert (Y.detach().double() - X.detach()).abs().max().item() <= 2e-5 * max(1.0, X.abs().max().item())
    for k, prm in ffn.named_parameters():
        ref = P[k].grad
        err = (prm.grad.double() - ref).abs().max().item()
        assert err <= 2e-4 * max(1.0, ref.abs().max().item()), (name, k, err)
    fused_acts = [a for a in acts_seen if a[0] != emu.ACT_NONE]
    if negative or isinstance(tau, nn.Identity):
        assert not fused_acts, acts_seen
    else:
        code = emu.ACT_LEAKYRELU if isinstance(tau, nn.LeakyReLU) else emu.ACT_ELU
        p = tau.negative_slope if isinstance(tau, nn.LeakyReLU) else tau.alpha
        assert fused_acts == [(code, pytest.approx(p))] * 2, acts_seen
