"""CPU tier: Monte Carlo dropout and the uncertainty estimators, kernels emulated where a model runs.

- Dropout follows the nn.Dropout module's flag: an eval-mode model whose dropout modules are trained (chemprop's
  DropoutEstimator) samples the encoder, on the monolithic tier for forward-only bond calls; the same configuration with
  gradients keeps today's tier, and AtomMessagePassing / MABAtomMessagePassing keep the composed tier.
- A forward-only bond call with dropout, fused bf16 (tanh) and fp32, against the f64 restatement mask for mask.
- Every estimator against the reference's outputs on the same per-model predictions (tests/golden/fixture_uq_estimators.npz,
  tools/make_golden_uq_estimators.py), for EngineMPNN and EngineMolAtomBondMPNN stand-ins.
- DropoutEstimator restores `p` and every training flag after it returns and after it raises; `predict` restores the
  flags and runs under inference mode."""
import numpy as np
import pytest
import torch
from torch import nn

from tests import emu
from tests.util import load_golden


def _eval_with_dropout(mp):
    mp.eval()
    mp.dropout.train()
    return mp


@pytest.mark.parametrize("precision,act", [("bf16", "tanh"), ("bf16", "elu"), ("fp32", "relu"), ("fp32", "leakyrelu")])
def test_bond_tier_choice(precision, act):
    from chemprop_b200.nn import BondMessagePassing

    mp = _eval_with_dropout(BondMessagePassing(d_h=32, dropout=0.25, activation=act, precision=precision))
    assert mp.dropout_active()
    with torch.no_grad():
        assert not mp.uses_composed_tier()
    with torch.inference_mode():
        assert not mp.uses_composed_tier()
    for p in mp.parameters():
        p.requires_grad_(False)
    assert not mp.uses_composed_tier()                  # no parameter asks for a gradient: forward-only too
    for p in mp.parameters():
        p.requires_grad_(True)
    assert mp.uses_composed_tier()                       # with gradients: today's tier (no layout: composed)
    mp.dropout.p = 0.0
    assert not mp.dropout_active() and not mp.uses_composed_tier()
    mp.dropout.p = 0.25
    mp.dropout.eval()
    assert not mp.dropout_active() and not mp.uses_composed_tier()


def test_atom_tier_choice():
    from chemprop_b200.nn import AtomMessagePassing, MABAtomMessagePassing, MABBondMessagePassing

    mp = _eval_with_dropout(AtomMessagePassing(d_h=32, dropout=0.25))
    with torch.no_grad():
        assert mp.uses_composed_tier()                   # per-edge masks break the restatement on atoms
    mab = _eval_with_dropout(MABAtomMessagePassing(d_h=32, dropout=0.25, precision="bf16"))
    with torch.no_grad():
        assert mab.composed_reason() == "dropout on atom states"
    assert mab.composed_reason() == "training-mode dropout"
    mb = _eval_with_dropout(MABBondMessagePassing(d_h=32, dropout=0.25, precision="bf16", activation="tanh"))
    with torch.no_grad():
        assert mb.composed_reason() is None and not mb.uses_composed_tier()
    assert mb.composed_reason() == "training-mode dropout"


class _Masks:
    def __init__(self, p, seed):
        self.p, self.masks, self.g = p, [], torch.Generator().manual_seed(seed)

    def __call__(self, like):
        m = (torch.rand(like.shape, generator=self.g) >= self.p).to(like.dtype)
        self.masks.append(m)
        return m


@pytest.mark.parametrize("precision,act,undirected", [("bf16", "tanh", False), ("bf16", "elu", True), ("fp32", "tanh", False)])
def test_forward_only_bond_mask_for_mask(precision, act, undirected, monkeypatch):
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import get_layout
    from chemprop_b200.nn import BondMessagePassing
    from oracle import restatement as R

    emu.patch_engine(monkeypatch)
    calls = []
    monkeypatch.setattr("chemprop_b200.composed.bond_forward", lambda *a: calls.append(a))
    mgs = make_molecules(14, seed=3, mean_atoms=10, std_atoms=4, min_atoms=1, shuffle_edges=True)
    bmg, ref = BatchMolGraph(mgs), BatchMolGraph(mgs)
    torch.manual_seed(2)
    p, depth, h = 0.3, 3, 32
    mp = _eval_with_dropout(BondMessagePassing(d_h=h, depth=depth, bias=True, dropout=p, activation=act,
                                               undirected=undirected, precision=precision))
    mp._mask_fn = masks = _Masks(p, seed=1)
    P = {k: v.detach().double() for k, v in mp.state_dict().items()}
    with torch.inference_mode():
        H = mp(bmg)
    assert not calls
    lay = get_layout(bmg)
    perm = lay.perm.long()
    assert len(masks.masks) == depth
    s = 1.0 / (1.0 - p)
    ref_masks = []
    for m in masks.masks[: depth - 1]:
        m = m[: lay.E, :h].double()
        mm = torch.empty_like(m)
        mm[perm] = m
        ref_masks.append(mm * s)
    ref_masks.append(masks.masks[-1][: lay.V, :h].double() * s)
    H_ref = R.message_passing_forward("bond", ref.V.double(), ref.E.double(), ref.edge_index, ref.rev_edge_index,
                                      P["W_i.weight"], P["W_i.bias"], P["W_h.weight"], P["W_h.bias"], P["W_o.weight"],
                                      P["W_o.bias"], depth, act, undirected, dropout_masks=ref_masks,
                                      act_param={"elu": 1.0}.get(act))
    bar = 2e-2 if precision == "bf16" else 2e-5
    assert (H.double() - H_ref).abs().max().item() <= bar * max(1.0, H_ref.abs().max().item())
    assert bool((H.double()[ref_masks[-1] == 0] == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# estimators against the reference on fixed predictions
# ---------------------------------------------------------------------------------------------------------------------
GOLD = load_golden("fixture_uq_estimators")
KINDS = sorted({k.split(".")[0] for k in GOLD})


class _StandIn(nn.Module):
    """An engine model whose `predict` returns recorded per-batch predictions, pass after pass."""

    def __init__(self, passes: list, mab: bool):
        super().__init__()
        self.passes, self.mab, self.calls, self.drop = passes, mab, 0, nn.Dropout(0.1)
        self.active = []

    def predict(self, batches, *, active_dropout=False):
        self.active.append((active_dropout, self.drop.p))
        per_batch = self.passes[self.calls]
        self.calls += 1
        if self.mab:
            return [None if lv[0] is None else torch.cat(lv, 0) for lv in zip(*per_batch)]
        return torch.cat(per_batch, 0)


def _mab_stand_in(passes):
    from chemprop_b200.nn import EngineMolAtomBondMPNN

    m = EngineMolAtomBondMPNN.__new__(EngineMolAtomBondMPNN)
    nn.Module.__init__(m)
    s = _StandIn(passes, True)
    m.predict = s.predict
    m.stand_in = s
    return m


def _models(case: str, mab: bool) -> list:
    models = []
    i = 0
    while any(k.startswith(f"{case}.in.m{i}.") for k in GOLD):
        passes = []
        k = 0
        while True:
            suf = f".k{k}" if any(x.startswith(f"{case}.in.m{i}.") and ".k" in x for x in GOLD) else ""
            if suf == "" and k > 0 or f"{case}.in.m{i}.b0" + (".l0" if mab else "") + suf not in GOLD:
                break
            per_batch = []
            for j in range(2):
                if mab:
                    per_batch.append(tuple(torch.from_numpy(GOLD[f"{case}.in.m{i}.b{j}.l{lv}{suf}"])
                                           if f"{case}.in.m{i}.b{j}.l{lv}{suf}" in GOLD else None for lv in range(3)))
                else:
                    per_batch.append(torch.from_numpy(GOLD[f"{case}.in.m{i}.b{j}{suf}"]))
            passes.append(per_batch)
            k += 1
        models.append(_mab_stand_in(passes) if mab else _StandIn(passes, False))
        i += 1
    return models


def _with_dirichlet_predictor(models):
    """multiclass-dirichlet: the estimator replaces `predictor.forward`; the stand-in's predict calls it per batch on the
    recorded concentrations (its train_step)."""
    for m in models:
        alphas = [b for b in m.passes[0]]

        class Pred(nn.Module):
            def __init__(self, alphas):
                super().__init__()
                self.alphas, self.i = alphas, 0

            def train_step(self, Z):
                a = self.alphas[self.i % len(self.alphas)]
                self.i += 1
                return a

            def forward(self, Z):
                raise AssertionError("the estimator must replace forward")

        m.predictor = Pred(alphas)
        m.predict = (lambda mm: lambda batches, active_dropout=False: torch.cat([mm.predictor(None) for _ in range(2)], 0))(m)
    return models


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("family", ["mpnn", "mab"])
def test_estimator_matches_reference(kind, family):
    from chemprop_b200.uncertainty import EngineUncertaintyEstimatorRegistry as Reg

    case, mab = f"{kind}.{family}", family == "mab"
    outs = {k[len(case) + 5:]: v for k, v in GOLD.items() if k.startswith(f"{case}.out.")}
    if not outs:
        pytest.skip("the reference has no such case (multiclass-dirichlet reads model.predictor)")
    models = _models(case, mab)
    if kind == "multiclass-dirichlet":
        models = _with_dirichlet_predictor(models)
    est = Reg[kind](ensemble_size=4, dropout=0.3) if kind == "dropout" else Reg[kind]()
    preds, uncs = est([None, None], models)
    for name, val in (("preds", preds), ("uncs", uncs)):
        vals = list(val) if mab else [val]
        for lv, v in enumerate(vals):
            key = f"{name}.l{lv}" if mab else name
            if key not in outs:
                assert v is None, (case, key)
                continue
            want = torch.from_numpy(outs[key])
            assert v.shape == want.shape and v.dtype == want.dtype, (case, key, v.shape, want.shape, v.dtype)
            torch.testing.assert_close(v, want, rtol=1e-6, atol=1e-7, msg=lambda m: f"{case} {key}: {m}")
    if kind == "dropout":
        for m in models:
            s = m.stand_in if mab else m
            assert s.active and all(a and p == 0.3 for a, p in s.active)
            assert s.drop.p == 0.1


def test_ensemble_needs_several_models():
    from chemprop_b200.uncertainty import EnsembleEstimator

    with pytest.raises(ValueError, match="multiple models"):
        EnsembleEstimator()([None], [_StandIn([[torch.zeros(2, 1)]], False)])


# ---------------------------------------------------------------------------------------------------------------------
# restore
# ---------------------------------------------------------------------------------------------------------------------
def _small_model():
    from chemprop_b200.nn import BondMessagePassing, EngineMPNN, EngineRegressionFFN

    torch.manual_seed(0)
    mp = BondMessagePassing(d_h=16, depth=2, dropout=0.2, precision="bf16")
    return EngineMPNN(mp, predictor=EngineRegressionFFN(n_tasks=1, input_dim=16, hidden_dim=8, n_layers=2, dropout=0.1))


def _batches():
    from chemprop_b200.data import BatchMolGraph, TrainingBatch, make_molecules

    return [TrainingBatch(BatchMolGraph(make_molecules(5, seed=s, mean_atoms=6, min_atoms=1)), None, None, None, None,
                          None, None) for s in range(2)]


def _state(model):
    return [(m.training, getattr(m, "p", None)) for m in model.modules()]


def test_dropout_estimator_restores_p_and_flags(monkeypatch):
    from chemprop_b200.uncertainty import DropoutEstimator

    emu.patch_engine(monkeypatch)
    model = _small_model()
    model.predictor.train(False)                 # a mixed state to restore
    before = _state(model)
    seen = []
    orig = type(model).predict

    def spy(self, batches, *, active_dropout=False):
        drops = [m for m in self.modules() if isinstance(m, nn.Dropout)]
        out = orig(self, batches, active_dropout=active_dropout)
        seen.append([m.p for m in drops])
        return out

    monkeypatch.setattr(type(model), "predict", spy)
    mean, var = DropoutEstimator(ensemble_size=3, dropout=0.5)(_batches(), [model])
    assert mean.shape == var.shape == (1, 10, 1)
    assert len(seen) == 3 and all(all(p == 0.5 for p in ps) for ps in seen)
    assert _state(model) == before


def test_dropout_estimator_restores_after_error(monkeypatch):
    from chemprop_b200.uncertainty import DropoutEstimator

    emu.patch_engine(monkeypatch)
    model = _small_model()
    model.eval()
    model.message_passing.train()
    before = _state(model)
    n = []

    def boom(*a, **k):
        n.append(1)
        assert all(m.training for m in model.modules() if isinstance(m, nn.Dropout))
        assert not model.predictor.training
        if len(n) == 2:
            raise RuntimeError("boom")
        return torch.zeros(10, 1)

    monkeypatch.setattr(model, "fingerprint", lambda *a, **k: torch.zeros(5, 16))
    monkeypatch.setattr(model.predictor, "forward", boom)
    with pytest.raises(RuntimeError, match="boom"):
        DropoutEstimator(ensemble_size=3, dropout=0.6)(_batches(), [model])
    assert _state(model) == before


def test_predict_runs_in_inference_mode_and_restores(monkeypatch):
    emu.patch_engine(monkeypatch)
    model = _small_model()
    before = _state(model)
    modes = []
    fp = model.fingerprint
    monkeypatch.setattr(model, "fingerprint",
                        lambda *a: (modes.append((torch.is_inference_mode_enabled(), model.training,
                                                  model.message_passing.dropout.training)), fp(*a))[1])
    out = model.predict(_batches())
    assert out.shape == (10, 1) and modes == [(True, False, False)] * 2
    model.predict(_batches(), active_dropout=True)
    assert modes[2:] == [(True, False, True)] * 2
    assert _state(model) == before
