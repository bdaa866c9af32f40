"""CPU tier: EngineMolAtomBondMPNN (chemprop_b200/nn/mol_atom_bond_model.py) and csrc/row_head.cu's entry points
(dmpnn_edge_pair_mean(_bwd), dmpnn_regression_loss_rows, dmpnn_bce_loss_rows, dmpnn_ce_loss_rows) through torch emulations
of their wrappers, against the reference's own `MolAtomBondMPNN.training_step`, eval-mode predictions and trained
checkpoints (tests/golden/fixture_mab_{model,ckpt}_*.npz, written by tools/make_golden_mab_model.py); the constructor's
errors, and a launch census of the bond head.  The emulations and `check_training` are shared with
tests/test_gpu_mab_model.py."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from tests import emu_mab
from tests.test_classification_host import bce_loss as _bce_emu
from tests.test_classification_host import ce_loss as _ce_emu
from tests.test_spectral_host import _check_weights, patch_spectral
from tests.test_spectral_host import regression_loss as _regression_emu
from tests.util import golden_bmg, load_golden

LEVELS = ("mol", "atom", "bond")
TRAIN_CASES = ("reg", "bin_bounded", "constrained")
CKPT_CASES = ("regression", "regression_mve", "regression_constrained")
D_H = 32                                                        # tools/make_golden_mab_model.py


# ---- torch emulations of the new wrappers (the kernels' contract, include/dmpnn.h) ----------------------------------------
def ref_edge_pair_mean(P, rev):
    """(P[2i] + P[2i+1]) / 2, NaN rows where rev[2i] != 2i+1."""
    E = P.shape[0]
    out = (P[0::2] + P[1::2]) / 2
    ok = rev[0::2].long() == torch.arange(1, E, 2, device=rev.device)
    return torch.where(ok.view(-1, *([1] * (P.dim() - 1))), out, torch.full_like(out, float("nan")))


def edge_pair_mean(P, rev, out):
    assert P.shape[0] % 2 == 0 and rev.dtype == torch.int32
    out.copy_(ref_edge_pair_mean(P, rev))


def edge_pair_mean_bwd(G, dP):
    dP[0::2] = G / 2
    dP[1::2] = G / 2


def regression_loss_rows(P, Y, w, tw, lt_mask, gt_mask, kind, loss, dP):
    _regression_emu(P, Y, w, tw, lt_mask, gt_mask, kind, loss, dP)


def bce_loss_rows(P, Y, w, tw, loss, dP):
    _check_weights(P, w, tw)
    _bce_emu(P, Y, w, tw, loss, dP)


def ce_loss_rows(P, Y, w, tw, C, loss, dP):
    _check_weights(Y, w, tw)
    _ce_emu(P, Y, w, tw, C, loss, dP)


ROW_WRAPPERS = ("edge_pair_mean", "edge_pair_mean_bwd", "regression_loss_rows", "bce_loss_rows", "ce_loss_rows")


def patch_mab_model(monkeypatch, census: list | None = None):
    """patch_spectral, the bf16 read-out emulation and the five new wrappers; `census` (a list) records
    (wrapper name, rows and columns of its first operand, whether it gathers a second operand as wide as the first:
    [X || X[idx2]]) for every head wrapper called."""
    from chemprop_b200 import engine

    patch_spectral(monkeypatch)
    monkeypatch.setattr(engine, "linear_tc_rows", emu_mab.linear_tc_rows)
    for name in ROW_WRAPPERS:
        monkeypatch.setattr(engine, name, globals()[name])
    if census is None:
        return
    for name in ROW_WRAPPERS + ("linear_fwd", "linear_wgrad", "regression_loss", "mse_loss", "bce_loss", "ce_loss"):
        fn = getattr(engine, name)

        def recorded(*a, _fn=fn, _name=name, **k):
            pair = k.get("idx2") is not None and k.get("K2") == a[1 if _name == "linear_fwd" else 2]
            census.append((_name, int(a[0].shape[0]), int(a[0].shape[1]), pair))
            return _fn(*a, **k)

        monkeypatch.setattr(engine, name, recorded)


# ---- models of the fixtures ------------------------------------------------------------------------------------------------
def build_training_model(case: str, g: dict, precision: str = "fp32"):
    """EngineMolAtomBondMPNN of the fixture's configuration holding its initial state (strict load of the reference's state
    dict minus `metricss.*` and the criteria's torchmetrics states)."""
    import chemprop_b200.nn as N

    kw = dict(hidden_dim=24, n_layers=2)
    mods = {}
    if case in ("reg", "constrained"):
        mods["mol_predictor"] = N.EngineRegressionFFN(n_tasks=2, input_dim=D_H + (3 if case == "reg" else 0), **kw)
        mods["atom_predictor"] = N.EngineRegressionFFN(n_tasks=2, input_dim=D_H, **kw)
        mods["bond_predictor"] = N.EngineRegressionFFN(n_tasks=1, input_dim=2 * D_H, **kw)
        mods["agg"] = N.SumAggregation()
        if case == "constrained":
            mods["atom_constrainer"] = N.ConstrainerFFN(n_constraints=2, fp_dim=D_H, hidden_dim=16)
            mods["bond_constrainer"] = N.ConstrainerFFN(n_constraints=1, fp_dim=2 * D_H, hidden_dim=16)
    else:
        mods["atom_predictor"] = N.EngineBinaryClassificationFFN(n_tasks=2, input_dim=D_H, **kw)
        mods["bond_predictor"] = N.EngineRegressionFFN(n_tasks=1, input_dim=2 * D_H, **kw,
                                                       criterion=N.EngineBoundedMSE(torch.ones(1)))
    model = N.EngineMolAtomBondMPNN(N.MABBondMessagePassing(d_h=D_H, depth=3, precision=precision),
                                    batch_norm=bool(g["batch_norm"]), **mods)
    _load_strict(model, {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")})
    return model


def _load_strict(model, state):
    res = model.load_state_dict({k: v for k, v in state.items() if not k.endswith(("total_loss", "num_samples"))},
                                strict=True)
    assert not res.missing_keys and not res.unexpected_keys


def _level_inputs(g: dict, device: str):
    t = lambda k: torch.from_numpy(g[k]).to(device) if k in g else None  # noqa: E731
    targetss = [t(f"Y.{lv}") for lv in LEVELS]
    weightss = [t(f"w.{lv}") for lv in LEVELS]
    lts = [t(f"lt.{lv}") for lv in LEVELS]
    gts = [t(f"gt.{lv}") for lv in LEVELS]
    cons = None if "constraints.atom" not in g else [t("constraints.atom"), t("constraints.bond")]
    return targetss, weightss, lts, gts, cons, t("X_d")


def run_step(case: str, device: str, precision: str = "fp32") -> dict:
    """One training step and the eval-mode predictions of the fixture's model, in the fixture's key format (loss,
    grad.*, after.*, preds_eval.*), on numpy arrays."""
    g = load_golden(f"fixture_mab_model_{case}")
    model = build_training_model(case, g, precision).to(device).train()
    bmg = golden_bmg(g, device)
    targetss, weightss, lts, gts, cons, X_d = _level_inputs(g, device)
    loss = model.training_loss(bmg, targetss, weightss, None, None, X_d, lt_masks=lts, gt_masks=gts, constraints=cons)
    loss.backward()
    out = {"loss": loss.detach().cpu().numpy()}
    out.update({"grad." + k: p.grad.cpu().numpy() for k, p in model.named_parameters() if p.grad is not None})
    out.update({"after." + k[len("after."):]: model.state_dict()[k[len("after."):]].cpu().numpy() for k in g
                if k.startswith("after.")})
    model.eval()
    with torch.no_grad():
        for lv, p in zip(LEVELS, model(bmg, None, None, X_d, cons)):
            if p is not None:
                out[f"preds_eval.{lv}"] = p.cpu().numpy()
    return out


def check_training(case: str, device: str, precision: str = "fp32", rtol: float = 2e-4, atol: float = 2e-6,
                   graph: bool = False, scaled: bool = False, expect: dict | None = None):
    """EngineMolAtomBondMPNN.training_loss against the reference's `training_step`: loss, every gradient, the batch norms'
    running statistics after the step, and the eval-mode predictions (with the fixture's constraints).  `graph`: the
    constraint-free step also runs as one captured CUDA graph, whose replay must be bit-identical to the eager step.
    `expect` (a run_step result) replaces the fixture's recorded results; `scaled`: every comparison is
    |a - b| <= rtol * max|b| elementwise and in Frobenius norm relative to |b|."""
    g = load_golden(f"fixture_mab_model_{case}")
    if expect is not None:
        g = {**{k: v for k, v in g.items() if not k.startswith(("loss", "grad.", "after.", "preds_eval."))}, **expect}
    model = build_training_model(case, g, precision).to(device).train()
    bmg = golden_bmg(g, device)
    targetss, weightss, lts, gts, cons, X_d = _level_inputs(g, device)

    def step(m, b):
        return m.training_loss(b, targetss, weightss, None, None, X_d, lt_masks=lts, gt_masks=gts, constraints=cons)

    def close(a, b, rt, at, name):
        if scaled:
            a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
            s = max(float(np.abs(b).max(initial=0.0)), 1e-6)
            err, fro = float(np.abs(a - b).max(initial=0.0)), float(np.linalg.norm(a - b)) / max(float(np.linalg.norm(b)), 1e-12)
            assert err <= rtol * s and (fro <= rtol or err <= 1e-5), (name, err, s, fro)
        else:
            np.testing.assert_allclose(a, b, rtol=rt, atol=at, err_msg=name)

    loss = step(model, bmg)
    loss.backward()
    close(loss.detach().cpu().numpy(), g["loss"], rtol, atol, "loss")
    grads = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    assert set(grads) == {k[len("grad."):] for k in g if k.startswith("grad.")}
    for k, v in grads.items():
        close(v.cpu().numpy(), g["grad." + k], rtol, atol, k)
    for k in (k for k in g if k.startswith("after.")):
        close(model.state_dict()[k[len("after."):]].cpu().numpy(), g[k], 1e-5, 1e-6, k)
    if graph:
        from chemprop_b200.graph import CudaGraphStep

        assert cons is None, "steps with constraints are eager only"
        eager = loss.detach().clone()
        eager_grads = {k: v.clone() for k, v in grads.items()}
        stepped = model                     # its running statistics have seen one step: the eval check below uses it
        model = build_training_model(case, g, precision).to(device).train()
        for p in model.parameters():
            p.grad = torch.zeros_like(p)

        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            out = step(model, b)
            out.backward()
            return out

        cg = CudaGraphStep(fn)
        for _ in range(2):
            out = cg(bmg)
            assert torch.equal(out, eager)
            for k, p in model.named_parameters():
                if k in eager_grads:
                    assert torch.equal(p.grad, eager_grads[k]), k
        assert cg.replays >= 1
        model = stepped
    model.eval()
    with torch.no_grad():
        predss = model(bmg, None, None, X_d, cons)
    for lv, preds in zip(LEVELS, predss):
        if f"preds_eval.{lv}" in g:
            close(preds.cpu().numpy(), g[f"preds_eval.{lv}"], rtol, 1e-5, lv)
        else:
            assert preds is None
    return model, bmg, predss, cons


class _FixedFingerprints(torch.nn.Module):
    """Stands in for the encoder: returns the reference's recorded (H_v, H_e)."""

    def __init__(self, H_v, H_e):
        super().__init__()
        self.H_v, self.H_e = H_v, H_e

    def forward(self, bmg, V_d=None, E_d=None):
        return self.H_v, self.H_e


def build_checkpoint_model(g: dict, hidden: int | None = None):
    """The checkpoint's model on the engine, predictors and constrainers from its hparams.  `hidden` None: the trained
    widths, and a state dict of exactly the checkpoint's keys and shapes (zeros) loads with strict=True.  `hidden` set:
    every head MLP with that many hidden units, loaded strictly with the fixture's cut of the trained heads (the encoder's
    weights as zeros of the recorded shapes)."""
    import chemprop_b200.nn as N

    width = (lambda h: int(h)) if hidden is None else (lambda h: hidden)  # noqa: E731
    cls = {"RegressionFFN": N.EngineRegressionFFN, "MveFFN": N.EngineMveFFN}
    mods = {}
    for lv in LEVELS:
        mean, scale = g[f"param.{lv}_predictor.output_transform.mean"], g[f"param.{lv}_predictor.output_transform.scale"]
        mods[f"{lv}_predictor"] = cls[str(g[f"hp.{lv}.cls"])](
            n_tasks=int(g[f"hp.{lv}.n_tasks"]), input_dim=int(g[f"hp.{lv}.input_dim"]),
            hidden_dim=width(g[f"hp.{lv}.hidden_dim"]), n_layers=int(g[f"hp.{lv}.n_layers"]),
            output_transform=N.UnscaleTransform(mean[0].tolist(), scale[0].tolist()))
    for lv in ("atom", "bond"):
        if f"hp.{lv}_constrainer.n_constraints" in g:
            kw = {k: int(g[f"hp.{lv}_constrainer.{k}"]) for k in ("n_constraints", "fp_dim", "hidden_dim", "n_layers")}
            kw["hidden_dim"] = width(kw["hidden_dim"])
            mods[f"{lv}_constrainer"] = N.ConstrainerFFN(**kw)
    model = N.EngineMolAtomBondMPNN(N.MABBondMessagePassing(d_h=int(g["hp.d_h"])), N.NormAggregation(norm=float(g["hp.norm"])),
                                    batch_norm=bool(g["hp.batch_norm"]), **mods)
    shapes = {k[len("shape."):]: tuple(int(s) for s in v) for k, v in g.items() if k.startswith("shape.")}
    if hidden is None:
        assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == {
            k: v for k, v in shapes.items() if not k.endswith(("total_loss", "num_samples"))}
        _load_strict(model, {k: torch.zeros(v) for k, v in shapes.items()})
        return model
    state = {k: torch.zeros(v) for k, v in shapes.items() if k.startswith("message_passing.")}
    state.update({k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")})
    _load_strict(model, state)
    return model


def check_checkpoint(name: str, device: str, rtol: float = 1e-4, atol: float = 1e-5):
    """The checkpoint's keys and shapes load strictly into the engine model its hparams rebuild; with the fixture's cut of
    the trained heads and the reference's fingerprints of its trained encoder, the engine's heads (aggregation, pair mean,
    target unscaling, constraints) predict as the reference's."""
    g = load_golden(f"fixture_mab_ckpt_{name}")
    build_checkpoint_model(g)
    model = build_checkpoint_model(g, hidden=int(g["hp.hidden_kept"])).to(device).eval()
    bmg = golden_bmg(g, device)
    model.message_passing = _FixedFingerprints(torch.from_numpy(g["H_v"]).to(device), torch.from_numpy(g["H_e"]).to(device))
    cons = None
    if "constraints.atom" in g:
        cons = [torch.from_numpy(g["constraints.atom"]).to(device), torch.from_numpy(g["constraints.bond"]).to(device)]
    with torch.no_grad():
        H_g = model.fingerprint(bmg)[0]
        predss = model(bmg, constraints=cons)
    np.testing.assert_allclose(H_g.cpu().numpy(), g["H_g"], rtol=rtol, atol=atol)
    for lv, preds in zip(LEVELS, predss):
        np.testing.assert_allclose(preds.cpu().numpy(), g[f"preds_eval.{lv}"], rtol=rtol, atol=atol, err_msg=lv)
    return model, bmg, predss, cons


def assert_constraints_met(bmg, predss, cons, atol=1e-4):
    """The constrained sums equal the constraints, per molecule and constrained column."""
    n = cons[0].shape[0]
    for level, c in ((1, cons[0]), (2, cons[1])):
        P = predss[level][..., 0] if predss[level].dim() > 2 else predss[level]
        seg = bmg.batch if level == 1 else bmg.batch[bmg.edge_index[0, ::2]]
        sums = torch.zeros((n, P.shape[1]), dtype=P.dtype, device=P.device).index_add_(0, seg, P)
        has = ~torch.isnan(c[0])
        torch.testing.assert_close(sums[:, has], c[:, has], rtol=1e-4, atol=atol)


# ---- the tests ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", TRAIN_CASES)
def test_training_fixture_matches_the_reference(case, monkeypatch):
    patch_mab_model(monkeypatch)
    model, bmg, predss, cons = check_training(case, "cpu")
    if cons is not None:
        assert_constraints_met(bmg, predss, cons)


@pytest.mark.parametrize("name", CKPT_CASES)
def test_checkpoint_loads_strictly_and_predicts_as_the_reference(name, monkeypatch):
    patch_mab_model(monkeypatch)
    model, bmg, predss, cons = check_checkpoint(name, "cpu")
    if cons is not None:
        assert_constraints_met(bmg, predss, cons)


def test_constructor_errors():
    import chemprop_b200.nn as N

    mp = N.MABBondMessagePassing(d_h=16)
    with pytest.raises(ValueError, match="At least one of"):
        N.EngineMolAtomBondMPNN(mp, N.MeanAggregation())
    with pytest.raises(ValueError, match="agg must also be provided"):
        N.EngineMolAtomBondMPNN(mp, None, mol_predictor=N.EngineRegressionFFN(input_dim=16))


def test_state_dict_keys_are_the_reference_model_keys():
    """Key for key the reference's MolAtomBondMPNN without `metricss.*` (and the criteria's torchmetrics states)."""
    from oracle.ref_shim import import_reference, reference_available

    if not reference_available():
        pytest.skip("reference tree not present")
    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.models import MolAtomBondMPNN
    from chemprop.nn.ffn import ConstrainerFFN as RefConstrainer
    from chemprop.nn.message_passing import MABBondMessagePassing

    import chemprop_b200.nn as N

    ref = MolAtomBondMPNN(MABBondMessagePassing(d_h=16), ref_nn.MeanAggregation(), ref_nn.RegressionFFN(input_dim=16),
                          ref_nn.MveFFN(input_dim=16), ref_nn.RegressionFFN(input_dim=32), RefConstrainer(fp_dim=16),
                          RefConstrainer(fp_dim=32), batch_norm=True)
    ours = N.EngineMolAtomBondMPNN(N.MABBondMessagePassing(d_h=16), N.MeanAggregation(), N.EngineRegressionFFN(input_dim=16),
                                   N.EngineMveFFN(input_dim=16), N.EngineRegressionFFN(input_dim=32), N.ConstrainerFFN(fp_dim=16),
                                   N.ConstrainerFFN(fp_dim=32), batch_norm=True)
    strip = lambda sd: {k for k in sd if not k.startswith("metricss.") and not k.endswith(("total_loss", "num_samples"))}  # noqa: E731
    assert strip(ref.state_dict()) == set(ours.state_dict())
    ours.load_state_dict({k: v for k, v in ref.state_dict().items() if k in strip(ref.state_dict())}, strict=True)


def test_launch_census_bond_head_gathers_and_rows_criteria_at_atom_and_bond_level(monkeypatch):
    """The bond predictor's first layer reads H_e twice through idx2 = rev (forward, weight gradient, dH) and no E x 2h
    operand is ever built; the atom and bond levels use the _rows criteria, the molecule level its single-block kernel."""
    from chemprop_b200.nn.head import EdgePairOperand

    census = []
    patch_mab_model(monkeypatch, census)
    monkeypatch.setattr(EdgePairOperand, "materialize", lambda self: pytest.fail("E x 2h operand materialised"))
    g = load_golden("fixture_mab_model_reg")
    model = build_training_model("reg", g).train()
    bmg = golden_bmg(g, "cpu")
    targetss, weightss, lts, gts, cons, X_d = _level_inputs(g, "cpu")
    model.training_loss(bmg, targetss, weightss, None, None, X_d).backward()
    E, V, B = int(bmg.E.shape[0]), int(bmg.V.shape[0]), len(bmg)
    assert not [c for c in census if c[1] == E and c[2] == 2 * D_H], "an E x 2h operand reached a kernel"
    gathered = [c[0] for c in census if c[3]]
    assert sorted(gathered) == ["linear_fwd", "linear_fwd", "linear_wgrad"], census
    losses = [(c[0], c[1]) for c in census if "loss" in c[0]]
    assert sorted(losses) == sorted([("mse_loss", B), ("regression_loss_rows", V), ("regression_loss_rows", E // 2)]), losses
    assert ("edge_pair_mean", E) in [(c[0], c[1]) for c in census]
    assert ("edge_pair_mean_bwd", E // 2) in [(c[0], c[1]) for c in census]


def test_pair_mean_refuses_odd_edge_counts_and_marks_unpaired_rows(monkeypatch):
    from chemprop_b200.nn.mol_atom_bond_model import EdgePairMeanFunction

    patch_mab_model(monkeypatch)
    with pytest.raises(ValueError, match="even number"):
        EdgePairMeanFunction.apply(torch.zeros(5, 2), torch.zeros(5, dtype=torch.int32))
    P = torch.randn(6, 3)
    rev = torch.tensor([1, 0, 3, 2, 5, 4], dtype=torch.int32)
    torch.testing.assert_close(EdgePairMeanFunction.apply(P, rev), (P[::2] + P[1::2]) / 2, rtol=0, atol=0)
    out = EdgePairMeanFunction.apply(P, torch.tensor([2, 3, 0, 1, 5, 4], dtype=torch.int32))
    assert torch.isnan(out[:2]).all() and torch.isfinite(out[2]).all()


def test_row_loss_refuses_masks_for_non_bounded_criteria(monkeypatch):
    """`_Criterion.row_loss`, which EngineMolAtomBondMPNN calls at atom and bond level, refuses lt_mask / gt_mask for a
    criterion that is not bounded, and takes them for a bounded one."""
    import chemprop_b200.nn as N

    patch_mab_model(monkeypatch)
    P, Y = torch.randn(8, 2), torch.randn(8, 2)
    m = torch.zeros(8, 2, dtype=torch.bool)
    with pytest.raises(NotImplementedError):
        N.EngineMAE(torch.ones(2)).row_loss(P, Y, None, m, m)
    assert torch.isfinite(N.EngineBoundedMAE(torch.ones(2)).row_loss(P, Y, None, m, m))
