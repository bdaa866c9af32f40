"""CPU tier: the classification heads (EngineBinaryClassificationFFN, EngineMulticlassClassificationFFN; csrc/head.cu's
dmpnn_bce_loss / dmpnn_ce_loss / dmpnn_class_probs) through torch emulations of their kernel wrappers, against the
reference's own `MPNN.training_step` (tests/golden/fixture_mpnn_binary.npz, fixture_mpnn_multiclass.npz, written by
tools/make_golden_classification.py), and the host-side argument checks of the three entry points."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import emu
from tests.util import golden_bmg, load_golden


# ---- torch emulations of engine.bce_loss / ce_loss / class_probs (the kernels' contract, include/dmpnn.h) ----------------
def _weights(Y, w, tw):
    m = torch.isfinite(Y)
    ww = (w.view(-1, 1) if w is not None else 1.0) * (tw.view(1, -1) if tw is not None else 1.0) * m
    return m, ww, m.sum().clamp(min=1)


def bce_loss(P, Y, w, tw, loss, dP):
    m, ww, n = _weights(Y, w, tw)
    y = torch.where(m, Y, torch.zeros_like(Y))
    L = F.binary_cross_entropy_with_logits(P, y, reduction="none")
    loss.copy_((torch.where(m, ww * L, torch.zeros_like(L)).sum() / n).reshape(1))
    dP.copy_((torch.sigmoid(P) - y) * ww / n)


def ce_loss(P, Y, w, tw, C, loss, dP):
    B = P.shape[0]
    X = P.reshape(B, -1, C)
    m, ww, n = _weights(Y, w, tw)
    k = torch.where(m, Y, torch.zeros_like(Y)).trunc()
    valid = (k >= 0) & (k < C)
    idx = k.clamp(0, C - 1).long()
    L = torch.logsumexp(X, -1) - X.gather(-1, idx[..., None])[..., 0]
    L = torch.where(valid, L, torch.full_like(L, float("nan")))
    loss.copy_((torch.where(m, ww * L, torch.zeros_like(L)).sum() / n).reshape(1))
    d = (X.softmax(-1) - F.one_hot(idx, C).to(X.dtype)) * (ww / n)[..., None]
    d = torch.where(valid[..., None], d, torch.full_like(d, float("nan")))
    dP.copy_(torch.where(m[..., None], d, torch.zeros_like(d)).reshape(B, -1))


def class_probs(P, C, softmax, out):
    out.copy_(P.reshape(P.shape[0], -1, C).softmax(-1).reshape(P.shape) if softmax else torch.sigmoid(P))


def patch_classification(monkeypatch):
    """emu.patch_engine plus the three classification wrappers."""
    from chemprop_b200 import engine

    emu.patch_engine(monkeypatch)
    for name in ("bce_loss", "ce_loss", "class_probs"):
        monkeypatch.setattr(engine, name, globals()[name])


# ---- the reference fixtures ---------------------------------------------------------------------------------------------
FIXTURES = {"binary": "fixture_mpnn_binary", "multiclass": "fixture_mpnn_multiclass"}


def build_model(kind: str, g: dict, precision: str = "fp32"):
    """EngineMPNN of the fixture's configuration holding its initial state (strict load of the reference's state dict minus
    the criterion's torchmetrics states)."""
    import chemprop_b200.nn as N

    if kind == "binary":
        pred = N.EngineBinaryClassificationFFN(n_tasks=3, input_dim=40, hidden_dim=24, n_layers=2)
    else:
        pred = N.EngineMulticlassClassificationFFN(n_classes=4, n_tasks=2, input_dim=40, hidden_dim=24, n_layers=2)
    model = N.EngineMPNN(N.BondMessagePassing(d_h=40, depth=3, precision=precision), N.MeanAggregation(), pred,
                         batch_norm=True)
    state = {k[len("param."):]: torch.from_numpy(np.asarray(v)) for k, v in g.items() if k.startswith("param.")}
    res = model.load_state_dict({k: v for k, v in state.items() if not k.endswith(("total_loss", "num_samples"))},
                                strict=True)
    assert not res.missing_keys and not res.unexpected_keys
    return model


def check_classification_head(kind: str, device: str, rtol: float = 2e-4, atol: float = 2e-6, graph: bool = False):
    """EngineMPNN.training_loss with a classification head (encoder -> aggregation -> batch norm -> FFN -> masked, weighted
    BCE / cross-entropy) against the reference's `MPNN.training_step`: loss, every gradient, the batch-norm running statistics
    after the step, eval-mode probabilities.  `graph`: the step runs as a captured CUDA graph (the recipe of
    tests/util.py::check_mpnn_head)."""
    g = load_golden(FIXTURES[kind])
    model = build_model(kind, g).to(device)
    model.train()
    bmg = golden_bmg(g, device)
    Y, w = torch.from_numpy(g["Y"]).to(device), torch.from_numpy(g["w"]).to(device)
    if graph:
        from chemprop_b200.graph import CudaGraphStep

        for p in model.parameters():
            p.grad = torch.zeros_like(p)
        rm0, rv0, nb0 = model.bn.running_mean.clone(), model.bn.running_var.clone(), model.bn.num_batches_tracked.clone()

        def fn(b):
            for p in model.parameters():
                p.grad.zero_()
            loss = model.training_loss(b, Y, w)
            loss.backward()
            return loss

        step = CudaGraphStep(fn)
        step(bmg)
        model.bn.running_mean.copy_(rm0); model.bn.running_var.copy_(rv0); model.bn.num_batches_tracked.copy_(nb0)
        loss = step(bmg).clone()
        assert step.captures == 1 and step.replays == 2
    else:
        loss = model.training_loss(bmg, Y, w)
        loss.backward()
    np.testing.assert_allclose(loss.detach().cpu().numpy(), g["loss"], rtol=rtol, atol=atol)
    for k, p in model.named_parameters():
        np.testing.assert_allclose(p.grad.cpu().numpy(), g["grad." + k], rtol=rtol, atol=atol, err_msg=k)
    for k in ("running_mean", "running_var", "num_batches_tracked"):
        np.testing.assert_allclose(getattr(model.bn, k).cpu().numpy(), g["after.bn." + k], rtol=1e-5, atol=1e-6, err_msg=k)
    model.eval()
    with torch.no_grad():
        probs = model(bmg)
    assert probs.shape == g["preds_eval"].shape
    np.testing.assert_allclose(probs.cpu().numpy(), g["preds_eval"], rtol=rtol, atol=1e-5)


@pytest.mark.parametrize("kind", sorted(FIXTURES))
def test_engine_mpnn_classification_matches_reference_training_step(kind, monkeypatch):
    patch_classification(monkeypatch)
    check_classification_head(kind, "cpu")


@pytest.mark.parametrize("kind", sorted(FIXTURES))
def test_reference_state_dict_loads_strictly_and_round_trips(kind):
    g = load_golden(FIXTURES[kind])
    model = build_model(kind, g)
    ref_keys = {k[len("param."):] for k in g if k.startswith("param.") and not k.endswith(("total_loss", "num_samples"))}
    assert set(model.state_dict()) == ref_keys
    tw = model.predictor.criterion.task_weights
    assert tw.shape == g["param.predictor.criterion.task_weights"].shape and not bool((tw == 1).all())


def test_fixtures_cover_the_cases_the_heads_must_handle():
    b, m = load_golden("fixture_mpnn_binary"), load_golden("fixture_mpnn_multiclass")
    for g in (b, m):
        assert np.isnan(g["Y"]).any() and g["w"].std() > 0
    soft = b["Y"][np.isfinite(b["Y"])]
    assert b["Y"].shape == (14, 3) and ((soft > 0) & (soft < 1)).any()
    assert m["Y"].shape == (14, 2) and m["preds_eval"].shape == (14, 2, 4)
    np.testing.assert_allclose(m["preds_eval"].sum(-1), 1.0, rtol=1e-6)


def test_predictor_shapes_hparams_and_n_tasks():
    import chemprop_b200.nn as N

    b = N.EngineBinaryClassificationFFN(n_tasks=12, input_dim=16, hidden_dim=8)
    assert b.n_tasks == 12 and b.output_dim == 12 and b.criterion.task_weights.shape == (1, 12)
    m = N.EngineMulticlassClassificationFFN(n_classes=5, n_tasks=3, input_dim=16, hidden_dim=8)
    assert m.n_tasks == 3 and m.n_classes == 5 and m.output_dim == 15 and m.criterion.task_weights.shape == (1, 3)
    for mod in (b, m):
        back = mod.hparams["cls"](**{k: v for k, v in mod.hparams.items() if k != "cls"})
        assert type(back) is type(mod) and back.n_tasks == mod.n_tasks and back.output_dim == mod.output_dim
    r = N.EngineRegressionFFN(n_tasks=2, input_dim=16, hidden_dim=8)
    assert set(r.hparams) == {"n_tasks", "input_dim", "hidden_dim", "n_layers", "dropout", "activation", "cls"}


@pytest.mark.parametrize("kind", ["binary", "multiclass"])
def test_criterion_mask_argument_and_bounded_masks(kind, monkeypatch):
    """`mask=` selects the same terms as NaN targets; lt_mask / gt_mask are refused."""
    import chemprop_b200.nn as N

    patch_classification(monkeypatch)
    torch.manual_seed(0)
    if kind == "binary":
        crit = N.EngineBinaryClassificationFFN(n_tasks=3, input_dim=4).criterion
        preds, Y = torch.randn(6, 3, dtype=torch.float64).float(), torch.randint(0, 2, (6, 3)).float()
    else:
        crit = N.EngineMulticlassClassificationFFN(n_classes=3, n_tasks=3, input_dim=4).criterion
        preds, Y = torch.randn(6, 3, 3), torch.randint(0, 3, (6, 3)).float()
    mask = torch.rand(6, 3) > 0.3
    a = crit(preds, Y, mask)
    b = crit(preds, torch.where(mask, Y, torch.full_like(Y, float("nan"))))
    assert torch.equal(a, b)
    with pytest.raises(NotImplementedError):
        crit(preds, Y, lt_mask=mask)


@pytest.mark.parametrize("kind", ["binary", "multiclass"])
def test_probability_outputs_carry_the_gradient_of_sigmoid_and_softmax(kind, monkeypatch):
    """chemprop's predictor `forward` is differentiable: the probabilities' mirror equals torch autograd through
    sigmoid / softmax."""
    from chemprop_b200.nn.head import ClassProbsFunction

    patch_classification(monkeypatch)
    torch.manual_seed(1)
    C = 1 if kind == "binary" else 4
    X = (torch.randn(7, 3 * C) * 3).requires_grad_(True)
    G = torch.randn(7, 3 * C)
    p = ClassProbsFunction.apply(X, C, kind != "binary")
    (p * G).sum().backward()
    X2 = X.detach().clone().requires_grad_(True)
    ref = torch.sigmoid(X2) if kind == "binary" else X2.view(7, 3, C).softmax(-1).view(7, -1)
    (ref * G).sum().backward()
    torch.testing.assert_close(p, ref.detach())
    torch.testing.assert_close(X.grad, X2.grad, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("fill", [float("nan"), 1e30], ids=["nan", "huge"])
@pytest.mark.parametrize("kind", ["binary", "multiclass"])
def test_classification_step_does_not_depend_on_uninitialised_memory(kind, fill, monkeypatch):
    """The poisoned-allocation differential on one classification training step, through the emulations: every dP entry and
    every probability is written."""
    from tests.uninit_matrix import assert_bit_identical, install_poison

    patch_classification(monkeypatch)
    g = load_golden(FIXTURES[kind])

    def run(f):
        with monkeypatch.context() as m:
            install_poison(m, f)
            model = build_model(kind, g).train()
            bmg = golden_bmg(g, "cpu")
            loss = model.training_loss(bmg, torch.from_numpy(g["Y"]), torch.from_numpy(g["w"]))
            loss.backward()
            out = {"loss": loss.detach().reshape(1)}
            out.update({"grad." + k: p.grad.detach() for k, p in model.named_parameters()})
            model.eval()
            with torch.no_grad():
                out["probs"] = model(bmg)
        return out

    assert_bit_identical(run(0.0), run(fill), f"{fill} fill")


def test_entry_points_validate_their_arguments_before_touching_the_device():
    """dmpnn_bce_loss / dmpnn_ce_loss / dmpnn_class_probs check their arguments on the host, before any CUDA call: callable
    (and failing cleanly, naming the entry point) without a GPU."""
    from chemprop_b200 import _lib

    lib = _lib.load()
    loss = np.zeros(1, dtype=np.float32)
    L = loss.ctypes.data
    # bce: T = 0, negative B, missing loss, null P with B > 0, short strides
    assert lib.dmpnn_bce_loss(None, 1, None, 1, None, None, 4, 0, L, None, 1, None) != 0
    assert b"bce_loss" in lib.dmpnn_last_error()
    assert lib.dmpnn_bce_loss(None, 1, None, 1, None, None, -1, 1, L, None, 1, None) != 0
    assert lib.dmpnn_bce_loss(None, 3, None, 3, None, None, 0, 3, None, None, 3, None) != 0
    assert lib.dmpnn_bce_loss(None, 3, None, 3, None, None, 5, 3, L, None, 3, None) != 0
    assert lib.dmpnn_bce_loss(L, 2, L, 3, None, None, 5, 3, L, None, 3, None) != 0
    assert b"bce_loss: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_bce_loss(L, 3, L, 3, None, None, 5, 3, L, L, 2, None) != 0
    # ce: C = 0, P's stride below T * C, dP's stride below T * C, Y's stride below T
    assert lib.dmpnn_ce_loss(L, 8, L, 2, None, None, 5, 2, 0, L, None, 8, None) != 0
    assert b"ce_loss" in lib.dmpnn_last_error()
    assert lib.dmpnn_ce_loss(L, 7, L, 2, None, None, 5, 2, 4, L, None, 8, None) != 0
    assert b"ce_loss: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_ce_loss(L, 8, L, 2, None, None, 5, 2, 4, L, L, 7, None) != 0
    assert lib.dmpnn_ce_loss(L, 8, L, 1, None, None, 5, 2, 4, L, None, 8, None) != 0
    assert lib.dmpnn_ce_loss(L, 2 ** 40, L, 2 ** 20, None, None, 5, 2 ** 20, 2 ** 20, L, None, 2 ** 40, None) != 0
    # probs: softmax flag outside {0, 1}, C = 0, null output, short strides; B = 0 needs no launch
    assert lib.dmpnn_class_probs(L, 4, 3, 4, 1, 2, L, 4, None) != 0
    assert b"class_probs" in lib.dmpnn_last_error()
    assert lib.dmpnn_class_probs(L, 4, 3, 4, 0, 1, L, 4, None) != 0
    assert lib.dmpnn_class_probs(L, 4, 3, 4, 1, 0, None, 4, None) != 0
    assert lib.dmpnn_class_probs(L, 4, 3, 2, 3, 1, L, 6, None) != 0
    assert lib.dmpnn_class_probs(L, 6, 3, 2, 3, 1, L, 5, None) != 0
    assert b"class_probs: row strides" in lib.dmpnn_last_error()
    assert lib.dmpnn_class_probs(None, 6, 0, 2, 3, 1, None, 6, None) == 0
