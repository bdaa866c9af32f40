"""GPU tier: the classification heads on the H100 kernels (csrc/head.cu: dmpnn_bce_loss, dmpnn_ce_loss, dmpnn_class_probs)
-- the reference's own training step (tests/golden/fixture_mpnn_binary.npz, fixture_mpnn_multiclass.npz) eager and as one
CUDA graph, the kernels against f64 torch, a bf16 encoder with each head on a packed-loader batch as one graph, and the
poisoned-allocation differential on a classification step."""
from __future__ import annotations

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_classification_host import FIXTURES, check_classification_head

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind", sorted(FIXTURES))
def test_engine_mpnn_classification_matches_reference_training_step(kind, graph):
    check_classification_head(kind, "cuda", graph=graph)


# ---- kernels against f64 torch --------------------------------------------------------------------------------------------
def _close(got, ref, rtol=2e-5):
    """Elementwise, with an absolute floor scaled to the reference's magnitude (dP entries are O(1 / sum m))."""
    ref = ref.to(got.dtype)
    torch.testing.assert_close(got, ref, rtol=rtol, atol=rtol * float(ref.abs().max().clamp(min=1e-30)), equal_nan=True)


def _inputs(B, T, C, scale, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    P = torch.randn(B, T * C, device="cuda", generator=g) * scale
    w = torch.rand(B, device="cuda", generator=g) * 1.5 + 0.5
    tw = torch.rand(T, device="cuda", generator=g) * 1.5 + 0.5
    drop = torch.rand(B, T, device="cuda", generator=g) < 0.2
    return P, w, tw, drop, g


def _ref_loss(L, Y, w, tw):
    """f64 reduction of the unreduced loss L (b x T): sum w tw m L / sum m, 0 when every target is masked."""
    m = torch.isfinite(Y)
    n = m.sum().clamp(min=1)
    return torch.where(m, L * w.double().view(-1, 1) * tw.double().view(1, -1), torch.zeros_like(L)).sum() / n


def _run_bce(P, Y, w, tw):
    from chemprop_b200 import engine as K

    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    K.bce_loss(P, Y, w, tw, loss, dP)
    return loss, dP


def _run_ce(P, Y, w, tw, C):
    from chemprop_b200 import engine as K

    loss, dP = torch.empty(1, device="cuda"), torch.empty_like(P)
    K.ce_loss(P, Y, w, tw, C, loss, dP)
    return loss, dP


def _ref_bce(P, Y, w, tw):
    X = P.double().requires_grad_(True)
    m = torch.isfinite(Y)
    y = torch.where(m, Y, torch.zeros_like(Y)).double()
    loss = _ref_loss(F.binary_cross_entropy_with_logits(X, y, reduction="none"), Y, w, tw)
    loss.backward()
    return loss.detach(), X.grad


def _ref_ce(P, Y, w, tw, C):
    B = P.shape[0]
    X = P.double().requires_grad_(True)
    m = torch.isfinite(Y)
    lab = torch.where(m, Y, torch.zeros_like(Y)).long()            # targets.long(): truncation toward zero
    L = F.cross_entropy(X.view(B, -1, C).transpose(1, 2), lab, reduction="none")
    loss = _ref_loss(L, Y, w, tw)
    loss.backward()
    return loss.detach(), X.grad


@pytest.mark.parametrize("B", [1, 7, 10000])
@pytest.mark.parametrize("T", [1, 12])
@pytest.mark.parametrize("scale", [1.0, 100.0], ids=["logits1", "logits100"])
def test_bce_loss_kernel_vs_f64_torch(B, T, scale):
    P, w, tw, drop, g = _inputs(B, T, 1, scale, seed=B * 31 + T)
    Y = (torch.rand(B, T, device="cuda", generator=g) < 0.5).float()
    soft = torch.rand(B, T, device="cuda", generator=g) < 0.3
    Y = torch.where(soft, torch.rand(B, T, device="cuda", generator=g), Y)       # soft labels in [0, 1]
    Y[drop] = float("nan")
    if T == 12:
        Y[:, 5] = float("nan")                                                    # an all-masked task
    loss, dP = _run_bce(P, Y, w, tw)
    ref_loss, ref_dP = _ref_bce(P, Y, w, tw)
    assert bool(torch.isfinite(loss).all()) and bool(torch.isfinite(dP).all())
    _close(loss[0], ref_loss)
    _close(dP, ref_dP)
    assert not bool(dP[~torch.isfinite(Y)].ne(0).any())
    loss2, dP2 = _run_bce(P, Y, w, tw)
    assert torch.equal(loss, loss2) and torch.equal(dP, dP2)                      # fixed reduction order
    _close(_run_bce(P, Y, None, None)[0][0], _ref_bce(P, Y, torch.ones_like(w), torch.ones_like(tw))[0])


@pytest.mark.parametrize("B", [1, 7, 10000])
@pytest.mark.parametrize("T", [1, 12])
@pytest.mark.parametrize("C", [1, 2, 3, 10])
def test_ce_loss_kernel_vs_f64_torch(B, T, C):
    P, w, tw, drop, g = _inputs(B, T, C, 3.0, seed=B * 37 + T * 5 + C)
    Y = torch.randint(0, C, (B, T), device="cuda", generator=g).float()
    Y = Y + torch.rand(B, T, device="cuda", generator=g) * 0.99                  # fractional labels: truncated like .long()
    Y[drop] = float("nan")
    if T == 12:
        Y[:, 3] = float("nan")
    loss, dP = _run_ce(P, Y, w, tw, C)
    ref_loss, ref_dP = _ref_ce(P, Y, w, tw, C)
    _close(loss[0], ref_loss)
    _close(dP, ref_dP)
    masked = (~torch.isfinite(Y)).repeat_interleave(C, dim=1)
    assert not bool(dP[masked].ne(0).any())
    if C == 1:
        assert float(loss) == 0.0 and not bool(dP.ne(0).any())
    loss2, dP2 = _run_ce(P, Y, w, tw, C)
    assert torch.equal(loss, loss2) and torch.equal(dP, dP2)


def test_losses_with_every_target_masked_and_empty_batches():
    """The engine's convention (as dmpnn_mse_loss): no finite target -> loss 0 and every dP entry 0."""
    P = torch.randn(9, 12, device="cuda")
    Y = torch.full((9, 4), float("nan"), device="cuda")
    loss, dP = _run_ce(P, Y, None, None, 3)
    assert float(loss) == 0.0 and not bool(dP.ne(0).any())
    loss, dP = _run_bce(P[:, :4], Y, None, None)
    assert float(loss) == 0.0 and not bool(dP.ne(0).any())
    E = torch.empty(0, 6, device="cuda")
    assert float(_run_bce(E, torch.empty(0, 6, device="cuda"), None, None)[0]) == 0.0
    assert float(_run_ce(E, torch.empty(0, 2, device="cuda"), None, None, 3)[0]) == 0.0


def test_ce_out_of_range_labels_give_nan_in_their_row_only():
    P = torch.randn(6, 8, device="cuda")
    Y = torch.tensor([[0.0, 1.0], [3.9, 2.0], [4.0, 1.0], [-1.0, 0.0], [-0.5, 3.0], [float("nan"), 1.0]], device="cuda")
    loss, dP = _run_ce(P, Y, None, None, 4)
    assert bool(torch.isnan(loss).all())
    bad = torch.zeros(6, 2, dtype=torch.bool, device="cuda")
    bad[2, 0] = bad[3, 0] = True                            # 4.0 -> 4 and -1.0 -> -1 are outside [0, 4); -0.5 -> 0 is class 0
    nan_rows = torch.isnan(dP.view(6, 2, 4)).all(-1)
    assert torch.equal(nan_rows, bad) and bool(torch.isfinite(dP.view(6, 2, 4)[~bad]).all())
    ok = ~bad.any(1)
    loss_ok, _ = _run_ce(P[ok], Y[ok], None, None, 4)
    _close(loss_ok[0], _ref_ce(P[ok], Y[ok], torch.ones(int(ok.sum()), device="cuda"), torch.ones(2, device="cuda"), 4)[0])


def test_extreme_logits_stay_finite():
    P = torch.tensor([[1e4, -1e4, 100.0, -100.0]], device="cuda").repeat(3, 1)
    Y = torch.tensor([[0.0, 1.0, 0.0, 1.0], [1.0, 0.0, 1.0, 0.0], [0.5, 0.5, 0.5, 0.5]], device="cuda")
    loss, dP = _run_bce(P, Y, None, None)
    ref_loss, ref_dP = _ref_bce(P, Y, torch.ones(3, device="cuda"), torch.ones(4, device="cuda"))
    assert bool(torch.isfinite(loss).all()) and bool(torch.isfinite(dP).all())
    _close(loss[0], ref_loss)
    _close(dP, ref_dP)
    Yc = torch.tensor([[1.0, 0.0], [0.0, 1.0], [1.0, 1.0]], device="cuda")
    loss, dP = _run_ce(P, Yc, None, None, 2)
    ref_loss, ref_dP = _ref_ce(P, Yc, torch.ones(3, device="cuda"), torch.ones(2, device="cuda"), 2)
    assert bool(torch.isfinite(loss).all()) and bool(torch.isfinite(dP).all())
    _close(loss[0], ref_loss)
    _close(dP, ref_dP)


@pytest.mark.parametrize("B", [1, 7, 10000])
@pytest.mark.parametrize("T", [1, 12])
@pytest.mark.parametrize("C", [1, 2, 3, 10])
def test_class_probs_kernel_vs_f64_torch(B, T, C):
    from chemprop_b200 import engine as K

    g = torch.Generator(device="cuda").manual_seed(B + 13 * T + C)
    P = torch.randn(B, T * C, device="cuda", generator=g) * 5
    P[0, 0] = 1e4
    P[-1, -1] = -1e4
    out = torch.empty_like(P)
    K.class_probs(P, C, True, out)
    ref = P.double().view(B, T, C).softmax(-1).view(B, -1)
    assert bool(torch.isfinite(out).all())
    _close(out, ref, rtol=1e-5)
    torch.testing.assert_close(out.double().view(B, T, C).sum(-1), torch.ones(B, T, dtype=torch.float64, device="cuda"),
                               rtol=0, atol=1e-6)
    if C == 1:
        sig = torch.empty_like(P)
        K.class_probs(P, 1, False, sig)
        assert bool(torch.isfinite(sig).all())
        _close(sig, torch.sigmoid(P.double()), rtol=1e-5)
        out2 = torch.empty_like(P)
        K.class_probs(P, 1, False, out2)
        assert torch.equal(sig, out2)


# ---- a bf16 encoder with each head: one CUDA graph on a packed-loader batch ------------------------------------------------
def _loader_batch(kind):
    from chemprop_b200.data import PackedBatchLoader, PackedMolGraphDataset, make_molecules

    mgs = make_molecules(900, seed=41, shuffle_edges=True, min_atoms=1)
    rng = np.random.default_rng(5)
    T = 12 if kind == "binary" else 1
    Y = (rng.integers(0, 2, size=(900, T)) if kind == "binary" else rng.integers(0, 10, size=(900, T))).astype(np.float32)
    Y[rng.random(Y.shape) < 0.15] = np.nan
    w = rng.uniform(0.5, 2.0, size=900).astype(np.float32)
    ds = PackedMolGraphDataset.from_molgraphs(mgs).to("cuda")
    loader = PackedBatchLoader(ds, batch_size=512, shuffle=True, seed=3, device="cuda", arrays={"Y": Y, "w": w})
    it = iter(loader)
    batch = next(it)
    it.close()                                              # stops the loader's planner thread
    return batch, ds


def _head(kind, d_h):
    import chemprop_b200.nn as N

    if kind == "binary":
        return N.EngineBinaryClassificationFFN(n_tasks=12, input_dim=d_h, task_weights=torch.linspace(0.5, 2.0, 12))
    return N.EngineMulticlassClassificationFFN(n_classes=10, n_tasks=1, input_dim=d_h)


@pytest.mark.parametrize("kind", ["binary", "multiclass"])
def test_bf16_encoder_with_classification_head_in_a_cuda_graph(kind):
    """EngineMPNN(BondMessagePassing(precision="bf16"), MeanAggregation(), <classification head>, batch_norm=True) trains as
    ONE CudaGraphStep on a packed-loader batch; the replay equals the eager step bit for bit."""
    import chemprop_b200.nn as N
    from chemprop_b200.graph import CudaGraphStep

    batch, ds = _loader_batch(kind)
    torch.manual_seed(0)
    model = N.EngineMPNN(N.BondMessagePassing(d_v=ds.d_v, d_e=ds.d_e, precision="bf16"), N.MeanAggregation(),
                         _head(kind, 300), batch_norm=True).cuda().train()
    Y, w = batch.extras["Y"], batch.extras["w"]
    for p in model.parameters():
        p.grad = torch.zeros_like(p)

    def fn(b):
        for p in model.parameters():
            p.grad.zero_()
        loss = model.training_loss(b, Y, w)
        loss.backward()
        return loss

    eager = fn(batch.bmg).detach().clone()
    eager_grads = {k: p.grad.clone() for k, p in model.named_parameters()}
    assert bool(torch.isfinite(eager)) and float(eager) > 0
    step = CudaGraphStep(fn)
    for _ in range(2):
        out = step(batch.bmg).clone()
        assert torch.equal(out, eager)
        for k, p in model.named_parameters():
            assert torch.equal(p.grad, eager_grads[k]), k
    assert step.captures == 1 and step.replays == 2
    model.eval()
    with torch.no_grad():
        probs = model(batch.bmg)
    assert bool(torch.isfinite(probs).all())
    if kind == "multiclass":
        assert probs.shape == (len(batch.ids), 1, 10)
        torch.testing.assert_close(probs.sum(-1), torch.ones_like(probs[..., 0]), rtol=0, atol=1e-5)
    else:
        assert probs.shape == (len(batch.ids), 12) and bool(((probs >= 0) & (probs <= 1)).all())


# ---- poisoned allocations: every dP entry and every probability is written --------------------------------------------------
@pytest.mark.parametrize("kind", ["binary", "multiclass"])
def test_classification_step_does_not_depend_on_uninitialised_memory(kind, monkeypatch):
    import chemprop_b200.nn as N
    from tests.uninit_matrix import POISONS, assert_bit_identical, install_poison, make_batch

    bmg = make_batch({}, "cuda", n_mols=150)
    g = torch.Generator().manual_seed(9)
    T = 12 if kind == "binary" else 2
    Y = (torch.rand(150, T, generator=g) < 0.5).float() if kind == "binary" else torch.randint(0, 10, (150, T), generator=g).float()
    Y[torch.rand(150, T, generator=g) < 0.2] = float("nan")
    Y, w = Y.cuda(), (torch.rand(150, generator=g) + 0.5).cuda()

    def run(fill):
        with monkeypatch.context() as m:
            install_poison(m, fill)
            torch.manual_seed(1234)
            head = (N.EngineBinaryClassificationFFN(n_tasks=T, n_layers=2) if kind == "binary"
                    else N.EngineMulticlassClassificationFFN(n_classes=10, n_tasks=T, n_layers=2))
            model = N.EngineMPNN(N.BondMessagePassing(precision="bf16"), N.MeanAggregation(), head,
                                 batch_norm=True).cuda().train()
            loss = model.training_loss(bmg, Y, w)
            loss.backward()
            out = {"loss": loss.detach().reshape(1)}
            out.update({"grad." + k: p.grad.detach() for k, p in model.named_parameters()})
            model.eval()
            with torch.no_grad():
                out["probs"] = model(bmg)
        torch.cuda.synchronize()
        return {k: v.cpu() for k, v in out.items()}

    ref = run(0.0)
    for name in sorted(POISONS):
        assert_bit_identical(ref, run(POISONS[name]), f"{name} fill")
