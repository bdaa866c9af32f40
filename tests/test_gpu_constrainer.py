"""GPU tier: dmpnn_constrain_fwd / dmpnn_constrain_bwd and the constrained EngineMolAtomBondMPNN training step on the device.

- ConstrainerFFN (engine MLP + the two kernels) against the reference's op sequence in float64 for every case of
  tests/test_constrainer_host.py, with and without caller offsets; the kernels alone (forward, dP, dKl) against the
  float64 restatement, including a molecule of more than 1024 rows; constrained sums equal the constraints and
  unconstrained columns are bit-equal to the input.
- A shape the reference rejects, under graph capture: NaN in the constrained columns and the status word, no host read.
- The constrained training step of the fixture_mab_model_constrained configuration (fp32 and bf16 encoders) captured by
  CudaGraphStep: replayed loss and every gradient bit-identical to the eager step; one eager step under
  torch.cuda.set_sync_debug_mode("error")."""
from __future__ import annotations

import numpy as np
import pytest
import torch

from tests.test_constrainer_host import CASES, check_against_reference, constrain_bwd, constrain_fwd
from tests.test_mab_model_host import _level_inputs, assert_constraints_met, build_training_model
from tests.util import golden_bmg, load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("name,rows,t,n_c,cols", CASES, ids=[c[0] for c in CASES])
def test_constrainer_matches_the_reference_op_sequence(name, rows, t, n_c, cols):
    check_against_reference(name, rows, t, n_c, cols, DEV, atol=2e-5)


KERNEL_CASES = CASES + [("large_molecules", [1500, 3, 1, 2049, 0], 3, 3, [0, 2, 1]),
                        ("large_broadcast", [4000, 7], 2, 1, [1])]


@pytest.mark.parametrize("name,rows,t,n_c,cols", KERNEL_CASES, ids=[c[0] for c in KERNEL_CASES])
def test_kernels_against_float64(name, rows, t, n_c, cols):
    from chemprop_b200.nn.constrainer import ConstrainFunction

    g = torch.Generator().manual_seed(3)
    m, R = len(rows), sum(rows)
    Kl = torch.randn((R, n_c), generator=g) * 0.5
    P = torch.randn((R, t), generator=g)
    C = torch.randn((m, t), generator=g) * 3
    if cols is not None:
        C[0, [j for j in range(t) if j not in cols]] = float("nan")
    G = torch.randn((R, t), generator=g)
    ptr = torch.tensor([0] + np.cumsum(rows).tolist(), dtype=torch.int32)
    # float64 restatement of the contract
    out64, st = torch.empty((R, t), dtype=torch.float64), torch.zeros(1, dtype=torch.int32)
    dP64, dK64 = torch.empty((R, t), dtype=torch.float64), torch.empty((R, n_c), dtype=torch.float64)
    constrain_fwd(Kl.double(), P.double(), ptr, C.double(), out64, st)
    constrain_bwd(G.double(), Kl.double(), P.double(), ptr, C.double(), dP64, dK64)
    # the kernels
    Kd, Pd = Kl.to(DEV).requires_grad_(True), P.to(DEV).requires_grad_(True)
    out, status = ConstrainFunction.apply(Kd, Pd, ptr.to(DEV), C.to(DEV))
    out.backward(G.to(DEV))
    assert int(status.item()) == 0
    scale = lambda x: max([1.0] + x.abs().flatten().tolist())  # noqa: E731
    tol = lambda ref, n: 8 * n * 2.0 ** -24 * scale(ref)  # noqa: E731   f32 sums over n rows, in units of the output's scale
    n = max(rows) if rows else 1
    for got, ref, what in ((out, out64, "P'"), (Pd.grad, dP64, "dP"), (Kd.grad, dK64, "dKl")):
        err = max([0.0] + (got.detach().double().cpu() - ref).abs().flatten().tolist())
        assert err <= tol(ref, n), (name, what, err, tol(ref, n))
    unset = [j for j in range(t) if cols is not None and j not in cols]
    assert torch.equal(out.detach()[:, unset].cpu(), P[:, unset])
    assert torch.equal(Pd.grad[:, unset].cpu(), G[:, unset])
    setc = list(range(t)) if cols is None else cols
    if R and setc:
        seg = torch.repeat_interleave(torch.arange(m), torch.tensor(rows))
        sums = torch.zeros((m, t), dtype=torch.float64).index_add_(0, seg, out.detach().double().cpu())
        own = torch.tensor(rows) > 0
        torch.testing.assert_close(sums[own][:, setc], C.double()[own][:, setc], rtol=1e-5, atol=1e-4 * n ** 0.5)
    # repeated launches give the same bits
    out2, _ = ConstrainFunction.apply(Kl.to(DEV), P.to(DEV), ptr.to(DEV), C.to(DEV))
    assert torch.equal(out2, out.detach())


def test_rejected_shape_under_capture_gives_nan_and_the_status_word():
    import chemprop_b200.nn as N

    torch.manual_seed(0)
    rows, t = [3, 5, 2], 4
    R = sum(rows)
    mod = N.ConstrainerFFN(n_constraints=2, fp_dim=8, hidden_dim=8).to(DEV)
    fp, preds = torch.randn(R, 8, device=DEV), torch.randn(R, t, device=DEV)
    batch = torch.repeat_interleave(torch.arange(3), torch.tensor(rows)).to(DEV)
    cons = torch.randn(3, t, device=DEV)
    cons[0, 1] = float("nan")                                       # 3 set columns, 2 MLP outputs
    offsets = torch.tensor([0, 3, 8, 10], dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="2 outputs and the constraints 3 set columns"):
        mod(fp, preds, batch, cons, offsets=offsets)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph):
        out = mod(fp, preds, batch, cons, offsets=offsets)
    status = mod.status
    graph.replay()
    torch.cuda.synchronize()
    assert int(status.item()) == 3
    assert torch.isnan(out[:, [0, 2, 3]]).all()
    assert torch.equal(out[:, 1], preds[:, 1])


def _constrained_step(precision):
    g = load_golden("fixture_mab_model_constrained")
    bmg = golden_bmg(g, DEV)
    targetss, weightss, lts, gts, cons, X_d = _level_inputs(g, DEV)

    def make():
        return build_training_model("constrained", g, precision).to(DEV).train()

    def step(m, b):
        return m.training_loss(b, targetss, weightss, None, None, X_d, lt_masks=lts, gt_masks=gts, constraints=cons)

    return make, step, bmg, cons


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_constrained_mab_training_step_replays_as_a_graph(precision):
    from chemprop_b200.graph import CudaGraphStep

    make, step, bmg, cons = _constrained_step(precision)
    eager_model = make()
    loss = step(eager_model, bmg)
    loss.backward()
    eager = loss.detach().clone()
    eager_grads = {k: p.grad.clone() for k, p in eager_model.named_parameters() if p.grad is not None}
    assert any(k.startswith("atom_constrainer.") for k in eager_grads)
    assert any(k.startswith("bond_constrainer.") for k in eager_grads)

    model = make()
    for p in model.parameters():
        p.grad = torch.zeros_like(p)

    def fn(b):
        for p in model.parameters():
            p.grad.zero_()
        out = step(model, b)
        out.backward()
        return out

    cg = CudaGraphStep(fn)
    for _ in range(3):
        out = cg(bmg)
        assert torch.equal(out, eager)
        for k, p in model.named_parameters():
            if k in eager_grads:
                assert torch.equal(p.grad, eager_grads[k]), k
    assert cg.captures == 1 and cg.replays >= 1
    model.eval()
    with torch.no_grad():
        assert_constraints_met(bmg, model(bmg, constraints=cons), cons)


def test_constrained_mab_eager_step_never_synchronises():
    make, step, bmg, cons = _constrained_step("fp32")
    model = make()
    step(model, bmg)                           # first call: builds and caches the batch layout
    for p in model.parameters():
        p.grad = None
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = step(model, bmg)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(loss).item()
    assert model.atom_constrainer.status is not None and int(model.atom_constrainer.status.item()) == 0
