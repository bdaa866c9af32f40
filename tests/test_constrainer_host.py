"""CPU tier: ConstrainerFFN's engine path (ConstrainFunction over dmpnn_constrain_fwd / dmpnn_constrain_bwd, the MLP on
EngineLinear) through torch emulations of the two new wrappers, against the reference's op sequence (oracle.restatement.
constrain) in float64: predictions and the gradients of the fingerprints, the predictions and every MLP parameter.  The
emulations follow the kernels' contract in include/dmpnn.h and are shared with tests/test_gpu_constrainer.py."""
from __future__ import annotations

import pytest
import torch

from oracle import restatement as R
from tests import emu

NAN = float("nan")


# ---- torch emulations of the new wrappers (include/dmpnn.h) -----------------------------------------------------------------
def _pairing(Kl, Cn):
    """(constrained column indices, w column of each, whether the reference accepts the shape)."""
    cols = torch.nonzero(~torch.isnan(Cn[0])).flatten()
    n_c, nq = Kl.shape[1], int(cols.numel())
    ok = nq > 0 and (n_c == nq or n_c == 1)
    wcol = torch.zeros(nq, dtype=torch.long) if n_c == 1 or not ok else torch.arange(nq)
    return cols, wcol, ok


def _segments(ptr, m):
    cnt = (ptr[1:m + 1] - ptr[:m]).long().cpu()
    return torch.repeat_interleave(torch.arange(m), cnt).to(ptr.device)


def ref_constrain(Kl, P, ptr, Cn):
    """(P', dP(G), dKl(G)) of the kernels' contract in the dtype of the inputs; `status` as the kernel writes it."""
    m, t = Cn.shape
    cols, wcol, ok = _pairing(Kl, Cn)
    seg = _segments(ptr, m)
    e = Kl.exp()
    Z = torch.zeros((m, Kl.shape[1]), dtype=Kl.dtype, device=Kl.device).index_add_(0, seg, e)
    w = (e / Z[seg])[:, wcol]
    D = (Cn - torch.zeros((m, t), dtype=P.dtype, device=P.device).index_add_(0, seg, P))[:, cols]
    return cols, wcol, ok, seg, w, D


def constrain_fwd(Kl, P, ptr, Cn, out, status):
    cols, wcol, ok, seg, w, D = ref_constrain(Kl, P, ptr, Cn)
    status.fill_(0 if ok or cols.numel() == 0 else cols.numel())
    out.copy_(P)
    if cols.numel() == 0:
        return
    out[:, cols] = P[:, cols] + w * D[seg] if ok else NAN


def constrain_bwd(G, Kl, P, ptr, Cn, dP, dKl):
    cols, wcol, ok, seg, w, D = ref_constrain(Kl, P, ptr, Cn)
    dP.copy_(G)
    dKl.zero_()
    if cols.numel() == 0:
        return
    if not ok:
        dP[:, cols] = NAN
        dKl.fill_(NAN)
        return
    m = Cn.shape[0]
    Gc = G[:, cols]
    a = torch.zeros((m, cols.numel()), dtype=G.dtype, device=G.device).index_add_(0, seg, Gc * w)
    dP[:, cols] = Gc - a[seg]
    dKl.index_add_(1, wcol, D[seg] * w * (Gc - a[seg]))


def patch_constrainer(monkeypatch):
    """emu.patch_engine, the two new wrappers, and the constrainer's engine path on CPU tensors (eager: it may read)."""
    from chemprop_b200 import engine
    import chemprop_b200.nn.constrainer as con_mod

    emu.patch_engine(monkeypatch)
    monkeypatch.setattr(engine, "constrain_fwd", constrain_fwd)
    monkeypatch.setattr(engine, "constrain_bwd", constrain_bwd)
    monkeypatch.setattr(con_mod, "_on_engine", lambda t: True)
    monkeypatch.setattr(con_mod, "_may_synchronise", lambda: True)


# ---- cases ---------------------------------------------------------------------------------------------------------------
# (name, molecule row counts, t, n_c, constrained columns or None = all)
CASES = [
    ("all_constrained", [3, 1, 5, 2], 3, 3, None),
    ("some_nan", [4, 2, 6], 4, 2, [0, 2]),
    ("broadcast_n_c_1", [2, 5, 1, 3], 3, 1, [1, 2]),
    ("trailing_empty", [3, 0, 4, 0, 0], 2, 2, None),
    ("no_rows", [0, 0, 0], 2, 2, None),
    ("no_constrained_column", [3, 4], 3, 2, []),
]


def make_case(rows, t, n_c, cols, device="cpu", fp_dim=12, seed=0):
    g = torch.Generator().manual_seed(seed)
    m, R_ = len(rows), sum(rows)
    batch = torch.repeat_interleave(torch.arange(m), torch.tensor(rows, dtype=torch.long))
    fp = torch.randn((R_, fp_dim), generator=g)
    preds = torch.randn((R_, t), generator=g)
    cons = torch.randn((m, t), generator=g) * 3
    if cols is not None:
        unset = [j for j in range(t) if j not in cols]
        cons[0, unset] = NAN                  # row 0 decides (ffn.py:135); the other rows of an unset column are ignored
    mod = __import__("chemprop_b200.nn", fromlist=["ConstrainerFFN"]).ConstrainerFFN(
        n_constraints=n_c, fp_dim=fp_dim, hidden_dim=8, n_layers=2, activation="tanh")
    for p in mod.parameters():
        with torch.no_grad():
            p.copy_(torch.randn(p.shape, generator=g) * 0.5)
    G = torch.randn((R_, t), generator=g)
    return [x.to(device) for x in (fp, preds, batch, cons, G)] + [mod.to(device)]


def reference(mod, fp, preds, batch, cons, G):
    """The reference's forward (MLP then ffn.py:120-141) and its gradients, in float64 on the CPU."""
    ref = {k: v.detach().double().cpu().requires_grad_(True) for k, v in mod.named_parameters()}
    fp64 = fp.detach().double().cpu().requires_grad_(True)
    p64 = preds.detach().double().cpu().requires_grad_(True)
    X = fp64
    blocks = list(mod.ffn)
    for k, block in enumerate(blocks):
        if k > 0:
            X = torch.tanh(X)
        X = X @ ref[f"ffn.{k}.{len(block) - 1}.weight"].t() + ref[f"ffn.{k}.{len(block) - 1}.bias"]
    if torch.isnan(cons[0]).all():    # the engine keeps the parent's P' = P here for any n_c; the reference's broadcast
        out = p64 + 0 * X.sum()          # only copes with n_c == 1
    else:
        out = R.constrain(X, p64, batch.cpu(), cons.detach().double().cpu())
    (out * G.double().cpu()).sum().backward()
    return out.detach(), fp64.grad, p64.grad, {k: v.grad for k, v in ref.items()}


def check_against_reference(name, rows, t, n_c, cols, device, atol):
    fp, preds, batch, cons, G, mod = make_case(rows, t, n_c, cols, device)
    want, dfp, dpreds, dparams = reference(mod, fp, preds, batch, cons, G)
    fp.requires_grad_(True)
    preds.requires_grad_(True)
    m = cons.shape[0]
    offsets = torch.tensor([0] + list(torch.tensor(rows).cumsum(0)), dtype=torch.int32, device=device)
    for kw in ({}, {"offsets": offsets}):
        fp.grad = preds.grad = None
        mod.zero_grad(set_to_none=True)
        out = mod(fp, preds, batch, cons, **kw)
        (out * G).sum().backward()
        torch.testing.assert_close(out.detach().double().cpu(), want, rtol=1e-5, atol=atol, msg=name)
        unset = [j for j in range(t) if cols is not None and j not in cols]
        assert torch.equal(out.detach()[:, unset], preds.detach()[:, unset]), name     # copied bit for bit
        if sum(rows) and cols != []:
            sums = torch.zeros((m, t), dtype=torch.float64).index_add_(0, batch.cpu(), out.detach().double().cpu())
            setc = list(range(t)) if cols is None else cols
            own = torch.tensor(rows) > 0                  # an empty molecule has nothing to adjust
            torch.testing.assert_close(sums[own][:, setc], cons.double().cpu()[own][:, setc], rtol=1e-5, atol=1e-4)
        torch.testing.assert_close(fp.grad.double().cpu(), dfp, rtol=1e-4, atol=atol, msg=name)
        torch.testing.assert_close(preds.grad.double().cpu(), dpreds, rtol=1e-4, atol=atol, msg=name)
        for k, p in mod.named_parameters():
            got = torch.zeros_like(p) if p.grad is None else p.grad
            torch.testing.assert_close(got.double().cpu(), dparams[k], rtol=1e-4, atol=atol, msg=f"{name} {k}")
        assert int(mod.status.item()) == 0


@pytest.mark.parametrize("name,rows,t,n_c,cols", CASES, ids=[c[0] for c in CASES])
def test_engine_path_matches_the_reference_op_sequence(name, rows, t, n_c, cols, monkeypatch):
    patch_constrainer(monkeypatch)
    check_against_reference(name, rows, t, n_c, cols, "cpu", atol=2e-5)


def test_mismatched_mlp_width_raises_eagerly_as_the_reference_does(monkeypatch):
    patch_constrainer(monkeypatch)
    fp, preds, batch, cons, G, mod = make_case([3, 2, 4], 4, 2, [0, 1, 3])
    with pytest.raises(RuntimeError):                  # the reference: w (R x 2) * deviation[batch] (R x 3)
        R.constrain(mod.ffn[0][-1](fp).detach(), preds, batch, cons)
    with pytest.raises(RuntimeError, match="2 outputs and the constraints 3 set columns"):
        mod(fp, preds, batch, cons)
    assert int(mod.status.item()) == 3


def test_offsets_are_checked_and_the_mlp_runs_on_the_engine_gemms(monkeypatch):
    from chemprop_b200 import engine

    patch_constrainer(monkeypatch)
    fp, preds, batch, cons, G, mod = make_case([3, 2], 2, 2, None)
    with pytest.raises(ValueError, match="offsets"):
        mod(fp, preds, batch, cons, offsets=torch.tensor([0, 3], dtype=torch.int32))
    calls = []
    f = engine.linear_fwd
    monkeypatch.setattr(engine, "linear_fwd", lambda *a, **k: (calls.append(k.get("act")), f(*a, **k))[1])
    mod(fp, preds, batch, cons)
    assert calls == [engine.ACT_TANH, engine.ACT_TANH, engine.ACT_NONE]    # tanh fused into the two hidden GEMMs
    assert sorted(mod.state_dict()) == ["ffn.0.0.bias", "ffn.0.0.weight", "ffn.1.2.bias", "ffn.1.2.weight",
                                        "ffn.2.2.bias", "ffn.2.2.weight"]


def test_constrained_mab_step_through_the_engine_path(monkeypatch):
    """The constrained MolAtomBond training fixture with the constrainers on the engine path and the layout's offsets."""
    from tests.test_mab_model_host import assert_constraints_met, check_training, patch_mab_model

    patch_mab_model(monkeypatch)
    patch_constrainer(monkeypatch)
    calls = []
    import chemprop_b200.nn.constrainer as con_mod
    f = con_mod.ConstrainFunction.apply
    monkeypatch.setattr(con_mod.ConstrainFunction, "apply", lambda *a: (calls.append(a[2]), f(*a))[1])
    model, bmg, predss, cons = check_training("constrained", "cpu")
    assert_constraints_met(bmg, predss, cons)
    assert len(calls) == 4 and all(c.dtype == torch.int32 for c in calls)       # atoms and bonds, train and eval
