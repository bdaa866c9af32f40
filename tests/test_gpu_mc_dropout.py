"""GPU tier: Monte Carlo dropout on the engine -- forward-only calls with the nn.Dropout modules in training mode.

(a) The 32 fused bond-step instantiations with keep bits that only forward-only calls launch (every activation but ReLU x
    FIRST x BIAS x FAR), with fixed keep bits, against float64 at the bound of test_gpu_fused_activations.py (half a bf16
    ulp + Lip(tau) x 2 h u sum |a w|).  Dropped elements must be exactly 0; kept ones carry the exact f32 scale 1 / (1 - p).
    `test_cases_cover_every_new_instantiation` fails when one of them has no case.
(b) Every forward-only path, mask for mask: BondMessagePassing fp32 (3xTF32 and SIMT GEMMs) and bf16 (fused step,
    directed and undirected, windows of molecules of more than 128 edges, the unfused step at depth 1 and with fused=False)
    and MABBondMessagePassing bf16, against oracle/restatement.py in float64 with the masks the run drew (the `_mask_fn`
    hook), at the bars of tests/test_gpu_zy_paths.py.
(c) Sampling: p = 0 or dropout in eval mode is bit-identical to the eval forward; two seeded DropoutEstimator runs are
    bit-identical, different seeds differ; with p > 0 the encoder alone gives a nonzero sample variance."""
import gc

import numpy as np
import pytest
import torch
from torch import nn

from tests.test_gpu_fused_activations import (ACTS, NAN, U, _banded, _batch, _buffer, _check_bound, _check_operand, _code,
                                              _lip, _operand_ref, _param, _tau64, _weights)

pytestmark = pytest.mark.gpu

P_DROP = 0.2
SCALE = float(np.float32(1.0) / np.float32(1.0 - P_DROP))      # the exact f32 1 / (1 - p) the engine passes


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------------
# (a) the new instantiations: keep bits with every activation but ReLU (which training already launches)
# ---------------------------------------------------------------------------------------------------------------------
def _new_instantiations():
    return {(a, first, bias, far) for a in ACTS if a != "relu" for first in (0, 1) for bias in (0, 1) for far in (0, 1)}


CASES = sorted(_new_instantiations(), key=str)


def _case_id(c):
    act, first, bias, far = c
    return "-".join(x for x in (act, "first" if first else "", "bias" if bias else "", "far" if far else "") if x)


def test_cases_cover_every_new_instantiation():
    assert len(_new_instantiations()) == 32 and set(CASES) == _new_instantiations()


@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_keep_bit_instantiation_vs_f64(case):
    from chemprop_b200.engine import bond_step_fused, pack_weight_bf16

    act, first, bias, far = case
    h = 300
    p = _param(act, len(_case_id(case)))
    what = _case_id(case)
    lay, lay_cpu = _batch(0, far, "")
    trp, tap, nt, wf, nw, dr = lay.step_tables()
    assert (wf is not None) == bool(far)
    rows, hp = lay.E, (h + 15) // 16 * 16
    ld = hp + 32
    g = torch.Generator(device="cuda").manual_seed(77 + len(what))
    W, b = _weights(h, g)
    Wb = W.bfloat16().double()
    H0 = _buffer(rows, h, ld, _banded(rows, h, g))
    Hin = H0 if first else _buffer(rows, h, ld, torch.randn(rows, h, device="cuda", generator=g) * 0.5)
    out = _buffer(rows, h, ld)
    out[:, h:hp] = NAN
    Mk = _buffer(rows, h, ld)
    Mk[:, h:hp] = NAN
    nj = hp // 16
    bits = torch.randint(-32768, 32768, (rows, nj), device="cuda", dtype=torch.int32, generator=g)
    keep = (((bits & 0xFFFF).unsqueeze(-1) >> torch.arange(16, device="cuda")) & 1).reshape(rows, hp)[:, :h].double()
    Wpk = pack_weight_bf16(W)
    bond_step_fused(Hin, H0, out, h, Wpk, b if bias else None, lay, _code(act), p, bool(first),
                    M_out=Mk if first else None, drop_bits=bits.to(torch.int16).contiguous(), drop_scale=SCALE)
    if not first:
        scratch = _buffer(rows, h, ld)
        bond_step_fused(Hin, H0, scratch, h, Wpk, None, lay, _code("none"), 0.0, True, M_out=Mk)
    torch.cuda.synchronize()
    X = Hin[:, :h].double()
    if first:
        X = _tau64(act, p, X)
    _check_operand(Mk, _operand_ref(lay, lay_cpu, X.bfloat16().float(), h, False, through_rev=False), h, what)
    A = Mk[:, :h].double()
    Z = A @ Wb.t()
    Ua = A.abs() @ Wb.abs().t()
    h0 = H0[:, :h].double()
    bd = b.double() if bias else torch.zeros(h, dtype=torch.float64, device="cuda")
    z = Z + h0 + bd
    y = _tau64(act, p, z) * keep * SCALE
    delta = SCALE * (_lip(act, p) * (h * 2 * U * Ua + 3 * U * (Z.abs() + h0.abs() + bd.abs())) + 8 * U * y.abs() / SCALE)
    got = out[:, :h]
    dropped = keep == 0
    assert 0.3 < float(dropped.double().mean()) < 0.7
    assert bool((got.float()[dropped] == 0).all()), f"{what}: a dropped element is not exactly 0"
    worst, mean = _check_bound(got, y, delta * keep, what)
    # kept elements carry 1 / (1 - p): without it they would sit ~20 % below the reference, far outside the bound
    assert worst <= 1.0
    hp_cols = out[:, h:hp].float()
    assert not bool(hp_cols.ne(0).any()), f"{what}: columns [h, pad16(h)) not zero"
    assert bool(torch.isnan(out[:, hp:].float()).all()), f"{what}: stray writes past pad16(h)"
    print(f"[mc-dropout] {what}: worst err / bound {worst:.3f}, mean {mean:.3f}")


# ---------------------------------------------------------------------------------------------------------------------
# (b) every forward-only path, mask for mask against the f64 restatement
# ---------------------------------------------------------------------------------------------------------------------
class _Masks:
    """The `_mask_fn` hook: draws a {0, 1} keep mask like the buffer it is given and records it."""

    def __init__(self, p: float, seed: int):
        self.p, self.masks = p, []
        self.g = torch.Generator(device="cuda").manual_seed(seed)

    def __call__(self, like):
        m = (torch.rand(like.shape, device=like.device, generator=self.g) >= self.p).to(like.dtype)
        self.masks.append(m)
        return m


def _mol_batch(n_mols: int, seed: int, big: int = 0, oversized: bool = False):
    from chemprop_b200.data import make_molecule, make_molecules

    rng = np.random.default_rng(seed)
    mgs = make_molecules(n_mols, seed=seed, mean_atoms=22, std_atoms=6, min_atoms=1, shuffle_edges=True)
    mgs += [make_molecule(rng, int(rng.integers(70, 140)), 72, 14) for _ in range(big)]
    if oversized:
        mgs.append(make_molecule(rng, 160, 72, 14))
    return mgs


PATHS = {
    # name: (module kind, precision, depth, undirected, activation, extra constructor kwargs, batch kwargs, bar)
    "bond-fp32-x3-relu": ("bond", "fp32", 3, False, "relu", {}, {}, 1e-5),
    "bond-fp32-simt-tanh-h30": ("bond", "fp32", 3, False, "tanh", dict(d_h=30), {}, 1e-5),
    "bond-fp32-undirected-elu": ("bond", "fp32", 3, True, "elu", {}, {}, 1e-5),
    "bond-bf16-fused-tanh": ("bond", "bf16", 3, False, "tanh", {}, {}, 1e-2),
    "bond-bf16-fused-relu": ("bond", "bf16", 3, False, "relu", {}, {}, 1e-2),
    "bond-bf16-fused-undirected-leakyrelu": ("bond", "bf16", 3, True, "leakyrelu", {}, {}, 1e-2),
    "bond-bf16-fused-windows-elu": ("bond", "bf16", 3, False, "elu", {}, dict(big=12, oversized=True), 1e-2),
    "bond-bf16-unfused-tanh": ("bond", "bf16", 3, False, "tanh", dict(fused=False), {}, 1e-2),
    "bond-bf16-depth1-tanh": ("bond", "bf16", 1, False, "tanh", {}, {}, 1e-2),
    "mab-bond-bf16-tanh": ("mab", "bf16", 3, False, "tanh", {}, {}, 1e-2),
}


@pytest.mark.parametrize("name", sorted(PATHS))
def test_forward_only_path_mask_for_mask(name):
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.engine import get_layout
    from chemprop_b200.nn import BondMessagePassing, MABBondMessagePassing
    from oracle import restatement as R

    kind, precision, depth, undirected, act, extra, bkw, bar = PATHS[name]
    torch.manual_seed(5)
    mgs = _mol_batch(1500, seed=9, **bkw)
    bmg, ref = BatchMolGraph(mgs), BatchMolGraph(mgs)
    d_h = extra.get("d_h", 300)
    cls = MABBondMessagePassing if kind == "mab" else BondMessagePassing
    mp = cls(d_h=d_h, depth=depth, bias=True, dropout=P_DROP, activation=act, undirected=undirected, precision=precision)
    if kind != "mab":
        mp.fused = extra.get("fused", True)
    P = {k: v.detach().double() for k, v in mp.state_dict().items()}
    mp = mp.cuda().eval()
    mp.dropout.train()
    masks = _Masks(P_DROP, seed=len(name))
    mp._mask_fn = masks
    bmg.to("cuda")
    with torch.inference_mode():
        assert not mp.uses_composed_tier() if kind == "mab" else not mp.uses_composed_tier(get_layout(bmg))
        out = mp(bmg)
    torch.cuda.synchronize()
    lay = get_layout(bmg)
    perm = lay.perm.long().cpu()
    n_edge_sites = depth - 1
    assert len(masks.masks) == n_edge_sites + (2 if kind == "mab" else 1)
    E, V = lay.E, lay.V
    ref_masks = []
    for m in masks.masks[:n_edge_sites]:          # drawn over the dst-sorted rows: back to the caller's edge order
        m = m[:E, :d_h].double().cpu()
        mm = torch.empty_like(m)
        mm[perm] = m
        ref_masks.append(mm)
    ref_masks.append(masks.masks[n_edge_sites][:V, :d_h].double().cpu())
    if kind == "mab":
        ref_masks.append(masks.masks[-1][:E, :d_h].double().cpu())      # H_e is in the caller's edge order already
    s = 1.0 / (1.0 - float(np.float32(P_DROP)))
    ref_masks = [m * s for m in ref_masks]
    ap = {"leakyrelu": 0.1, "elu": 1.0}.get(act)
    args = (ref.V.double(), ref.E.double(), ref.edge_index, ref.rev_edge_index, P["W_i.weight"], P.get("W_i.bias"),
            P["W_h.weight"], P.get("W_h.bias"))
    if kind == "mab":
        H_v, H_e = out
        Hv_ref, He_ref = R.mab_forward("bond", *args, P["W_vo.weight"], P["W_vo.bias"], P["W_eo.weight"], P["W_eo.bias"],
                                       depth, act, dropout_masks=ref_masks, act_param=ap)
        pairs = [(H_v, Hv_ref), (H_e, He_ref)]
    else:
        H_ref = R.message_passing_forward("bond", *args, P["W_o.weight"], P["W_o.bias"], depth, act, undirected,
                                          dropout_masks=ref_masks, act_param=ap)
        pairs = [(out, H_ref)]
    for got, want in pairs:
        got = got.double().cpu()
        scale = max(1.0, float(want.abs().max()))
        err = (got - want).abs().max().item()
        print(f"[mc-dropout] {name}: max err {err:.3e}, bar {bar * scale:.3e}")
        assert err <= bar * scale, (name, err, bar * scale)


# ---------------------------------------------------------------------------------------------------------------------
# (c) sampling
# ---------------------------------------------------------------------------------------------------------------------
def _model(precision: str, act: str = "relu", p: float = P_DROP, head_p: float = 0.0):
    from chemprop_b200.nn import BondMessagePassing, EngineMPNN, EngineRegressionFFN

    torch.manual_seed(0)
    mp = BondMessagePassing(d_h=300, depth=3, dropout=p, activation=act, precision=precision)
    return EngineMPNN(mp, predictor=EngineRegressionFFN(n_tasks=2, input_dim=300, dropout=head_p)).cuda()


def _batches(n: int = 3):
    from chemprop_b200.data import BatchMolGraph, TrainingBatch

    out = []
    for i in range(n):
        bmg = BatchMolGraph(_mol_batch(400, seed=20 + i))
        bmg.to("cuda")
        out.append(TrainingBatch(bmg, None, None, None, None, None, None))
    return out


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_inactive_dropout_is_the_eval_forward(precision):
    from chemprop_b200.uncertainty import DropoutEstimator

    batches = _batches()
    model = _model(precision)
    ref = model.predict(batches)
    zero = DropoutEstimator(ensemble_size=2, dropout=None)
    for m in model.modules():
        if isinstance(m, nn.Dropout):
            m.p = 0.0
    mean, var = zero(batches, [model])
    assert torch.equal(mean[0], ref.float()) and bool((var == 0).all())
    for m in model.modules():
        if isinstance(m, nn.Dropout):
            m.p = P_DROP
    assert torch.equal(model.predict(batches), ref)          # dropout configured, eval mode: the eval forward


@pytest.mark.parametrize("precision,act", [("fp32", "relu"), ("bf16", "tanh"), ("bf16", "relu")])
def test_seeded_samples_repeat_and_vary(precision, act):
    from chemprop_b200.uncertainty import DropoutEstimator

    batches = _batches()
    model = _model(precision, act)
    est = DropoutEstimator(ensemble_size=4)
    torch.manual_seed(123)
    a = est(batches, [model])
    torch.manual_seed(123)
    b = est(batches, [model])
    torch.manual_seed(124)
    c = est(batches, [model])
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not torch.equal(a[0], c[0])
    # the head has no dropout here: the whole sample variance comes from the encoder
    assert float(a[1].mean()) > 0 and bool((a[1] >= 0).all())
    assert a[0].shape == (1, 1200, 2) and a[1].shape == (1, 1200, 2)
    assert all(m.training for m in model.modules())          # flags restored (the model was built in train mode)
