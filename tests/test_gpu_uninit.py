"""GPU tier: the poisoned-allocation differential (tests/uninit_matrix.py) on the H100 kernels -- every module configuration
run with the library's uninitialised floating-point buffers zero-filled, NaN-filled and 1e30-filled must give bit-identical,
finite outputs and gradients -- and the fused depth step's own contract on the columns it may not read: NaN in the row
padding [pad16(h), ld) of every input changes no bit of its output, and columns [h, pad16(h)) of every output are zeros."""
from __future__ import annotations

import pytest
import torch

from tests.uninit_matrix import CASES, POISONS, assert_bit_identical, case_id, install_poison, make_batch, run_case

pytestmark = pytest.mark.gpu


@pytest.fixture
def run_filled(monkeypatch):
    """run_filled(case, bmg, fill): the case with every floating-point torch.empty / empty_like / engine._empty_hidden of the
    library filled with `fill` (0.0 for the reference run)."""

    def run(c, bmg, fill):
        with monkeypatch.context() as m:
            install_poison(m, fill)
            out = run_case(c, bmg, "cuda")
        torch.cuda.synchronize()
        return out

    return run


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_outputs_do_not_depend_on_uninitialised_memory(case, run_filled):
    bmg = make_batch(case, "cuda", n_mols=150)
    ref = run_filled(case, bmg, 0.0)
    for name in sorted(POISONS):
        assert_bit_identical(ref, run_filled(case, bmg, POISONS[name]), f"{name} fill")


# ---- kernel level: the fused step never reads past pad16(h), and writes zeros in [h, pad16(h)) ---------------------------
def _inputs(lay_rows, h, n, seed):
    """n bf16 hidden buffers [rows, ld] with data in [0, h) and zeros past it (the engine's row stride ld = pad64(h))."""
    from chemprop_b200.engine import pad_hidden

    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for _ in range(n):
        t = torch.zeros(lay_rows, pad_hidden(h), dtype=torch.bfloat16, device="cuda")
        t[:, :h] = (torch.randn(lay_rows, h, device="cuda", generator=g) * 0.7).bfloat16()
        out.append(t)
    return out


def _check_padding_contract(launch, ins, outs, h):
    """launch() twice: with zeros and with NaN in columns [pad16(h), ld) of every input.  Outputs are NaN-filled before each
    launch; columns [0, pad16(h)) must come out finite, identical bit for bit, and zero in [h, pad16(h))."""
    hp = (h + 15) // 16 * 16
    results = []
    for poison in (False, True):
        for t in ins:
            t[:, hp:] = float("nan") if poison else 0.0
        for t in outs:
            t.fill_(float("nan"))
        launch()
        torch.cuda.synchronize()
        results.append([t[:, :hp].clone() for t in outs])
    for i, (a, b) in enumerate(zip(*results)):
        assert bool(torch.isfinite(a.float()).all()), f"output {i}: columns below pad16(h) left unwritten or NaN"
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"output {i}: depends on columns past pad16(h)"
        assert hp == h or not bool(a[:, h:].float().ne(0).any()), f"output {i}: columns [h, pad16(h)) not zero"


def _bond_layout(big):
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.engine import get_layout

    mgs = make_molecules(400, seed=5, shuffle_edges=True, min_atoms=1)
    if big:
        mgs += make_molecules(6, seed=6, mean_atoms=90.0, std_atoms=10.0, min_atoms=70, max_atoms=120, shuffle_edges=True)
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = get_layout(bmg)
    assert (lay.max_tile_rows > 128) == big
    return lay


def _weights(h, seed):
    from chemprop_b200.engine import pack_weight_bf16

    g = torch.Generator(device="cuda").manual_seed(seed)
    W = torch.randn(h, h, device="cuda", generator=g) / h ** 0.5
    b = torch.randn(h, device="cuda", generator=g) * 0.1
    return pack_weight_bf16(W), pack_weight_bf16(W.t().contiguous()), b


@pytest.mark.parametrize("h", [300, 100])
@pytest.mark.parametrize("big", [False, True], ids=["tiles", "windows"])
def test_bond_step_ignores_row_padding(h, big):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import bond_step_bwd_fused, bond_step_fused

    lay = _bond_layout(big)
    Wpk, WpkT, b = _weights(h, 1)
    H0, Hp, dZ, a0, a1 = _inputs(lay.E, h, 5, seed=2)
    Hp.relu_()
    Hn, M1, dO, G = (torch.empty_like(H0) for _ in range(4))
    R, T = _lib.ACT_RELU, _lib.ACT_TANH
    _check_padding_contract(lambda: bond_step_fused(H0, H0, Hn, h, Wpk, b, lay, R, 0.0, True, M_out=M1), [H0], [Hn, M1], h)
    _check_padding_contract(lambda: bond_step_fused(Hp, H0, Hn, h, Wpk, b, lay, T, 0.0, False), [Hp, H0], [Hn], h)
    _check_padding_contract(lambda: bond_step_bwd_fused(dZ, Hp, dO, h, WpkT, lay, R, 0.0, G_out=G), [dZ, Hp], [dO, G], h)
    _check_padding_contract(lambda: bond_step_bwd_fused(dZ, None, dO, h, WpkT, lay, R, 0.0, G_out=G), [dZ], [dO, G], h)
    _check_padding_contract(lambda: bond_step_bwd_fused(dZ, H0, dO, h, WpkT, lay, T, 0.0, y_is_preact=True, addends=(a0, a1)),
                            [dZ, H0, a0, a1], [dO], h)


@pytest.mark.parametrize("h", [300, 100])
def test_atom_step_ignores_row_padding(h):
    from chemprop_b200 import _lib
    from chemprop_b200.data import BatchMolGraph, make_cgr_graphs
    from chemprop_b200.engine import atom_step_bwd_fused, atom_step_fused, get_layout

    bmg = BatchMolGraph(make_cgr_graphs(60, seed=3))
    bmg.to("cuda")
    lay = get_layout(bmg)
    Wpk, WpkT, b = _weights(h, 4)
    H0, Hp, dZ = _inputs(lay.V, h, 3, seed=5)
    Hp.relu_()
    Hn, N1, dO, G = (torch.empty_like(H0) for _ in range(4))
    R, E = _lib.ACT_RELU, _lib.ACT_ELU
    _check_padding_contract(lambda: atom_step_fused(H0, H0, Hn, h, Wpk, b, lay, R, 0.0, True, N_out=N1), [H0], [Hn, N1], h)
    _check_padding_contract(lambda: atom_step_fused(Hp, H0, Hn, h, Wpk, None, lay, E, 1.0, False), [Hp, H0], [Hn], h)
    for Y, pre in ((Hp, False), (None, False), (H0, True)):
        _check_padding_contract(lambda: atom_step_bwd_fused(dZ, Y, dO, h, WpkT, lay, R, 0.0, G_out=G, y_is_preact=pre),
                                [dZ] + ([Y] if Y is not None else []), [dO, G], h)
