"""CPU tier: the poisoned-allocation differential (tests/uninit_matrix.py) on the kernel emulations of tests/emu.py +
tests/emu_mab.py.  The fused-step emulations read the padding columns [h, pad16(h)) the kernel reads, so a buffer that
reaches a fused step with those columns unwritten shows here as NaN rows (NaN fill) or changed bits, without a GPU."""
from __future__ import annotations

import pytest

from tests import emu_mab
from tests.uninit_matrix import CASES, POISONS, assert_bit_identical, case_id, install_poison, make_batch, run_case


@pytest.fixture
def run_filled(monkeypatch):
    """run_filled(case, bmg, fill): the case on the emulated kernels, with every floating-point torch.empty / empty_like /
    engine._empty_hidden of the library filled with `fill` (0.0 for the reference run)."""
    emu_mab.patch_engine(monkeypatch)

    def run(c, bmg, fill):
        with monkeypatch.context() as m:
            install_poison(m, fill)
            return run_case(c, bmg, "cpu")

    return run


@pytest.mark.parametrize("poison", sorted(POISONS))
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_outputs_do_not_depend_on_uninitialised_memory(case, poison, run_filled):
    bmg = make_batch(case, "cpu", n_mols=24)
    ref = run_filled(case, bmg, 0.0)
    got = run_filled(case, bmg, POISONS[poison])
    assert_bit_identical(ref, got, f"{poison} fill")
