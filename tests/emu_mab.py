"""TEST INFRASTRUCTURE ONLY.  torch-CPU emulation of dmpnn_linear_tc_rows_bf16 (engine.linear_tc_rows, the read-out
epilogues of the bf16 mol-atom-bond path), written from its contract in include/dmpnn.h, and `patch_engine`, which routes
engine.py's wrappers to tests/emu.py's emulations plus this one.  Rounds to bf16 exactly where the kernel stores bf16."""
from __future__ import annotations

import torch

from chemprop_b200 import engine
from tests import emu


def linear_tc_rows(A, K, Wpk, N, out, *, R=None, bias=None, act=emu.ACT_NONE, act_param=0.0, Y=None, from_preact=False,
                   out_row=None, res=None, res_row=None):
    R = A.shape[0] if R is None else R
    assert A.dtype == torch.bfloat16 and Wpk.shape == (N, K)
    if R == 0:
        return
    acc = A[:R, :K].float() @ Wpk.t()
    n16 = (N + 15) // 16 * 16
    if Y is None:                                   # forward mode
        assert out_row is None and res is None and res_row is None and not from_preact
        if bias is not None:
            acc = acc + bias.float()
        out[:R, :N] = emu._act(acc, act, act_param).to(out.dtype)
        if out.dtype == torch.bfloat16 and n16 > N:
            out[:R, N:n16] = 0
        return
    assert out.dtype == torch.bfloat16 and Y.dtype == torch.bfloat16 and bias is None   # mirror mode
    assert res_row is None or res is not None
    q = torch.arange(R) if out_row is None else out_row[:R].long()
    assert q.unique().numel() == R, "out_row repeats a row"
    if res is not None:
        s = torch.arange(R) if res_row is None else res_row[:R].long()
        acc = acc + res[s, :N].float()
    out[q, :N] = (acc * emu._dact(Y[q, :N].float(), act, act_param, from_preact)).to(out.dtype)
    if n16 > N:
        out[q, N:n16] = 0


def patch_engine(monkeypatch):
    """tests/emu.py's patch_engine plus the read-out epilogues of the mol-atom-bond path."""
    emu.patch_engine(monkeypatch)
    monkeypatch.setattr(engine, "linear_tc_rows", linear_tc_rows)
