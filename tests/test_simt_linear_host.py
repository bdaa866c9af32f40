"""CPU tier: which instantiations of the SIMT f32 GEMMs (csrc/linear.cu: `dmpnn_linear_fwd`, `dmpnn_linear_wgrad`) the
engine launches, and whether tests/test_gpu_simt_linear.py has a case for each of them.

The census drives the engine's host logic through the kernel emulation (tests/emu.py) with a spy on `engine.linear_fwd` /
`engine.linear_wgrad`, over the configurations that reach these kernels:

- BondMessagePassing and AtomMessagePassing, fp32 and bf16, d_h in {300, 302, 2048}, d_v in {72, 133} (chemprop's v1 atom
  featuriser), f32 and bf16 feature transfer, forward and backward;
- an EngineMPNN with batch norm and a 3-layer EngineRegressionFFN at n_tasks 1 and 12 on each of them.

An entry is the operand types, which optional operands are present, `accumulate`, and whether N or K is 1 (the key of
`tests.test_gpu_simt_linear.fwd_key` / `wgrad_key`).  The GPU module's case table is imported without running it."""
import functools

import pytest
import torch

from tests import emu

KINDS = ("bond", "atom")
PRECISIONS = ("fp32", "bf16")
D_H = (300, 302, 2048)
D_V = (72, 133)
TRANSFER = (None, torch.bfloat16)


def _dt(t):
    return None if t is None else {torch.float32: "f32", torch.bfloat16: "bf16"}[t.dtype]


@functools.lru_cache(maxsize=None)
def census():
    """{key: first configuration that launched it} over the configuration grid of the module docstring."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph, make_molecules
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, EngineMPNN, EngineRegressionFFN
    from tests.test_gpu_simt_linear import fwd_key, wgrad_key

    seen: dict = {}
    with pytest.MonkeyPatch.context() as mp:
        emu.patch_engine(mp)
        mp.setattr(engine, "_WARNED", set())
        fwd, wgrad = engine.linear_fwd, engine.linear_wgrad
        where = [None]

        def spy_fwd(X1, K1, W, out, N, *, idx1=None, X2=None, K2=0, idx2=None, bias=None, res=None, **k):
            key = fwd_key(_dt(X1), _dt(X2) if K2 else None, _dt(res), _dt(out), idx1 is not None or idx2 is not None,
                          bias is not None, N, K1 + K2)
            seen.setdefault(key, where[0])
            return fwd(X1, K1, W, out, N, idx1=idx1, X2=X2, K2=K2, idx2=idx2, bias=bias, res=res, **k)

        def spy_wgrad(dY, X1, K1, dW, N, *, idx1=None, X2=None, K2=0, idx2=None, dbias=None, accumulate=False, R=None):
            key = wgrad_key(_dt(dY), _dt(X1), _dt(X2) if K2 else None, idx1 is not None or idx2 is not None,
                            dbias is not None, accumulate, N, K1 + K2)
            seen.setdefault(key, where[0])
            return wgrad(dY, X1, K1, dW, N, idx1=idx1, X2=X2, K2=K2, idx2=idx2, dbias=dbias, accumulate=accumulate, R=R)

        mp.setattr(engine, "linear_fwd", spy_fwd)
        mp.setattr(engine, "linear_wgrad", spy_wgrad)
        for kind in KINDS:
            for precision in PRECISIONS:
                for d_h in D_H:
                    for d_v in D_V:
                        for transfer in TRANSFER:
                            torch.manual_seed(0)
                            mgs = make_molecules(6, seed=d_h + d_v, mean_atoms=6.0, std_atoms=2.0, d_v=d_v)
                            bmg = BatchMolGraph(mgs, transfer_dtype=transfer)
                            cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
                            for n_tasks in (1, 12):
                                where[0] = (kind, precision, d_h, d_v, None if transfer is None else "bf16", n_tasks)
                                mpn = cls(d_v=d_v, d_h=d_h, depth=3, precision=precision)
                                model = EngineMPNN(mpn, predictor=EngineRegressionFFN(n_tasks=n_tasks, input_dim=d_h,
                                                                                     n_layers=3), batch_norm=True)
                                Y = torch.randn(len(mgs), n_tasks)
                                model.training_loss(bmg, Y).backward()
    return seen


def test_census_of_simt_linear_launches():
    """The census holds the paths the kernels serve: the head's GEMMs (N = 1 output, K = 1 input gradient at n_tasks 1),
    the atom fp32 tier's two-source W_h / W_o, the bond tier's gathered W_i, the bf16 tier's storage types past the
    tensor-core limits, and accumulation into dW_h."""
    from tests.test_gpu_simt_linear import fwd_key, wgrad_key

    seen = census()
    for key in seen:
        print("[simt-linear census]", key, "<-", seen[key])
    want = [
        fwd_key("f32", None, None, "f32", False, True, 1, 300),              # head: last layer, n_tasks 1
        fwd_key("f32", None, None, "f32", False, False, 300, 1),             # head: dX of the last layer, n_tasks 1
        fwd_key("f32", "f32", "f32", "f32", False, False, 300, 314),         # atom fp32: W_h on [N_b || SE] + H_0
        fwd_key("f32", "f32", None, "f32", True, False, 300, 147),           # bond fp32 off x3: W_i on V[src] || E[perm]
        fwd_key("f32", "bf16", None, "bf16", False, True, 2048, 2120),       # bf16 past the tensor-core limits: W_o
        fwd_key("bf16", None, "bf16", "bf16", False, False, 2048, 2048),     # ... W_h with a bf16 residual
        wgrad_key("f32", "f32", "f32", True, False, False, 300, 147),        # bond fp32: dW_i on gathered V[src] || E
        wgrad_key("bf16", "bf16", None, False, False, True, 2048, 2048),     # bf16 storage: dW_h accumulated
        wgrad_key("f32", "f32", None, False, True, False, 1, 300),           # head: dW and db of the last layer, n_tasks 1
    ]
    missing = [k for k in want if k not in seen]
    assert not missing, missing


def test_gpu_cases_cover_the_census():
    """Every census entry has a case in tests/test_gpu_simt_linear.py (FWD_CASES / WGRAD_CASES); deleting the only case of an
    entry fails here."""
    from tests.test_gpu_simt_linear import FWD_CASES, WGRAD_CASES

    have = {c.key for c in FWD_CASES} | {c.key for c in WGRAD_CASES}
    missing = sorted((k for k in census() if k not in have), key=str)
    assert not missing, missing
    print(f"[simt-linear census] {len(census())} entries, all covered by {len(FWD_CASES) + len(WGRAD_CASES)} GPU cases")
