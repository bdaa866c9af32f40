"""CPU tier: which execution path each message-passing call takes outside the bf16 tier's main line -- the fp32 SIMT and
3xTF32 GEMMs, bf16 past the tensor-core limits, the fused forward with the generic mirror, undirected bonds off the fused
step, batches without edges or atoms, the two-launch atom step, the export op -- and the one-time RuntimeWarnings each call
emits.  Kernel wrappers are emulated (tests/emu.py); a call is recorded as in tests/test_host_logic.py's launch sequence.
The golden, tests/golden/launch_sequences_paths.json, is written by `python -m tests.test_path_plan_host`."""
import json
import os
import warnings

import pytest
import torch

from tests.test_host_logic import _LAUNCH_WRAPPERS, _launch_record

PATH_GOLDEN = "launch_sequences_paths.json"

# kind, precision, d_h, extra; patches: engine switches set for the case
PATH_CASES = {
    "bond-fp32-simt": ("bond", "fp32", 34, {}),
    "bond-fp32-x3": ("bond", "fp32", 36, {}),
    "bond-fp32-x3-disabled": ("bond", "fp32", 36, dict(patch={"X3_ENABLED": False})),
    "bond-bf16-over-limits": ("bond", "bf16", 320, {}),
    "bond-bf16-dh34": ("bond", "bf16", 34, {}),
    "bond-bf16-undirected-dh34": ("bond", "bf16", 34, dict(undirected=True)),
    "bond-bf16-noedges": ("bond", "bf16", 36, dict(noedges=True)),
    "bond-fp32-noedges": ("bond", "fp32", 36, dict(noedges=True)),
    "atom-fp32": ("atom", "fp32", 36, {}),
    "atom-bf16-over-limits": ("atom", "bf16", 320, {}),
    "atom-bf16-atom-fused-disabled": ("atom", "bf16", 36, dict(patch={"ATOM_FUSED_ENABLED": False})),
    "atom-bf16-noatoms": ("atom", "bf16", 36, dict(noatoms=True)),
    "atom-bf16-bigatom": ("atom", "bf16", 36, dict(bigatom=True)),
    "export-bond-bf16": ("bond", "bf16", 36, dict(export=True)),
    "export-bond-fp32": ("bond", "fp32", 36, dict(export=True)),
    "export-atom-bf16": ("atom", "bf16", 36, dict(export=True)),
    "export-atom-fp32": ("atom", "fp32", 36, dict(export=True)),
    "dropout-tier-relu": ("bond", "bf16", 36, dict(probe="relu")),
    "dropout-tier-tanh": ("bond", "bf16", 36, dict(probe="tanh")),
    "dropout-tier-relu-over-limits": ("bond", "bf16", 320, dict(probe="relu")),
    "dropout-tier-tanh-over-limits": ("bond", "bf16", 320, dict(probe="tanh")),
}


def _batch(kind, x):
    from chemprop_b200.data import BatchMolGraph, make_molecule, make_molecules

    d_v, d_e = (72, 14) if kind == "bond" else (106, 14)
    if x.get("noatoms"):
        return BatchMolGraph.from_tensors(torch.zeros((0, d_v)), torch.zeros((0, d_e)), torch.zeros((2, 0), dtype=torch.int64),
                                          torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64), 0), d_v, d_e
    if x.get("noedges"):
        import numpy as np

        rng = np.random.default_rng(2)
        return BatchMolGraph([make_molecule(rng, 1, d_v, d_e) for _ in range(3)]), d_v, d_e
    mgs = make_molecules(9, seed=3, mean_atoms=10, std_atoms=4, min_atoms=2, d_v=d_v, d_e=d_e, shuffle_edges=True)
    if x.get("bigatom"):
        mgs += make_molecules(1, seed=4, mean_atoms=135.0, std_atoms=3.0, min_atoms=130, max_atoms=140, d_v=d_v, d_e=d_e)
    return BatchMolGraph(mgs), d_v, d_e


def path_record(case: str, monkeypatch) -> dict:
    """Kernel-wrapper calls (forward and backward; forward only for the export op) and RuntimeWarning messages of one case;
    the dropout cases record the tier BondMessagePassing picks for a training batch instead of launches."""
    import inspect

    from chemprop_b200 import engine
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing, MeanAggregation
    from tests import emu_mab

    kind, precision, d_h, x = PATH_CASES[case]
    sigs = {n: inspect.signature(getattr(engine, n)) for n in _LAUNCH_WRAPPERS}
    emu_mab.patch_engine(monkeypatch)
    monkeypatch.setattr(engine, "_WARNED", set())
    for k, v in x.get("patch", {}).items():
        monkeypatch.setattr(engine, k, v)
    seq = []
    for n in _LAUNCH_WRAPPERS:
        f0 = getattr(engine, n)
        monkeypatch.setattr(engine, n, lambda *a, _f=f0, _n=n, **k: (seq.append(_launch_record(_n, sigs[_n], a, k)),
                                                                     _f(*a, **k))[1])
    torch.manual_seed(5)
    bmg, d_v, d_e = _batch(kind, x)
    cls = BondMessagePassing if kind == "bond" else AtomMessagePassing
    mp = cls(d_v=d_v, d_e=d_e, d_h=d_h, depth=3, bias=True, precision=precision, undirected=x.get("undirected", False),
             activation=x.get("probe", "relu"), dropout=0.2 if "probe" in x else 0.0)
    mp.train()
    out = {}
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        if "probe" in x:
            out["composed"] = mp.uses_composed_tier(engine.get_layout(bmg))
        elif x.get("export"):
            from chemprop_b200 import export

            cfg = mp._config()
            H = export.mp_forward(bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch, mp.W_i.weight, mp.W_i.bias,
                                  mp.W_h.weight, mp.W_h.bias, mp.W_o.weight, mp.W_o.bias, type(mp)._kind, cfg.depth, cfg.act,
                                  cfg.act_param, cfg.undirected, precision == "bf16", True)
            out["dtype"] = str(H.dtype)
        else:
            assert not mp.uses_composed_tier(engine.get_layout(bmg))
            H = mp(bmg)
            MeanAggregation()(H, bmg.batch).float().square().sum().backward()
            out["dtype"] = str(H.dtype)
    out["launches"] = seq
    out["warnings"] = [str(w.message) for w in caught if issubclass(w.category, RuntimeWarning)]
    return json.loads(json.dumps(out))


@pytest.mark.parametrize("case", list(PATH_CASES))
def test_execution_path_launch_sequence(case, monkeypatch):
    """The kernel launches, in order and with their sizes and flags, and the one-time RuntimeWarnings of every execution path
    the bf16 launch-sequence golden does not cover: a refactor of the host code's path choice must leave both as they are."""
    from tests.util import GOLDEN_DIR

    with open(os.path.join(GOLDEN_DIR, PATH_GOLDEN)) as fh:
        want = json.load(fh)[case]
    got = path_record(case, monkeypatch)
    assert got["warnings"] == want["warnings"]
    assert {k: v for k, v in got.items() if k != "launches"} == {k: v for k, v in want.items() if k != "launches"}
    for i, (g, w) in enumerate(zip(got["launches"], want["launches"])):
        assert g == w, (i, g, w)
    assert len(got["launches"]) == len(want["launches"])


if __name__ == "__main__":
    from tests.util import GOLDEN_DIR

    res = {}
    for c in PATH_CASES:
        with pytest.MonkeyPatch.context() as m:
            res[c] = path_record(c, m)
    with open(os.path.join(GOLDEN_DIR, PATH_GOLDEN), "w") as fh:
        json.dump(res, fh, indent=0)
        fh.write("\n")
