"""CPU tier: every execution path of MABBond / MABAtomMessagePassing has a batch-scale float64 case on the GPU.

`mab_plan_key` (tests/test_gpu_zy_mab_paths.py, imported without running it) is evaluated over a grid -- kind, precision,
d_h in {298, 300, 320, 600}, depth 1 and 3, ReLU / tanh / PReLU, directed and undirected, training dropout or none, batches
with and without edges, with and without a molecule of more than 128 atoms, ATOM_FUSED_ENABLED on and off, the three
read-out combinations, d_e = 0, and d_v above the tensor-core GEMMs' K limit -- with a stub layout and the tensor-core
kernels reported available (modules on the meta device: no weights are initialised).  The set of keys it produces must
equal the set `CASES` declares: a path added to `plan()` or to the module fails here until a GPU case covers it, and a case
whose path went away fails too.

Some paths differ inside one key in ways a host bug can hide in -- why the composed tier was chosen, the GEMM kernels of the
composed tier, why the atom step took two launches, tau' of a non-idempotent activation at the edge head's entry, the bias,
descriptors, the PReLU weight.  `FACETS` names those, and each must be a case as well.  Every case must be needed for a key
or a facet, so deleting any case fails this module.

`test_case_through_emulation_vs_f64_oracle` runs every case at ~200 molecules on the CPU, the kernels replaced by the
rounding-aware emulation (tests/emu.py, tests/emu_mab.py), against the same float64 oracle and bars as the GPU run."""
import functools
import itertools
import warnings
from types import SimpleNamespace

import pytest
import torch

from tests.test_gpu_zy_mab_paths import CASES, case_dims, mab_plan_key, make_module, run_case

KINDS = ("bond", "atom")
PRECISIONS = ("bf16", "fp32")
D_H = (298, 300, 320, 600)
DEPTHS = (1, 3)
ACTS = ("relu", "tanh", "prelu")
READOUTS = ((True, True), (True, False), (False, True))


@functools.lru_cache(maxsize=None)
def _case_reason(name: str) -> str | None:
    return _reason(CASES[name])


def _reason(c: dict) -> str | None:
    """What composed_reason() of the case's module says, the tensor-core kernels reported available (None: the bf16 tier,
    or precision="fp32")."""
    from chemprop_b200 import engine

    if c["precision"] != "bf16":
        return None
    with torch.device("meta"):
        mp = make_module(c, device="meta")
    with pytest.MonkeyPatch.context() as m:
        m.setattr(engine, "_fused_available", lambda: True)
        return mp.train().composed_reason()


def _tc(c):
    return c["key"][1] == "tc"


def _non_idempotent(c):
    return c["act"] in ("tanh", "elu") and c["depth"] >= 3


def _two_launch(c):
    return c["key"][:3] == ("atom", "tc", False) and not c["key"][5]


# facet: predicate over a case's configuration (its declared key included)
FACETS = {
    "bf16 tier with bias": lambda c: _tc(c) and c["bias"],
    "bf16 tier without bias": lambda c: _tc(c) and not c["bias"],
    "bf16 LeakyReLU at a non-default slope": lambda c: _tc(c) and "act_param" in c,
    "bf16 bond with d_vd and d_ed descriptors": lambda c: _tc(c) and c["kind"] == "bond" and c.get("d_vd") and c.get("d_ed"),
    "bf16 atom with d_vd and d_ed descriptors": lambda c: _tc(c) and c["kind"] == "atom" and c.get("d_vd") and c.get("d_ed"),
    # the edge head's entry applies tau' of H^{T-1} from the stored output: an idempotent tau cannot show it taken twice
    "bf16 fused bond step, edge head, non-idempotent tau, depth >= 3":
        lambda c: c["key"][:3] == ("bond", "tc", True) and c["edge"] and _non_idempotent(c),
    "bf16 fused atom step, edge head, non-idempotent tau, depth >= 3":
        lambda c: c["key"][:3] == ("atom", "tc", True) and c["edge"] and _non_idempotent(c),
    "two-launch atom step, edge head, non-idempotent tau, depth >= 3":
        lambda c: _two_launch(c) and c["edge"] and _non_idempotent(c),
    "two-launch atom step from a molecule of more than 128 atoms, edge head":
        lambda c: _two_launch(c) and c.get("batch") == "oversized" and c["edge"],
    "two-launch atom step from ATOM_FUSED_ENABLED=False":
        lambda c: _two_launch(c) and c.get("patch", {}).get("ATOM_FUSED_ENABLED") is False,
    "two-launch atom step at depth 1, edge head": lambda c: _two_launch(c) and c["depth"] == 1 and c["edge"],
    "bond at depth 1, edge head (H^0 recomputed with tau)":
        lambda c: c["key"][:2] == ("bond", "tc") and c["depth"] == 1 and c["edge"] and not c["key"][5],
    "composed fp32 bond, d_h % 4 == 0 (3xTF32 W_h GEMM)":
        lambda c: c["precision"] == "fp32" and c["kind"] == "bond" and c["d_h"] % 4 == 0 and not c["key"][5],
    "composed fp32 bond, d_h % 4 != 0 (SIMT GEMMs)":
        lambda c: c["precision"] == "fp32" and c["kind"] == "bond" and c["d_h"] % 4 != 0 and not c["key"][5],
    "composed fp32 atom, d_h % 4 == 0": lambda c: c["precision"] == "fp32" and c["kind"] == "atom" and c["d_h"] % 4 == 0
                                                  and not c["key"][5],
    "composed fp32 atom, d_h % 4 != 0": lambda c: c["precision"] == "fp32" and c["kind"] == "atom" and c["d_h"] % 4 != 0
                                                  and not c["key"][5],
    "composed with d_vd and d_ed descriptors": lambda c: c["key"][1] == "composed" and c.get("d_vd") and c.get("d_ed"),
    "the PReLU weight's own gradient": lambda c: c["act"] == "prelu" and not c["key"][5],
}
# precision="bf16" on the composed tier: one facet per reason composed_reason() gives
DROPS = {"activation": "activation ", "undirected": "undirected=True", "dropout": "training-mode dropout",
         "d_h > 304": "> 304", "d_h % 4": "not a multiple of 4", "d_e = 0": "d_e = 0", "K limit": "GEMM inner dimensions"}
for _what, _text in DROPS.items():
    FACETS[f"bf16 on the composed tier: {_what}"] = (lambda t: lambda c: t in (c["_reason"] or ""))(_text)


@pytest.fixture
def stub(monkeypatch):
    """mab_plan_key with the tensor-core kernels reported available; `switch` sets ATOM_FUSED_ENABLED."""
    from chemprop_b200 import engine

    monkeypatch.setattr(engine, "_fused_available", lambda: True)
    monkeypatch.setattr(engine, "_WARNED", set())

    def key(mp, lay, atom_fused=True):
        monkeypatch.setattr(engine, "ATOM_FUSED_ENABLED", atom_fused)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            return mab_plan_key(mp, lay)
    return key


def grid_keys(key) -> set:
    keys = set()
    for kind, precision, h, act, undirected, dropout, (vertex, edge), d_e, d_v in itertools.product(
            KINDS, PRECISIONS, D_H, ACTS, (False, True), (0.0, 0.2), READOUTS, (14, 0), (72, 160)):
        c = dict(kind=kind, precision=precision, d_h=h, depth=1, act=act, bias=True, undirected=undirected, dropout=dropout,
                 vertex=vertex, edge=edge, dims=(d_v, d_e))
        with torch.device("meta"):
            mp = make_module(c, device="meta")
        mp.train()
        for depth, edges, big, atom_fused in itertools.product(DEPTHS, (True, False), (False, True), (True, False)):
            mp.depth = depth
            lay = SimpleNamespace(V=60, E=120 if edges else 0, max_tile_atoms=140 if big else 60)
            keys.add(key(mp, lay, atom_fused))
    return keys


def _covers(cases: dict) -> tuple:
    keys = {c["key"] for c in cases.values()}
    facets = {f for f, pred in FACETS.items() if any(pred(dict(c, _reason=_case_reason(n))) for n, c in cases.items())}
    return keys, facets


def test_every_mab_plan_key_has_a_gpu_case(stub):
    keys = grid_keys(stub)
    declared = {c["key"] for c in CASES.values()}
    assert keys - declared == set(), f"paths without a case in tests/test_gpu_zy_mab_paths.py: {sorted(keys - declared)}"
    assert declared - keys == set(), f"cases of paths the module no longer takes: {sorted(declared - keys)}"


def test_every_mab_facet_has_a_case():
    _, facets = _covers(CASES)
    assert set(FACETS) - facets == set(), sorted(set(FACETS) - facets)


@pytest.mark.parametrize("name", list(CASES))
def test_every_mab_case_is_needed(name):
    """Without this case a key or a facet goes uncovered: deleting it from CASES fails the two tests above."""
    rest = {n: c for n, c in CASES.items() if n != name}
    assert _covers(rest) != _covers(CASES), f"{name} covers nothing another case does not"


@pytest.mark.parametrize("name", list(CASES))
def test_mab_case_takes_its_declared_key(name, stub):
    """The configuration of each case, on a stub of its batch, plans to the key it declares (the GPU test asserts the same
    on the real batch)."""
    c = CASES[name]
    batch = c.get("batch", "mixed")
    lay = SimpleNamespace(V=60, E=0 if batch == "edgeless" else 120, max_tile_atoms=140 if batch == "oversized" else 100)
    with torch.device("meta"):
        mp = make_module(c, device="meta")
    got = stub(mp.train(), lay, c.get("patch", {}).get("ATOM_FUSED_ENABLED", True))
    assert got == c["key"], (got, c["key"])
    assert case_dims(c)[1] != 0 or _case_reason(name) == "d_e = 0"


@pytest.mark.parametrize("name", list(CASES))
def test_case_through_emulation_vs_f64_oracle(name, monkeypatch):
    from chemprop_b200 import composed
    from tests import emu_mab

    emu_mab.patch_engine(monkeypatch)
    monkeypatch.setattr(composed, "_X3_STATE", {"ok": None})     # the emulated first-use check must not outlive the test
    run_case(name, "cpu", 200, monkeypatch)
