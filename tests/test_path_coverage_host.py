"""CPU tier: every execution path `engine.plan()` can choose has a batch-scale float64 case on the GPU.

`engine.plan` is called over a grid of configurations -- Bond / AtomMessagePassing (atoms directed only), bf16 and fp32,
d_h in {298, 300, 320, 600}, depth 1 and 3, directed and undirected, batches with and without edges, with and without a
molecule of more than 128 atoms, each of the switches UNDIRECTED_FUSED, X3_ENABLED and ATOM_FUSED_ENABLED on and off --
with a stub layout and the tensor-core kernels reported available.  The set of plan keys it produces must equal the set
`tests.test_gpu_zy_paths.CASES` declares (imported without running it): a path added to `plan()` fails here until a GPU
case covers it, and a case whose path went away fails too.

Some paths differ inside one key in ways a host bug can hide in -- the activation (ReLU is idempotent, so a ReLU case cannot
see tau applied twice), the bias, d_h % 4 (vector or scalar kernels), bf16 or f32 storage, more terms than one multi-term
weight-gradient launch takes.  `FACETS` names those, and each must be a case as well.  Every case must be needed for a key
or a facet, so deleting any case fails this module, and no composition runs twice."""
import importlib
import itertools
import warnings
from types import SimpleNamespace

import pytest
import torch

from tests.test_gpu_zy_paths import _ATOM_TC, _FUSED_UND, _SIMT_DIR, _SIMT_UND, _TC_UND, CASES, plan_key

KINDS = ("bond", "atom")
PRECISIONS = ("bf16", "fp32")
D_H = (298, 300, 320, 600)
DEPTHS = (1, 3)
SWITCHES = ("UNDIRECTED_FUSED", "X3_ENABLED", "ATOM_FUSED_ENABLED")

# facet: (key, predicate over the case's configuration)
FACETS = {
    "fused undirected mirror with db_h (its column sum of dZ)": (_FUSED_UND, lambda c: c["bias"]),
    "fused undirected step, non-idempotent tau, depth >= 4": (_FUSED_UND, lambda c: c["act"] != "relu" and c["depth"] >= 4),
    "undirected W_h on the tensor-core linear (d_h % 4 == 0)": (_TC_UND, lambda c: c["d_h"] % 4 == 0),
    "undirected scalar rev_average / message (d_h % 4 != 0)": (_TC_UND, lambda c: c["d_h"] % 4 != 0),
    "undirected on the SIMT GEMMs, bf16 storage": (_SIMT_UND, lambda c: c["precision"] == "bf16"),
    "undirected on the SIMT GEMMs, f32 storage": (_SIMT_UND, lambda c: c["precision"] == "fp32"),
    "directed on the SIMT GEMMs, bf16 storage": (_SIMT_DIR, lambda c: c["precision"] == "bf16"),
    "directed on the SIMT GEMMs, f32 at d_h % 4 == 0": (_SIMT_DIR, lambda c: c["precision"] == "fp32" and c["d_h"] % 4 == 0),
    "two-launch atom step, a molecule of more than 128 atoms": (_ATOM_TC, lambda c: c.get("batch") == "oversized"),
    # dW_i takes `depth` terms, at most three per wgrad_tc_multi launch: depth >= 4 issues an accumulating second group
    "two-launch atom step, dW_i in two multi-term groups": (_ATOM_TC, lambda c: c["depth"] >= 4),
    "two-launch atom step at depth 1 (no depth loop)": (_ATOM_TC, lambda c: c["depth"] == 1),
}


def _cfg(precision, depth, undirected, act="relu"):
    from chemprop_b200 import _lib, engine

    return engine.MPConfig(depth=depth, act={"relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act], act_param=0.0,
                           undirected=undirected, hidden_dtype=torch.bfloat16 if precision == "bf16" else torch.float32)


def _key(monkeypatch, kind, cfg, lay, h, d_v, d_e, switches):
    from chemprop_b200 import engine

    for k, v in switches.items():
        monkeypatch.setattr(engine, k, v)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return plan_key(kind, cfg, lay, engine.plan(kind, cfg, lay, h, d_v, d_e))


@pytest.fixture
def planner(monkeypatch):
    from chemprop_b200 import engine

    monkeypatch.setattr(engine, "_fused_available", lambda: True)
    monkeypatch.setattr(engine, "_WARNED", set())
    return lambda *a: _key(monkeypatch, *a)


def grid_keys(planner) -> set:
    keys = set()
    for kind, precision, h, depth, undirected, edges, big, *sw in itertools.product(
            KINDS, PRECISIONS, D_H, DEPTHS, (False, True), (True, False), (False, True), *[(True, False)] * len(SWITCHES)):
        if kind == "atom" and undirected:
            continue                      # AtomMessagePassing(undirected=True) runs on the composed tier, outside plan()
        lay = SimpleNamespace(V=60, E=120 if edges else 0, max_tile_atoms=140 if big else 60)
        keys.add(planner(kind, _cfg(precision, depth, undirected), lay, h, 72, 14, dict(zip(SWITCHES, sw))))
    return keys


def _covers(cases: dict) -> tuple:
    keys = {c["key"] for c in cases.values()}
    facets = {f for f, (k, pred) in FACETS.items() if any(c["key"] == k and pred(c) for c in cases.values())}
    return keys, facets


def test_every_plan_key_has_a_gpu_case(planner):
    keys = grid_keys(planner)
    declared = {c["key"] for c in CASES.values()}
    assert keys - declared == set(), f"paths without a case in tests/test_gpu_zy_paths.py: {sorted(keys - declared)}"
    assert declared - keys == set(), f"cases of paths plan() no longer produces: {sorted(declared - keys)}"


def test_every_facet_has_a_case():
    _, facets = _covers(CASES)
    assert set(FACETS) - facets == set(), sorted(set(FACETS) - facets)


@pytest.mark.parametrize("name", list(CASES))
def test_every_case_is_needed(name):
    """Without this case a key or a facet goes uncovered: deleting it from CASES fails the two tests above."""
    rest = {n: c for n, c in CASES.items() if n != name}
    assert _covers(rest) != _covers(CASES), f"{name} covers nothing another case does not"


@pytest.mark.parametrize("name", list(CASES))
def test_case_takes_its_declared_key(name, planner):
    """The configuration of each case, on a stub of its batch, plans to the key it declares (the GPU test asserts the same
    on the real batch)."""
    c = CASES[name]
    d_v, d_e = c.get("dims", (72, 14))
    batch = c.get("batch", "mixed")
    lay = SimpleNamespace(V=60, E=0 if batch == "edgeless" else 120, max_tile_atoms=140 if batch == "oversized" else 100)
    switches = {k: c.get("patch", {}).get(k, True) for k in SWITCHES}
    got = planner(c["kind"], _cfg(c["precision"], c["depth"], c["undirected"], c["act"]), lay, c["d_h"], d_v, d_e, switches)
    assert got == c["key"], (got, c["key"])


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if "covered_by" in c])
def test_covering_test_exists(name):
    path, test = CASES[name]["covered_by"].split("::")
    mod = importlib.import_module(path[:-len(".py")].replace("/", "."))
    assert callable(getattr(mod, test, None)), CASES[name]["covered_by"]
