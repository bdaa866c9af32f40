"""CPU tier: every host-side argument of a training step is a function of the batch signature.

`CudaGraphStep` (chemprop_b200/graph.py) captures a step once per `batch_signature` and replays it for every later batch of
that signature, so every launch of the step must take its sizes, flags, path choices and workspace shapes from the
signature alone, and everything that depends on the batch's contents must be rebuilt on the device from the graph's static
inputs.  Here each configuration runs one full training step (forward, loss, backward) through the emulated kernel
wrappers (tests/emu.py and the head emulations of the *_host.py files) on a batch A and on two same-signature twins B and
C (tests/graph_twins.py), recording every wrapper call with its scalar arguments, the shapes and dtypes of its tensors, and
the host fields of the layout.  The three sequences must be identical.

Configurations: every plan key of tests/test_gpu_zy_paths.py and of tests/test_gpu_zy_mab_paths.py (the cases those files
declare, so a new path joins here too; training-mode dropout is left out, `engine.dropout_keep_bits` refuses capture on
purpose), EngineMPNN with batch norm and one criterion per kernel family (MSE, BCE, CE, MVE, Dirichlet, spectral),
EngineMolAtomBondMPNN with atom and bond targets and constraints, and EngineMulticomponentMPNN on the union and list paths.
Each twin's differences from A -- (a) the atom-tile count, (b) the window count, (c) where the atoms of in-degree > 4 and the
edgeless molecules sit, (d) mol_atom_ptr -- are declared per configuration and asserted through oracle/layout_np.py.

`test_a_content_derived_host_argument_is_caught` shows the check has teeth: one wrapper's host argument is made to read
the batch's molecule offsets, and the comparison fails on each named configuration."""
from __future__ import annotations

import dataclasses
import warnings

import numpy as np
import pytest
import torch

from tests import graph_twins as T
from tests.test_gpu_zy_mab_paths import CASES as MAB_CASES
from tests.test_gpu_zy_mab_paths import _inputs as mab_inputs
from tests.test_gpu_zy_mab_paths import _loss as mab_loss
from tests.test_gpu_zy_mab_paths import make_module as make_mab_module
from tests.test_gpu_zy_paths import CASES as PATH_CASES
from tests.test_gpu_zy_paths import _module_factory, molecules
from tests.test_host_logic import _LAUNCH_WRAPPERS

HEAD_WRAPPERS = ("bn_train_fwd", "bn_bwd", "mse_loss", "bce_loss", "ce_loss", "class_probs", "pred_transform",
                 "pred_transform_bwd", "mve_loss", "evidential_loss", "quantile_loss", "dirichlet_loss", "regression_loss",
                 "spectral_transform", "spectral_transform_bwd", "sid_loss", "wasserstein_loss", "edge_pair_mean",
                 "edge_pair_mean_bwd", "regression_loss_rows", "bce_loss_rows", "ce_loss_rows", "constrain_fwd",
                 "constrain_bwd", "build_layout", "atom_tables")
WRAPPERS = _LAUNCH_WRAPPERS + HEAD_WRAPPERS
N_MOLS = 16


# ---- the batches -----------------------------------------------------------------------------------------------------------
def batches(kind: str, batch: str, dims: tuple, seed: int, n: int = N_MOLS, paired: bool = False) -> tuple:
    """(A, B, C, what B and C differ in): A is the batch of a path case (tests/test_gpu_zy_paths.py::molecules at n
    molecules) plus three edgeless molecules and the pair of `graph_twins.window_molecules`; B holds the other pair, so every
    batch with edges has twins that differ in (a), (b) and (d), and in (c) where it holds K_k.  An edgeless batch holds
    molecules of 1-3 atoms: (d) only.
    `paired`: the featuriser's paired edge order (the mol-atom-bond bond head needs it), no K_k; batch "cgr": condensed
    reaction graphs (chemprop_b200.data.make_cgr_graphs), no K_k."""
    d_v, d_e = dims
    if d_e == 0:                                   # no bond features: the generators' molecules with E cut to zero columns
        from chemprop_b200.data import MolGraph

        A, B, C, want = batches(kind, batch, (d_v, 1), seed, n, paired)
        cut = lambda mgs: [MolGraph(m.V, m.E[:, :0], m.edge_index, m.rev_edge_index) for m in mgs]  # noqa: E731
        return cut(A), cut(B), cut(C), want
    if batch == "edgeless":
        want = dict(B="d", C="d")
        return (*T.twins(T.edgeless_molecules(n, seed, d_v, d_e), want, seed), want)
    if paired:
        from chemprop_b200.data import make_molecules

        base = make_molecules(n, seed=seed, mean_atoms=20.0, d_v=d_v, d_e=d_e)
    elif batch == "cgr":
        from chemprop_b200.data import make_cgr_graphs

        base = make_cgr_graphs(n, seed=seed, d_v=d_v, d_e=d_e)
    else:
        base = molecules(dict(kind=kind, batch=batch, dims=dims), seed, n)
    pa, pb, big = T.window_molecules(seed, d_v, d_e)
    # edgeless molecules, except beside the mol-atom-bond bond constraints (a set constraint on a molecule without bonds
    # cannot be met: the reference gives NaN there)
    base = base[:3] + pa + [big] + base[3:] + ([] if paired else T.edgeless_molecules(3, seed, d_v, d_e))
    # (c) needs atoms of in-degree > 4 (the K_k of the mixed batches): the edgeless molecules alone seldom leave their place
    # under a shuffle that keeps every tile's first molecule
    c = "c" if batch in ("mixed", "oversized") and not paired else ""
    want = dict(B="abd" + c, C="ad" + c)
    return (*T.twins(base, want, seed, paired=paired, windows=(3, pb)), want)


def _device_batch(mgs, device):
    from chemprop_b200.data import BatchMolGraph

    b = BatchMolGraph(mgs)
    b.to(device)
    return b


# ---- the configurations: make(device) -> (model, step(model, bmg, inputs) -> loss, inputs(mgs, seed, device)) -------------
def _path_config(c):
    def make(device):
        torch.manual_seed(3)
        return _module_factory(c, None)(device)

    def inputs(mgs, seed, device):
        return torch.randn(len(mgs), c["d_h"], generator=torch.Generator().manual_seed(seed)).to(device)

    def step(mp, bmg, G):
        from chemprop_b200.nn import MeanAggregation

        return (MeanAggregation()(mp(bmg), bmg.batch).float() * G).sum()

    return dict(make=make, inputs=inputs, step=step, kind=c["kind"], batch=c.get("batch", "mixed"), dims=c.get("dims", (72, 14)),
                patch=c.get("patch", {}), train=True)


def _mab_config(c):
    def make(device):
        torch.manual_seed(3)
        return make_mab_module(c, device)

    def inputs(mgs, seed, device):
        return [None if t is None else t.to(device) for t in mab_inputs(c, mgs, seed)]

    def step(mp, bmg, x):
        V_d, E_d, G, G_e = x
        H_v, H_e = mp(bmg, V_d, E_d)
        return mab_loss(H_v, H_e, bmg, G, G_e)

    return dict(make=make, inputs=inputs, step=step, kind=c["kind"], batch=c.get("batch", "mixed"), dims=c.get("dims", (72, 14)),
                patch=c.get("patch", {}), train=True)


HEADS = ("mse", "bce", "ce", "mve", "dirichlet", "spectral")
N_CLASSES, N_TASKS = 3, 2


def make_head_model(head: str, precision: str = "bf16", d_h: int = 64):
    import chemprop_b200.nn as N

    kw = dict(n_tasks=N_TASKS, input_dim=d_h, hidden_dim=32, n_layers=2)
    pred = {"mse": lambda: N.EngineRegressionFFN(**kw), "bce": lambda: N.EngineBinaryClassificationFFN(**kw),
            "ce": lambda: N.EngineMulticlassClassificationFFN(n_classes=N_CLASSES, **kw), "mve": lambda: N.EngineMveFFN(**kw),
            "dirichlet": lambda: N.EngineMulticlassDirichletFFN(n_classes=N_CLASSES, **kw),
            "spectral": lambda: N.EngineSpectralFFN(**dict(kw, n_tasks=8))}[head]()
    return N.EngineMPNN(N.BondMessagePassing(d_h=d_h, depth=3, precision=precision), N.MeanAggregation(), pred,
                        batch_norm=True)


def head_targets(head: str, n: int, gen: torch.Generator) -> tuple:
    """(targets, weights) of n molecules, a few targets masked (NaN)."""
    if head in ("ce", "dirichlet"):
        Y = torch.randint(0, N_CLASSES, (n, N_TASKS), generator=gen).float()
    elif head == "bce":
        Y = torch.randint(0, 2, (n, N_TASKS), generator=gen).float()
    elif head == "spectral":
        Y = torch.rand(n, 8, generator=gen) + 0.05
        Y = Y / Y.sum(1, keepdim=True)
    else:
        Y = torch.randn(n, N_TASKS, generator=gen)
    if head != "spectral":
        Y[torch.rand(Y.shape, generator=gen) < 0.1] = float("nan")
    return Y, torch.rand(n, 1, generator=gen) + 0.5


def _head_config(head):
    def make(device):
        torch.manual_seed(3)
        return make_head_model(head).to(device)

    def inputs(mgs, seed, device):
        return [t.to(device) for t in head_targets(head, len(mgs), torch.Generator().manual_seed(seed))]

    def step(model, bmg, x):
        return model.training_loss(bmg, *x)

    return dict(make=make, inputs=inputs, step=step, kind="bond", batch="mixed", dims=(72, 14), patch={}, train=True)


def make_mab_model(precision: str, d_h: int = 32):
    import chemprop_b200.nn as N

    kw = dict(hidden_dim=24, n_layers=2)
    return N.EngineMolAtomBondMPNN(
        N.MABBondMessagePassing(d_h=d_h, depth=3, precision=precision), agg=N.SumAggregation(), batch_norm=True,
        mol_predictor=N.EngineRegressionFFN(n_tasks=2, input_dim=d_h, **kw),
        atom_predictor=N.EngineRegressionFFN(n_tasks=2, input_dim=d_h, **kw),
        bond_predictor=N.EngineRegressionFFN(n_tasks=1, input_dim=2 * d_h, **kw),
        atom_constrainer=N.ConstrainerFFN(n_constraints=2, fp_dim=d_h, hidden_dim=16),
        bond_constrainer=N.ConstrainerFFN(n_constraints=1, fp_dim=2 * d_h, hidden_dim=16))


def mab_model_inputs(mgs, seed: int, device) -> list:
    """targets and weights per level (molecule, atom, bond) and the atom / bond constraints (every column set: a
    constrainer of two outputs takes two set columns)."""
    g = torch.Generator().manual_seed(seed)
    B, nV, nB = len(mgs), sum(m.V.shape[0] for m in mgs), sum(m.edge_index.shape[1] for m in mgs) // 2
    Ys = [torch.randn(B, 2, generator=g), torch.randn(nV, 2, generator=g), torch.randn(nB, 1, generator=g)]
    ws = [torch.rand(B, 1, generator=g) + 0.5, torch.rand(nV, 1, generator=g) + 0.5, torch.rand(nB, 1, generator=g) + 0.5]
    cons = [torch.randn(B, 2, generator=g), torch.randn(B, 1, generator=g)]
    return [[t.to(device) for t in ts] for ts in (Ys, ws, cons)]


def mab_model_step(model, bmg, x):
    Ys, ws, cons = x
    return model.training_loss(bmg, Ys, ws, constraints=cons)


def _mab_model_config(precision):
    def make(device):
        torch.manual_seed(3)
        return make_mab_model(precision).to(device)

    return dict(make=make, inputs=mab_model_inputs, step=mab_model_step, kind="bond", batch="mixed", dims=(72, 14), patch={},
                train=True, paired=True)


def make_mc_model(precision: str = "bf16", d_h: int = 32):
    import chemprop_b200.nn as N

    mcmp = N.EngineMulticomponentMessagePassing([N.BondMessagePassing(d_h=d_h, precision=precision)], n_components=2,
                                                shared=True)
    return N.EngineMulticomponentMPNN(mcmp, N.MeanAggregation(), N.EngineRegressionFFN(n_tasks=2, input_dim=2 * d_h),
                                      batch_norm=True)


def _mc_config(union):
    def make(device):
        torch.manual_seed(3)
        return make_mc_model().to(device)

    def inputs(mgs, seed, device):
        g = torch.Generator().manual_seed(seed)
        n = len(mgs) // 2 if union else len(mgs[0])
        return [torch.randn(n, 2, generator=g).to(device), (torch.rand(n, 1, generator=g) + 0.5).to(device)]

    def step(model, bmg, x):
        return model.training_loss(bmg, *x)

    return dict(make=make, inputs=inputs, step=step, kind="bond", batch="mixed", dims=(72, 14), patch={}, train=True,
                components=None if union else 2)


CONFIGS = {}
CONFIGS.update({f"path:{n}": _path_config(c) for n, c in PATH_CASES.items()})
CONFIGS.update({f"mab:{n}": _mab_config(c) for n, c in MAB_CASES.items() if not c.get("dropout")})
CONFIGS.update({f"mpnn-bn-{h}": _head_config(h) for h in HEADS})
CONFIGS.update({f"mab-model-constrained-{p}": _mab_model_config(p) for p in ("bf16", "fp32")})
CONFIGS.update({"mc-union": _mc_config(True), "mc-list": _mc_config(False)})


def config_batches(name: str, seed: int, n: int = N_MOLS) -> tuple:
    """([A, B, C], want): each of A, B, C a list of MolGraphs, or for the multicomponent list path a list of the two
    components' lists (each component twinned on its own, both with n molecules)."""
    cfg = CONFIGS[name]
    if cfg.get("components"):
        comps = [batches(cfg["kind"], cfg["batch"], cfg["dims"], seed + 17 * k, n // 2 - 4) for k in range(cfg["components"])]
        n_min = min(len(c[0]) for c in comps)
        assert all(len(x) == n_min for c in comps for x in c[:3]), "components of different sizes"
        return [[c[i] for c in comps] for i in range(3)], comps[0][3]
    A, B, C, want = batches(cfg["kind"], cfg["batch"], cfg["dims"], seed, n, cfg.get("paired", False))
    if name == "mc-union" and len(A) % 2:
        raise AssertionError("a union batch needs an even molecule count")
    return [A, B, C], want


# ---- the recorder ----------------------------------------------------------------------------------------------------------
def _value(v):
    from chemprop_b200 import engine

    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), str(v.dtype))
    if isinstance(v, engine.Layout):
        return ("Layout", v.V, v.E, v.B, tuple(v._host()),
                tuple(_value(getattr(v, f.name)) for f in dataclasses.fields(v) if isinstance(getattr(v, f.name), torch.Tensor)))
    if dataclasses.is_dataclass(v) and not isinstance(v, type):
        return (type(v).__name__,) + tuple(_value(getattr(v, f.name)) for f in dataclasses.fields(v))
    if isinstance(v, (list, tuple)):
        return tuple(_value(x) for x in v)
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    return type(v).__name__


def patch_all(monkeypatch):
    """Every emulation the *_host.py files use: the engine kernels, the mol-atom-bond read-out, the head, row-head and
    constrainer wrappers; the constrainer on its engine path (it must not read the status word: a captured step cannot)."""
    import chemprop_b200.nn.constrainer as con_mod
    from chemprop_b200 import composed, engine
    from tests.test_constrainer_host import constrain_bwd, constrain_fwd
    from tests.test_mab_model_host import patch_mab_model

    patch_mab_model(monkeypatch)
    monkeypatch.setattr(engine, "constrain_fwd", constrain_fwd)
    monkeypatch.setattr(engine, "constrain_bwd", constrain_bwd)
    monkeypatch.setattr(con_mod, "_on_engine", lambda t: True)
    monkeypatch.setattr(con_mod, "_may_synchronise", lambda: False)
    monkeypatch.setattr(engine, "_WARNED", set())
    monkeypatch.setattr(composed, "_X3_STATE", {"ok": None})     # the emulated first-use check must not outlive the test


def install_recorder(monkeypatch, seq: list):
    import chemprop_b200.nn.agg as agg_mod
    import chemprop_b200.nn.constrainer as con_mod
    from chemprop_b200 import engine

    for n in WRAPPERS:
        f0 = getattr(engine, n)
        monkeypatch.setattr(engine, n, lambda *a, _f=f0, _n=n, **k: (seq.append((_n, _value(a), _value(sorted(k.items())))),
                                                                     _f(*a, **k))[1])
    seg0 = engine.segments_of
    rec_seg = lambda *a, **k: (seq.append(("segments_of", _value(a), _value(sorted(k.items())))), seg0(*a, **k))[1]  # noqa: E731
    for mod in (engine, agg_mod, con_mod):
        monkeypatch.setattr(mod, "segments_of", rec_seg)


def launch_sequences(name: str, monkeypatch, seed: int = 11, fault=None) -> tuple:
    """The recorded wrapper calls of one training step on each of A, B, C, and the twins' declared differences."""
    from chemprop_b200 import engine

    cfg = CONFIGS[name]
    patch_all(monkeypatch)
    for k, v in cfg["patch"].items():
        monkeypatch.setattr(engine, k, v)
    seq = []
    install_recorder(monkeypatch, seq)
    if fault is not None:                  # between the callers and the recorded wrapper
        fault(monkeypatch)
    trio, want = config_batches(name, seed)
    model = cfg["make"]("cpu")
    model.train(cfg["train"])
    out = []
    for mgs in [trio[0]] + trio:           # a warm-up step first, as CudaGraphStep takes before its capture (the composed
        bmg = [_device_batch(m, "cpu") for m in mgs] if cfg.get("components") else _device_batch(mgs, "cpu")
        x = cfg["inputs"](mgs, seed, "cpu")
        model.zero_grad(set_to_none=False)
        del seq[:]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            loss = cfg["step"](model, bmg, x)
            loss.backward()
        assert torch.isfinite(loss).all()
        out.append(list(seq))               # tier's one-time 3xTF32 check runs there)
    return out[1:], want


def assert_same_sequences(seqs: list):
    a = seqs[0]
    assert a, "no wrapper call recorded"
    for twin, s in zip("BC", seqs[1:]):
        for i, (x, y) in enumerate(zip(a, s)):
            assert x == y, f"twin {twin}, call {i}: {x} != {y}"
        assert len(a) == len(s), (twin, len(a), len(s))


def test_atom_tile_constants_match_the_engine():
    from chemprop_b200 import engine

    assert (T.ATOM_TILE_ATOMS, T.ATOM_TILE_EDGES) == (engine.ATOM_TILE_ATOMS, engine.ATOM_TILE_EDGES)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_twins_have_one_signature_and_their_declared_differences(name):
    """Through oracle/layout_np.py, and the signature also through the library's host meta words (graph.batch_signature)."""
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.graph import batch_signature

    trio, want = config_batches(name, 11)
    comps = trio if CONFIGS[name].get("components") else [[b] for b in trio]
    for k in range(len(comps[0])):
        fa = T.facts(comps[0][k])
        for twin, mgs in zip("BC", comps[1:]):
            got = T.differences(fa, T.facts(mgs[k]))
            assert set(want[twin]) <= got, (twin, want[twin], got)
            assert batch_signature(BatchMolGraph(mgs[k])) == batch_signature(BatchMolGraph(comps[0][k])) == fa["signature"]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_host_arguments_are_a_function_of_the_signature(name, monkeypatch):
    seqs, _ = launch_sequences(name, monkeypatch)
    assert_same_sequences(seqs)


def _content_derived_scale(monkeypatch):
    """The fault: segment_sum's `scale` (unused unless the mode is SCALE_DIV_CONST) read from the molecule offsets on the
    host -- a value a capture would freeze for every later batch of the signature."""
    from chemprop_b200 import _lib, engine

    f0 = engine.segment_sum

    def segment_sum(X, ptr, n_seg, Ccols, out, **k):
        if k.get("scale_mode", _lib.SCALE_NONE) != _lib.SCALE_DIV_CONST:
            k["scale"] = float((ptr[:n_seg + 1].double() * torch.arange(n_seg + 1, dtype=torch.float64)).sum())
        return f0(X, ptr, n_seg, Ccols, out, **k)

    monkeypatch.setattr(engine, "segment_sum", segment_sum)


@pytest.mark.parametrize("name", ["path:D1-bond-bf16-fused-generic-mirror-dh298-tanh", "path:atom-bf16-fused-step",
                                  "mab:B1-bond-fused-relu-descriptors", "mpnn-bn-mse", "mab-model-constrained-bf16",
                                  "mc-union", "mc-list"])
def test_a_content_derived_host_argument_is_caught(name, monkeypatch):
    seqs, _ = launch_sequences(name, monkeypatch, fault=_content_derived_scale)
    with pytest.raises(AssertionError, match="segment_sum"):
        assert_same_sequences(seqs)
