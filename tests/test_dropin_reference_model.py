"""CPU tier, reference tree required (skipped on the GPU box): the north-star claim "drops into the existing MPNN /
Lightning model as-is", checked literally.  The reference's own `chemprop.models.MPNN` (unmodified, imported through
oracle/ref_shim.py) is built twice on the same weights -- once with the reference's BondMessagePassing + MeanAggregation,
once with the engine's modules plugged into the same constructor -- and fed the reference's own BatchMolGraph; the
engine side runs with the kernel wrappers emulated (tests/emu.py).  Predictions, the training loss and every gradient
must agree, and the reference state dict must load into the drop-in model unchanged."""
import copy

import numpy as np
import pytest
import torch

from oracle.ref_shim import reference_available
from tests import emu

pytestmark = pytest.mark.skipif(not reference_available(), reason="needs the unmodified reference package (CHEMPROP_REFERENCE_ROOT)")


@pytest.mark.parametrize("kind,agg,act,undirected", [("bond", "mean", "relu", False), ("atom", "sum", "tanh", False),
                                                     ("bond", "norm", "prelu", True)])
def test_engine_modules_inside_the_reference_mpnn(kind, agg, act, undirected, monkeypatch):
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MPNN

    import chemprop_b200.nn as ours
    from chemprop_b200.data import make_molecules
    from chemprop_b200.integrate import register_with_chemprop

    emu.patch_engine(monkeypatch)
    torch.manual_seed(0)
    mgs = make_molecules(16, seed=3, mean_atoms=9, std_atoms=3, shuffle_edges=True, min_atoms=1)
    bmg = RefBMG([RefMG(*m) for m in mgs])                                   # the REFERENCE's batch object
    targets = torch.from_numpy(np.random.default_rng(0).normal(size=(16, 1)).astype(np.float32))
    kw = dict(d_h=48, depth=3, bias=True, activation=act, undirected=undirected)
    ref_mp = (ref_nn.BondMessagePassing if kind == "bond" else ref_nn.AtomMessagePassing)(**kw)
    ref_agg = {"mean": ref_nn.MeanAggregation, "sum": ref_nn.SumAggregation, "norm": ref_nn.NormAggregation}[agg]()
    ref = MPNN(ref_mp, ref_agg, ref_nn.RegressionFFN(input_dim=48), batch_norm=True)
    our_mp = (ours.BondMessagePassing if kind == "bond" else ours.AtomMessagePassing)(**kw)
    our_agg = ours.AggregationRegistry[agg]()
    drop = MPNN(our_mp, our_agg, copy.deepcopy(ref.predictor), batch_norm=True)          # same constructor, engine modules
    assert set(drop.state_dict()) == set(ref.state_dict())
    drop.load_state_dict(ref.state_dict())                                             # strict: keys and shapes identical
    reg = register_with_chemprop()
    assert isinstance(our_mp, type(ref_mp)) and isinstance(our_agg, ref_nn.Aggregation) and len(reg) >= 9
    assert isinstance(our_mp, ref_nn.BondMessagePassing) == (kind == "bond")           # chemprop/cli/predict.py:256
    rebuilt = our_mp.hparams["cls"](**{k: v for k, v in our_mp.hparams.items() if k != "cls"})   # models/model.py:267-271
    assert type(rebuilt) is type(our_mp) and rebuilt.output_dim == drop.message_passing.output_dim == 48
    before = [t.clone() for t in (bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch)]
    for model in (ref, drop):
        model.train()
    outs, grads = [], []
    for model in (ref, drop):
        model.zero_grad()
        Z = model.fingerprint(bmg)                                                     # message passing + agg + batch norm
        preds = model.predictor.train_step(Z)
        loss = torch.nn.functional.mse_loss(preds, targets)
        loss.backward()
        outs.append((Z.detach(), preds.detach(), loss.detach()))
        grads.append({k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None})
    for a, b in zip(outs[0], outs[1]):
        torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-5)
    assert set(grads[0]) == set(grads[1])
    for k in grads[0]:
        torch.testing.assert_close(grads[1][k], grads[0][k], rtol=2e-3, atol=2e-5, msg=k)
    for a, b in zip(before, (bmg.V, bmg.E, bmg.edge_index, bmg.rev_edge_index, bmg.batch)):
        assert torch.equal(a, b)                                                       # the caller's batch is untouched
    for model in (ref, drop):
        model.eval()
    with torch.inference_mode():
        torch.testing.assert_close(drop(bmg), ref(bmg), rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("shared", [False, True])
def test_engine_blocks_inside_the_reference_multicomponent_mpnn(shared, monkeypatch):
    """chemprop.models.MulticomponentMPNN (models/multi.py) over the REFERENCE's own MulticomponentMessagePassing
    container (a list-in / list-out wrapper, SURVEY.md section 2 row 6: "works unchanged on top of a replaced block")
    holding the engine's blocks: two components (e.g. solute / solvent), per-component or shared encoder."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MulticomponentMPNN

    import chemprop_b200.nn as ours
    from chemprop_b200.data import make_molecules

    emu.patch_engine(monkeypatch)
    torch.manual_seed(1)
    bmgs = [RefBMG([RefMG(*m) for m in make_molecules(10, seed=s, mean_atoms=7, std_atoms=2, min_atoms=1)]) for s in (4, 5)]
    targets = torch.from_numpy(np.random.default_rng(1).normal(size=(10, 1)).astype(np.float32))
    if shared:
        ref_blocks, our_blocks = [ref_nn.BondMessagePassing(d_h=24)], [ours.BondMessagePassing(d_h=24)]
    else:
        ref_blocks = [ref_nn.BondMessagePassing(d_h=24), ref_nn.AtomMessagePassing(d_h=16, activation="elu")]
        our_blocks = [ours.BondMessagePassing(d_h=24), ours.AtomMessagePassing(d_h=16, activation="elu")]
    ref_mc = ref_nn.MulticomponentMessagePassing(ref_blocks, n_components=2, shared=shared)
    our_mc = ref_nn.MulticomponentMessagePassing(our_blocks, n_components=2, shared=shared)
    assert our_mc.output_dim == ref_mc.output_dim and len(our_mc) == len(ref_mc) == 2
    ref = MulticomponentMPNN(ref_mc, ref_nn.MeanAggregation(), ref_nn.RegressionFFN(input_dim=ref_mc.output_dim), batch_norm=True)
    drop = MulticomponentMPNN(our_mc, ours.MeanAggregation(), copy.deepcopy(ref.predictor), batch_norm=True)
    drop.load_state_dict(ref.state_dict())
    results = []
    for model in (ref, drop):
        model.train()
        model.zero_grad()
        preds = model.predictor.train_step(model.fingerprint(bmgs))
        loss = torch.nn.functional.mse_loss(preds, targets)
        loss.backward()
        results.append((preds.detach(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}))
    torch.testing.assert_close(results[1][0], results[0][0], rtol=1e-4, atol=1e-5)
    assert set(results[0][1]) == set(results[1][1])
    for k in results[0][1]:
        torch.testing.assert_close(results[1][1][k], results[0][1][k], rtol=2e-3, atol=2e-5, msg=k)


def test_reference_checkpoint_round_trip_rebuilds_the_engine_modules(tmp_path):
    """chemprop.models.utils.save_model / load_model (hparams["cls"](**hparams), models/model.py:267-271): a model saved
    with the engine's modules comes back with the engine's modules -- `precision` and `norm` included."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.models import MPNN
    from chemprop.models.utils import load_model, save_model

    import chemprop_b200.nn as ours

    torch.manual_seed(2)
    model = MPNN(ours.BondMessagePassing(d_h=16, depth=4, precision="bf16", activation="tanh", bias=True, d_vd=3),
                 ours.NormAggregation(norm=50.0), ref_nn.RegressionFFN(input_dim=19))
    path = tmp_path / "model.pt"
    save_model(path, model)
    back = load_model(path)
    mp = back.message_passing
    assert type(mp) is ours.BondMessagePassing and mp.precision == "bf16" and mp.depth == 4 and isinstance(mp.tau, torch.nn.Tanh)
    assert mp.W_d is not None and mp.output_dim == 19 and mp.W_i.bias is not None
    assert type(back.agg) is ours.NormAggregation and back.agg.norm == 50.0
    for (ka, a), (kb, b) in zip(model.state_dict().items(), back.state_dict().items()):
        assert ka == kb and torch.equal(a, b)


@pytest.mark.parametrize("kind", ["bond", "atom"])
def test_engine_mab_modules_inside_the_reference_mol_atom_bond_mpnn(kind, monkeypatch):
    """chemprop.models.MolAtomBondMPNN (models/mol_atom_bond.py:215-238) with the engine's MAB message passing: the
    molecule-, atom- and bond-level fingerprints (the last one pairs every directed edge with its reverse, so the
    per-edge embeddings must come back in the caller's edge order) and the gradients of a loss on all three."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data.collate import BatchMolAtomBondGraph
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MolAtomBondMPNN
    from chemprop.nn.message_passing import MABAtomMessagePassing, MABBondMessagePassing

    import chemprop_b200.nn as ours
    from chemprop_b200.data import make_molecules

    emu.patch_engine(monkeypatch)
    torch.manual_seed(4)
    bmg = BatchMolAtomBondGraph([RefMG(*m) for m in make_molecules(9, seed=6, mean_atoms=8, std_atoms=3, shuffle_edges=True)])
    kw = dict(d_h=32, depth=3, bias=True, activation="elu")
    ref_mp = (MABBondMessagePassing if kind == "bond" else MABAtomMessagePassing)(**kw)
    our_mp = (ours.MABBondMessagePassing if kind == "bond" else ours.MABAtomMessagePassing)(**kw)
    preds = lambda: dict(mol_predictor=ref_nn.RegressionFFN(input_dim=32), atom_predictor=ref_nn.RegressionFFN(input_dim=32),  # noqa: E731
                         bond_predictor=ref_nn.RegressionFFN(input_dim=64))
    ref = MolAtomBondMPNN(ref_mp, ref_nn.SumAggregation(), batch_norm=True, **preds())
    drop = MolAtomBondMPNN(our_mp, ours.SumAggregation(), batch_norm=True, **preds())
    assert set(drop.state_dict()) == set(ref.state_dict())
    drop.load_state_dict(ref.state_dict())
    results = []
    for model in (ref, drop):
        model.train()
        model.zero_grad()
        H_g, H_v, H_e = model.fingerprint(bmg)
        assert H_e.shape == (bmg.E.shape[0], 64) and H_v.shape == (bmg.V.shape[0], 32) and H_g.shape == (9, 32)
        loss = H_g.square().mean() + H_v.tanh().mean() + (H_e * torch.linspace(-1, 1, 64)).mean()
        loss.backward()
        results.append(([t.detach() for t in (H_g, H_v, H_e)],
                        {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}))
    for a, b in zip(results[0][0], results[1][0]):
        torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-5)
    assert set(results[0][1]) == set(results[1][1])
    for k in results[0][1]:
        torch.testing.assert_close(results[1][1][k], results[0][1][k], rtol=2e-3, atol=2e-5, msg=k)


def test_engine_constrainer_inside_the_reference_mol_atom_bond_mpnn(monkeypatch):
    """MolAtomBondMPNN.forward with an atom constrainer (models/mol_atom_bond.py:255-290): the engine's ConstrainerFFN in
    the reference model == the reference's own, and the constrained atom predictions sum to the constraint per molecule."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data.collate import BatchMolAtomBondGraph
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MolAtomBondMPNN
    from chemprop.nn.ffn import ConstrainerFFN as RefConstrainer
    from chemprop.nn.message_passing import MABBondMessagePassing

    import chemprop_b200.nn as ours
    from chemprop_b200.data import make_molecules
    from chemprop_b200.integrate import register_with_chemprop

    emu.patch_engine(monkeypatch)
    torch.manual_seed(5)
    bmg = BatchMolAtomBondGraph([RefMG(*m) for m in make_molecules(7, seed=9, mean_atoms=7, std_atoms=2)])
    constraints = [torch.from_numpy(np.random.default_rng(2).normal(size=(7, 1)).astype(np.float32)), None]
    ref = MolAtomBondMPNN(MABBondMessagePassing(d_h=32), ref_nn.SumAggregation(), atom_predictor=ref_nn.RegressionFFN(input_dim=32),
                          atom_constrainer=RefConstrainer(n_constraints=1, fp_dim=32, hidden_dim=16))
    drop = MolAtomBondMPNN(ours.MABBondMessagePassing(d_h=32), ours.SumAggregation(), atom_predictor=ref_nn.RegressionFFN(input_dim=32),
                           atom_constrainer=ours.ConstrainerFFN(n_constraints=1, fp_dim=32, hidden_dim=16))
    assert set(drop.state_dict()) == set(ref.state_dict())
    drop.load_state_dict(ref.state_dict())
    assert isinstance(drop.atom_constrainer, RefConstrainer) or register_with_chemprop() and isinstance(drop.atom_constrainer, RefConstrainer)
    for model in (ref, drop):
        model.eval()
    with torch.no_grad():
        a = ref(bmg, constraints=constraints)[1]
        b = drop(bmg, constraints=constraints)[1]
    torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-5)
    sums = torch.zeros(7, 1).index_add_(0, bmg.batch, b)
    torch.testing.assert_close(sums, constraints[0], rtol=1e-4, atol=1e-4)


def test_the_maintainer_side_subclass_of_integration_md_runs_as_written(monkeypatch):
    """INTEGRATION.md section 2 shows the binding a chemprop maintainer would add: a subclass of the REFERENCE's
    `BondMessagePassing` whose `forward` calls the engine.  The code block is taken from the document verbatim, executed,
    and the resulting class -- reference constructor, reference parameters, reference BatchMolGraph -- is compared with the
    reference module on the same weights (forward incl. the `V_d` branch, and every gradient)."""
    import os
    import re

    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG

    from chemprop_b200.data import make_molecules

    doc = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "INTEGRATION.md")).read()
    block = re.search(r"```python\n(# chemprop/nn/message_passing/fused\.py.*?)```", doc, re.S).group(1)
    ns = {"torch": torch}
    exec(compile(block, "INTEGRATION.md#fused.py", "exec"), ns)              # noqa: S102 -- our own document
    Fused = ns["FusedBondMessagePassing"]
    assert issubclass(Fused, ref_nn.BondMessagePassing)

    emu.patch_engine(monkeypatch)
    torch.manual_seed(1)
    mgs = make_molecules(12, seed=5, mean_atoms=8, std_atoms=3, min_atoms=1)
    bmg = RefBMG([RefMG(*m) for m in mgs])
    V_d = torch.randn(bmg.V.shape[0], 3)
    kw = dict(d_h=32, depth=3, bias=True, activation="elu", d_vd=3)
    ref = ref_nn.BondMessagePassing(**kw)
    fused = Fused(**kw)
    fused.precision = "fp32"                                                # the sketch's class attribute: bf16 by default
    fused.load_state_dict(ref.state_dict())
    G = torch.randn(bmg.V.shape[0], ref.output_dim)
    res = []
    for m in (ref, fused):
        m.zero_grad()
        H = m(bmg, V_d)
        (H * G).sum().backward()
        res.append((H.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}))
    torch.testing.assert_close(res[1][0], res[0][0], rtol=1e-4, atol=1e-5)
    assert set(res[0][1]) == set(res[1][1])
    for k in res[0][1]:
        torch.testing.assert_close(res[1][1][k], res[0][1][k], rtol=2e-3, atol=2e-5, msg=k)
    torch.testing.assert_close(fused(bmg), ref(bmg), rtol=1e-4, atol=1e-5)  # without descriptors


@pytest.mark.parametrize("ref_agg", [False, True])
def test_bf16_engine_module_inside_the_reference_mpnn(ref_agg, monkeypatch):
    """precision="bf16" inside the unmodified reference MPNN (its f32 BatchNorm / FFN follow): with the engine's aggregation
    (which always returns f32) as is; with the REFERENCE's aggregation -- a scatter on whatever dtype it is given -- through
    `output_dtype=torch.float32`.  Predictions within the bf16 tier's tolerance of the all-reference model."""
    from oracle.ref_shim import import_reference

    import_reference()
    import chemprop.nn as ref_nn
    from chemprop.data import BatchMolGraph as RefBMG
    from chemprop.data.molgraph import MolGraph as RefMG
    from chemprop.models import MPNN

    import chemprop_b200.nn as ours
    from chemprop_b200.data import make_molecules

    emu.patch_engine(monkeypatch)
    torch.manual_seed(0)
    bmg = RefBMG([RefMG(*m) for m in make_molecules(16, seed=7, mean_atoms=9, std_atoms=3, min_atoms=1)])
    kw = dict(d_h=64, depth=3)
    ref = MPNN(ref_nn.BondMessagePassing(**kw), ref_nn.MeanAggregation(), ref_nn.RegressionFFN(input_dim=64), batch_norm=False)
    our_mp = ours.BondMessagePassing(precision="bf16", output_dtype=torch.float32 if ref_agg else None, **kw)
    agg = ref_nn.MeanAggregation() if ref_agg else ours.MeanAggregation()
    drop = MPNN(our_mp, agg, copy.deepcopy(ref.predictor), batch_norm=False)
    drop.load_state_dict(ref.state_dict())
    for m in (ref, drop):
        m.eval()
    with torch.no_grad():
        Z_ref, Z = ref.fingerprint(bmg), drop.fingerprint(bmg)
        assert Z.dtype == torch.float32
        assert float((Z - Z_ref).abs().max()) <= 1e-2
        torch.testing.assert_close(drop(bmg), ref(bmg), rtol=0, atol=2e-2)
    drop.train()
    targets = torch.zeros(16, 1)
    loss = torch.nn.functional.mse_loss(drop.predictor.train_step(drop.fingerprint(bmg)), targets)
    loss.backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in drop.parameters())
