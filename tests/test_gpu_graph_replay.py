"""GPU tier: one captured training step replayed across same-signature batches of different topology equals the eager
steps bit for bit, and float64.

For each configuration, at a few thousand molecules: batches A, B, C of one `batch_signature` (tests/graph_twins.py: B and C
relabel, reorder and rewire A's molecules, so the layout, the fused step's window table, the atom tiles, the segment pointers
and the mol-atom-bond index maps all differ; the differences (a)-(d) each pair shows are asserted through
oracle/layout_np.py and printed), and a training step with `torch.optim.Adam(capturable=True)` inside it.  The step is
captured on A by `CudaGraphStep` and replayed on A, B, C, A, B, per-step targets copied into static buffers; the same five
steps run eagerly on an identical copy of the model.  Asserted:

  * bit equality with the eager sequence: the loss, every `.grad`, every parameter and buffer after the step (batch-norm
    running statistics included) -- the library is deterministic, so a replay on a stale table or a frozen host argument
    cannot hide here;
  * the encoder's output of the first replay on each twin against the float64 restatement on that twin
    (oracle/restatement.py, restatement.mab_forward) with the parameters of that step, at the bars of the path tests:
    1e-2 * max(1, max|H|) for the bf16 tier, 1e-5 * max(1, max|H|) for fp32;
  * one capture for the whole sequence, and every eager step after the first launching as many library kernels as one
    replay (`cap.launches`).

And training-mode dropout on the fused step refuses capture (DmpnnError) instead of replaying frozen masks."""
from __future__ import annotations

import copy
import time

import pytest
import torch

from tests import graph_twins as T
from tests.test_graph_signature_host import (batches, head_targets, make_head_model, make_mab_model, make_mc_model,
                                             mab_model_inputs, mab_model_step)

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_MOLS = 2000
SEQUENCE = (0, 1, 2, 0, 1)          # A, B, C, A, B


def _mpnn(mp_cls, head="mse", **kw):
    def make():
        import chemprop_b200.nn as N

        model = make_head_model(head, d_h=kw.get("d_h", 300))
        model.message_passing = getattr(N, mp_cls)(**kw)
        return model
    return make


def _head_inputs(head):
    return lambda mgs, seed: [t.to(DEV) for t in head_targets(head, len(mgs), torch.Generator().manual_seed(seed))]


def _head_step(model, bmg, x):
    return model.training_loss(bmg, *x)


def _mc_inputs(union):
    def inputs(mgs, seed):
        g = torch.Generator().manual_seed(seed)
        n = len(mgs) // 2 if union else len(mgs[0])
        return [torch.randn(n, 2, generator=g).to(DEV), (torch.rand(n, 1, generator=g) + 0.5).to(DEV)]
    return inputs


# make() -> model; inputs(mgs, seed) -> the step's targets (regression targets and weights when absent); step(model, bmg,
# inputs) -> loss; batch: (kind, batch of test_graph_signature_host.batches, dims[, paired]); mab / mc: the encoder's kind;
# components: the multicomponent list path
CONFIGS = {
    "bond-bf16-fused": dict(make=_mpnn("BondMessagePassing", d_h=300, precision="bf16"), batch=("bond", "mixed", (72, 14))),
    "bond-fp32-x3-dh600": dict(make=_mpnn("BondMessagePassing", d_h=600, precision="fp32"), batch=("bond", "mixed", (72, 14))),
    "bond-bf16-windows": dict(make=_mpnn("BondMessagePassing", d_h=300, precision="bf16"), batch=("bond", "windows", (72, 14))),
    "bond-bf16-undirected": dict(make=_mpnn("BondMessagePassing", d_h=300, precision="bf16", undirected=True),
                                 batch=("bond", "mixed", (72, 14)), undirected=True),
    "atom-bf16-fused-cgr": dict(make=_mpnn("AtomMessagePassing", d_v=106, d_e=28, d_h=300, precision="bf16"),
                                batch=("atom", "cgr", (106, 28))),
    "atom-fp32": dict(make=_mpnn("AtomMessagePassing", d_h=300, precision="fp32"), batch=("atom", "mixed", (72, 14))),
    "mab-bf16-constrained": dict(make=lambda: make_mab_model("bf16", d_h=300), inputs=lambda m, s: mab_model_inputs(m, s, DEV),
                                 step=mab_model_step, batch=("bond", "mixed", (72, 14), True), mab=True),
    "mab-fp32-constrained": dict(make=lambda: make_mab_model("fp32", d_h=300), inputs=lambda m, s: mab_model_inputs(m, s, DEV),
                                 step=mab_model_step, batch=("bond", "mixed", (72, 14), True), mab=True),
    "mc-union": dict(make=lambda: make_mc_model("bf16", d_h=300), inputs=_mc_inputs(True), batch=("bond", "mixed", (72, 14)),
                     mc=True),
    "mc-list": dict(make=lambda: make_mc_model("bf16", d_h=300), inputs=_mc_inputs(False), batch=("bond", "mixed", (72, 14)),
                    mc=True, components=2),
    "mpnn-mve": dict(make=_mpnn("BondMessagePassing", head="mve", d_h=300, precision="bf16"), inputs=_head_inputs("mve"),
                     batch=("bond", "mixed", (72, 14))),
    "mpnn-multiclass": dict(make=_mpnn("BondMessagePassing", head="ce", d_h=300, precision="bf16"), inputs=_head_inputs("ce"),
                            batch=("bond", "mixed", (72, 14))),
}


def _trio(cfg, seed):
    """([A, B, C] molecule lists -- for the list path, lists of the two components' lists -- and the declared differences)."""
    kind, batch, dims, *paired = cfg["batch"]
    if cfg.get("components"):
        comps = [batches(kind, batch, dims, seed + 17 * k, N_MOLS // 2 - 4) for k in range(cfg["components"])]
        assert len({len(x) for c in comps for x in c[:3]}) == 1
        return [[c[i] for c in comps] for i in range(3)], comps[0][3]
    A, B, C, want = batches(kind, batch, dims, seed, N_MOLS, bool(paired and paired[0]))
    if cfg.get("mc") and len(A) % 2:
        A, B, C = (x + T.edgeless_molecules(1, seed, *dims) for x in (A, B, C))
    return [A, B, C], want


def _device_batch(mgs):
    from chemprop_b200.data import BatchMolGraph

    b = BatchMolGraph(mgs)
    b.to(DEV)
    return b


def _encoder(model, cfg):
    return model.message_passing.blocks[0] if cfg.get("mc") else model.message_passing


def _f64(cfg, enc, state, mgs):
    """The encoder's output on `mgs` in float64 with the parameters `state` (restatement of the reference's op sequence)."""
    from chemprop_b200.data import BatchMolGraph
    from oracle import restatement as R

    bm = BatchMolGraph(mgs)
    bm.to(DEV)
    P = {k: v.to(DEV, torch.float64) for k, v in state.items()}
    V, E = bm.V.double(), bm.E.double()
    if cfg.get("mab"):
        return R.mab_forward(enc._kind, V, E, bm.edge_index, bm.rev_edge_index, P["W_i.weight"], P.get("W_i.bias"),
                             P["W_h.weight"], P.get("W_h.bias"), P.get("W_vo.weight"), P.get("W_vo.bias"), P.get("W_eo.weight"),
                             P.get("W_eo.bias"), enc.depth, "relu")
    kind = "bond" if type(enc).__name__.startswith("Bond") else "atom"
    return (R.message_passing_forward(kind, V, E, bm.edge_index, bm.rev_edge_index, P["W_i.weight"], P.get("W_i.bias"),
                                      P["W_h.weight"], P.get("W_h.bias"), P["W_o.weight"], P["W_o.bias"], enc.depth, "relu",
                                      cfg.get("undirected", False)),)


def _flat(outs):
    return [t for o in outs for t in (o if isinstance(o, tuple) else (o,)) if t is not None]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_replay_across_twins_equals_eager_and_float64(name):
    from chemprop_b200 import _lib
    from chemprop_b200.graph import CudaGraphStep

    t0 = time.perf_counter()
    cfg = CONFIGS[name]
    seed = 31 + list(CONFIGS).index(name)
    trio, want = _trio(cfg, seed)
    comps = trio if cfg.get("components") else [[m] for m in trio]
    fa = [T.facts(c) for c in comps[0]]
    diffs = {tw: set.union(*(T.differences(fa[k], T.facts(c)) for k, c in enumerate(comps[i])))
             for tw, i in (("B", 1), ("C", 2))}
    for tw in "BC":
        assert set(want[tw]) <= diffs[tw], (tw, want[tw], diffs[tw])
    bmgs = [[_device_batch(c) for c in cs] if cfg.get("components") else _device_batch(cs[0]) for cs in comps]
    inputs_of = cfg.get("inputs", _head_inputs("mse"))
    xs = [inputs_of(trio[i], seed + 100 * i) for i in range(3)]
    step_fn = cfg.get("step", _head_step)

    torch.manual_seed(seed)
    model_e = cfg["make"]().to(DEV).train()
    model_g = copy.deepcopy(model_e)
    lib = _lib.load()

    def runner(model, box):
        """The step `fn(b)` of `model`, its inputs read from box["x"] (eager: the step's own; graph: static buffers)."""
        params = list(model.parameters())
        for p in params:
            p.grad = torch.zeros_like(p)
        opt = torch.optim.Adam(params, lr=1e-3, capturable=True)
        outs = []
        _encoder(model, cfg).register_forward_hook(lambda m, i, o: outs.append(o))

        def fn(b):
            del outs[:]
            for p in params:
                p.grad.zero_()
            loss = step_fn(model, b, box["x"])
            loss.backward()
            opt.step()
            return (loss.detach(), *[t.detach() for t in _flat(outs)])
        return fn, opt

    # the eager sequence; the encoder's parameters before each step for the float64 restatement
    box_e = {}
    fn_e, _ = runner(model_e, box_e)
    eager, states, n_eager = [], [], []
    for i in SEQUENCE:
        states.append({k: v.detach().clone() for k, v in _encoder(model_e, cfg).state_dict().items()})
        box_e["x"] = xs[i]
        fresh = [_device_batch(c) for c in comps[i]] if cfg.get("components") else _device_batch(comps[i][0])
        l0 = lib.dmpnn_launch_count()
        out = fn_e(fresh)                       # a fresh batch object: nothing cached from an earlier step
        n_eager.append(int(lib.dmpnn_launch_count() - l0))
        eager.append(_snapshot(model_e, out))

    # the graph: captured on A, the state put back to the initial one, then A, B, C, A, B
    x_static = [None if t is None else t.clone() for t in _flat_inputs(xs[0])]
    box_g = {"x": _unflat_inputs(xs[0], x_static)}
    fn_g, opt_g = runner(model_g, box_g)
    init = {k: v.clone() for k, v in model_g.state_dict().items()}
    step = CudaGraphStep(fn_g)
    step(bmgs[0])                                 # two eager warm-up steps, the capture, one replay
    model_g.load_state_dict(init)                 # in place: the graph keeps its pointers
    for st in opt_g.state.values():
        for v in st.values():
            v.zero_()
    replayed = []
    for i in SEQUENCE:
        for s_, t in zip(x_static, _flat_inputs(xs[i])):
            if s_ is not None:
                s_.copy_(t)
        out = step(bmgs[i])
        replayed.append(_snapshot(model_g, out))
    torch.cuda.synchronize()
    assert step.captures == 1 and step.replays == 1 + len(SEQUENCE)
    launches = step.last_launches
    print(f"[graph-replay] {name}: twins B {sorted(diffs['B'])}, C {sorted(diffs['C'])}; launches per replay {launches}, "
          f"eager {n_eager}")
    assert all(n == launches for n in n_eager[1:]), (n_eager, launches)

    for k, (e, g) in enumerate(zip(eager, replayed)):
        assert [w for w, _ in e] == [w for w, _ in g]
        for (what, te), (_, tg) in zip(e, g):
            assert torch.equal(te, tg), (name, "step", k, "twin", "ABC"[SEQUENCE[k]], what)

    bf16 = _encoder(model_e, cfg).precision == "bf16"
    worst = 0.0
    for k in range(3):
        got = [t for w, t in replayed[k] if w.startswith("out.")]
        ref = []
        for c in comps[k]:
            ref += [r for r in _f64(cfg, _encoder(model_e, cfg), states[k], c) if r is not None]
        assert len(got) == len(ref), (len(got), len(ref))
        for tg, tr in zip(got, ref):
            hmax = max(1.0, tr.abs().max().item())
            bar = (1e-2 if bf16 else 1e-5) * hmax
            err = (tg.double() - tr).abs().max().item()
            worst = max(worst, err / bar)
            assert err <= bar, (name, "twin", "ABC"[k], err, bar)
    print(f"[graph-replay] {name}: worst float64 error {worst:.3f} of its bar ({'bf16' if bf16 else 'fp32'} tier); "
          f"{time.perf_counter() - t0:.1f} s")


def _flat_inputs(x):
    out = []
    for t in (x if isinstance(x, (list, tuple)) else [x]):
        out += _flat_inputs(t) if isinstance(t, (list, tuple)) else [t]
    return out


def _unflat_inputs(x, flat):
    it = iter(flat)

    def go(v):
        if isinstance(v, (list, tuple)):
            return [go(t) for t in v]
        return next(it)
    return go(x)


def _snapshot(model, out):
    return ([("loss", out[0].clone())] + [(f"out.{j}", t.clone()) for j, t in enumerate(out[1:])]
            + [(f"grad.{k}", p.grad.clone()) for k, p in model.named_parameters()]
            + [(f"state.{k}", v.clone()) for k, v in model.state_dict().items()])


def test_training_dropout_on_the_fused_step_refuses_capture():
    """The fused step's dropout masks come from a Philox offset held on the host: a captured step would replay the same
    masks every time, so dropout_keep_bits refuses capture (engine.py) and CudaGraphStep passes the error on."""
    import chemprop_b200.nn as N
    from chemprop_b200 import DmpnnError, engine
    from chemprop_b200.graph import CudaGraphStep

    torch.manual_seed(0)
    model = N.EngineMPNN(N.BondMessagePassing(d_h=64, dropout=0.2, precision="bf16"), N.MeanAggregation(),
                         N.EngineRegressionFFN(input_dim=64)).to(DEV).train()
    mgs = batches("bond", "windows", (72, 14), 5, 200)[0]
    bmg = _device_batch(mgs)
    Y = torch.randn(len(mgs), 1, device=DEV)
    for p in model.parameters():
        p.grad = torch.zeros_like(p)

    def fn(b):
        loss = model.training_loss(b, Y)
        loss.backward()
        return loss

    fn(bmg)                                     # eagerly the step runs, on the fused path's dropout
    assert model.message_passing._dropout_on_fused_path(engine.get_layout(bmg))
    with pytest.raises(DmpnnError, match="dropout inside a captured CUDA graph"):
        CudaGraphStep(fn)(bmg)
    torch.cuda.synchronize()
