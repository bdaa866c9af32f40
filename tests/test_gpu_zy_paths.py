"""GPU tier: every execution path `engine.plan()` can choose for a message-passing call, at batch scale, against float64.

A path is a host composition of kernels -- forward function, mirror function, GEMM family, fused or unfused depth loop -- and
its plan key is  (kind, gemm, fused, forward.__name__, mirror.__name__, undirected and E > 0, E == 0).  The kernels have
their own float64 tests; this file runs each composition end to end on ~1 500 molecules with shuffled edge order, so that
the persistent tile loop, the 128-row windows of molecules with more than 128 directed edges, atoms of in-degree up to 11
(K_6 .. K_12) and the weight-gradient launches over many row blocks are all reached.  Each case

  * asserts that the call took the plan key `CASES` declares for it, and that its batch has what the case is for (windows
    and in-degree > 4, an oversized molecule, no edges);
  * runs forward, MeanAggregation, a fixed random projection (agg . G).sum() -- every gradient term gets an independent
    weight -- and backward;
  * compares H_v, the aggregate and all six parameter gradients with oracle/restatement.py in float64 on the same weights,
    and, for precision="bf16", with the rounding-aware emulation of the same tier (tests/emu.py).

Keys that an earlier test already runs at batch scale against float64 are declared with that test's name (`covered_by`)
and not run again.  tests/test_path_coverage_host.py checks on the CPU that the keys of `CASES` are exactly the keys
`plan()` can produce, so a new path fails there until a case here covers it.  This module imports nothing CUDA at import.

Bars (those of tests/test_gpu_fp32_wide.py::test_module_wide_vs_f64_oracle and
tests/test_gpu_parity.py::test_bf16_mirror_vs_rounding_aware_emulation):
  * fp32: H_v and the aggregate within 1e-5 * max(1, max|H|) (5e-5 at depth >= 6); each gradient within 2e-4 of its
    max-abs, and 2e-5 in the relative Frobenius norm;
  * bf16 against the emulation: |dH| <= 4e-2 (times |H| / 2 where the element exceeds 2: the ReLU cases reach |H| ~ 40, and
    4e-2 is 2.5 ulps of the stored bf16 at |H| in [2, 4)), with at most 1 % of the elements above 1e-3; gradients within 2 %
    (max-abs of the tensor's scale, and Frobenius);
  * bf16 against float64: H_v and the aggregate within 1e-2 * max(1, max|H|); gradients within 6 % (max-abs and Frobenius;
    the max-abs bar is 20 % on batches with K_k, as in tests/test_gpu_high_degree.py).
A case that needs a wider bar says why beside it.
Each case prints its plan key and its worst error as a fraction of each bar."""
from __future__ import annotations

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N_MOLS = 1500

# fp32 tier: SIMT f32 GEMMs / 3xTF32 tensor-core GEMMs; bf16 tier: "tc" = bf16 tensor cores
_FUSED_UND = ("bond", "tc", True, "bond_forward", "bond_backward", True, False)
_TC_UND = ("bond", "tc", False, "bond_forward", "bond_backward", True, False)
_SIMT_UND = ("bond", "simt", False, "bond_forward", "bond_backward", True, False)
_SIMT_DIR = ("bond", "simt", False, "bond_forward", "bond_backward", False, False)
_ATOM_TC = ("atom", "tc", False, "atom_forward_tc", "atom_backward_tc", False, False)

# kind, precision, d_h, depth, activation, bias, undirected; batch: see `molecules` ("mixed" when absent); dims: (d_v, d_e);
# patch: engine switches set for the call
CASES = {
    # undirected bonds, on every tier
    "U1-bond-bf16-fused-undirected-relu-bias": dict(
        kind="bond", precision="bf16", d_h=300, depth=3, act="relu", bias=True, undirected=True, key=_FUSED_UND),
    "U2-bond-bf16-fused-undirected-tanh-d4": dict(
        kind="bond", precision="bf16", d_h=300, depth=4, act="tanh", bias=False, undirected=True, batch="windows",
        key=_FUSED_UND),
    "U3-bond-bf16-undirected-fused-switch-off": dict(
        kind="bond", precision="bf16", d_h=300, depth=3, act="relu", bias=True, undirected=True,
        patch=dict(UNDIRECTED_FUSED=False), key=_TC_UND),
    "U4-bond-bf16-undirected-dh298": dict(
        kind="bond", precision="bf16", d_h=298, depth=3, act="tanh", bias=True, undirected=True, batch="windows",
        key=_TC_UND),
    "U5-bond-bf16-undirected-simt-dh320": dict(
        kind="bond", precision="bf16", d_h=320, depth=3, act="relu", bias=True, undirected=True, key=_SIMT_UND),
    # grad_bars: at depth 6 the random projection's gradients cancel over five mirror steps, and plain f32 arithmetic (torch on
    # the CPU, every GEMM in f32) already lands 8.0e-4 of the max-abs and 2.1e-4 in Frobenius from float64 on this batch --
    # 4x and 10x the fp32 bars, which were set on a square().sum() loss at depth <= 6.  Held to twice that f32 floor.
    "U6-bond-fp32-undirected-x3-dh600-d6": dict(
        kind="bond", precision="fp32", d_h=600, depth=6, act="relu", bias=True, undirected=True, batch="windows",
        grad_bars=(1.6e-3, 4.2e-4), key=("bond", "x3", False, "bond_forward", "bond_backward", True, False)),
    "U7-bond-fp32-undirected-simt-dh298": dict(
        kind="bond", precision="fp32", d_h=298, depth=3, act="tanh", bias=True, undirected=True, key=_SIMT_UND),
    # directed bonds off the benchmarked path
    "D1-bond-bf16-fused-generic-mirror-dh298-tanh": dict(
        kind="bond", precision="bf16", d_h=298, depth=3, act="tanh", bias=True, undirected=False, batch="windows",
        key=("bond", "tc", True, "bond_forward", "bond_backward", False, False)),
    "D2-bond-bf16-depth1": dict(
        kind="bond", precision="bf16", d_h=300, depth=1, act="relu", bias=True, undirected=False,
        key=("bond", "tc", False, "bond_forward", "bond_backward_tc", False, False)),
    "D3-bond-fp32-simt-x3-switch-off": dict(
        kind="bond", precision="fp32", d_h=300, depth=3, act="relu", bias=True, undirected=False,
        patch=dict(X3_ENABLED=False), key=_SIMT_DIR),
    "D4-bond-bf16-depth1-dh298": dict(
        kind="bond", precision="bf16", d_h=298, depth=1, act="tanh", bias=True, undirected=False,
        key=("bond", "tc", False, "bond_forward", "bond_backward", False, False)),
    # the two-launch atom step
    "A1-atom-bf16-oversized-molecule": dict(
        kind="atom", precision="bf16", d_h=300, depth=3, act="relu", bias=True, undirected=False, batch="oversized",
        key=_ATOM_TC),
    "A2-atom-bf16-cgr-d5-fused-switch-off": dict(
        kind="atom", precision="bf16", d_h=300, depth=5, act="relu", bias=True, undirected=False, dims=(106, 28), batch="windows",
        patch=dict(ATOM_FUSED_ENABLED=False), key=_ATOM_TC),
    "A3-atom-bf16-depth1": dict(
        kind="atom", precision="bf16", d_h=300, depth=1, act="relu", bias=True, undirected=False, key=_ATOM_TC),
    "A4-atom-bf16-simt-dh298": dict(
        kind="atom", precision="bf16", d_h=298, depth=3, act="relu", bias=True, undirected=False,
        key=("atom", "simt", False, "atom_forward", "atom_backward", False, False)),
    # batches without edges: one case per key
    "E1-bond-bf16-edgeless": dict(
        kind="bond", precision="bf16", d_h=300, depth=3, act="tanh", bias=True, undirected=True, batch="edgeless",
        key=("bond", "tc", False, "bond_forward", "bond_backward", False, True)),
    "E2-bond-fp32-x3-edgeless": dict(
        kind="bond", precision="fp32", d_h=300, depth=3, act="relu", bias=True, undirected=False, batch="edgeless",
        key=("bond", "x3", False, "bond_forward", "bond_backward", False, True)),
    "E3-bond-fp32-simt-edgeless": dict(
        kind="bond", precision="fp32", d_h=298, depth=3, act="relu", bias=True, undirected=False, batch="edgeless",
        key=("bond", "simt", False, "bond_forward", "bond_backward", False, True)),
    "E4-atom-bf16-edgeless": dict(
        kind="atom", precision="bf16", d_h=300, depth=3, act="tanh", bias=True, undirected=False, batch="edgeless",
        key=("atom", "tc", False, "atom_forward_tc", "atom_backward_tc", False, True)),
    "E5-atom-fp32-edgeless": dict(
        kind="atom", precision="fp32", d_h=300, depth=3, act="relu", bias=True, undirected=False, batch="edgeless",
        key=("atom", "simt", False, "atom_forward", "atom_backward", False, True)),
    # keys an existing test already runs at batch scale against float64 (one of its configurations)
    "bond-bf16-fused-tc-mirror": dict(
        kind="bond", precision="bf16", d_h=300, depth=3, act="relu", bias=True, undirected=False,
        key=("bond", "tc", True, "bond_forward", "bond_backward_tc", False, False),
        covered_by="tests/test_gpu_parity.py::test_bf16_mirror_vs_rounding_aware_emulation"),
    "bond-fp32-x3": dict(
        kind="bond", precision="fp32", d_h=600, depth=6, act="relu", bias=True, undirected=False,
        key=("bond", "x3", False, "bond_forward", "bond_backward", False, False),
        covered_by="tests/test_gpu_fp32_wide.py::test_module_wide_vs_f64_oracle"),
    "bond-bf16-over-tc-limits": dict(
        kind="bond", precision="bf16", d_h=2048, depth=3, act="tanh", bias=True, undirected=False,
        key=_SIMT_DIR, covered_by="tests/test_gpu_fp32_wide.py::test_module_wide_vs_f64_oracle"),
    "atom-bf16-fused-step": dict(
        kind="atom", precision="bf16", d_h=300, depth=3, act="relu", bias=True, undirected=False,
        key=("atom", "tc", True, "atom_forward_fused", "atom_backward_fused", False, False),
        covered_by="tests/test_gpu_fused_activations.py::test_module_vs_f64_oracle"),
}

GPU_CASES = [n for n, c in CASES.items() if "covered_by" not in c]


def plan_key(kind: str, cfg, lay, p) -> tuple:
    """The plan key of one `engine.plan(kind, cfg, lay, ...)` call that returned `p`."""
    return (kind, p.gemm, p.fused, p.forward.__name__, p.mirror.__name__, bool(cfg.undirected and lay.E > 0), lay.E == 0)


def case_dims(c: dict) -> tuple:
    return c.get("dims", (72, 14))


def molecules(c: dict, seed: int, n_mols: int = N_MOLS) -> list:
    """The batch of case `c`, shuffled edge and molecule order.  "mixed": n_mols molecules of ~25 atoms, 20 of 66-200 atoms (more
    than 128 directed edges: the fused step's 128-row windows), and two copies of each K_6 .. K_12 (in-degree up to 11);
    "windows": the same without the K_k; "oversized": mixed plus one molecule of 130-140 atoms (more than an atom tile);
    "edgeless": n_mols single atoms (its bf16 cases use tanh: with ReLU, a kink flip of one single-atom molecule
    moves the W_o gradient by 8 % of its scale).

    The K_k stay out of the tanh cases of the bf16 tier and of the deepest ones (depth 5 and 6): on a K_k every step multiplies a perturbation of H by
    up to (k - 1) * ||W_h|| ~ 10, so after two or three steps the bf16 storage error of those molecules' H_v reaches several
    percent of |tanh| <= 1 (measured through the emulation: 9.5x the 1e-2 bar at U2) -- the conditioning of the input, not a
    property of the path -- and at depth 5-6 their H grows to ~1 000-2 400, where plain f32 arithmetic exceeds the fp32
    tier's Frobenius bar.  ReLU cases at depth <= 3 scale their bars with max|H| and keep the K_k."""
    from chemprop_b200.data import make_molecule, make_molecules
    from tests.test_gpu_high_degree import high_degree_molecules

    d_v, d_e = case_dims(c)
    rng = np.random.default_rng(seed)
    batch = c.get("batch", "mixed")
    if batch == "edgeless":
        return [make_molecule(rng, 1, d_v, d_e) for _ in range(n_mols)]
    mgs = make_molecules(n_mols, seed=seed, d_v=d_v, d_e=d_e, shuffle_edges=True)
    big = 200 if c["kind"] == "bond" else 128        # an atom tile holds 128 atoms: larger is the "oversized" batch
    mgs += make_molecules(20, seed=seed + 1, mean_atoms=110.0, std_atoms=40.0, min_atoms=66, max_atoms=big, d_v=d_v, d_e=d_e,
                          shuffle_edges=True)
    if batch != "windows":
        mgs += high_degree_molecules(0, seed=seed + 2, kmax=12, reps=2, d_v=d_v, d_e=d_e)
    if batch == "oversized":
        mgs += make_molecules(1, seed=seed + 3, mean_atoms=135.0, std_atoms=3.0, min_atoms=130, max_atoms=140, d_v=d_v,
                              d_e=d_e, shuffle_edges=True)
    return [mgs[i] for i in rng.permutation(len(mgs))]


def _check_batch(c: dict, lay, n_mols: int = N_MOLS):
    """The batch really has what the case is for, whatever the generators do."""
    batch = c.get("batch", "mixed")
    if batch == "edgeless":
        assert lay.E == 0 and lay.V == n_mols
        return
    assert (lay.max_indeg > 4) == (batch != "windows"), lay.max_indeg
    if c["kind"] == "bond":
        assert lay.max_tile_rows > 128, lay.max_tile_rows
    else:
        assert (lay.max_tile_atoms > 128) == (batch == "oversized"), lay.max_tile_atoms


def _report(name, what, err, bar):
    print(f"[zy-paths] {name} {what}: {err:.3e} of bar {bar:.3e} ({err / bar if bar else 0.0:.3f})")
    return err / bar if bar else 0.0


def _close_h(name, what, got, ref, bar):
    err = (got.double().cpu() - ref.double().cpu()).abs().max().item()
    frac = _report(name, what, err, bar)
    assert err <= bar, (name, what, err, bar)
    return frac


def _close_grad(name, what, got, ref, rel_max, rel_fro):
    got, ref = got.double().cpu(), ref.double().cpu()
    scale = max(1e-6, ref.abs().max().item())
    err = (got - ref).abs().max().item()
    fro = ((got - ref).norm() / max(1e-12, ref.norm().item())).item()
    frac = max(_report(name, f"{what} max", err / scale, rel_max), _report(name, f"{what} frob", fro, rel_fro))
    assert err <= rel_max * scale and fro <= rel_fro, (name, what, err, scale, fro)
    return frac


def _f64_oracle(c, mgs, state, Gm):
    """H_v, the mean aggregate and the six parameter gradients of oracle/restatement.py in float64 (on the GPU)."""
    from chemprop_b200.data import BatchMolGraph
    from oracle import restatement as R

    bm = BatchMolGraph(mgs)
    bm.to("cuda")
    P = {k: v.double().cuda().requires_grad_(True) for k, v in state.items()}
    H_ref = R.message_passing_forward(c["kind"], bm.V.double(), bm.E.double(), bm.edge_index, bm.rev_edge_index,
                                      P["W_i.weight"], P.get("W_i.bias"), P["W_h.weight"], P.get("W_h.bias"),
                                      P["W_o.weight"], P["W_o.bias"], c["depth"], c["act"], c["undirected"])
    a_ref = R.aggregate(H_ref, bm.batch, "mean", n_mols=len(mgs))
    (a_ref * Gm.double().cuda()).sum().backward()
    # a parameter the oracle never uses (W_h at depth 1, W_i and W_h without edges) has a zero gradient
    out = (H_ref.detach().cpu(), a_ref.detach().cpu(),
           {k: (p.grad if p.grad is not None else torch.zeros_like(p)).cpu() for k, p in P.items()})
    del P, H_ref, a_ref
    torch.cuda.empty_cache()
    return out


def _module_factory(c, state):
    from chemprop_b200.nn import AtomMessagePassing, BondMessagePassing

    cls = BondMessagePassing if c["kind"] == "bond" else AtomMessagePassing
    d_v, d_e = case_dims(c)

    def make(device):
        mp = cls(d_v=d_v, d_e=d_e, d_h=c["d_h"], depth=c["depth"], bias=c["bias"], activation=c["act"],
                 undirected=c["undirected"], precision=c["precision"])
        if state is not None:
            mp.load_state_dict(state)
        return mp.to(device)

    return make


def _initial_state(c, seed):
    """The module's own initialisation under a fixed seed, as f32 tensors on the CPU."""
    torch.manual_seed(seed)
    return {k: v.detach().clone() for k, v in _module_factory(c, None)("cpu").state_dict().items()}


@pytest.mark.parametrize("name", GPU_CASES)
def test_execution_path_vs_f64_oracle(name, monkeypatch):
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.nn import MeanAggregation
    from tests.test_gpu_parity import _emulated_run

    c = CASES[name]
    seed = 101 + 7 * GPU_CASES.index(name)
    for k, v in c.get("patch", {}).items():
        monkeypatch.setattr(engine, k, v)
    mgs = molecules(c, seed)
    state = _initial_state(c, seed)
    make = _module_factory(c, state)
    Gm = torch.randn(len(mgs), c["d_h"], generator=torch.Generator().manual_seed(seed + 3))
    loss_fn = lambda H, b: (MeanAggregation()(H, b.batch).float() * Gm.to(H.device)).sum()  # noqa: E731

    H_ref, a_ref, g_ref = _f64_oracle(c, mgs, state, Gm)

    keys = []
    plan0 = engine.plan

    def spy(kind, cfg, lay, *a):
        p = plan0(kind, cfg, lay, *a)
        keys.append(plan_key(kind, cfg, lay, p))
        return p

    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    mp = make("cuda")
    with monkeypatch.context() as m:
        m.setattr(engine, "plan", spy)
        assert not mp.uses_composed_tier(engine.get_layout(bmg))
        H = mp(bmg)
        a = MeanAggregation()(H, bmg.batch)
        (a.float() * Gm.cuda()).sum().backward()
        torch.cuda.synchronize()
    lay = engine.get_layout(bmg)
    print(f"[zy-paths] {name}: plan key {keys[0] if keys else None}; E = {lay.E}, V = {lay.V}, max in-degree "
          f"{lay.max_indeg}, max tile rows {lay.max_tile_rows}, max tile atoms {lay.max_tile_atoms}")
    assert keys == [c["key"]], keys
    _check_batch(c, lay)
    grads = {k: p.grad for k, p in mp.named_parameters()}
    assert set(grads) == set(g_ref) and all(g is not None for g in grads.values())

    bf16 = c["precision"] == "bf16"
    hmax = max(1.0, H_ref.abs().max().item())
    worst = {}
    if bf16:
        # with the K_k in the batch the max-abs bar is 20 %, as in test_module_high_indegree_vs_oracle_and_emulation: bf16
        # storage flips ReLU kinks of their |H| ~ 40-60 states and moves single entries of the atom kinds' W_i / W_o gradients
        # 7-11 % from float64 (measured through the emulation); the Frobenius bar stays 6 %, the emulation's 2 %
        tol, gmax, gfro = 1e-2 * hmax, (0.2 if c.get("batch", "mixed") in ("mixed", "oversized") else 6e-2), 6e-2
    else:
        tol, (gmax, gfro) = (5e-5 if c["depth"] >= 6 else 1e-5) * hmax, c.get("grad_bars", (2e-4, 2e-5))
    worst["H_v vs f64"] = _close_h(name, "H_v vs f64", H.detach(), H_ref, tol)
    worst["agg vs f64"] = _close_h(name, "agg vs f64", a.detach(), a_ref, tol)
    worst["grads vs f64"] = max(_close_grad(name, f"{k} vs f64", grads[k], g_ref[k], gmax, gfro) for k in grads)
    if bf16:
        H_e, egrads = _emulated_run(lambda: make("cpu"), lambda: BatchMolGraph(mgs), None, loss_fn)
        dH = (H.detach().float().cpu() - H_e).abs()
        # 4e-2 is 2.5 bf16 ulps at |H| in [2, 4); the K_k molecules reach |H| ~ 40, where one ulp of the stored H_v is 0.25,
        # so the bar grows with the element's magnitude above 2: at least 2.5 ulps of it everywhere
        bar = 4e-2 * (H_e.abs() / 2).clamp_min(1.0)
        worst["H_v vs emulation"] = _report(name, "H_v vs emulation (of the element's bar)", (dH / bar).max().item(), 1.0)
        assert bool((dH <= bar).all()), (name, dH.max().item())
        above = (dH > 1e-3).float().mean().item()
        worst["H_v above 1e-3"] = _report(name, "H_v share above 1e-3 vs emulation", above, 1e-2)
        assert above <= 1e-2, above
        worst["grads vs emulation"] = max(_close_grad(name, f"{k} vs emulation", grads[k], egrads[k], 2e-2, 2e-2)
                                          for k in grads)
    print(f"[zy-paths] {name}: worst fraction of each bar " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_undirected_atom_message_passing_on_the_composed_tier_vs_f64_oracle(precision, monkeypatch):
    """AtomMessagePassing(undirected=True) does not go through `plan()`: averaging H with its reverse breaks the atom-granular
    restatement of the monolithic tiers, so it runs on the composed tier (composed.atom_forward, f32 hidden states whatever
    the precision).  Eval mode, the mixed batch of the cases above, against float64.

    fp32: H_v and the aggregate at the fp32 bar.  The gradients of W_i / W_h / b_i / b_h have an f32 floor on the atom kind:
    restatement.py itself run in float32 lands 2.3e-3 of the max-abs and 2.4e-4 in Frobenius from float64 on a batch
    without the K_k, and this batch measures 3.3e-4 / 4.6e-5 (identical digits from the composed tier on the device and in
    the emulation on the CPU): an atom state whose pre-activation lies within f32 rounding of a ReLU kink feeds every one of
    its out-edges.  They are held to 1e-3 of the max-abs (test_cgr_dims_vs_oracle's bar for fp32 atoms) and 1e-4 in
    Frobenius, about twice the floor; W_o and b_o, which see no kink, keep the fp32 bars (measured ~4e-7).
    bf16: the module returns H_v in bf16 (H_v and the aggregate within 1e-2 * max(1, max|H|)), and the gradient arriving at
    H_v is bf16, each element within 2^-9 of its f32 value; everything after it is f32, so the gradients are held to 1e-2
    (max-abs and Frobenius) -- a sixth of the bf16 tier's 6e-2, and far above the f32 round-off."""
    from chemprop_b200 import engine
    from chemprop_b200.data import BatchMolGraph
    from chemprop_b200.nn import MeanAggregation

    name = f"composed-atom-undirected-{precision}"
    c = dict(kind="atom", precision=precision, d_h=300, depth=3, act="relu", bias=True, undirected=True)
    seed = 977
    mgs = molecules(c, seed)
    state = _initial_state(c, seed)
    Gm = torch.randn(len(mgs), c["d_h"], generator=torch.Generator().manual_seed(seed + 3))
    H_ref, a_ref, g_ref = _f64_oracle(c, mgs, state, Gm)

    calls = []
    plan0 = engine.plan
    monkeypatch.setattr(engine, "plan", lambda *a, **k: (calls.append(a[0]), plan0(*a, **k))[1])
    bmg = BatchMolGraph(mgs)
    bmg.to("cuda")
    lay = engine.get_layout(bmg)
    _check_batch(c, lay)
    mp = _module_factory(c, state)("cuda").eval()
    assert mp.uses_composed_tier(lay)
    H = mp(bmg)
    a = MeanAggregation()(H, bmg.batch)
    (a.float() * Gm.cuda()).sum().backward()
    torch.cuda.synchronize()
    assert not calls, calls
    assert H.dtype == (torch.bfloat16 if precision == "bf16" else torch.float32)
    hmax = max(1.0, H_ref.abs().max().item())
    tol, gmax, gfro = (1e-2 * hmax, 1e-2, 1e-2) if precision == "bf16" else (1e-5 * hmax, 2e-4, 2e-5)
    worst = {"H_v vs f64": _close_h(name, "H_v vs f64", H.detach().float(), H_ref, tol),
             "agg vs f64": _close_h(name, "agg vs f64", a.detach(), a_ref, tol)}
    grads = {k: p.grad for k, p in mp.named_parameters()}
    assert set(grads) == set(g_ref)
    if precision == "fp32":
        floor = {k: (1e-3, 1e-4) for k in ("W_i.weight", "W_i.bias", "W_h.weight", "W_h.bias")}
        worst["grads vs f64"] = max(_close_grad(name, f"{k} vs f64", grads[k], g_ref[k], *floor.get(k, (gmax, gfro)))
                                    for k in grads)
    else:
        worst["grads vs f64"] = max(_close_grad(name, f"{k} vs f64", grads[k], g_ref[k], gmax, gfro) for k in grads)
    print(f"[zy-paths] {name}: worst fraction of each bar " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
