"""TEST INFRASTRUCTURE ONLY -- the oracle.  A CPU restatement, in plain torch ops, of the reference
algorithm for the D-MPNN hot path (chemprop v2.3.1).  It exists because `/root/reference` does not
travel to the GPU box; it is the checker the CUDA path is compared with, never the thing measured or
shipped, and nothing under ``chemprop_b200/`` imports it.

PARITY PINNING: this restatement is pinned against the *real* reference in two ways:
  (1) tests/golden/*.npz were produced by running the unmodified reference modules
      (oracle/make_golden.py, via oracle/ref_shim.py) -- tests/test_oracle.py checks the restatement
      against every golden case (forward outputs, aggregation outputs, weight gradients);
  (2) when /root/reference is reachable the same test also runs the reference live on fresh seeds.
The reference has no numeric known-answer test for BondMessagePassing.forward itself
(SURVEY.md section 8c); its structural fixtures (chain graph, E=0 batch, collate values) are among
the golden cases.

Every function cites the reference lines it follows (paths relative to the chemprop repo root).
Works in float32 or float64 (pass tensors of that dtype); autograd gives the reference gradients.
"""
from __future__ import annotations

import numpy as np
import torch
from torch import Tensor
from torch.nn import functional as F


# --- activations: chemprop/nn/utils.py:43-55 ------------------------------------------------
def activation(name, prelu_weight: Tensor | None = None, param: float | None = None):
    """utils.py:19-55.  `name` may also be a callable (utils.py:37-42 passes modules through, e.g. nn.LeakyReLU(0.3));
    "prelu" takes the learnable slope (nn.PReLU: one parameter, initial value 0.25); `param` replaces the default
    negative slope of "leakyrelu" (0.1) and alpha of "elu" (1.0)."""
    if callable(name):
        return name
    name = name.lower()
    if name == "relu":
        return torch.relu
    if name == "leakyrelu":
        return lambda x: F.leaky_relu(x, 0.1 if param is None else param)
    if name == "prelu":
        assert prelu_weight is not None, "prelu needs its weight"
        return lambda x: F.prelu(x, prelu_weight)
    if name == "tanh":
        return torch.tanh
    if name == "elu":
        return F.elu if param is None else (lambda x: F.elu(x, param))
    if name == "selu":
        return F.selu
    if name == "softplus":
        return F.softplus
    raise KeyError(name)


# --- collate: chemprop/data/collate.py:37-62 ------------------------------------------------
def collate(mgs):
    """Returns (V f32, E f32, edge_index i64 2xE, rev_edge_index i64, batch i64) as numpy arrays."""
    Vs, Es, eis, revs, batch = [], [], [], [], []
    num_nodes = 0
    num_edges = 0
    for i, mg in enumerate(mgs):
        Vs.append(mg.V)
        Es.append(mg.E)
        eis.append(mg.edge_index + num_nodes)            # collate.py:51
        revs.append(mg.rev_edge_index + num_edges)       # collate.py:52
        batch.append(np.full(len(mg.V), i, dtype=np.int64))  # collate.py:53
        num_nodes += mg.V.shape[0]
        num_edges += mg.edge_index.shape[1]
    return (np.concatenate(Vs).astype(np.float32), np.concatenate(Es).astype(np.float32),
            np.hstack(eis).astype(np.int64), np.concatenate(revs).astype(np.int64),
            np.concatenate(batch).astype(np.int64))


def collate_torch(mgs):
    """collate.py:40-62 operation for operation (Python lists for `batch`, `torch.from_numpy(...).float()` / `.long()`
    conversions): the version bench.py times as the reference's batch assembly."""
    Vs, Es, edge_indexes, rev_edge_indexes, batch_indexes = [], [], [], [], []
    num_nodes = 0
    num_edges = 0
    for i, mg in enumerate(mgs):
        Vs.append(mg.V)
        Es.append(mg.E)
        edge_indexes.append(mg.edge_index + num_nodes)
        rev_edge_indexes.append(mg.rev_edge_index + num_edges)
        batch_indexes.append([i] * len(mg.V))
        num_nodes += mg.V.shape[0]
        num_edges += mg.edge_index.shape[1]
    return (torch.from_numpy(np.concatenate(Vs)).float(), torch.from_numpy(np.concatenate(Es)).float(),
            torch.from_numpy(np.hstack(edge_indexes)).long(), torch.from_numpy(np.concatenate(rev_edge_indexes)).long(),
            torch.tensor(np.concatenate(batch_indexes)).long())


# --- scatter-sum idiom: mixins.py:12-15, base.py:208-211 -----------------------------------
def _scatter_sum_rows(H: Tensor, index: Tensor, n_rows: int) -> Tensor:
    index_torch = index.unsqueeze(1).repeat(1, H.shape[1])
    return torch.zeros(n_rows, H.shape[1], dtype=H.dtype, device=H.device).scatter_reduce_(
        0, index_torch, H, reduce="sum", include_self=False)


# --- bond message passing -------------------------------------------------------------------
def bond_initialize(V, E, edge_index, W_i, b_i=None):
    """mixins.py:8-9"""
    return F.linear(torch.cat([V[edge_index[0]], E], dim=1), W_i, b_i)


def bond_message(H, edge_index, rev_edge_index, n_atoms):
    """mixins.py:11-18"""
    M_all = _scatter_sum_rows(H, edge_index[1], n_atoms)[edge_index[0]]
    M_rev = H[rev_edge_index]
    return M_all - M_rev


def atom_initialize(V, edge_index, W_i, b_i=None):
    """mixins.py:22-23"""
    return F.linear(V[edge_index[0]], W_i, b_i)


def atom_message(H, E, edge_index, n_atoms):
    """mixins.py:25-30  (concat order is (H, E))"""
    HE = torch.cat((H, E), dim=1)
    return _scatter_sum_rows(HE, edge_index[1], n_atoms)[edge_index[0]]


def _no_dropout(H):
    return H


def update(M_t, H_0, W_h, b_h, tau, dropout=_no_dropout):
    """base.py:135-141"""
    return dropout(tau(H_0 + F.linear(M_t, W_h, b_h)))


def finalize(M, V, W_o, b_o, tau, V_d=None, W_d=None, b_d=None, dropout=_no_dropout):
    """base.py:143-194 (note: no activation after W_d)"""
    H = dropout(tau(F.linear(torch.cat((V, M), dim=1), W_o, b_o)))
    if V_d is not None:
        H = dropout(F.linear(torch.cat((H, V_d), dim=1), W_d, b_d))
    return H


def message_passing_forward(kind, V, E, edge_index, rev_edge_index, W_i, b_i, W_h, b_h, W_o, b_o, depth, act="relu",
                            undirected=False, V_d=None, W_d=None, b_d=None, return_intermediates=False,
                            prelu_weight=None, dropout_masks=None, act_param=None):
    """_MessagePassingBase.forward, base.py:196-212.  kind in {"bond", "atom"}.
    `dropout_masks`: training-mode dropout with the masks given explicitly -- a list of already scaled
    (0 or 1/(1-p)) tensors consumed in call order (one E x h mask per depth step, base.py:139; one V x h mask after
    W_o, base.py:182; one after W_d, base.py:188), so a run can be compared mask for mask.
    `act_param`: the LeakyReLU slope / ELU alpha when `act` is a name."""
    tau = activation(act, prelu_weight, act_param)
    masks = list(dropout_masks) if dropout_masks is not None else None
    dropout = _no_dropout if masks is None else (lambda H: H * masks.pop(0))
    n_atoms = V.shape[0]
    H_0 = bond_initialize(V, E, edge_index, W_i, b_i) if kind == "bond" else atom_initialize(V, edge_index, W_i, b_i)
    H = tau(H_0)                                                   # base.py:200
    inter = {"H_0": H_0, "H": [H], "M": []}
    for _ in range(1, depth):                                      # base.py:201
        if undirected:
            H = (H + H[rev_edge_index]) / 2                        # base.py:202-203
        if kind == "bond":
            M = bond_message(H, edge_index, rev_edge_index, n_atoms)
        else:
            M = atom_message(H, E, edge_index, n_atoms)
        H = update(M, H_0, W_h, b_h, tau, dropout)                 # base.py:206
        inter["M"].append(M)
        inter["H"].append(H)
    M_v = _scatter_sum_rows(H, edge_index[1], n_atoms)             # base.py:208-211
    out = finalize(M_v, V, W_o, b_o, tau, V_d, W_d, b_d, dropout)
    if return_intermediates:
        inter["M_v"] = M_v
        return out, inter
    return out


def mab_forward(kind, V, E, edge_index, rev_edge_index, W_i, b_i, W_h, b_h, W_vo, b_vo, W_eo, b_eo, depth, act="relu",
                undirected=False, V_d=None, W_vd=None, b_vd=None, E_d=None, W_ed=None, b_ed=None, prelu_weight=None,
                return_vertex=True, return_edge=True, dropout_masks=None, act_param=None):
    """_MABMessagePassingBase.forward (chemprop/nn/message_passing/mol_atom_bond.py): the loop of base.py:196-206,
    then vertex_finalize (same as `finalize`) and edge_finalize: tau(W_eo([E || H])) [-> W_ed([. || E_d])] per directed
    edge.  kind in {"bond", "atom"}.  Returns (H_v | None, H_e | None).
    `dropout_masks`: training-mode dropout with the masks given explicitly, already scaled (0 or 1/(1-p)), in the order
    the reference draws them: one E x h mask per depth step, then vertex_finalize's (after W_vo, after W_vd) when the vertex
    read-out exists, then edge_finalize's (after W_eo, after W_ed) when the edge read-out does.
    `act_param`: the LeakyReLU slope / ELU alpha when `act` is a name."""
    tau = activation(act, prelu_weight, act_param)
    masks = list(dropout_masks) if dropout_masks is not None else None
    loop_masks = None
    if masks is not None:
        n = max(depth - 1, 0) + ((1 + (V_d is not None)) if W_vo is not None else 0)
        # without a vertex read-out the dummy one below still consumes a mask: a scalar one
        loop_masks, masks = masks[:n] + ([] if W_vo is not None else [torch.ones((), dtype=V.dtype, device=V.device)]), masks[n:]
    if W_vo is None:   # edge embeddings only: the vertex read-out does not exist; run the loop with a dummy W_o
        W_vo_, b_vo_ = torch.zeros(1, V.shape[1] + W_h.shape[0], dtype=V.dtype, device=V.device), None
    else:
        W_vo_, b_vo_ = W_vo, b_vo
    H_v, inter = message_passing_forward(kind, V, E, edge_index, rev_edge_index, W_i, b_i, W_h, b_h, W_vo_, b_vo_, depth,
                                         act, undirected, V_d if W_vo is not None else None, W_vd, b_vd,
                                         return_intermediates=True, prelu_weight=prelu_weight, dropout_masks=loop_masks,
                                         act_param=act_param)
    H = inter["H"][-1]
    H_e = None
    if return_edge:
        dropout = _no_dropout if masks is None else (lambda X: X * masks.pop(0))
        H_e = dropout(tau(F.linear(torch.cat((E, H), dim=1), W_eo, b_eo)))
        if E_d is not None:
            H_e = dropout(F.linear(torch.cat((H_e, E_d), dim=1), W_ed, b_ed))
    return (H_v if (return_vertex and W_vo is not None) else None), H_e


# --- aggregation: chemprop/nn/agg.py:65-113 --------------------------------------------------
def aggregate(H, batch, mode="mean", norm=100.0, n_mols=None):
    index_torch = batch.unsqueeze(1).repeat(1, H.shape[1])
    dim_size = int(batch.max()) + 1 if n_mols is None else n_mols    # agg.py:75
    red = "mean" if mode == "mean" else "sum"
    out = torch.zeros(dim_size, H.shape[1], dtype=H.dtype, device=H.device).scatter_reduce_(
        0, index_torch, H, reduce=red, include_self=False)           # agg.py:76-78 / 93-95
    if mode == "norm":
        out = out / norm                                             # agg.py:112-113
    return out


def attentive_aggregate(H, batch, W, b, n_mols=None):
    """AttentiveAggregation.forward, chemprop/nn/agg.py:121-133 (no max-subtraction, as in the reference)."""
    dim_size = int(batch.max()) + 1 if n_mols is None else n_mols
    logits = F.linear(H, W, b).exp()                                                        # agg.py:123
    Z = torch.zeros(dim_size, 1, dtype=H.dtype).scatter_reduce_(0, batch.unsqueeze(1), logits, reduce="sum",
                                                                include_self=False)         # agg.py:124-126
    alphas = logits / Z[batch]                                                              # agg.py:127
    index_torch = batch.unsqueeze(1).repeat(1, H.shape[1])
    return torch.zeros(dim_size, H.shape[1], dtype=H.dtype).scatter_reduce_(0, index_torch, alphas * H, reduce="sum",
                                                                            include_self=False)   # agg.py:128-131


def constrain(k, preds, batch, constraints):
    """ConstrainerFFN.forward after its MLP (chemprop/nn/ffn.py:120-142): k = ffn(fp)."""
    expk = k.exp()
    n_mols = constraints.shape[0]
    idx = batch.unsqueeze(1).repeat(1, k.shape[1])
    per_mol_sum_expk = torch.zeros(n_mols, expk.shape[1], dtype=expk.dtype).scatter_reduce_(0, idx, expk, reduce="sum",
                                                                                           include_self=False)
    w = expk / per_mol_sum_expk[batch]
    idx = batch.unsqueeze(1).repeat(1, preds.shape[1])
    per_mol_preds = torch.zeros(n_mols, preds.shape[1], dtype=preds.dtype).scatter_reduce_(0, idx, preds, reduce="sum",
                                                                                          include_self=False)
    has = ~torch.isnan(constraints)[0]
    deviation = constraints[:, has] - per_mol_preds[:, has]
    corrections = w * deviation[batch]
    cor = torch.zeros_like(preds)
    cor[:, has] = corrections
    return preds + cor
