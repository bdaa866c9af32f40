"""Molecule-level head of the training step on the engine's kernels (SURVEY.md section 8f-2): what chemprop's `MPNN` does
after the encoder -- `H = agg(H_v, batch)`, `H = bn(H)`, `preds = predictor(H)`, `loss = criterion(preds, targets, mask, w)`
(chemprop/models/model.py:126-161, nn/ffn.py:38-61, nn/predictors.py:101-170, 231-317, nn/metrics.py:78-123, 139-141,
291-303) -- for regression and classification: Mean / Sum / Norm aggregation, optional BatchNorm1d, the MLP of
`RegressionFFN` / `BinaryClassificationFFN` / `MulticlassClassificationFFN`, masked + weighted MSE, BCE or cross-entropy;
and for chemprop's uncertainty predictors `MveFFN` / `EvidentialFFN` / `QuantileFFN` / `BinaryDirichletFFN` /
`MulticlassDirichletFFN` (predictors.py:172-228, 250-270, 319-336) with their criteria (metrics.py:202-257, 502-544,
588-613): the MLP output goes through dmpnn_pred_transform (softplus, + 1, eval-mode unscaling; mirror
dmpnn_pred_transform_bwd), the criterion is one launch (dmpnn_mve_loss / dmpnn_evidential_loss / dmpnn_quantile_loss /
dmpnn_dirichlet_loss).

Every arithmetic step is a libdmpnn launch (aggregation: dmpnn_segment_sum; batch norm: dmpnn_bn_train_fwd / dmpnn_bn_bwd;
the MLP's GEMMs: dmpnn_linear_fwd / dmpnn_linear_wgrad with the activation in the epilogue; the criterion and its gradient:
dmpnn_mse_loss / dmpnn_bce_loss / dmpnn_ce_loss; eval-mode probabilities: dmpnn_class_probs), none synchronises with the
host, so the encoder + head + backward (+ a capturable optimizer) replay as ONE CUDA graph (`chemprop_b200.graph.CudaGraphStep`).

Module tree and state-dict keys are the reference's: `bn.{weight,bias,running_mean,running_var,num_batches_tracked}`,
`predictor.ffn.<i>.<j>.{weight,bias}`, `predictor.criterion.task_weights` -- a reference `MPNN` state dict loads with
`strict=True` into `EngineMPNN` (tests/test_dropin_reference_model.py) and vice versa."""
from __future__ import annotations

from typing import Sequence

import torch
from torch import Tensor, nn

from .. import _lib
from .. import engine as K
from .agg import Aggregation, MeanAggregation
from .constrainer import build_mlp
from .message_passing import DEFAULT_HIDDEN_DIM, engine_activation, is_fused_activation
from .transforms import UnscaleTransform


class BatchNormTrainFunction(torch.autograd.Function):
    """nn.BatchNorm1d in training mode on a b x d f32 matrix: dmpnn_bn_train_fwd / dmpnn_bn_bwd."""

    @staticmethod
    def forward(ctx, X, gamma, beta, running_mean, running_var, eps, momentum):
        K._require_cuda(X)
        Xc = X.float().contiguous()
        d = Xc.shape[1]
        Y, Xhat = torch.empty_like(Xc), torch.empty_like(Xc)
        mean, invstd = torch.empty(d, device=X.device), torch.empty(d, device=X.device)
        g = None if gamma is None else gamma.detach().float().contiguous()
        b = None if beta is None else beta.detach().float().contiguous()
        K.bn_train_fwd(Xc, g, b, running_mean, running_var, eps, momentum, Y, Xhat, mean, invstd)
        ctx.save_for_backward(Xhat, invstd, g)
        ctx.has = (gamma is not None, beta is not None)
        return Y

    @staticmethod
    def backward(ctx, dY):
        Xhat, invstd, g = ctx.saved_tensors
        dYc = dY.float().contiguous()
        d = dYc.shape[1]
        dX = torch.empty_like(dYc)
        dg = torch.empty(d, device=dYc.device) if ctx.has[0] else None
        db = torch.empty(d, device=dYc.device) if ctx.has[1] else None
        K.bn_bwd(dYc, Xhat, g, invstd, dX, dg, db)
        return dX, dg, db, None, None, None, None


class LinearActFunction(torch.autograd.Function):
    """Y = act(X . W^T + b) with the activation in the GEMM epilogue (dmpnn_linear_fwd); mirror: dZ = dY * act'(Y)
    (dmpnn_act_bwd), dW / db (dmpnn_linear_wgrad), dX = dZ . W (dmpnn_linear_fwd)."""

    @staticmethod
    def forward(ctx, X, W, b, act, act_param):
        K._require_cuda(X, W)
        Xc, Wc = X.float().contiguous(), W.detach().float().contiguous()
        bc = None if b is None else b.detach().float().contiguous()
        R, Kd = Xc.shape
        N = Wc.shape[0]
        Y = torch.empty((R, N), dtype=torch.float32, device=X.device)
        if R > 0:
            K.linear_fwd(Xc, Kd, Wc, Y, N, bias=bc, act=act, act_param=act_param, R=R, pad_to=N)
        ctx.save_for_backward(Xc, Wc, Y)
        ctx.cfg = (act, act_param, b is not None, W.dtype, None if b is None else b.dtype)
        return Y

    @staticmethod
    def backward(ctx, dY):
        Xc, Wc, Y = ctx.saved_tensors
        act, ap, has_b, wdt, bdt = ctx.cfg
        R, Kd = Xc.shape
        N = Wc.shape[0]
        dYc = dY.float().contiguous()
        dZ = dYc
        if act != _lib.ACT_NONE and R > 0:
            dZ = torch.empty_like(dYc)
            K.act_bwd(dYc, Y, R, N, act=act, act_param=ap, dZ=dZ)
        dW = torch.zeros_like(Wc)
        db = torch.zeros(N, dtype=torch.float32, device=Wc.device) if has_b else None
        dX = torch.zeros_like(Xc) if ctx.needs_input_grad[0] else None
        if R > 0:
            K.linear_wgrad(dZ, Xc, Kd, dW, N, dbias=db, R=R)
            if dX is not None:
                K.linear_fwd(dZ, N, Wc.t().contiguous(), dX, Kd, R=R, pad_to=Kd)
        return dX, dW.to(wdt), (None if db is None else db.to(bdt)), None, None


class EdgePairOperand:
    """The bond-level fingerprint `[H_e || H_e[rev]]` of chemprop's MolAtomBondMPNN (E x 2h) without the E x 2h buffer:
    H (E x h) and the int32 reverse-edge index.  EngineLinear consumes it through PairLinearFunction; `materialize()` gives
    the concatenation for code that needs a tensor."""

    def __init__(self, H: Tensor, rev: Tensor):
        self.H, self.rev = H, rev

    @property
    def shape(self) -> torch.Size:
        return torch.Size((self.H.shape[0], 2 * self.H.shape[1]))

    def dim(self) -> int:
        return 2

    def __len__(self) -> int:
        return self.H.shape[0]

    def materialize(self) -> Tensor:
        return torch.cat((self.H, self.H[self.rev.long()]), dim=1)


class PairLinearFunction(torch.autograd.Function):
    """Y = act([H || H[rev]] . W^T + b) with the second half of the operand gathered by the GEMM (dmpnn_linear_fwd,
    X2 = H, idx2 = rev); mirror: dW / db from the same gathered operand (dmpnn_linear_wgrad), and
    dH = [dZ || dZ[rev]] . [W_a^T | W_b^T] in one dmpnn_linear_fwd (W = [W_a | W_b]; rev is an involution)."""

    @staticmethod
    def forward(ctx, H, rev, W, b, act, act_param):
        K._require_cuda(H, W)
        Hc, Wc = H.float().contiguous(), W.detach().float().contiguous()
        bc = None if b is None else b.detach().float().contiguous()
        E, h = Hc.shape
        N = Wc.shape[0]
        if Wc.shape[1] != 2 * h:
            raise ValueError(f"the bond-level fingerprint has {2 * h} columns, the layer takes {Wc.shape[1]}")
        Y = torch.empty((E, N), dtype=torch.float32, device=H.device)
        if E > 0:
            K.linear_fwd(Hc, h, Wc, Y, N, X2=Hc, K2=h, idx2=rev, bias=bc, act=act, act_param=act_param, R=E, pad_to=N)
        ctx.save_for_backward(Hc, rev, Wc, Y)
        ctx.cfg = (act, act_param, b is not None, W.dtype, None if b is None else b.dtype, H.dtype)
        return Y

    @staticmethod
    def backward(ctx, dY):
        Hc, rev, Wc, Y = ctx.saved_tensors
        act, ap, has_b, wdt, bdt, hdt = ctx.cfg
        E, h = Hc.shape
        N = Wc.shape[0]
        dZ = dY.float().contiguous()
        if act != _lib.ACT_NONE and E > 0:
            dZ = torch.empty_like(dZ)
            K.act_bwd(dY.float().contiguous(), Y, E, N, act=act, act_param=ap, dZ=dZ)
        dW = torch.zeros_like(Wc)
        db = torch.zeros(N, dtype=torch.float32, device=Wc.device) if has_b else None
        dH = torch.zeros_like(Hc) if ctx.needs_input_grad[0] else None
        if E > 0:
            K.linear_wgrad(dZ, Hc, h, dW, N, X2=Hc, K2=h, idx2=rev, dbias=db, R=E)
            if dH is not None:
                WT = torch.cat((Wc[:, :h].t(), Wc[:, h:].t()), dim=1).contiguous()     # h x 2N
                K.linear_fwd(dZ, N, WT, dH, h, X2=dZ, K2=N, idx2=rev, R=E, pad_to=h)
        return (None if dH is None else dH.to(hdt)), None, dW.to(wdt), (None if db is None else db.to(bdt)), None, None


class EngineLinear(nn.Linear):
    """nn.Linear (same parameters / state-dict keys) executed by dmpnn_linear_fwd / dmpnn_linear_wgrad (f32).  An
    EdgePairOperand input runs PairLinearFunction: the pair concatenation is gathered, never stored."""

    def forward(self, x: Tensor, act: int = _lib.ACT_NONE, act_param: float = 0.0) -> Tensor:
        return linear_act(self, x, act, act_param)


def linear_act(lin: nn.Linear, x, act: int = _lib.ACT_NONE, act_param: float = 0.0) -> Tensor:
    """act(lin(x)) on the engine's GEMMs with the activation in the epilogue, for any nn.Linear; x may be an
    EdgePairOperand (PairLinearFunction)."""
    if isinstance(x, EdgePairOperand):
        return PairLinearFunction.apply(x.H, x.rev, lin.weight, lin.bias, act, act_param)
    return LinearActFunction.apply(x, lin.weight, lin.bias, act, act_param)


def engine_mlp(ffn: nn.Sequential, Z) -> Tensor:
    """`ffn(Z)` for an MLP of chemprop's module tree (nn/ffn.py:38-61: Linear, then [act, dropout, Linear] per further
    layer) on the engine's GEMMs, with every activation the engine fuses folded into the epilogue of the GEMM before it.
    The Linear layers may be plain nn.Linear (run through linear_act); EngineLinear layers are called as modules, so their
    hooks run.  Z may be an EdgePairOperand."""
    blocks = [list(b) for b in ffn if isinstance(b, nn.Sequential)]
    X = Z
    for k, block in enumerate(blocks):
        lin = block[-1]
        run = lin if isinstance(lin, EngineLinear) else (lambda x, *a, lin=lin: linear_act(lin, x, *a))
        if k + 1 == len(blocks):
            X = run(X)
            break
        tau, drop = blocks[k + 1][0], blocks[k + 1][1]
        if is_fused_activation(tau):
            X = run(X, *engine_activation(tau))              # act(W x + b) in the GEMM epilogue
        else:
            X = tau(run(X))
        X = drop(X)                                          # identity when p = 0 or in eval mode
    return X


class ClassProbsFunction(torch.autograd.Function):
    """Eval-mode outputs of the classification predictors (dmpnn_class_probs): sigmoid of every logit, or the softmax of every
    group of C columns.  The mirror (torch elementwise ops) is off the training path; it exists because chemprop's `forward`
    is differentiable."""

    @staticmethod
    def forward(ctx, logits, C, softmax):
        K._require_cuda(logits)
        X = logits.float().contiguous()
        out = torch.empty_like(X)
        K.class_probs(X, C, softmax, out)
        ctx.save_for_backward(out)
        ctx.cfg = (C, softmax, logits.dtype)
        return out

    @staticmethod
    def backward(ctx, g):
        (p,) = ctx.saved_tensors
        C, softmax, dt = ctx.cfg
        g = g.float()
        if not softmax:
            return (g * p * (1 - p)).to(dt), None, None
        b, n = p.shape
        p3, g3 = p.view(b, n // C, C), g.reshape(b, n // C, C)
        return (p3 * (g3 - (g3 * p3).sum(-1, keepdim=True))).view(b, n).to(dt), None, None


class PredTransformFunction(torch.autograd.Function):
    """Raw MLP output X (b x T*u) -> the predictor output (b x T x u) of `kind` (_lib.PRED_*) in one launch
    (dmpnn_pred_transform), with UnscaleTransform's eval mode when mean / scale are given.  Mirror: dmpnn_pred_transform_bwd
    for the training outputs; the eval-only Dirichlet probabilities take theirs in torch, as ClassProbsFunction does."""

    @staticmethod
    def forward(ctx, X, kind, u, mean, scale):
        K._require_cuda(X)
        Xc = X.float().contiguous()
        m = None if mean is None else mean.detach().float().reshape(-1).contiguous()
        s = None if scale is None else scale.detach().float().reshape(-1).contiguous()
        out = torch.empty_like(Xc)
        K.pred_transform(Xc, kind, u, m, s, out)
        ctx.save_for_backward(Xc, s)
        ctx.cfg = (kind, u, X.dtype)
        return out.view(Xc.shape[0], Xc.shape[1] // u, u)

    @staticmethod
    def backward(ctx, g):
        Xc, s = ctx.saved_tensors
        kind, u, dt = ctx.cfg
        b, n = Xc.shape
        g = g.float().reshape(b, n).contiguous()
        if kind <= _lib.PRED_DIRICHLET or kind == _lib.PRED_SOFTPLUS:
            dX = torch.empty_like(Xc)
            K.pred_transform_bwd(Xc, g, kind, u, s, dX)
        else:
            with torch.enable_grad():
                x = Xc.detach().requires_grad_(True)
                a = torch.nn.functional.softplus(x.view(b, n // u, u)) + 1
                S = a.sum(-1, keepdim=True)
                y = a / S if kind == _lib.PRED_DIRICHLET_PROBS else torch.stack(((a / S)[..., 1], 2 / S[..., 0]), 2)
                (dX,) = torch.autograd.grad(y, x, g.view_as(y))
        return dX.to(dt), None, None, None, None


def _loss_weights(weights, task_weights, b: int, T: int):
    """Per-molecule and per-task weights as contiguous f32 vectors of exactly b and T entries (or None), as the kernels read
    them.  A 1-entry task weight (the criteria's default `task_weights=1.0`) broadcasts, as in the reference; any other size
    is refused."""
    w = None if weights is None else weights.float().reshape(-1)
    tw = None if task_weights is None else task_weights.float().reshape(-1)
    if tw is not None and tw.numel() == 1:
        tw = tw.expand(T)
    if (w is not None and w.numel() != b) or (tw is not None and tw.numel() != T):
        raise ValueError(f"weights must have {b} entries and task_weights 1 or {T}, got "
                         f"{None if w is None else w.numel()} and {None if tw is None else tw.numel()}")
    return (None if w is None else w.contiguous()), (None if tw is None else tw.contiguous())


class CriterionLossFunction(torch.autograd.Function):
    """A criterion's loss and dLoss/dPreds in one launch, at any level.  `preds` is b x T, or b x T x u (u values per task:
    class logits, the uncertainty predictors' outputs), and `targets` b x T' -- which shapes go together is the criterion's
    rule, checked before this runs (_Criterion._check_shapes).  `launch(P, Y, w, tw, lt, gt, loss, dP)` (_Criterion._loss)
    gets them as b x (T*u) and b x T' f32, the weights as exactly b and T' entries (_loss_weights) and the bound masks as
    b x T' uint8 (None where not given); it writes loss[0] and dP."""

    @staticmethod
    def forward(ctx, preds, targets, weights, task_weights, lt_mask, gt_mask, launch):
        K._require_cuda(preds, targets, lt_mask, gt_mask)
        b, T = targets.shape
        P, Y = preds.float().flatten(1).contiguous(), targets.float().contiguous()
        w, tw = _loss_weights(weights, task_weights, b, T)
        lt, gt = (None if m is None else m.to(torch.uint8).expand(b, T).contiguous() for m in (lt_mask, gt_mask))
        loss = torch.empty(1, device=P.device)
        dP = torch.empty_like(P)
        launch(P, Y, w, tw, lt, gt, loss, dP)
        ctx.save_for_backward(dP.view(preds.shape))
        ctx.pdtype = preds.dtype
        return loss.reshape(())

    @staticmethod
    def backward(ctx, g):
        (dP,) = ctx.saved_tensors
        return (dP * g).to(ctx.pdtype), None, None, None, None, None, None


# the engine wrappers that take the b x T bound masks and a _lib.LOSS_* kind after `tw`
_REGRESSION_WRAPPERS = ("regression_loss", "regression_loss_rows")


class _Criterion(nn.Module):
    """chemprop's `ChempropMetric` interface (nn/metrics.py:59-123) around one loss kernel: `task_weights` buffer (1 x T),
    NaN targets or `mask` select the terms, `weights` are per molecule.  This class is chemprop's MSE.

    Each criterion names its engine wrappers: `_kernel` for molecules (a single-block kernel of csrc/head.cu) and
    `_row_kernel` for atom or bond rows (a row-parallel one of csrc/row_head.cu), None where it has none and `row_loss`
    runs `forward`.  `_args(preds)` are the wrapper's arguments between `tw` and `loss`; the regression wrappers take the
    bound masks and `_kind` there instead."""
    _kernel = "mse_loss"
    _row_kernel = "regression_loss_rows"
    _kind = _lib.LOSS_MSE
    _bounded = False                      # takes lt_mask / gt_mask (BoundedMixin, nn/metrics.py:142-149)
    _grouped = False                      # b x T x u predictions

    def __init__(self, task_weights):
        super().__init__()
        self.register_buffer("task_weights", torch.as_tensor(task_weights, dtype=torch.float).view(1, -1))

    def forward(self, preds, targets, mask=None, weights=None, lt_mask=None, gt_mask=None):
        return self._loss(self._kernel, preds, self._masked(targets, mask), weights, lt_mask, gt_mask)

    def row_loss(self, preds, targets, weights=None, lt_mask=None, gt_mask=None):
        """The criterion over atom or bond rows (`weights` per row, NaN targets masked) on `_row_kernel`, or through
        `forward` where there is none."""
        if self._row_kernel is None:
            return self(preds, targets, None, weights, lt_mask, gt_mask)
        return self._loss(self._row_kernel, preds, targets, weights, lt_mask, gt_mask)

    @staticmethod
    def _masked(targets, mask):
        return targets if mask is None else torch.where(mask, targets, torch.full_like(targets, float("nan")))

    def _args(self, preds) -> tuple:
        return ()

    def nan_error(self) -> str | None:
        """The reference's error message where it raises on a NaN loss instead of returning it; None for the criteria
        whose reference returns the NaN."""
        return None

    def _check_shapes(self, preds, targets):
        """b x T predictions (b x T x u when `_grouped`) and b x T targets."""
        if preds.dim() != (3 if self._grouped else 2) or targets.shape != preds.shape[:2]:
            raise ValueError(f"expected {'b x T x u' if self._grouped else 'b x T'} predictions and b x T targets, got "
                             f"{tuple(preds.shape)} and {tuple(targets.shape)}")

    def _loss(self, kernel, preds, targets, weights, lt_mask, gt_mask):
        if not self._bounded and (lt_mask is not None or gt_mask is not None):
            raise NotImplementedError(f"{type(self).__name__} takes no lt_mask / gt_mask; the bounded criteria "
                                      "(EngineBoundedMSE, EngineBoundedMAE, EngineBoundedRMSE) do")
        self._check_shapes(preds, targets)
        fn, regression = getattr(K, kernel), kernel in _REGRESSION_WRAPPERS
        args = () if regression else self._args(preds)          # a criterion refuses its bad arguments before any launch

        def launch(P, Y, w, tw, lt, gt, loss, dP):
            fn(P, Y, w, tw, *((lt, gt, self._kind) if regression else args), loss, dP)

        return CriterionLossFunction.apply(preds, targets, weights, self.task_weights, lt_mask, gt_mask, launch)


class _BCECriterion(_Criterion):
    """chemprop's BCELoss (nn/metrics.py:291-294): soft labels allowed."""
    _kernel = "bce_loss"
    _row_kernel = "bce_loss_rows"


class _CrossEntropyCriterion(_Criterion):
    """chemprop's CrossEntropyLoss (nn/metrics.py:297-303) on b x T x C logits and b x T class labels (truncated like
    `targets.long()`)."""
    _kernel = "ce_loss"
    _row_kernel = "ce_loss_rows"
    _grouped = True

    def _args(self, preds) -> tuple:
        return (preds.shape[2],)


class EngineMVELoss(_Criterion):
    """chemprop's MVELoss (nn/metrics.py:202-219) on b x T x 2 (mean, var) predictions (dmpnn_mve_loss)."""
    _kernel = "mve_loss"
    _row_kernel = None
    _grouped = True

    def __init__(self, task_weights=1.0):
        super().__init__(task_weights)


class EngineEvidentialLoss(_Criterion):
    """chemprop's EvidentialLoss (nn/metrics.py:222-260) on b x T x 4 (mean, v, alpha, beta) predictions
    (dmpnn_evidential_loss)."""
    _kernel = "evidential_loss"
    _row_kernel = None
    _grouped = True

    def __init__(self, task_weights=1.0, v_kl: float = 0.2, eps: float = 1e-8):
        super().__init__(task_weights)
        self.v_kl = v_kl
        self.eps = eps

    def _args(self, preds) -> tuple:
        return self.v_kl, self.eps

    def extra_repr(self) -> str:
        return f"v_kl={self.v_kl}, eps={self.eps}"


class EngineQuantileLoss(_Criterion):
    """chemprop's QuantileLoss (nn/metrics.py:588-613) on b x T x 2 (mean, interval) predictions (dmpnn_quantile_loss); the
    `bounds` and `tau` buffers are the reference's, so that its state dicts load strictly."""
    _kernel = "quantile_loss"
    _row_kernel = None
    _grouped = True

    def __init__(self, task_weights=1.0, alpha: float = 0.1):
        super().__init__(task_weights)
        self.alpha = alpha
        self.register_buffer("bounds", torch.tensor([-1 / 2, 1 / 2]).view(-1, 1, 1))
        self.register_buffer("tau", torch.tensor([[alpha / 2, 1 - alpha / 2], [alpha / 2 - 1, -alpha / 2]]).view(2, 2, 1, 1))

    def _args(self, preds) -> tuple:
        return (self.alpha,)

    def extra_repr(self) -> str:
        return f"alpha={self.alpha}"


class EngineDirichletLoss(_Criterion):
    """chemprop's DirichletLoss (nn/metrics.py:502-544) on b x T x C concentrations alpha and b x T class labels
    (dmpnn_dirichlet_loss)."""
    _kernel = "dirichlet_loss"
    _row_kernel = None
    _grouped = True

    def __init__(self, task_weights=1.0, v_kl: float = 0.2):
        super().__init__(task_weights)
        self.v_kl = v_kl

    def _args(self, preds) -> tuple:
        return preds.shape[2], self.v_kl

    def extra_repr(self) -> str:
        return f"v_kl={self.v_kl}"


class EnginePointQuantileLoss(_Criterion):
    """chemprop's PointQuantileLoss (nn/metrics.py:264-288): the pinball loss of b x T point predictions at `alpha`, alpha
    (y - p) above the target and (1 - alpha)(p - y) elsewhere.  One row-parallel kernel at every level
    (dmpnn_pinball_loss_rows)."""
    _kernel = "pinball_loss_rows"
    _row_kernel = "pinball_loss_rows"

    def __init__(self, task_weights=1.0, alpha: float = 0.1):
        super().__init__(task_weights)
        self.alpha = alpha

    def _args(self, preds) -> tuple:
        return (self.alpha,)

    def extra_repr(self) -> str:
        return f"alpha={self.alpha}"


class EngineNLogProbEnrichment(_Criterion):
    """chemprop's NLogProbEnrichment (nn/metrics.py:616-692), the loss of DNA-encoded-library screening counts, on b x 1
    predicted enrichments R (EngineRegressionFFN with its Softplus output) and b x 2 count targets (k1 in the positive
    sample, k2 in the counter sample; NaN = masked, counted as 0 in z as training_step's nan_to_num does): -log of the
    two-sided Poisson-ratio p-value of z = get_zstats(R, k1, k2, n1, n2, method), clamped at +-zinterval after dividing by
    zscale; the molecule's loss counts once per unmasked count, as the reference broadcasts its b x 1 loss against the
    b x 2 mask.  Task weights have 1 or 2 entries.  One launch (dmpnn_enrichment_loss); no row kernel.

    Where the reference raises ("Got nan loss": a NaN z anywhere in the batch, e.g. method "score" or "wald" with a row of
    zero counts) the loss is NaN instead, so that a training step never synchronises with the host and captures into a
    CUDA graph; `EngineMPNN.evaluate` raises the reference's ValueError at its one host sync."""
    _kernel = "enrichment_loss"
    _row_kernel = None

    def __init__(self, task_weights=1.0, n1: int = 1, n2: int = 1, method: str = "sqrt", zscale: float = 1.0,
                 zinterval: float = 5.0):
        super().__init__(task_weights)
        self.n1 = n1
        self.n2 = n2
        self.method = method
        self.zscale = zscale
        self.zinterval = zinterval

    def nan_error(self) -> str:
        """The reference's message where a z is NaN."""
        return (f"Got nan loss with method '{self.method}', ensure row-wise sum of counts are nonzero or use "
                "method='sqrt'")

    def _check_shapes(self, preds, targets):
        if preds.dim() != 2 or preds.shape[1] != 1 or targets.dim() != 2 or targets.shape != (preds.shape[0], 2):
            raise ValueError(f"NLogProbEnrichment takes b x 1 predictions and b x 2 count targets (k1, k2), got "
                             f"{tuple(preds.shape)} and {tuple(targets.shape)}")

    def _args(self, preds) -> tuple:
        if self.method not in _lib.ENRICH_METHODS:
            raise ValueError(f"Unsupported method: {self.method}")
        return self.n2 / self.n1, _lib.ENRICH_METHODS[self.method], self.zscale, self.zinterval

    def extra_repr(self) -> str:
        return f"n1={self.n1}, n2={self.n2}, method='{self.method}', zscale={self.zscale}, zinterval={self.zinterval}"


class SpectralTransformFunction(torch.autograd.Function):
    """SpectralFFN's output from the raw MLP output X (b x T): a(a(X)) normalised per row, a = softplus or exp
    (_lib.SPEC_*), in one launch (dmpnn_spectral_transform; mirror dmpnn_spectral_transform_bwd)."""

    @staticmethod
    def forward(ctx, X, act):
        K._require_cuda(X)
        Xc = X.float().contiguous()
        out = torch.empty_like(Xc)
        K.spectral_transform(Xc, act, out)
        ctx.save_for_backward(Xc)
        ctx.cfg = (act, X.dtype)
        return out

    @staticmethod
    def backward(ctx, g):
        (Xc,) = ctx.saved_tensors
        act, dt = ctx.cfg
        dX = torch.empty_like(Xc)
        K.spectral_transform_bwd(Xc, g.float().contiguous(), act, dX)
        return dX.to(dt), None


class _RegressionCriterion(_Criterion):
    """MSE / MAE / RMSE (`_kind`, _lib.LOSS_*) on b x T predictions, one launch of dmpnn_regression_loss; the `_bounded`
    ones take the batch's `lt_mask` / `gt_mask` (BoundedMixin, nn/metrics.py:142-149), the others refuse them."""
    _kernel = "regression_loss"

    def __init__(self, task_weights=1.0):
        super().__init__(task_weights)


class EngineMAE(_RegressionCriterion):
    """chemprop's MAE (nn/metrics.py:128-132): |preds - targets|."""
    _kind = _lib.LOSS_MAE


class EngineRMSE(_RegressionCriterion):
    """chemprop's RMSE (nn/metrics.py:135-139): sqrt of the MSE value, the gradient through the sqrt."""
    _kind = _lib.LOSS_RMSE


class EngineBoundedMSE(_RegressionCriterion):
    """chemprop's BoundedMSE (nn/metrics.py:142-157): MSE where a prediction on the allowed side of a censored target
    (`lt_mask` and preds < targets, or `gt_mask` and preds > targets) counts as exact."""
    _kind = _lib.LOSS_MSE
    _bounded = True


class EngineBoundedMAE(_RegressionCriterion):
    """chemprop's BoundedMAE (nn/metrics.py:160-163)."""
    _kind = _lib.LOSS_MAE
    _bounded = True


class EngineBoundedRMSE(_RegressionCriterion):
    """chemprop's BoundedRMSE (nn/metrics.py:166-169)."""
    _kind = _lib.LOSS_RMSE
    _bounded = True


class EngineSID(_Criterion):
    """chemprop's SID (nn/metrics.py:547-566) on b x T spectra: predictions clamped at `threshold` (None: not clamped),
    normalised over the masked-in bins, symmetric KL against the targets (dmpnn_sid_loss)."""
    _kernel = "sid_loss"
    _row_kernel = None

    def __init__(self, task_weights=1.0, threshold: float | None = None):
        super().__init__(task_weights)
        self.threshold = threshold

    def _args(self, preds) -> tuple:
        return (self.threshold,)

    def extra_repr(self) -> str:
        return f"threshold={self.threshold}"


class EngineWasserstein(EngineSID):
    """chemprop's Wasserstein (nn/metrics.py:569-585): |cumsum(targets) - cumsum(normalised preds)| per bin
    (dmpnn_wasserstein_loss).  A masked bin -- a NaN target, or one `mask` excludes -- adds 0 to the target cumsum, as in
    the reference's `MPNN.training_step`, whose criterion sees `targets.nan_to_num(0)`.  Called directly with a `mask` and
    finite targets at the masked bins, the reference criterion would add those targets to its cumsum instead; the engine
    does not read them."""
    _kernel = "wasserstein_loss"


class _EngineFFNPredictor(nn.Module):
    """`_FFNPredictorBase` (chemprop/nn/predictors.py:101-157) with the reference's module tree; GEMMs on the engine.  The
    MLP has n_tasks * n_targets outputs.  `criterion` replaces the default criterion (built from `task_weights`), and
    `output_transform` (an UnscaleTransform) unscales the regression predictors' outputs in eval mode; each is recorded in
    `hparams` when given."""
    n_targets = 1
    _criterion_cls = _Criterion

    def __init__(self, n_tasks: int = 1, input_dim: int = DEFAULT_HIDDEN_DIM, hidden_dim: int | Sequence[int] = 300,
                 n_layers: int = 1, dropout: float = 0.0, activation="relu", task_weights=None, *, criterion=None,
                 output_transform=None):
        super().__init__()
        self.hparams = dict(n_tasks=n_tasks, input_dim=input_dim, hidden_dim=hidden_dim, n_layers=n_layers, dropout=dropout,
                            activation=activation, cls=self.__class__)
        if criterion is not None:
            self.hparams["criterion"] = criterion
        if output_transform is not None:
            self.hparams["output_transform"] = output_transform
        ffn = build_mlp(input_dim, n_tasks * self.n_targets, hidden_dim, n_layers, dropout, activation)
        for block in ffn:                         # same tree, engine-backed Linear layers
            for i, m in enumerate(block):
                if isinstance(m, nn.Linear):
                    e = EngineLinear(m.in_features, m.out_features, m.bias is not None)
                    e.load_state_dict(m.state_dict())
                    block[i] = e
        self.ffn = ffn
        self.criterion = criterion if criterion is not None else self._criterion_cls(
            torch.ones(n_tasks) if task_weights is None else task_weights)
        self.output_transform = output_transform if output_transform is not None else nn.Identity()

    @property
    def input_dim(self) -> int:
        return self.ffn[0][-1].in_features

    @property
    def output_dim(self) -> int:
        return self.ffn[-1][-1].out_features

    @property
    def n_tasks(self) -> int:
        return self.output_dim // self.n_targets

    def _mlp(self, Z: Tensor) -> Tensor:
        return engine_mlp(self.ffn, Z)


def _is_default_softplus(t: nn.Module) -> bool:
    return isinstance(t, nn.Softplus) and t.beta == 1 and t.threshold == 20


class EngineRegressionFFN(_EngineFFNPredictor):
    """`RegressionFFN` (chemprop/nn/predictors.py:160-169) with the reference's module tree; GEMMs on the engine.  With an
    UnscaleTransform as `output_transform`, eval-mode predictions are `Y * scale + mean` (dmpnn_pred_transform); with
    `nn.Softplus()` (beta 1, threshold 20: the output of NLogProbEnrichment's enrichment ratios) they are softplus(Y) in
    training and eval mode alike.  Any other output transform is refused: the engine would not apply it.  The uncertainty
    predictors below take only an UnscaleTransform."""
    _kind = _lib.PRED_REGRESSION

    def _unscale(self):
        t = self.output_transform
        if not isinstance(t, (nn.Identity, UnscaleTransform)):
            allowed = "nn.Identity, UnscaleTransform" + (" or nn.Softplus()" if self._kind == _lib.PRED_REGRESSION else "")
            raise ValueError(f"{type(self).__name__} runs the output transforms {allowed} (beta 1, threshold 20) on its "
                             f"kernels; got {t!r}")
        if isinstance(t, nn.Identity) or t.training:      # UnscaleTransform is the identity in training mode
            return None, None
        return t.mean, t.scale

    def forward(self, Z: Tensor) -> Tensor:
        Y = self._mlp(Z)
        if self._kind == _lib.PRED_REGRESSION and _is_default_softplus(self.output_transform):
            return PredTransformFunction.apply(Y, _lib.PRED_SOFTPLUS, 1, None, None).view(Y.shape)
        mean, scale = self._unscale()
        if self._kind == _lib.PRED_REGRESSION:
            return Y if mean is None else PredTransformFunction.apply(Y, self._kind, 1, mean, scale).view(Y.shape)
        return PredTransformFunction.apply(Y, self._kind, self.n_targets, mean, scale)

    train_step = forward


class EngineMveFFN(EngineRegressionFFN):
    """`MveFFN` (chemprop/nn/predictors.py:172-188): b x T x 2 (mean, softplus(var)); in eval mode with an output transform
    the mean is unscaled and the variance multiplied by scale^2.  Criterion: EngineMVELoss."""
    n_targets = 2
    _kind = _lib.PRED_MVE
    _criterion_cls = EngineMVELoss


class EngineEvidentialFFN(EngineRegressionFFN):
    """`EvidentialFFN` (chemprop/nn/predictors.py:191-209): b x T x 4 (mean, softplus(v), softplus(alpha) + 1,
    softplus(beta)); in eval mode with an output transform the mean is unscaled and beta multiplied by scale^2.
    Criterion: EngineEvidentialLoss."""
    n_targets = 4
    _kind = _lib.PRED_EVIDENTIAL
    _criterion_cls = EngineEvidentialLoss


class EngineQuantileFFN(EngineRegressionFFN):
    """`QuantileFFN` (chemprop/nn/predictors.py:212-228): b x T x 2 (mean, interval) of the two predicted bounds, each
    unscaled in eval mode with an output transform.  Criterion: EngineQuantileLoss."""
    n_targets = 2
    _kind = _lib.PRED_QUANTILE
    _criterion_cls = EngineQuantileLoss


class EngineBinaryClassificationFFN(_EngineFFNPredictor):
    """`BinaryClassificationFFN` (chemprop/nn/predictors.py:235-247): `train_step` gives the b x T logits, `forward` their
    sigmoid (dmpnn_class_probs; no output transform, as in the reference); criterion: masked, weighted BCE (dmpnn_bce_loss)."""
    _criterion_cls = _BCECriterion

    def forward(self, Z: Tensor) -> Tensor:
        return ClassProbsFunction.apply(self._mlp(Z), 1, False)

    def train_step(self, Z: Tensor) -> Tensor:
        return self._mlp(Z)


class EngineMulticlassClassificationFFN(_EngineFFNPredictor):
    """`MulticlassClassificationFFN` (chemprop/nn/predictors.py:272-316): the MLP has n_tasks * n_classes outputs, task t in
    columns [t * n_classes, (t + 1) * n_classes); `train_step` gives the logits as b x T x C, `forward` their softmax over
    the classes (dmpnn_class_probs); criterion: masked, weighted cross-entropy (dmpnn_ce_loss)."""
    _criterion_cls = _CrossEntropyCriterion

    def __init__(self, n_classes: int, n_tasks: int = 1, input_dim: int = DEFAULT_HIDDEN_DIM,
                 hidden_dim: int | Sequence[int] = 300, n_layers: int = 1, dropout: float = 0.0, activation="relu",
                 task_weights=None, *, criterion=None, output_transform=None):
        task_weights = torch.ones(n_tasks) if task_weights is None else task_weights
        super().__init__(n_tasks * n_classes, input_dim, hidden_dim, n_layers, dropout, activation, task_weights,
                         criterion=criterion, output_transform=output_transform)
        self.n_classes = n_classes
        self.hparams.update(n_tasks=n_tasks, n_classes=n_classes)

    @property
    def n_tasks(self) -> int:
        return self.output_dim // (self.n_targets * self.n_classes)

    def forward(self, Z: Tensor) -> Tensor:
        return ClassProbsFunction.apply(self._mlp(Z), self.n_classes, True).reshape(Z.shape[0], -1, self.n_classes)

    def train_step(self, Z: Tensor) -> Tensor:
        return self._mlp(Z).reshape(Z.shape[0], -1, self.n_classes)


class EngineBinaryDirichletFFN(_EngineFFNPredictor):
    """`BinaryDirichletFFN` (chemprop/nn/predictors.py:250-269): the MLP has 2 outputs per task, task t in columns
    [2t, 2t + 2); `train_step` gives alpha = softplus + 1 as b x T x 2, `forward` the b x T x 2 pair (alpha_1 / S, 2 / S)
    (dmpnn_pred_transform).  Criterion: EngineDirichletLoss."""
    n_targets = 2
    _criterion_cls = EngineDirichletLoss

    def forward(self, Z: Tensor) -> Tensor:
        return PredTransformFunction.apply(self._mlp(Z), _lib.PRED_DIRICHLET_BINARY, 2, None, None)

    def train_step(self, Z: Tensor) -> Tensor:
        return PredTransformFunction.apply(self._mlp(Z), _lib.PRED_DIRICHLET, 2, None, None)


class EngineMulticlassDirichletFFN(EngineMulticlassClassificationFFN):
    """`MulticlassDirichletFFN` (chemprop/nn/predictors.py:319-336): `train_step` gives alpha = softplus + 1 as b x T x C,
    `forward` alpha / sum(alpha) (dmpnn_pred_transform).  Criterion: EngineDirichletLoss."""
    _criterion_cls = EngineDirichletLoss

    def forward(self, Z: Tensor) -> Tensor:
        return PredTransformFunction.apply(self._mlp(Z), _lib.PRED_DIRICHLET_PROBS, self.n_classes, None, None)

    def train_step(self, Z: Tensor) -> Tensor:
        return PredTransformFunction.apply(self._mlp(Z), _lib.PRED_DIRICHLET, self.n_classes, None, None)


class _Exp(nn.Module):
    """`_Exp` of chemprop/nn/predictors.py:337-339 (SpectralFFN's "exp" activation)."""

    def forward(self, X: Tensor) -> Tensor:
        return X.exp()


class EngineSpectralFFN(_EngineFFNPredictor):
    """`SpectralFFN` (chemprop/nn/predictors.py:342-376): the MLP's b x T output goes through the spectral activation twice
    (the reference appends it to `ffn` as `ffn.spectral_activation` and applies it again in `forward`) and is normalised
    to sum 1 per row (dmpnn_spectral_transform); `train_step` is `forward`.  `spectral_activation` is "softplus" (or None)
    or "exp".  Criterion: EngineSID(task_weights, threshold)."""
    _criterion_cls = EngineSID

    def __init__(self, n_tasks: int = 1, input_dim: int = DEFAULT_HIDDEN_DIM, hidden_dim: int | Sequence[int] = 300,
                 n_layers: int = 1, dropout: float = 0.0, activation="relu", task_weights=None,
                 threshold: float | None = None, spectral_activation: str | None = "softplus", *, criterion=None,
                 output_transform=None):
        if spectral_activation not in ("softplus", "exp", None):
            raise ValueError(f"Unknown spectral activation: {spectral_activation}. "
                             "Expected one of 'exp', 'softplus' or None.")
        given = criterion
        if criterion is None:
            criterion = EngineSID(torch.ones(n_tasks) if task_weights is None else task_weights, threshold)
        super().__init__(n_tasks, input_dim, hidden_dim, n_layers, dropout, activation, task_weights, criterion=criterion,
                         output_transform=output_transform)
        # every key the reference records (criterion and output_transform even when None), and what rebuilds the default
        # criterion
        self.hparams.update(criterion=given, output_transform=output_transform, task_weights=task_weights,
                            threshold=threshold, spectral_activation=spectral_activation)
        self._act = _lib.SPEC_EXP if spectral_activation == "exp" else _lib.SPEC_SOFTPLUS
        self.ffn.add_module("spectral_activation", _Exp() if self._act == _lib.SPEC_EXP else nn.Softplus())

    @property
    def output_dim(self) -> int:
        return self.ffn[-2][-1].out_features

    def forward(self, Z: Tensor) -> Tensor:
        return SpectralTransformFunction.apply(self._mlp(Z), self._act)

    train_step = forward


class EngineBatchNorm1d(nn.BatchNorm1d):
    """nn.BatchNorm1d (same parameters / buffers); training mode runs dmpnn_bn_train_fwd / dmpnn_bn_bwd."""

    def forward(self, x: Tensor) -> Tensor:
        # torch's own path where the kernel has no equivalent: eval mode, CPU tensors, no running statistics, and
        # momentum=None (cumulative average: the factor 1 / num_batches_tracked is host state, a sync per step)
        if not self.training or not x.is_cuda or self.running_mean is None or self.momentum is None:
            return super().forward(x)
        if x.dim() != 2:
            raise ValueError(f"expected a 2D input (molecules x features), got {x.dim()}D")
        if x.shape[0] <= 1:                       # as torch: the batch variance of one row is undefined (the reference's
            raise ValueError(f"Expected more than 1 value per channel when training, got input size {tuple(x.shape)}")  # loader drops such a batch, dataloader.py:77-86)
        if self.num_batches_tracked is not None:
            self.num_batches_tracked.add_(1)
        return BatchNormTrainFunction.apply(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps,
                                            self.momentum)


def _predict(model: nn.Module, batches, step, active_dropout: bool, gather):
    """The predict loop of EngineMPNN / EngineMolAtomBondMPNN: `step(batch)` per batch in eval mode (nn.Dropout modules
    trained when `active_dropout`) under torch.inference_mode(), `gather(outputs)`; training flags restored even on error."""
    flags = [(m, m.training) for m in model.modules()]
    try:
        model.eval()
        if active_dropout:
            for m in model.modules():
                if isinstance(m, nn.Dropout):
                    m.train()
        with torch.inference_mode():
            outs = [step(b) for b in batches]
            if not outs:
                raise ValueError("predict: no batches")
            return gather(outs)
    finally:
        for m, f in flags:
            m.training = f


class EngineMPNN(nn.Module):
    """`chemprop.models.MPNN` reduced to the path (models/model.py:66-161): message passing -> aggregation -> batch norm ->
    predictor -> criterion, all on the engine.  The predictor is EngineRegressionFFN (the default),
    EngineBinaryClassificationFFN, EngineMulticlassClassificationFFN or one of the uncertainty predictors (EngineMveFFN,
    EngineEvidentialFFN, EngineQuantileFFN, EngineBinaryDirichletFFN, EngineMulticlassDirichletFFN) or EngineSpectralFFN.
    `training_loss(bmg, targets, weights=None, lt_mask=None, gt_mask=None)` is `MPNN.training_step` without Lightning's
    logging (the b x T boolean lt / gt masks go to the bounded criteria); `forward(bmg)` gives
    the predictions (probabilities for the classification predictors).  `X_d_transform` (a ScaleTransform, as
    models/model.py:97) scales extra molecule descriptors X_d in eval mode before they join the fingerprint."""

    def __init__(self, message_passing: nn.Module, agg: Aggregation | None = None, predictor: nn.Module | None = None,
                 batch_norm: bool = False, X_d_transform: nn.Module | None = None):
        super().__init__()
        self.message_passing = message_passing
        self.agg = agg if agg is not None else MeanAggregation()
        self.bn = EngineBatchNorm1d(message_passing.output_dim) if batch_norm else nn.Identity()
        self.predictor = predictor if predictor is not None else EngineRegressionFFN(input_dim=message_passing.output_dim)
        self.X_d_transform = X_d_transform if X_d_transform is not None else nn.Identity()

    def fingerprint(self, bmg, V_d: Tensor | None = None, X_d: Tensor | None = None) -> Tensor:
        H = self.bn(self.agg(self.message_passing(bmg, V_d), bmg.batch))
        return H if X_d is None else torch.cat((H, self.X_d_transform(X_d)), dim=1)

    def forward(self, bmg, V_d: Tensor | None = None, X_d: Tensor | None = None) -> Tensor:
        return self.predictor(self.fingerprint(bmg, V_d, X_d))

    def training_loss(self, bmg, targets: Tensor, weights: Tensor | None = None, V_d=None, X_d=None, *,
                      lt_mask: Tensor | None = None, gt_mask: Tensor | None = None) -> Tensor:
        preds = self.predictor.train_step(self.fingerprint(bmg, V_d, X_d))
        if lt_mask is None and gt_mask is None:
            return self.predictor.criterion(preds, targets, None, weights)  # NaN targets are the mask (model.py:140-141)
        return self.predictor.criterion(preds, targets, None, weights, lt_mask, gt_mask)

    def predict(self, batches, *, active_dropout: bool = False) -> Tensor:
        """chemprop's `predict_step` over `batches` (TrainingBatch, or MulticomponentTrainingBatch for
        EngineMulticomponentMPNN), concatenated along molecules: `trainer.predict` followed by `torch.concat(preds, 0)`
        (models/model.py:203-206).  Eval mode under torch.inference_mode(); `active_dropout` then trains every nn.Dropout
        module, as chemprop's DropoutEstimator does for each pass.  Every module's training flag is restored, even on error.
        No host synchronisation: the result is a device tensor, ready when the stream is."""
        return _predict(self, batches, lambda b: self(b[0], b[1], b[2]), active_dropout,
                        lambda outs: torch.cat(outs, 0))

    def _eval_modules(self) -> list[nn.Module]:
        """The modules `on_validation_model_eval` (models/model.py:162-167, models/multi.py) keeps in training mode: every
        encoder block's V_d and graph transforms, the X_d transform and the predictor's output transform."""
        blocks = [getattr(b, n) for b in self.message_passing.modules() for n in ("V_d_transform", "graph_transform")
                  if isinstance(getattr(b, n, None), nn.Module)]
        return blocks + [self.X_d_transform, self.predictor.output_transform]

    def evaluate(self, batches, metrics=None, *, stage: str = "val") -> dict[str, float]:
        """chemprop's `validation_step` / `test_step` over `batches` (TrainingBatch, or MulticomponentTrainingBatch for
        EngineMulticomponentMPNN), then each metric's epoch value (models/model.py:162-202).

        stage="val": eval mode except the input and output transforms (V_d / graph / X_d transforms and the predictor's
        output transform stay in training mode, so predictions are compared to the scaled targets), `val_loss` from
        `predictor.train_step` and the criterion with the batch's weights, and every metric on `forward`'s output with
        weights of one.  stage="test": eval mode, metrics only.  Both take `preds[..., 0]` when the predictor has several
        targets per task, and mask non-finite targets.  `metrics` (EngineMetric objects, reset here) default to the
        predictor's default metric (nn.metrics.default_metric).  Runs under no_grad, restores every module's training flag,
        and synchronises with the host once, at the end.  Returns {"val_loss": .., "val/<alias>": ..} or
        {"test/<alias>": ..}; raises ValueError where an update met a target its metric cannot take, or where the
        NLogProbEnrichment criterion (as the loss or as a metric) met a NaN z, with the reference's message."""
        from .metrics import EngineCriterionMetric, default_metric

        if stage not in ("val", "test"):
            raise ValueError(f"stage must be 'val' or 'test', got {stage!r}")
        metrics = [default_metric(self.predictor)] if metrics is None else list(metrics)
        loss = EngineCriterionMetric(self.predictor.criterion) if stage == "val" else None
        for m in metrics:
            m.reset()
        flags = [(m, m.training) for m in self.modules()]
        try:
            self.eval()
            if stage == "val":
                for m in self._eval_modules():
                    m.train()
            with torch.no_grad():
                for bmg, V_d, X_d, targets, weights, lt_mask, gt_mask in batches:
                    mask = targets.isfinite()
                    targets = targets.nan_to_num(nan=0.0)
                    Z = self.fingerprint(bmg, V_d, X_d)
                    preds = self.predictor(Z)
                    if self.predictor.n_targets > 1:
                        preds = preds[..., 0]
                    ones = torch.ones_like(weights)
                    for m in metrics:
                        m.update(preds, targets, mask, ones, lt_mask, gt_mask)
                    if loss is not None:     # validation_step: the same fingerprint through train_step
                        loss.update(self.predictor.train_step(Z), targets, mask, weights, lt_mask, gt_mask)
                values = [m.compute() for m in metrics] + ([] if loss is None else [loss.compute()])
                checked = [m for m in metrics + ([] if loss is None else [loss]) if m._status is not None]
                host = torch.stack([v.double().reshape(()) for v in values]
                                   + [m._status.double().reshape(()) for m in checked]).tolist()
        finally:
            for m, f in flags:
                m.training = f
        bad = [m for m, s in zip(checked, host[len(values):]) if s]
        for m in bad:                   # a criterion whose reference raises on a NaN loss (EngineNLogProbEnrichment)
            if isinstance(m, EngineCriterionMetric):
                raise ValueError(m.criterion.nan_error())
        if bad:
            raise ValueError(f"metric(s) {[m.alias for m in bad]}: a target is not a valid label (binary targets must be 0 "
                             "or 1, class targets in [-C, C))")
        out = {f"{stage}/{m.alias}": v for m, v in zip(metrics, host)}
        if loss is not None:
            out = {"val_loss": host[len(metrics)], **out}
        return out
