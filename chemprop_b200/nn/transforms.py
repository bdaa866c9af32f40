"""`ScaleTransform` / `UnscaleTransform` / `GraphTransform` with the behaviour of chemprop/nn/transforms.py:11-74:
identity in training mode, `(X - mean) / scale` (or `X * scale + mean`) in eval mode, on a shallow copy of the graph.
Thin and not on the hot path (only used with extra atom/bond features)."""
from __future__ import annotations

import copy

import torch
from torch import Tensor, nn


class _ScaleTransformMixin(nn.Module):
    def __init__(self, mean, scale, pad: int = 0):
        super().__init__()
        mean = torch.cat([torch.zeros(pad), torch.as_tensor(mean, dtype=torch.float)])
        scale = torch.cat([torch.ones(pad), torch.as_tensor(scale, dtype=torch.float)])
        if mean.shape != scale.shape:
            raise ValueError(f"uneven shapes for 'mean' and 'scale'! got: mean={mean.shape}, scale={scale.shape}")
        self.register_buffer("mean", mean.unsqueeze(0))
        self.register_buffer("scale", scale.unsqueeze(0))

    @classmethod
    def from_standard_scaler(cls, scaler, pad: int = 0):
        return cls(scaler.mean_, scaler.scale_, pad=pad)


class ScaleTransform(_ScaleTransformMixin):
    def forward(self, X: Tensor) -> Tensor:
        if self.training:
            return X
        return (X - self.mean) / self.scale


class UnscaleTransform(_ScaleTransformMixin):
    """chemprop/nn/transforms.py:45-55: the target scaler a regression checkpoint carries (`predictor.output_transform.
    {mean,scale}`, 1 x T).  Identity in training mode; in eval mode `X * scale + mean`, and `transform_variance(var)` gives
    `var * scale^2`.  The engine's predictors apply it inside dmpnn_pred_transform; these torch forms are its definition."""

    def forward(self, X: Tensor) -> Tensor:
        if self.training:
            return X
        return X * self.scale + self.mean

    def transform_variance(self, var: Tensor) -> Tensor:
        if self.training:
            return var
        return var * (self.scale ** 2)


class GraphTransform(nn.Module):
    def __init__(self, V_transform: nn.Module, E_transform: nn.Module):
        super().__init__()
        self.V_transform = V_transform
        self.E_transform = E_transform

    def forward(self, bmg):
        if self.training:
            return bmg
        bmg = copy.copy(bmg)  # never mutate the caller's graph (tests/integration/test_regression_mol.py:143-226)
        bmg.V = self.V_transform(bmg.V)
        bmg.E = self.E_transform(bmg.E)
        return bmg
