"""Distance criteria of src/criterion/distance.py: ``MeanAbsoluteError`` and ``MeanSquaredError`` (the criterion of the MUSDB18
Conv-TasNet recipe, ``criterion='mse'``), with the reference's semantics:

    loss = mean over ``dim`` of |input - target| (or its square)          (batch_size, *rest)
    reduction 'mean' / 'sum' over every remaining axis but the batch axis  (batch_size,)   ; None keeps them
    batch_mean: mean over the batch axis                                   ()

Plain torch operations on whatever device the tensors live on (one elementwise pass and a reduction: not a hot path); autograd
goes through them, so ``loss.backward()`` hands the model its cotangent directly."""
import torch
import torch.nn as nn


def _reduce(loss, reduction):
    if reduction:
        dim = tuple(range(1, loss.dim()))
        if reduction == 'mean':
            loss = loss.mean(dim=dim)
        elif reduction == 'sum':
            loss = loss.sum(dim=dim)
        else:
            raise NotImplementedError("Not support self.reduction={}.".format(reduction))
    return loss


class MeanAbsoluteError(nn.Module):
    def __init__(self, dim=1, reduction=None):
        """dim <int> or <tuple<int>>: the axes averaged first; reduction: None, 'mean' or 'sum' over the axes left after that"""
        super().__init__()
        self.dim = dim
        self.reduction = reduction

    def forward(self, input, target, batch_mean=True):
        """input, target (batch_size, *) -> () with batch_mean, else (batch_size,) or (batch_size, *rest)"""
        loss = torch.mean(torch.abs(input - target), dim=self.dim)
        loss = _reduce(loss, self.reduction)
        if batch_mean:
            loss = loss.mean(dim=0)
        return loss

    @property
    def maximize(self):
        return False


class MeanSquaredError(nn.Module):
    def __init__(self, dim=1, reduction=None):
        """dim <int> or <tuple<int>>: the axes averaged first; reduction: None, 'mean' or 'sum' over the axes left after that"""
        super().__init__()
        self.dim = dim
        self.reduction = reduction

    def forward(self, input, target, batch_mean=True):
        """input, target (batch_size, *) -> () with batch_mean, else (batch_size,) or (batch_size, *rest)"""
        loss = torch.mean((input - target) ** 2, dim=self.dim)
        loss = _reduce(loss, self.reduction)
        if batch_mean:
            loss = loss.mean(dim=0)
        return loss

    @property
    def maximize(self):
        return False
