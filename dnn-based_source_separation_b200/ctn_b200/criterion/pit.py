"""Permutation-invariant training, mirroring src/criterion/pit.py: ``pit`` (:9-44), ``PIT`` (:46-69), ``PIT1d``
(:71-77).  When the criterion is (Neg)SISDR or (Neg)SDR with reduction 'mean'/'sum' on (batch_size, n_sources, T) tensors,
n_sources <= 6, the whole thing is ONE fused call (ctn_sisdr_pit_fwd / ctn_sdr_pit_fwd): the S x S table of pair statistics is
computed in streaming passes and the S! permutations are scored from it (lexicographic order, first minimum).  Any other
criterion, or a subset of the permutations, goes through the generic loop of the reference semantics."""
import itertools

import torch
import torch.nn as nn

from .. import _native as N
from .sdr import NegSDR, NegSISDR, SDR, SISDR

# (forward, backward, scratch bytes) of the fused PIT, by criterion
_SISDR_PIT = (N.ctn_sisdr_pit_fwd, N.ctn_sisdr_pit_bwd, N.ctn_sisdr_pit_scratch_bytes)
_SDR_PIT = (N.ctn_sdr_pit_fwd, N.ctn_sdr_pit_bwd, N.ctn_sdr_pit_scratch_bytes)


def _fused_ok(criterion, input, target):
    return (isinstance(criterion, (NegSISDR, SISDR, NegSDR, SDR)) and criterion.reduction in ('mean', 'sum') and input.dim() == 3
            and input.shape == target.shape and input.is_cuda and input.size(1) <= 6)


def _pit_fwd(kernels, x, t, eps, loss_mean=None):
    """(loss_b, perm, scratch) of the fused forward: loss_b (B) = min_perm -mean_i criterion(est_i, tgt_perm[i])"""
    fwd, _, scratch_bytes = kernels
    dev = N.require_cuda(x, t)
    B, S, T = x.shape
    loss_b = torch.empty(B, dtype=torch.float32, device=dev)
    perm = torch.empty(B, S, dtype=torch.int64, device=dev)
    scratch = torch.empty(scratch_bytes(B, S) // 8, dtype=torch.float64, device=dev)
    N.check(fwd(x.data_ptr(), t.data_ptr(), B, S, T, float(eps), loss_b.data_ptr(), perm.data_ptr(), N.ptr(loss_mean), None,
                scratch.data_ptr(), N.stream_ptr(dev)), fwd.__name__)
    return loss_b, perm, scratch


def _pit_fn_forward(ctx, kernels, x, t, eps):
    loss_b, perm, scratch = _pit_fwd(kernels, x, t, eps)
    ctx.save_for_backward(x, t, perm, scratch)
    ctx.eps, ctx.bwd = float(eps), kernels[1]
    ctx.mark_non_differentiable(perm)
    return loss_b, perm


class _PitNegSisdrFn(torch.autograd.Function):
    """loss_b (B) = min_perm -mean_i SI-SDR(est_i, tgt_perm[i]) with its gradient w.r.t. the estimate through the selected
    permutation (the indices carry no gradient, pit.py:36-44); ctn_sisdr_pit_fwd / ctn_sisdr_pit_bwd."""
    kernels = _SISDR_PIT

    @staticmethod
    def forward(ctx, x, t, eps):
        return _pit_fn_forward(ctx, _SISDR_PIT, x, t, eps)

    @staticmethod
    def backward(ctx, g_loss_b, _g_perm):
        x, t, perm, scratch = ctx.saved_tensors
        B, S, T = x.shape
        g = g_loss_b.contiguous().to(torch.float32)
        d_est = torch.empty_like(x)
        N.check(ctx.bwd(x.data_ptr(), t.data_ptr(), perm.data_ptr(), B, S, T, ctx.eps, scratch.data_ptr(), g.data_ptr(), -1.0 / S,
                        d_est.data_ptr(), N.stream_ptr(x.device)), ctx.bwd.__name__)
        return d_est, None, None


class _PitNegSdrFn(_PitNegSisdrFn):
    """loss_b (B) = min_perm -mean_i SDR(est_i, tgt_perm[i]) with its gradient w.r.t. the estimate through the selected
    permutation; ctn_sdr_pit_fwd / ctn_sdr_pit_bwd."""
    kernels = _SDR_PIT

    @staticmethod
    def forward(ctx, x, t, eps):
        return _pit_fn_forward(ctx, _SDR_PIT, x, t, eps)


def _fused(criterion, input, target, batch_mean):
    x, t = input.contiguous(), target.contiguous()
    if torch.is_grad_enabled() and target.requires_grad:
        raise NotImplementedError("gradient w.r.t. the PIT target is not built")
    fn = _PitNegSdrFn if isinstance(criterion, (NegSDR, SDR)) else _PitNegSisdrFn
    S = x.shape[1]
    # the kernels score -mean_i criterion; a maximised criterion (SISDR, SDR) is its negation, 'sum' = * S
    scale = (S if criterion.reduction == 'sum' else 1) * (-1.0 if criterion.maximize else 1.0)
    if torch.is_grad_enabled() and x.requires_grad:
        loss_b, perm = fn.apply(x, t, float(criterion.eps))
        loss = loss_b.mean(dim=0) if batch_mean else loss_b
    else:
        loss_mean = torch.empty(1, dtype=torch.float32, device=x.device)
        loss_b, perm, _ = _pit_fwd(fn.kernels, x, t, criterion.eps, loss_mean)
        loss = loss_mean[0] if batch_mean else loss_b
    if scale != 1:
        loss = loss * scale
    return loss, perm


def pit(criterion, input, target, n_sources=None, patterns=None, batch_mean=True):
    """Returns (loss, pattern): loss scalar or (batch_size,), pattern (batch_size, n_sources) int64 with
    estimate i <-> target pattern[i]."""
    if _fused_ok(criterion, input, target) and (patterns is None or len(patterns) == _nperm(input.size(1))):
        return _fused(criterion, input, target, batch_mean)
    return _pit_generic(criterion, input, target, n_sources, patterns, batch_mean)


def _pit_generic(criterion, input, target, n_sources=None, patterns=None, batch_mean=True):
    """the reference's loop over the permutations (pit.py:20-44)"""
    if patterns is None:
        if n_sources is None:
            n_sources = input.size(1)
        patterns = torch.tensor(list(itertools.permutations(range(n_sources))), dtype=torch.long)
    patterns = patterns.to(input.device)
    possible_loss = torch.stack([criterion(input, target[:, p], batch_mean=False) for p in patterns], dim=1)
    if hasattr(criterion, "maximize") and criterion.maximize:
        loss, indices = torch.max(possible_loss, dim=1)
    else:
        loss, indices = torch.min(possible_loss, dim=1)
    if batch_mean:
        loss = loss.mean(dim=0)
    return loss, patterns[indices]


def _nperm(S):
    n = 1
    for i in range(2, S + 1):
        n *= i
    return n


class PIT(nn.Module):
    def __init__(self, criterion, n_sources):
        super().__init__()
        self.criterion = criterion
        self.patterns = torch.tensor(list(itertools.permutations(range(n_sources))), dtype=torch.long)

    def forward(self, input, target, batch_mean=True):
        return pit(self.criterion, input, target, patterns=self.patterns, batch_mean=batch_mean)


class PIT1d(PIT):
    def __init__(self, criterion, n_sources):
        super().__init__(criterion, n_sources)


class PIT2d(PIT):
    def __init__(self, criterion, n_sources):
        super().__init__(criterion, n_sources)


# ---- ORPIT (src/criterion/pit.py:87-160) and Sinkhorn PIT (:162-213) ----------------------------------------------------
# Fused when the criterion is NegSISDR / SISDR on (batch_size, n, T) float32 CUDA tensors with n <= 16: the criterion is then
# applied to 2-D rows, so its `reduction` does not enter, and both losses are functions of the per-pair SI-SDR statistics
# (ctn_orpit_* / ctn_sinkpit_*).  Anything else runs the generic loop of the reference semantics.
_PITX_MAX = 16


def _pitx_fused_ok(criterion, input, n):
    return (isinstance(criterion, (NegSISDR, SISDR)) and input.dim() == 3 and input.is_cuda and input.dtype == torch.float32
            and n <= _PITX_MAX)


def _no_target_grad(target):
    if torch.is_grad_enabled() and target.requires_grad:
        raise NotImplementedError("gradient w.r.t. the PIT target is not built")


class _OrpitSisdrFn(torch.autograd.Function):
    """(loss_b (B), indices (B) int64) of ORPIT over SI-SDR with its gradient w.r.t. the estimate through the selected
    candidate; ctn_orpit_fwd / ctn_orpit_bwd."""

    @staticmethod
    def forward(ctx, x, t, n_b, eps, maximize):
        dev = N.require_cuda(x, t)
        B, n, T = t.shape
        loss_b = torch.empty(B, dtype=torch.float32, device=dev)
        idx = torch.empty(B, dtype=torch.int64, device=dev)
        scratch = torch.empty(N.ctn_orpit_scratch_bytes(B, n) // 4, dtype=torch.float32, device=dev)
        N.check(N.ctn_orpit_fwd(x.data_ptr(), t.data_ptr(), N.ptr(n_b), B, n, T, float(eps), int(maximize), loss_b.data_ptr(),
                                idx.data_ptr(), scratch.data_ptr(), N.stream_ptr(dev)), "ctn_orpit_fwd")
        ctx.save_for_backward(x, t, n_b, idx, scratch)
        ctx.eps, ctx.maximize = float(eps), int(maximize)
        ctx.mark_non_differentiable(idx)
        return loss_b, idx

    @staticmethod
    def backward(ctx, g_loss_b, _g_idx):
        x, t, n_b, idx, scratch = ctx.saved_tensors
        B, n, T = t.shape
        g = g_loss_b.contiguous().to(torch.float32)
        d_x = torch.empty_like(x)
        N.check(N.ctn_orpit_bwd(x.data_ptr(), t.data_ptr(), N.ptr(n_b), idx.data_ptr(), B, n, T, ctx.eps, ctx.maximize,
                                scratch.data_ptr(), g.data_ptr(), d_x.data_ptr(), N.stream_ptr(x.device)), "ctn_orpit_bwd")
        return d_x, None, None, None, None


def _orpit_generic(criterion, input, target, lens):
    """the reference's per-sample loop (pit.py:123-158); returns (loss_b, indices)"""
    losses, indices = [], []
    maximize = hasattr(criterion, "maximize") and criterion.maximize
    for b in range(input.size(0)):
        n = int(lens[b])
        _input, _target = input[b: b + 1], target[b: b + 1, :n]
        # copies: a row view starts at an odd offset when T is odd, and the native SI-SDR wants 16-byte aligned rows
        input_one, input_rest = (r.clone() for r in torch.unbind(_input, dim=1))
        possible = []
        for idx in range(n):
            mask_one = torch.zeros_like(_target)
            mask_one[:, idx] = 1.0
            mask_rest = torch.ones_like(_target) - mask_one
            target_one = torch.sum(mask_one * _target, dim=1)
            target_rest = torch.sum(mask_rest * _target, dim=1)
            loss_one = criterion(input_one, target_one, batch_mean=False)
            loss_rest = criterion(input_rest, target_rest, batch_mean=False)
            possible.append(loss_one + loss_rest / (n - 1))
        possible = torch.cat(possible, dim=0)
        loss, i = torch.max(possible, dim=0, keepdim=True) if maximize else torch.min(possible, dim=0, keepdim=True)
        losses.append(loss)
        indices.append(i)
    return torch.cat(losses, dim=0), torch.cat(indices, dim=0)


class ORPIT(nn.Module):
    """One-and-rest PIT (src/criterion/pit.py:87-160).  input (batch_size, 2, *): the first output is one speaker, the second
    the rest; target (batch_size, n, *) or a PackedSequence of per-sample (n_b, *) targets.  Returns (loss, indices): loss
    scalar (batch_mean) or (batch_size,), indices (batch_size,) int64, the target taken as 'one'.  Every sample needs
    n_b >= 2 (ValueError otherwise; the reference divides by n_b - 1)."""

    def __init__(self, criterion):
        super().__init__()
        self.criterion = criterion
        self.patterns = torch.tensor(list(itertools.permutations(range(2))), dtype=torch.long)

    def forward(self, input, target, batch_mean=True):
        assert input.size(1) == 2, "input.size() is expected (batch_size, 2, *), but given {}".format(input.size())
        if isinstance(target, torch.Tensor):
            lens = torch.full((target.size(0),), target.size(1), dtype=torch.int64)
            packed = False
        else:
            target, lens = nn.utils.rnn.pad_packed_sequence(target, batch_first=True)
            packed = True
        if lens.numel() != input.size(0):
            raise ValueError("ORPIT: {} targets for a batch of {}".format(lens.numel(), input.size(0)))
        if int(lens.min()) < 2:
            raise ValueError("ORPIT needs at least two targets per sample, got n_sources = {}".format(lens.tolist()))
        n = target.size(1)
        if _pitx_fused_ok(self.criterion, input, n) and target.shape[0::2] == input.shape[0::2]:
            _no_target_grad(target)
            x, t = input.contiguous(), target.contiguous()
            n_b = lens.to(device=x.device, dtype=torch.int32) if packed else None
            loss, indices = _OrpitSisdrFn.apply(x, t, n_b, float(self.criterion.eps), bool(self.criterion.maximize))
        else:
            loss, indices = _orpit_generic(self.criterion, input, target, lens)
        if batch_mean:
            loss = loss.mean(dim=0)
        return loss, indices


class _SinkPitSisdrFn(torch.autograd.Function):
    """(loss_b (B), P (B,S,S)) of Sinkhorn PIT over SI-SDR; the backward runs the K iterations back (the gradient of the
    unrolled loop, as autograd gives it) and accepts a gradient on P; ctn_sinkpit_fwd / ctn_sinkpit_bwd."""

    @staticmethod
    def forward(ctx, x, t, iteration, coldness, eps, maximize):
        dev = N.require_cuda(x, t)
        B, S, T = x.shape
        loss_b = torch.empty(B, dtype=torch.float32, device=dev)
        P = torch.empty(B, S, S, dtype=torch.float32, device=dev)
        scratch = torch.empty(N.ctn_sinkpit_scratch_bytes(B, S, iteration) // 4, dtype=torch.float32, device=dev)
        N.check(N.ctn_sinkpit_fwd(x.data_ptr(), t.data_ptr(), B, S, T, iteration, coldness, float(eps), int(maximize),
                                  loss_b.data_ptr(), P.data_ptr(), None, scratch.data_ptr(), N.stream_ptr(dev)), "ctn_sinkpit_fwd")
        ctx.save_for_backward(x, t, scratch)
        ctx.args = (iteration, coldness, float(eps), int(maximize))
        ctx.set_materialize_grads(False)  # an unused P passes no gradient (grad_P = null)
        return loss_b, P

    @staticmethod
    def backward(ctx, g_loss_b, g_P):
        x, t, scratch = ctx.saved_tensors
        B, S, T = x.shape
        iteration, coldness, eps, maximize = ctx.args
        g = None if g_loss_b is None else g_loss_b.contiguous().to(torch.float32)
        gP = None if g_P is None else g_P.contiguous().to(torch.float32)
        if g is None:
            g = torch.zeros(B, dtype=torch.float32, device=x.device)
        dL = torch.empty(B, S, S, dtype=torch.float32, device=x.device)
        d_x = torch.empty_like(x)
        N.check(N.ctn_sinkpit_bwd(x.data_ptr(), t.data_ptr(), B, S, T, iteration, coldness, eps, maximize, scratch.data_ptr(),
                                  g.data_ptr(), N.ptr(gP), dL.data_ptr(), d_x.data_ptr(), N.stream_ptr(x.device)),
                "ctn_sinkpit_bwd")
        return d_x, None, None, None, None, None


def sinkpit(criterion, input, target, n_sources=None, coldness=1e+0, iteration=10, batch_mean=True):
    """Sinkhorn PIT (src/criterion/pit.py:162-194).  Returns (loss, P): loss scalar (batch_mean) or (batch_size,), P
    (batch_size, n_sources, n_sources) the soft permutation matrix, which carries gradient."""
    S = input.size(1)
    if ((n_sources is None or n_sources == S) and _pitx_fused_ok(criterion, input, S) and target.shape == input.shape
            and float(coldness) > 0 and int(iteration) >= 0):
        _no_target_grad(target)
        loss, P = _SinkPitSisdrFn.apply(input.contiguous(), target.contiguous(), int(iteration), float(coldness),
                                        float(criterion.eps), bool(criterion.maximize))
    else:
        loss, P = _sinkpit_generic(criterion, input, target, n_sources, coldness, iteration)
    if batch_mean:
        loss = loss.mean(dim=0)
    return loss, P


def _sinkpit_generic(criterion, input, target, n_sources, coldness, iteration):
    """the reference's arithmetic (pit.py:162-194) without the batch mean"""
    if n_sources is None:
        n_sources = input.size(1)
    B = input.size(0)
    input_size, target_size = input.size()[2:], target.size()[2:]
    input = input.unsqueeze(dim=2).expand(-1, -1, n_sources, -1).contiguous()
    target = target.unsqueeze(dim=1).expand(-1, n_sources, -1, -1).contiguous()
    input, target = input.view(B * n_sources * n_sources, *input_size), target.view(B * n_sources * n_sources, *target_size)
    possible_loss = criterion(input, target, batch_mean=False).view(B, n_sources, n_sources)
    maximize = hasattr(criterion, "maximize") and criterion.maximize
    if maximize:
        possible_loss = -possible_loss
    Z = -coldness * possible_loss
    for _ in range(iteration):
        Z = Z - torch.logsumexp(Z, dim=1, keepdim=True)
        Z = Z - torch.logsumexp(Z, dim=2, keepdim=True)
    P = torch.exp(Z)
    loss = torch.sum((possible_loss + Z / coldness) * P, dim=(1, 2))
    if maximize:
        loss = -loss
    return loss, P


class SinkPIT(nn.Module):
    """Sinkhorn PIT (src/criterion/pit.py:196-213), "Towards Listening to 10 People Simultaneously"
    (https://arxiv.org/abs/2010.11871).  Returns (loss, pattern): pattern (batch_size, n_sources) int64 = argmax(P, dim=2)."""

    def __init__(self, criterion, n_sources=None, coldness=1, iteration=10):
        super().__init__()
        self.criterion = criterion
        self.n_sources = n_sources
        self.coldness = coldness
        self.iteration = iteration

    def forward(self, input, target, batch_mean=True):
        loss, P = sinkpit(self.criterion, input, target, n_sources=self.n_sources, coldness=self.coldness,
                          iteration=self.iteration, batch_mean=batch_mean)
        return loss, torch.argmax(P, dim=2)
