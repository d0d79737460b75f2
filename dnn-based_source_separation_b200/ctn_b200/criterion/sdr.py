"""SDR-family criteria on sm_90a kernels, mirroring src/criterion/sdr.py: ``sdr`` / ``SDR`` / ``NegSDR`` (:6-110), ``sisdr``
(:122-139), ``SISDR`` (:141-185), ``NegSISDR`` (:187-231), ``ClippedSISDR`` / ``ClippedNegSISDR`` (:233-327).
Inputs (batch_size, T), (batch_size, n_sources, T) or (batch_size, n_sources, n_mics, T).  ``sisdr`` is differentiable w.r.t. its
input.  The function ``sdr`` is forward only (an evaluation metric: it raises under autograd); the ``SDR`` / ``NegSDR`` modules,
which the recipes train with, are differentiable w.r.t. the estimate (ctn_sdr_fwd / ctn_sdr_bwd).  No criterion here
differentiates w.r.t. its target."""
import torch
import torch.nn as nn

from .. import _native as N

EPS = 1e-12


def sisdr(input, target, eps=EPS):
    n_dims = input.dim()
    assert n_dims in [2, 3, 4], "Only 2D or 3D or 4D tensor is acceptable, but given {}D tensor.".format(n_dims)
    if input.shape != target.shape:
        raise ValueError("input and target must have the same shape")
    if torch.is_grad_enabled() and target.requires_grad:
        raise NotImplementedError("gradient w.r.t. the SI-SDR target is not built")
    if torch.is_grad_enabled() and input.requires_grad:
        # autograd: every row is a 1-source PIT problem (identity permutation) -> the fused forward/backward pair
        # ctn_sisdr_pit_fwd / ctn_sisdr_pit_bwd; its loss is -SI-SDR
        from .pit import _PitNegSisdrFn
        T = input.shape[-1]
        x, t = input.contiguous().view(-1, 1, T), target.contiguous().view(-1, 1, T)
        N.require_cuda(x, t)
        neg, _ = _PitNegSisdrFn.apply(x, t, float(eps))
        return (-neg).view(input.shape[:-1])
    x, t = input.contiguous(), target.contiguous()
    dev = N.require_cuda(x, t)
    T = x.shape[-1]
    rows = x.numel() // T
    out = torch.empty(x.shape[:-1], dtype=torch.float32, device=dev)
    scratch = torch.empty(N.ctn_sisdr_pit_scratch_bytes(rows, 1) // 8, dtype=torch.float64, device=dev)
    N.check(N.ctn_sisdr_fwd(x.data_ptr(), t.data_ptr(), rows, T, float(eps), out.data_ptr(), scratch.data_ptr(),
                            N.stream_ptr(dev)), "ctn_sisdr_fwd")
    return out


def sdr(input, target, eps=EPS):
    n_dims = input.dim()
    assert n_dims in [2, 3, 4], "Only 2D or 3D or 4D tensor is acceptable, but given {}D tensor.".format(n_dims)
    if input.shape != target.shape:
        raise ValueError("input and target must have the same shape")
    if torch.is_grad_enabled() and (input.requires_grad or target.requires_grad):
        raise NotImplementedError("sdr() is forward only (an evaluation metric); train with the SDR / NegSDR modules")
    x, t = input.contiguous(), target.contiguous()
    dev = N.require_cuda(x, t)
    T = x.shape[-1]
    rows = x.numel() // T
    out = torch.empty(x.shape[:-1], dtype=torch.float32, device=dev)
    scratch = torch.empty(2 * rows, dtype=torch.float64, device=dev)
    N.check(N.ctn_sdr_fwd(x.data_ptr(), t.data_ptr(), rows, T, float(eps), out.data_ptr(), scratch.data_ptr(), N.stream_ptr(dev)), "ctn_sdr_fwd")
    return out


class _SdrFn(torch.autograd.Function):
    """sdr (rows) of (rows, T) estimates and targets with its gradient w.r.t. the estimate; ctn_sdr_fwd / ctn_sdr_bwd"""

    @staticmethod
    def forward(ctx, x, t, eps):
        dev = N.require_cuda(x, t)
        rows, T = x.shape
        out = torch.empty(rows, dtype=torch.float32, device=dev)
        scratch = torch.empty(2 * rows, dtype=torch.float64, device=dev)
        N.check(N.ctn_sdr_fwd(x.data_ptr(), t.data_ptr(), rows, T, float(eps), out.data_ptr(), scratch.data_ptr(), N.stream_ptr(dev)),
                "ctn_sdr_fwd")
        ctx.save_for_backward(x, t, scratch)
        ctx.eps = float(eps)
        return out

    @staticmethod
    def backward(ctx, g_out):
        x, t, scratch = ctx.saved_tensors
        rows, T = x.shape
        g = g_out.contiguous().to(torch.float32)
        d_x = torch.empty_like(x)
        N.check(N.ctn_sdr_bwd(x.data_ptr(), t.data_ptr(), rows, T, ctx.eps, scratch.data_ptr(), g.data_ptr(), 1.0, d_x.data_ptr(),
                              N.stream_ptr(x.device)), "ctn_sdr_bwd")
        return d_x, None, None


def _sdr_trainable(input, target, eps):
    """sdr() for the SDR / NegSDR modules: the same values, differentiable w.r.t. the estimate"""
    if not torch.is_grad_enabled() or not (input.requires_grad or target.requires_grad):
        return sdr(input, target, eps=eps)
    n_dims = input.dim()
    assert n_dims in [2, 3, 4], "Only 2D or 3D or 4D tensor is acceptable, but given {}D tensor.".format(n_dims)
    if input.shape != target.shape:
        raise ValueError("input and target must have the same shape")
    if target.requires_grad:
        raise NotImplementedError("gradient w.r.t. the SDR target is not built")
    T = input.shape[-1]
    return _SdrFn.apply(input.contiguous().view(-1, T), target.contiguous().view(-1, T), float(eps)).view(input.shape[:-1])


def _reduce(loss, n_dims, reduction, batch_mean):
    if reduction:
        dims = 1 if n_dims == 3 else ((1, 2) if n_dims == 4 else None)
        if dims is not None:
            loss = loss.mean(dim=dims) if reduction == 'mean' else loss.sum(dim=dims)
    if batch_mean:
        loss = loss.mean(dim=0)
    return loss


class SISDR(nn.Module):
    def __init__(self, reduction='mean', eps=EPS):
        super().__init__()
        if reduction not in ['mean', 'sum', None]:
            raise ValueError("Invalid reduction type")
        self.reduction, self.eps = reduction, eps

    def forward(self, input, target, batch_mean=True):
        return _reduce(sisdr(input, target, eps=self.eps), input.dim(), self.reduction, batch_mean)

    @property
    def maximize(self):
        return True


class NegSISDR(nn.Module):
    def __init__(self, reduction='mean', eps=EPS):
        super().__init__()
        if reduction not in ['mean', 'sum', None]:
            raise ValueError("Invalid reduction type")
        self.reduction, self.eps = reduction, eps

    def forward(self, input, target, batch_mean=True):
        return _reduce(-sisdr(input, target, eps=self.eps), input.dim(), self.reduction, batch_mean)

    @property
    def maximize(self):
        return False


class _Criterion(nn.Module):
    def __init__(self, reduction='mean', eps=EPS):
        super().__init__()
        if reduction not in ['mean', 'sum', None]:
            raise ValueError("Invalid reduction type")
        self.reduction, self.eps = reduction, eps


class SDR(_Criterion):
    def forward(self, input, target, batch_mean=True):
        return _reduce(_sdr_trainable(input, target, self.eps), input.dim(), self.reduction, batch_mean)

    @property
    def maximize(self):
        return True


class NegSDR(_Criterion):
    def forward(self, input, target, batch_mean=True):
        return _reduce(-_sdr_trainable(input, target, self.eps), input.dim(), self.reduction, batch_mean)

    @property
    def maximize(self):
        return False


class ClippedSISDR(_Criterion):
    def __init__(self, max=None, reduction='mean', eps=EPS):
        super().__init__(reduction=reduction, eps=eps)
        self.max = max

    def forward(self, input, target, batch_mean=True):
        return _reduce(torch.clamp(sisdr(input, target, eps=self.eps), max=self.max), input.dim(), self.reduction, batch_mean)

    @property
    def maximize(self):
        return True


class ClippedNegSISDR(_Criterion):
    def __init__(self, min=None, reduction='mean', eps=EPS):
        super().__init__(reduction=reduction, eps=eps)
        self.min = min

    def forward(self, input, target, batch_mean=True):
        return _reduce(torch.clamp(-sisdr(input, target, eps=self.eps), min=self.min), input.dim(), self.reduction, batch_mean)

    @property
    def maximize(self):
        return False
