"""Layer norms of the Conv-TasNet path, computed by sm_90a kernels.

Mirrors src/modules/norm.py of the reference: ``GlobalLayerNorm`` (:11-35, a GroupNorm(1, C) -> state_dict keys
``norm.weight`` / ``norm.bias``) and ``CumulativeLayerNorm1d`` (:42-101, parameters ``gamma`` / ``beta`` of shape
(1, C, 1), eps outside the sqrt).  Inside ConvTasNet the statistics are produced by the preceding kernel's epilogue
and the affine part is folded into the following 1x1 conv; these classes are the stand-alone module API.
"""
import torch
import torch.nn as nn

from .. import _native as N

EPS = 1e-12


class GlobalLayerNorm(nn.Module):
    def __init__(self, num_features, eps=EPS):
        super().__init__()
        self.num_features, self.eps = num_features, eps
        # parameter container only (keeps the reference's 'norm.weight' / 'norm.bias' keys); never called
        self.norm = nn.GroupNorm(1, num_features, eps=eps)

    def forward(self, input):
        """input (batch_size, C, *) -> same shape."""
        if input.dim() < 3:
            raise ValueError("Expected (batch_size, C, *) input, but given {}D".format(input.dim()))
        x = input.contiguous()
        dev = N.require_cuda(x, self.norm.weight)
        B, Cc = x.shape[0], x.shape[1]
        if Cc != self.num_features:
            raise ValueError("Expected {} channels, but given {}".format(self.num_features, Cc))
        T = x.numel() // (B * Cc)
        y = torch.empty_like(x)
        scratch = torch.empty(2 * B, dtype=torch.float64, device=dev)
        N.check(N.ctn_gln_fwd(x.data_ptr(), self.norm.weight.data_ptr(), self.norm.bias.data_ptr(), y.data_ptr(), B, Cc, T,
                              float(self.eps), scratch.data_ptr(), N.stream_ptr(dev)), "ctn_gln_fwd")
        return y

    def __repr__(self):
        return "{}({}, eps={})".format(self.__class__.__name__, self.num_features, self.eps)


class _CLNFn(torch.autograd.Function):
    """cLN under autograd: ctn_cln_fwd / ctn_cln_bwd on the (B, C, T) view of the input"""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        dev = N.require_cuda(x, gamma, beta)
        B, Cc = x.shape[0], x.shape[1]
        T = x.numel() // (B * Cc)
        y = torch.empty_like(x)
        scratch = torch.empty(2 * B * T, dtype=torch.float64, device=dev)
        N.check(N.ctn_cln_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), B, Cc, T, float(eps),
                              scratch.data_ptr(), N.stream_ptr(dev)), "ctn_cln_fwd")
        ctx.save_for_backward(x, gamma)
        ctx.eps = float(eps)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma = ctx.saved_tensors
        dev = x.device
        B, Cc = x.shape[0], x.shape[1]
        T = x.numel() // (B * Cc)
        dy = dy.contiguous()
        N.require_cuda(dy)
        dx = torch.empty_like(x)
        dg = torch.zeros(2, Cc, dtype=torch.float32, device=dev)  # dgamma, dbeta: accumulated by the kernel
        scratch = torch.empty(20 * B * T, dtype=torch.float64, device=dev)
        N.check(N.ctn_cln_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), scratch.data_ptr(), dx.data_ptr(), dg[0].data_ptr(),
                              dg[1].data_ptr(), B, Cc, T, ctx.eps, N.stream_ptr(dev)), "ctn_cln_bwd")
        return dx, dg[0].view(gamma.shape), dg[1].view(gamma.shape), None


class CumulativeLayerNorm1d(nn.Module):
    def __init__(self, num_features, eps=EPS):
        super().__init__()
        self.num_features, self.eps = num_features, eps
        self.gamma = nn.Parameter(torch.ones(1, num_features, 1))
        self.beta = nn.Parameter(torch.zeros(1, num_features, 1))

    def forward(self, input):
        """input (batch_size, C, T) or (batch_size, C, S, chunk_size) -> same shape."""
        n_dims = input.dim()
        if n_dims not in (3, 4):
            raise ValueError("Only support 3D or 4D input, but given {}D".format(n_dims))
        x = input.contiguous()
        dev = N.require_cuda(x, self.gamma)
        B, Cc = x.shape[0], x.shape[1]
        if torch.is_grad_enabled() and (x.requires_grad or self.gamma.requires_grad or self.beta.requires_grad):
            return _CLNFn.apply(x, self.gamma.contiguous(), self.beta.contiguous(), self.eps)
        T = x.numel() // (B * Cc)
        y = torch.empty_like(x)
        scratch = torch.empty(2 * B * T, dtype=torch.float64, device=dev)
        N.check(N.ctn_cln_fwd(x.data_ptr(), self.gamma.data_ptr(), self.beta.data_ptr(), y.data_ptr(), B, Cc, T,
                              float(self.eps), scratch.data_ptr(), N.stream_ptr(dev)), "ctn_cln_fwd")
        return y

    def __repr__(self):
        return "{}({}, eps={})".format(self.__class__.__name__, self.num_features, self.eps)
