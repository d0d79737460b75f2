"""Plain depthwise-separable convolution, mirroring src/modules/conv.py:13-29 of the reference (``DepthwiseSeparableConv1d``):
``depthwise_conv1d`` (Conv1d with groups = in_channels) followed by ``pointwise_conv1d`` (1x1 Conv1d), same constructor, parameter
names and shapes.  Not on Conv-TasNet's hot path (its blocks use the fused variant in models/tdcn.py); the two stages run in
ctn_depthwise_conv1d_fwd / ctn_pointwise_conv1d_fwd (csrc/ctn_conv.cu).  Inference only."""
import torch
import torch.nn as nn

from .. import _native as N
from ..models.tdcn import resolve_math


class DepthwiseSeparableConv1d(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=None, padding=0, dilation=1, bias=True):
        super().__init__()
        if stride is None:
            stride = kernel_size
        self.kernel_size, self.stride, self.dilation, self.padding = kernel_size, stride, dilation, padding
        self.depthwise_conv1d = nn.Conv1d(in_channels, in_channels, kernel_size=kernel_size, stride=stride, padding=padding,
                                          dilation=dilation, groups=in_channels, bias=bias)
        self.pointwise_conv1d = nn.Conv1d(in_channels, out_channels, kernel_size=1, stride=1, bias=bias)
        self.math = None

    def forward(self, input):
        """input (batch_size, in_channels, T) -> (batch_size, out_channels, T_out)"""
        if input.dim() != 3 or input.size(1) != self.depthwise_conv1d.in_channels:
            raise ValueError("input.size() is expected (?, {}, ?), but given {}".format(self.depthwise_conv1d.in_channels, tuple(input.size())))
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("modules.conv.DepthwiseSeparableConv1d is inference-only on the sm_90a path: call under torch.no_grad()")
        x = input.contiguous()
        dev = N.require_cuda(x)
        B, Cc, T = x.shape
        K, S, P, D = self.kernel_size, self.stride, self.padding, self.dilation
        span = D * (K - 1) + 1
        if T + 2 * P < span:
            raise ValueError("input is shorter than the dilated kernel")
        To = (T + 2 * P - span) // S + 1
        pitch = N.ctn_pitch(To)
        M = self.pointwise_conv1d.out_channels
        dw, pw = self.depthwise_conv1d, self.pointwise_conv1d
        u = torch.empty(B, Cc, pitch, dtype=torch.float32, device=dev)
        st = N.stream_ptr(dev)
        N.check(N.ctn_depthwise_conv1d_fwd(x.data_ptr(), dw.weight.data_ptr(), N.ptr(dw.bias), u.data_ptr(), B, Cc, T, K, S, P, D, pitch, st),
                "ctn_depthwise_conv1d_fwd")
        y = torch.empty(B, M, To, dtype=torch.float32, device=dev)
        need = 4 * B * M * pitch + N.ctn_stage_workspace_bytes(M, Cc) + 16 * B + 4096
        base, nbytes = N.aligned(N.workspace(dev, need, tag="conv"))
        N.check(N.ctn_pointwise_conv1d_fwd(u.data_ptr(), pw.weight.data_ptr(), N.ptr(pw.bias), y.data_ptr(), B, M, Cc, To, pitch,
                                           resolve_math(self.math), base, nbytes, st), "ctn_pointwise_conv1d_fwd")
        return y
