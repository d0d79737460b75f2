"""Trainable encoder / decoder filterbanks on sm_90a kernels.

Mirrors ``Encoder`` (src/models/filterbank.py:205-235) and ``Decoder`` (:237-251) of the reference: same constructor,
same ``conv1d.weight`` / ``conv_transpose1d.weight`` parameters, same forward shapes.  The nn.Conv1d /
nn.ConvTranspose1d members are parameter containers (identical default init and state_dict keys); the arithmetic
runs in ctn_encoder_fwd / ctn_decoder_fwd (csrc/ctn_encdec.cu).
"""
import torch
import torch.nn as nn

from .. import _native as N


class Encoder(nn.Module):
    def __init__(self, in_channels, n_basis, kernel_size=16, stride=8, nonlinear=None):
        super().__init__()
        if in_channels < 1 or in_channels > 64:
            raise NotImplementedError("in_channels={} is outside the sm_90a path (1 .. 64)".format(in_channels))
        self.in_channels, self.n_basis = in_channels, n_basis
        self.kernel_size, self.stride = kernel_size, stride
        self.conv1d = nn.Conv1d(in_channels, n_basis, kernel_size=kernel_size, stride=stride, bias=False)
        if nonlinear is None or nonlinear == '':
            self.nonlinear = False
        elif nonlinear == 'relu':
            self.nonlinear = True
        else:
            raise NotImplementedError("Not support {}".format(nonlinear))

    def forward(self, input):
        """input (batch_size, in_channels, T) -> (batch_size, n_basis, (T - kernel_size) // stride + 1)"""
        if input.dim() != 3 or input.size(1) != self.in_channels:
            raise ValueError("input.size() is expected (?, {}, ?), but given {}".format(self.in_channels, tuple(input.size())))
        if torch.is_grad_enabled() and self.in_channels > 1 and (input.requires_grad or self.conv1d.weight.requires_grad):
            raise NotImplementedError("the multichannel encoder is forward only: call under torch.no_grad()")
        x = input.contiguous()
        dev = N.require_cuda(x, self.conv1d.weight)
        B, _, T = x.shape
        L, S = self.kernel_size, self.stride
        if T < L:
            raise ValueError("input is shorter than the kernel")
        frames = (T - L) // S + 1
        T_used = (frames - 1) * S + L  # Conv1d drops the ragged tail
        w = torch.empty(B, self.n_basis, frames, dtype=torch.float32, device=dev)
        xin = x if T_used == T else x[..., :T_used].contiguous()
        if self.in_channels > 1:
            N.check(N.ctn_encoder_mc_fwd(xin.data_ptr(), self.conv1d.weight.data_ptr(), w.data_ptr(), B, self.in_channels, T_used, 0, 0,
                                         self.n_basis, L, S, int(self.nonlinear), frames, None, N.stream_ptr(dev)), "ctn_encoder_mc_fwd")
            return w
        N.check(N.ctn_encoder_fwd(xin.data_ptr(), self.conv1d.weight.data_ptr(), w.data_ptr(), B, T_used, 0, 0, self.n_basis,
                                  L, S, int(self.nonlinear), frames, None, N.stream_ptr(dev)), "ctn_encoder_fwd")
        return w

    def get_basis(self):
        return self.conv1d.weight


class Decoder(nn.Module):
    def __init__(self, n_basis, out_channels, kernel_size=16, stride=8):
        super().__init__()
        if out_channels < 1 or out_channels > 64:
            raise NotImplementedError("out_channels={} is outside the sm_90a path (1 .. 64)".format(out_channels))
        self.n_basis, self.out_channels = n_basis, out_channels
        self.kernel_size, self.stride = kernel_size, stride
        self.conv_transpose1d = nn.ConvTranspose1d(n_basis, out_channels, kernel_size=kernel_size, stride=stride, bias=False)

    def forward(self, input):
        """input (batch_size, n_basis, T') -> (batch_size, out_channels, (T' - 1) * stride + kernel_size)"""
        if input.dim() != 3 or input.size(1) != self.n_basis:
            raise ValueError("input.size() is expected (?, {}, ?), but given {}".format(self.n_basis, tuple(input.size())))
        x = input.contiguous()
        dev = N.require_cuda(x, self.conv_transpose1d.weight)
        BS, _, frames = x.shape
        L, S = self.kernel_size, self.stride
        if L % S != 0:
            raise NotImplementedError("kernel_size % stride != 0 is outside the sm_90a decoder envelope")
        T_out = (frames - 1) * S + L
        y = torch.empty(BS, self.out_channels, T_out, dtype=torch.float32, device=dev)
        if self.out_channels > 1:
            if torch.is_grad_enabled() and (input.requires_grad or self.conv_transpose1d.weight.requires_grad):
                raise NotImplementedError("the multichannel decoder is forward only: call under torch.no_grad()")
            N.check(N.ctn_decoder_mc_fwd(x.data_ptr(), self.conv_transpose1d.weight.data_ptr(), y.data_ptr(), BS, self.out_channels,
                                         self.n_basis, frames, frames, L, S, 0, T_out, N.stream_ptr(dev)), "ctn_decoder_mc_fwd")
            return y
        N.check(N.ctn_decoder_fwd(x.data_ptr(), self.conv_transpose1d.weight.data_ptr(), y.data_ptr(), BS, self.n_basis, frames,
                                  frames, L, S, 0, T_out, N.stream_ptr(dev)), "ctn_decoder_fwd")
        return y

    def get_basis(self):
        return self.conv_transpose1d.weight
