"""Time-dilated convolutional network (the Conv-TasNet separator core) on sm_90a kernels.

Mirrors src/models/tdcn.py of the reference -- ``TimeDilatedConvNet`` (:13-41), ``TimeDilatedConvBlock1d`` (:43-75),
``ResidualBlock1d`` (:77-147), ``DepthwiseSeparableConv1d`` (:149-196): same constructors, same module tree and
therefore the same ``state_dict`` keys.  The sub-modules are *parameter containers*: the whole stack is executed by
one C call (ctn_tcn_fwd) that runs, per residual block,

    1x1 conv (+bias, PReLU, gLN statistics)  ->  gLN-apply + dilated depthwise conv + PReLU (+ statistics)
      ->  [output;skip] 1x1 convs with the second gLN folded into the weights  ->  residual / skip accumulation.

Kernel envelope: dilated=True, separable=True, nonlinear='prelu', norm=True; causal=False (gLN, fused stack) or
causal=True (cLN, un-fused forward pipeline).  Anything else
raises NotImplementedError -- there is no eager fallback.
"""
import ctypes as C

import torch
import torch.nn as nn

from .. import _native as N
from ..utils.tasnet import choose_layer_norm

EPS = 1e-12
DEFAULT_MATH = None  # None -> 'f16x3' when the tensor-core family is built, else 'fp32'


def resolve_math(mode=None):
    if mode is None:
        mode = DEFAULT_MATH
    if mode is None:
        # 'f16x3': fp32-parity 3-pass split on fp16 pieces (same 11-bit pieces as 'tf32x3', twice the tensor rate).  Its envelope
        # (|activation|, |weight| < 65504) always holds behind the normalisations of this network; the one contraction that
        # sees un-normalised data (the separator head on the encoder output) stays on 'tf32x3' inside the library.
        mode = "f16x3" if N.ctn_has_tcgen05() else "fp32"
    return N.MATH_NAMES[mode]


class DepthwiseSeparableConv1d(nn.Module):
    """Parameter container for the depthwise stage + the two pointwise heads (tdcn.py:149-196)."""

    def __init__(self, in_channels, out_channels=256, skip_channels=256, kernel_size=3, stride=2, dilation=1, causal=True,
                 nonlinear=None, norm=True, dual_head=True, eps=EPS):
        super().__init__()
        self.dual_head, self.norm, self.eps = dual_head, norm, eps
        self.kernel_size, self.stride, self.dilation = kernel_size, stride, dilation
        self.depthwise_conv1d = nn.Conv1d(in_channels, in_channels, kernel_size=kernel_size, stride=stride, dilation=dilation,
                                          groups=in_channels)
        if nonlinear is not None:
            if nonlinear != 'prelu':
                raise ValueError("Not support {}".format(nonlinear))
            self.nonlinear1d = nn.PReLU()
        self.nonlinear = nonlinear is not None
        if norm:
            self.norm1d = choose_layer_norm('cLN' if causal else 'gLN', in_channels, causal=causal, eps=eps)
        if dual_head:
            self.output_pointwise_conv1d = nn.Conv1d(in_channels, out_channels, kernel_size=1, stride=1)
        self.skip_pointwise_conv1d = nn.Conv1d(in_channels, skip_channels, kernel_size=1, stride=1)

    def forward(self, input):
        raise NotImplementedError("DepthwiseSeparableConv1d is fused into TimeDilatedConvNet.forward on the sm_90a path")


class ResidualBlock1d(nn.Module):
    """Parameter container for one residual block (tdcn.py:77-147)."""

    def __init__(self, num_features, hidden_channels=256, skip_channels=256, kernel_size=3, stride=2, dilation=1,
                 separable=False, causal=True, nonlinear=None, norm=True, dual_head=True, eps=EPS):
        super().__init__()
        if not separable:
            raise NotImplementedError("separable=False is outside the sm_90a kernel envelope")
        self.kernel_size, self.stride, self.dilation = kernel_size, stride, dilation
        self.separable, self.causal, self.norm, self.dual_head = separable, causal, norm, dual_head
        self.bottleneck_conv1d = nn.Conv1d(num_features, hidden_channels, kernel_size=1, stride=1)
        if nonlinear is not None:
            if nonlinear != 'prelu':
                raise ValueError("Not support {}".format(nonlinear))
            self.nonlinear1d = nn.PReLU()
        self.nonlinear = nonlinear is not None
        if norm:
            self.norm1d = choose_layer_norm('cLN' if causal else 'gLN', hidden_channels, causal=causal, eps=eps)
        self.separable_conv1d = DepthwiseSeparableConv1d(
            hidden_channels, num_features, skip_channels=skip_channels, kernel_size=kernel_size, stride=stride,
            dilation=dilation, causal=causal, nonlinear=nonlinear, norm=norm, dual_head=dual_head, eps=eps)

    def forward(self, input):
        """input (batch_size, num_features, T) -> (output or None, skip): tdcn.py:107-147, one fused block through
        ctn_tcn_blocks_fwd (non-causal gLN, stride 1)."""
        return run_blocks([self], input, want_output=self.dual_head)

    def native_params(self):
        """Device pointers in the order of ctn_block_params_t (include/ctn_b200.h)."""
        sep = self.separable_conv1d
        g1, b1 = N.norm_affine(self.norm1d)
        g2, b2 = N.norm_affine(sep.norm1d)
        out_w = sep.output_pointwise_conv1d.weight if self.dual_head else None
        out_b = sep.output_pointwise_conv1d.bias if self.dual_head else None
        return (self.bottleneck_conv1d.weight, self.bottleneck_conv1d.bias, self.nonlinear1d.weight, g1, b1,
                sep.depthwise_conv1d.weight, sep.depthwise_conv1d.bias, sep.nonlinear1d.weight, g2, b2,
                out_w, out_b, sep.skip_pointwise_conv1d.weight, sep.skip_pointwise_conv1d.bias)


class TimeDilatedConvBlock1d(nn.Module):
    def __init__(self, num_features, hidden_channels=256, skip_channels=256, kernel_size=3, num_layers=10, dilated=True,
                 separable=False, causal=True, nonlinear=None, norm=True, dual_head=True, eps=EPS):
        super().__init__()
        if not dilated:
            raise NotImplementedError("dilated=False is outside the sm_90a kernel envelope")
        self.num_layers = num_layers
        net = []
        for idx in range(num_layers):
            last = (not dual_head) and idx == num_layers - 1  # tdcn.py:58-61
            net.append(ResidualBlock1d(num_features, hidden_channels=hidden_channels, skip_channels=skip_channels,
                                       kernel_size=kernel_size, stride=1, dilation=2 ** idx, separable=separable, causal=causal,
                                       nonlinear=nonlinear, norm=norm, dual_head=not last, eps=eps))
        self.net = nn.Sequential(*net)

    def forward(self, input):
        """input (batch_size, num_features, T) -> (output or None, skip sum of the layers): tdcn.py:65-75"""
        blocks = list(self.net)
        return run_blocks(blocks, input, want_output=blocks[-1].dual_head)


def run_blocks(blocks, input, want_output, math=None):
    """A run of ResidualBlock1d modules with their own dilations through ctn_tcn_blocks_fwd -> (output | None, skip)."""
    if input.dim() != 3:
        raise ValueError("input is expected 3-D (batch_size, num_features, T), but given {}".format(tuple(input.size())))
    if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for b in blocks for p in b.parameters())):
        raise NotImplementedError("block-level forward is inference-only: training goes through ConvTasNet.forward (one autograd node)")
    b0 = blocks[0]
    if b0.causal or b0.stride != 1 or not b0.norm or not b0.nonlinear:
        raise NotImplementedError("stand-alone blocks: non-causal gLN, stride 1, prelu only")
    x = input.contiguous()
    dev = N.require_cuda(x)
    B, F_in, frames = x.shape
    cfg = N.Config()
    cfg.bottleneck, cfg.hidden = b0.bottleneck_conv1d.in_channels, b0.bottleneck_conv1d.out_channels
    cfg.skip = b0.separable_conv1d.skip_pointwise_conv1d.out_channels
    cfg.sep_kernel, cfg.num_blocks, cfg.num_layers, cfg.causal = b0.kernel_size, 1, len(blocks), 0
    cfg.math = resolve_math(math)
    cfg.eps_tcn = cfg.eps = float(b0.separable_conv1d.eps)
    if F_in != cfg.bottleneck:
        raise ValueError("input.size() is expected (?, {}, ?), but given {}".format(cfg.bottleneck, tuple(input.size())))
    arr, keep = block_param_array(blocks, dev)
    dil = (C.c_int * len(blocks))(*[int(b.dilation) for b in blocks])
    cfg2 = N.Config.from_buffer_copy(cfg)
    cfg2.num_layers = len(blocks)
    need = C.c_size_t(0)
    N.check(N.ctn_tcn_workspace_bytes(C.byref(cfg2), B, frames, C.byref(need)), "ctn_tcn_workspace_bytes")
    base, nbytes = N.aligned(N.workspace(dev, need.value))
    skip = torch.empty(B, cfg.skip, frames, dtype=torch.float32, device=dev)
    out = torch.empty(B, cfg.bottleneck, frames, dtype=torch.float32, device=dev) if want_output else None
    N.check(N.ctn_tcn_blocks_fwd(C.byref(cfg2), arr, len(blocks), dil, x.data_ptr(), N.ptr(out), skip.data_ptr(), B, frames, base,
                                 nbytes, N.stream_ptr(dev)), "ctn_tcn_blocks_fwd")
    return out, skip


def block_slots(residual_blocks):
    """[((block index, block field name), tensor-or-None)] of a list of ResidualBlock1d, for N.build_params"""
    return [((i, name), t) for i, blk in enumerate(residual_blocks) for name, t in zip(N.BLOCK_FIELDS, blk.native_params())]


def block_param_array(residual_blocks, dev):
    """ctn_block_params_t array of a list of ResidualBlock1d -> (array pointer, keep)"""
    p, keep = N.build_params(block_slots(residual_blocks), dev)
    return p.blocks, keep


class TimeDilatedConvNet(nn.Module):
    def __init__(self, num_features, hidden_channels=256, skip_channels=256, kernel_size=3, num_blocks=3, num_layers=10,
                 dilated=True, separable=False, causal=True, nonlinear=None, norm=True, eps=EPS):
        super().__init__()
        if nonlinear != 'prelu' or not norm:
            raise NotImplementedError("the sm_90a TCN requires nonlinear='prelu' and norm=True")
        self.num_features, self.hidden_channels, self.skip_channels = num_features, hidden_channels, skip_channels
        self.kernel_size, self.num_blocks, self.num_layers = kernel_size, num_blocks, num_layers
        self.dilated, self.separable, self.causal, self.eps = dilated, separable, causal, eps
        self.math = None  # per-module override of the numeric mode ('fp32' | 'tf32x3' | 'tf32')
        net = []
        for idx in range(num_blocks):
            net.append(TimeDilatedConvBlock1d(num_features, hidden_channels=hidden_channels, skip_channels=skip_channels,
                                              kernel_size=kernel_size, num_layers=num_layers, dilated=dilated, separable=separable,
                                              causal=causal, nonlinear=nonlinear, norm=norm, dual_head=idx != num_blocks - 1, eps=eps))
        self.net = nn.Sequential(*net)

    def residual_blocks(self):
        return [blk for stage in self.net for blk in stage.net]

    def native_config(self, **extra):
        cfg = N.Config()
        cfg.bottleneck, cfg.hidden, cfg.skip = self.num_features, self.hidden_channels, self.skip_channels
        cfg.sep_kernel, cfg.num_blocks, cfg.num_layers = self.kernel_size, self.num_blocks, self.num_layers
        cfg.causal = int(self.causal)
        cfg.math = resolve_math(self.math)
        cfg.eps_tcn = float(self.eps)
        cfg.eps = float(self.eps)
        for k, v in extra.items():
            setattr(cfg, k, v)
        return cfg

    def forward(self, input):
        """input (batch_size, num_features, T) -> skip-connection sum (batch_size, skip_channels, T)"""
        if input.dim() != 3 or input.size(1) != self.num_features:
            raise ValueError("input.size() is expected (?, {}, ?), but given {}".format(self.num_features, tuple(input.size())))
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise NotImplementedError("stand-alone TimeDilatedConvNet.forward is inference-only (training runs through ConvTasNet.forward, one autograd node): call under torch.no_grad()")
        x = input.contiguous()
        dev = N.require_cuda(x)
        B, _, frames = x.shape
        cfg = self.native_config()
        arr, keep = block_param_array(self.residual_blocks(), dev)
        need = C.c_size_t(0)
        N.check(N.ctn_tcn_workspace_bytes(C.byref(cfg), B, frames, C.byref(need)), "ctn_tcn_workspace_bytes")
        base, nbytes = N.aligned(N.workspace(dev, need.value))
        out = torch.empty(B, self.skip_channels, frames, dtype=torch.float32, device=dev)
        N.check(N.ctn_tcn_fwd(C.byref(cfg), arr, x.data_ptr(), out.data_ptr(), B, frames, base, nbytes, N.stream_ptr(dev)), "ctn_tcn_fwd")
        return out
