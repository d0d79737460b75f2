"""GTU1d behind the reference's class API (src/models/gtu.py:10-44): same constructor and ``map`` / ``map_gate`` parameters.

Inside DPTNet the two 1x1 convolutions run as one contraction of 2N rows in ``ctn_dpt_tail_fwd`` (csrc/ctn_dptnet.cu), with
tanh(map) * sigmoid(map_gate), the mask nonlinearity and w * mask in the pass after it; the stand-alone module is a parameter
container.
"""
import torch.nn as nn


class GTU1d(nn.Module):
    """Gated Tanh Units for 1D inputs"""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1):
        super().__init__()
        if out_channels is None:
            out_channels = in_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        if kernel_size != 1 or stride != 1 or padding != 0 or dilation != 1:
            raise NotImplementedError("GTU1d runs as a 1x1 contraction only (kernel_size=1, stride=1, padding=0, dilation=1)")
        self.map = nn.Conv1d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding, dilation=dilation)
        self.map_gate = nn.Conv1d(in_channels, out_channels, kernel_size=kernel_size, stride=stride, padding=padding, dilation=dilation)

    def forward(self, input):
        raise NotImplementedError("the stand-alone GTU1d.forward is not built; it runs inside DPTNet's separator tail")
