"""Dual-path RNN blocks behind the reference's class API (src/models/dprnn.py:9-148).

``DPRNN`` / ``DPRNNBlock`` / ``IntraChunkRNN`` / ``InterChunkRNN`` keep the reference's constructors, module tree and
``state_dict`` keys (``rnn.weight_ih_l0`` ..., ``fc.weight/bias``, ``norm1d.norm.weight/bias``).

What runs where: the dual-path state lives CHANNELS-LAST, (batch, D1, D2, features) -- already the batch_first tensor the
path's LSTM consumes, so none of the reference's permute().contiguous() copies exist.  For num_features / hidden_channels in
{32, 64, 128} (cfg4: 64 / 128) the bi-LSTM recurrence AND the 2H -> F Linear run in one native wgmma kernel (3xTF32)
(``ctn_bilstm_proj_fwd``, csrc/ctn_lstm.cu): the (batch*D1, D2, 2H) LSTM output is never written.  gLN statistics,
normalisation, the sum of the two directions' partial projections + bias, the residual add and the intra <-> inter layout swap are
one more native call (``ctn_dprnn_norm_res2_fwd``).  Other sizes fall back to cuDNN's LSTM (IEEE fp32) + a library GEMM +
``ctn_dprnn_norm_res_fwd``; ``NATIVE_LSTM = False`` forces that path (it is the A/B baseline of bench.py --config cfg4).
Envelope: non-causal (gLN, bidirectional inter-chunk LSTM), rnn_type='lstm', norm=True; forward only.
"""
import contextlib

import torch
import torch.nn as nn
import torch.nn.functional as F_

from .. import _native as N
from ..utils.tasnet import choose_layer_norm
from .transform import ctn_dprnn_norm_res_fwd

EPS = 1e-12


NATIVE_LSTM = True  # native recurrence (csrc/ctn_lstm.cu) where the sizes allow; False = cuDNN + library GEMM everywhere
LSTM_TF32 = False  # cuDNN's RNN path defaults to TF32 tensor-core math (1e-3 relative): off = fp32 parity with the reference


@contextlib.contextmanager
def _rnn_precision():
    rnn = getattr(torch.backends.cudnn, "rnn", None)
    if LSTM_TF32 or rnn is None or not hasattr(rnn, "fp32_precision"):
        if LSTM_TF32 or not torch.backends.cudnn.allow_tf32:
            yield
            return
        old = torch.backends.cudnn.allow_tf32
        torch.backends.cudnn.allow_tf32 = False
        try:
            yield
        finally:
            torch.backends.cudnn.allow_tf32 = old
        return
    old = rnn.fp32_precision
    rnn.fp32_precision = "ieee"
    try:
        yield
    finally:
        rnn.fp32_precision = old


def choose_rnn(name, **kwargs):
    """src/utils/model.py:22-32"""
    if name == 'rnn':
        return nn.RNN(**kwargs)
    if name == 'lstm':
        return nn.LSTM(**kwargs)
    if name == 'gru':
        return nn.GRU(**kwargs)
    raise NotImplementedError("Invalid RNN is specified. Choose 'rnn', 'lstm', or 'gru' instead of {}.".format(name))


class _ChunkRNN(nn.Module):
    def __init__(self, num_features, hidden_channels, causal_rnn, norm=True, rnn_type='lstm', eps=EPS):
        super().__init__()
        self.num_features, self.hidden_channels = num_features, hidden_channels
        self.norm = norm
        if rnn_type != 'lstm':
            raise NotImplementedError("Not support {}.".format(rnn_type))
        if causal_rnn:
            raise NotImplementedError("causal DPRNN (uni-directional inter-chunk LSTM + cLN) is outside the sm_90a path")
        self.rnn = choose_rnn(rnn_type, input_size=num_features, hidden_size=hidden_channels, batch_first=True, bidirectional=True)
        self.fc = nn.Linear(2 * hidden_channels, num_features)
        if not norm:
            raise NotImplementedError("norm=False is outside the sm_90a path")
        self.norm1d = choose_layer_norm('gLN', num_features, causal=False, eps=eps)
        self.eps = eps

    def _step(self, z, swap, z_absmax=None):
        """z (B, D1, D2, F) channels-last -> gLN(fc(rnn(z))) + z, stored as (B, D2, D1, F) when swap.  z_absmax: optional device
        word with the bit pattern of max|z| (left by the previous block's step); the output's is left in ``self.last_absmax``."""
        B, D1, D2, F = z.shape
        dev = N.require_cuda(z)
        H = self.hidden_channels
        out = torch.empty((B, D2, D1, F) if swap else (B, D1, D2, F), dtype=torch.float32, device=dev)
        scratch = torch.empty(2 * B, dtype=torch.float64, device=dev)
        g, b = self.norm1d.norm.weight, self.norm1d.norm.bias
        if NATIVE_LSTM and N.ctn_bilstm_supported(F, H, F):
            r = self.rnn
            ptrs = (N._fp * 8)(*[t.data_ptr() for t in (r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0, r.weight_ih_l0_reverse,
                                                         r.weight_hh_l0_reverse, r.bias_ih_l0_reverse, r.bias_hh_l0_reverse)])
            nws = N.ctn_bilstm_workspace_bytes(F, H, F)
            ws = torch.empty(nws, dtype=torch.uint8, device=dev)
            P = torch.empty((2, B, D1, D2, F), dtype=torch.float32, device=dev)
            amax = torch.empty(1, dtype=torch.int32, device=dev)
            N.check(N.ctn_bilstm_proj_fwd(z.data_ptr(), B * D1, D2, F, H, ptrs, self.fc.weight.data_ptr(), F, P.data_ptr(), None,
                                          N.ptr(z_absmax), ws.data_ptr(), nws, N.stream_ptr(dev)), "ctn_bilstm_proj_fwd")
            N.check(N.ctn_dprnn_norm_res2_fwd(P.data_ptr(), self.fc.bias.data_ptr(), z.data_ptr(), g.data_ptr(), b.data_ptr(), out.data_ptr(),
                                              B, D1, D2, F, float(self.eps), int(swap), scratch.data_ptr(), amax.data_ptr(), N.stream_ptr(dev)),
                    "ctn_dprnn_norm_res2_fwd")
            self.last_absmax = amax
            return out
        self.last_absmax = None
        self.rnn.flatten_parameters()
        with _rnn_precision():
            y, _ = self.rnn(z.view(B * D1, D2, F))              # cuDNN bi-LSTM over D2, IEEE fp32 math
        y = F_.linear(y, self.fc.weight, self.fc.bias)           # (B*D1, D2, F)
        N.check(ctn_dprnn_norm_res_fwd(y.data_ptr(), z.data_ptr(), g.data_ptr(), b.data_ptr(), out.data_ptr(), B, D1, D2, F,
                                       float(self.eps), int(swap), scratch.data_ptr(), N.stream_ptr(dev)), "ctn_dprnn_norm_res_fwd")
        return out


class IntraChunkRNN(_ChunkRNN):
    def __init__(self, num_features, hidden_channels, norm=True, rnn_type='lstm', eps=EPS):
        super().__init__(num_features, hidden_channels, causal_rnn=False, norm=norm, rnn_type=rnn_type, eps=eps)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size) -- the reference layout (dprnn.py:70-94)"""
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("the DPRNN path is forward-only: call under torch.no_grad()")
        z = input.permute(0, 2, 3, 1).contiguous()
        return self._step(z, swap=False).permute(0, 3, 1, 2).contiguous()


class InterChunkRNN(_ChunkRNN):
    def __init__(self, num_features, hidden_channels, causal, norm=True, rnn_type='lstm', eps=EPS):
        super().__init__(num_features, hidden_channels, causal_rnn=causal, norm=norm, rnn_type=rnn_type, eps=eps)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size) (dprnn.py:122-148)"""
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("the DPRNN path is forward-only: call under torch.no_grad()")
        z = input.permute(0, 3, 2, 1).contiguous()             # (B, K, S, F)
        return self._step(z, swap=False).permute(0, 3, 2, 1).contiguous()


class DPRNNBlock(nn.Module):
    def __init__(self, num_features, hidden_channels, causal, norm=True, rnn_type='lstm', eps=EPS):
        super().__init__()
        self.intra_chunk_block = IntraChunkRNN(num_features, hidden_channels, norm=norm, rnn_type=rnn_type, eps=eps)
        self.inter_chunk_block = InterChunkRNN(num_features, hidden_channels, norm=norm, causal=causal, rnn_type=rnn_type, eps=eps)

    def forward(self, input):
        return self.inter_chunk_block(self.intra_chunk_block(input))

    def forward_channels_last(self, z, z_absmax=None):
        """z (B, S, K, F) -> (B, S, K, F): intra (swap to (B, K, S, F)), inter (swap back).  max|z| travels along as a device word
        (each gLN + residual kernel leaves it for the next LSTM's operand scale)."""
        y = self.intra_chunk_block._step(z, swap=True, z_absmax=z_absmax)
        y = self.inter_chunk_block._step(y, swap=True, z_absmax=self.intra_chunk_block.last_absmax)
        self.last_absmax = self.inter_chunk_block.last_absmax
        return y


class DPRNN(nn.Module):
    def __init__(self, num_features, hidden_channels, num_blocks=6, norm=True, causal=False, rnn_type='lstm', eps=EPS):
        super().__init__()
        self.net = nn.Sequential(*[DPRNNBlock(num_features, hidden_channels, norm=norm, causal=causal, rnn_type=rnn_type, eps=eps)
                                   for _ in range(num_blocks)])

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        if torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise NotImplementedError("the DPRNN path is forward-only: call under torch.no_grad()")
        z = input.permute(0, 2, 3, 1).contiguous()
        return self.forward_channels_last(z).permute(0, 3, 1, 2).contiguous()

    def forward_channels_last(self, z):
        amax = None
        for blk in self.net:
            z = blk.forward_channels_last(z, amax)
            amax = blk.last_absmax
        return z
