"""DPRNN-TasNet (BASELINE cfg4) behind the reference's class API (src/models/dprnn_tasnet.py:15-351).

Same constructors, ``forward`` / ``extract_latent`` / ``get_config`` / ``build_model`` and the same ``state_dict`` keys as the
reference, so its checkpoints load with ``load_state_dict``.  Forward = encoder kernel (+ gLN statistics) -> gLN folded
into the bottleneck 1x1 (wgmma) -> pad + Segment1d straight into the channels-last dual-path layout -> B x (intra, inter)
blocks (cuDNN LSTM + library GEMM between native gLN / residual / layout-swap calls, see dprnn.py) -> OverlapAdd1d + crop ->
PReLU + mask 1x1 + sigmoid + w * mask (wgmma) -> transposed-conv decoder + crop.
Envelope: trainable bases, monaural 3-D input, non-causal, rnn_type='lstm', sigmoid mask; forward only.
"""
import ctypes as C

import torch
import torch.nn as nn

from .. import _native as N
from ..utils.filterbank import choose_filterbank
from ..utils.tasnet import choose_layer_norm
from ._dual_path import forward_only, math_of, segment_geometry
from .dprnn import DPRNN
from .transform import (Segment1d, OverlapAdd1d, ctn_segment_fwd, ctn_overlap_add_fwd, ctn_stage_workspace_bytes, ctn_sep_head_fwd,
                        ctn_sep_tail_fwd)

EPS = 1e-12


class Separator(nn.Module):
    def __init__(self, num_features, bottleneck_channels=64, hidden_channels=128, chunk_size=100, hop_size=50, num_blocks=6,
                 norm=True, mask_nonlinear='sigmoid', causal=True, rnn_type='lstm', n_sources=2, eps=EPS):
        super().__init__()
        self.num_features, self.n_sources = num_features, n_sources
        self.bottleneck_channels = bottleneck_channels
        self.chunk_size, self.hop_size = chunk_size, hop_size
        self.norm, self.eps = norm, eps
        if causal:
            raise NotImplementedError("causal DPRNN-TasNet (cLN, uni-directional inter-chunk LSTM) is outside the sm_90a path")
        self.norm1d = choose_layer_norm('gLN', num_features, causal=False, eps=eps)
        self.bottleneck_conv1d = nn.Conv1d(num_features, bottleneck_channels, kernel_size=1, stride=1)
        self.segment1d = Segment1d(chunk_size, hop_size)
        self.dprnn = DPRNN(bottleneck_channels, hidden_channels, num_blocks=num_blocks, causal=causal, norm=norm, rnn_type=rnn_type, eps=eps)
        self.overlap_add1d = OverlapAdd1d(chunk_size, hop_size)
        self.prelu = nn.PReLU()
        self.mask_conv1d = nn.Conv1d(bottleneck_channels, n_sources * num_features, kernel_size=1, stride=1)
        if mask_nonlinear == 'sigmoid':
            pass
        elif mask_nonlinear == 'softmax':
            raise NotImplementedError("mask_nonlinear='softmax' is outside the sm_90a kernel envelope")
        else:
            raise ValueError("Cannot support {}".format(mask_nonlinear))
        self.math = None

    def segment_geometry(self, n_frames):
        """padding rule of dprnn_tasnet.py:339-341 -> (pad_left, pad_right, S)"""
        return segment_geometry(n_frames, self.chunk_size, self.hop_size)

    def run_pitched(self, w, stats0, frames, pitch, dev):
        """w (B, N, pitch) pitched encoder output (+ its statistics) -> y (B, Bc, pitch): everything between the encoder and the
        PReLU of dprnn_tasnet.py:348."""
        B = w.shape[0]
        Nf, Bc, K, P = self.num_features, self.bottleneck_channels, self.chunk_size, self.hop_size
        ws_bytes = max(ctn_stage_workspace_bytes(Bc, Nf), ctn_stage_workspace_bytes(self.n_sources * Nf, Bc)) + 512
        base, nbytes = N.aligned(N.workspace(dev, ws_bytes, tag="dprnn_stage"))
        st = N.stream_ptr(dev)
        x0 = torch.empty(B, Bc, pitch, dtype=torch.float32, device=dev)
        g0, b0 = self.norm1d.norm.weight, self.norm1d.norm.bias
        N.check(ctn_sep_head_fwd(w.data_ptr(), stats0.data_ptr(), g0.data_ptr(), b0.data_ptr(), self.bottleneck_conv1d.weight.data_ptr(),
                                 self.bottleneck_conv1d.bias.data_ptr(), x0.data_ptr(), B, Nf, Bc, frames, pitch, float(self.eps), math_of(self.math),
                                 base, nbytes, st), "ctn_sep_head_fwd")
        pl, pr, S = self.segment_geometry(frames)
        z = torch.empty(B, S, K, Bc, dtype=torch.float32, device=dev)
        N.check(ctn_segment_fwd(x0.data_ptr(), z.data_ptr(), B, Bc, frames, pitch, K, P, pl, pr, 1, st), "ctn_segment_fwd")
        z = self.dprnn.forward_channels_last(z)
        y = x0  # reuse: (B, Bc, pitch)
        N.check(ctn_overlap_add_fwd(z.data_ptr(), y.data_ptr(), B, Bc, S, K, P, pl, frames, pitch, 1, st), "ctn_overlap_add_fwd")
        return y, (base, nbytes)

    def forward(self, input):
        """input (batch_size, num_features, n_frames) -> mask (batch_size, n_sources, num_features, n_frames)"""
        raise NotImplementedError("the stand-alone DPRNN Separator.forward (materialised mask) is not built; use DPRNNTasNet")


class DPRNNTasNet(nn.Module):
    def __init__(self, n_basis, kernel_size, stride=None, enc_basis=None, dec_basis=None, sep_hidden_channels=128,
                 sep_bottleneck_channels=64, sep_chunk_size=100, sep_hop_size=50, sep_num_blocks=6, sep_norm=True,
                 mask_nonlinear='sigmoid', causal=True, rnn_type='lstm', n_sources=2, eps=EPS, **kwargs):
        super().__init__()
        if stride is None:
            stride = kernel_size // 2
        assert kernel_size % stride == 0, "kernel_size is expected divisible by stride"
        self.in_channels = kwargs.get('in_channels', 1)
        self.n_basis, self.kernel_size, self.stride = n_basis, kernel_size, stride
        self.enc_basis, self.dec_basis = enc_basis, dec_basis
        self.enc_nonlinear = kwargs['enc_nonlinear'] if (enc_basis == 'trainable' and dec_basis != 'pinv') else None
        self.window_fn, self.enc_onesided, self.enc_return_complex = None, None, None
        self.sep_hidden_channels, self.sep_bottleneck_channels = sep_hidden_channels, sep_bottleneck_channels
        self.sep_chunk_size, self.sep_hop_size, self.sep_num_blocks = sep_chunk_size, sep_hop_size, sep_num_blocks
        self.causal, self.sep_norm, self.mask_nonlinear, self.rnn_type = causal, sep_norm, mask_nonlinear, rnn_type
        self.n_sources, self.eps = n_sources, eps
        encoder, decoder = choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis, dec_basis=dec_basis, **kwargs)
        self.encoder = encoder
        self.separator = Separator(n_basis, bottleneck_channels=sep_bottleneck_channels, hidden_channels=sep_hidden_channels,
                                   chunk_size=sep_chunk_size, hop_size=sep_hop_size, num_blocks=sep_num_blocks, norm=sep_norm,
                                   mask_nonlinear=mask_nonlinear, causal=causal, rnn_type=rnn_type, n_sources=n_sources, eps=eps)
        self.decoder = decoder
        self.math = None

    def forward(self, input):
        output, _ = self._run(input, want_latent=False)
        return output

    def extract_latent(self, input):
        """input (batch_size, 1, T) -> output (batch_size, n_sources, T), latent (batch_size, n_sources, n_basis, T')"""
        return self._run(input, want_latent=True)

    def _run(self, input, want_latent):
        n_dim = input.dim()
        if n_dim == 3:
            assert input.size(1) == 1, "input.size() is expected (?, 1, ?), but given {}".format(input.size())
        elif n_dim == 4:
            assert input.size(1) == 1, "input.size() is expected (?, 1, ?, ?), but given {}".format(input.size())
            raise NotImplementedError("multichannel (4-D) input is outside the sm_90a kernel envelope")
        else:
            raise ValueError("Not support {} dimension input".format(n_dim))
        forward_only(self, input)
        x = input.contiguous()
        B, _, T = x.shape
        if B > 65535:  # segmentation, overlap-add and the gLN + residual put the batch on a grid axis of at most 65535 blocks
            raise NotImplementedError("batch_size={} is outside the DPRNN-TasNet kernels' launch limit (batch_size <= 65535)".format(B))
        dev = N.require_cuda(x)
        sep = self.separator
        sep.math = self.math if self.math is not None else sep.math
        frames, pl, pr = N.frames_of(T, self.kernel_size, self.stride)
        pitch = N.ctn_pitch(frames)
        st = N.stream_ptr(dev)
        Nb, S = self.n_basis, self.n_sources
        w = torch.empty(B, Nb, pitch, dtype=torch.float32, device=dev)
        stats0 = torch.zeros(2 * B, dtype=torch.float64, device=dev)
        N.check(N.ctn_encoder_fwd(x.data_ptr(), self.encoder.conv1d.weight.data_ptr(), w.data_ptr(), B, T, pl, pr, Nb, self.kernel_size,
                                  self.stride, int(self.encoder.nonlinear), pitch, stats0.data_ptr(), st), "ctn_encoder_fwd")
        y, (base, ws_bytes) = sep.run_pitched(w, stats0, frames, pitch, dev)
        out = torch.empty(B, S, T, dtype=torch.float32, device=dev)
        latent = torch.empty(B, S, Nb, frames, dtype=torch.float32, device=dev) if want_latent else None
        what = torch.empty(B, S * Nb, pitch, dtype=torch.float32, device=dev)
        N.check(ctn_sep_tail_fwd(y.data_ptr(), w.data_ptr(), sep.prelu.weight.data_ptr(), sep.mask_conv1d.weight.data_ptr(),
                                 sep.mask_conv1d.bias.data_ptr(), self.decoder.conv_transpose1d.weight.data_ptr(), out.data_ptr(),
                                 N.ptr(latent), what.data_ptr(), B, Nb, sep.bottleneck_channels, S, frames, pitch, self.kernel_size,
                                 self.stride, pl, T, math_of(sep.math), base, ws_bytes, st), "ctn_sep_tail_fwd")
        return out, latent

    def get_config(self):
        return {
            'in_channels': self.in_channels, 'n_basis': self.n_basis, 'kernel_size': self.kernel_size, 'stride': self.stride,
            'enc_basis': self.enc_basis, 'dec_basis': self.dec_basis, 'enc_nonlinear': self.enc_nonlinear,
            'window_fn': self.window_fn, 'enc_onesided': self.enc_onesided, 'enc_return_complex': self.enc_return_complex,
            'sep_hidden_channels': self.sep_hidden_channels, 'sep_bottleneck_channels': self.sep_bottleneck_channels,
            'sep_chunk_size': self.sep_chunk_size, 'sep_hop_size': self.sep_hop_size, 'sep_num_blocks': self.sep_num_blocks,
            'causal': self.causal, 'sep_norm': self.sep_norm, 'mask_nonlinear': self.mask_nonlinear, 'rnn_type': self.rnn_type,
            'n_sources': self.n_sources, 'eps': self.eps,
        }

    @classmethod
    def build_model(cls, model_path, load_state_dict=False):
        """dprnn_tasnet.py:181-221 (legacy keys n_bases / enc_bases / dec_bases tolerated)"""
        config = torch.load(model_path, map_location=lambda storage, loc: storage, weights_only=False)
        get = config.get
        model = cls(
            get('n_bases') or config['n_basis'], in_channels=get('in_channels') or 1, kernel_size=config['kernel_size'],
            stride=config['stride'], enc_basis=get('enc_bases') or config['enc_basis'], dec_basis=get('dec_bases') or config['dec_basis'],
            enc_nonlinear=config['enc_nonlinear'], window_fn=config['window_fn'], enc_onesided=get('enc_onesided') or None,
            enc_return_complex=get('enc_return_complex') or None, sep_hidden_channels=config['sep_hidden_channels'],
            sep_bottleneck_channels=config['sep_bottleneck_channels'], sep_chunk_size=config['sep_chunk_size'],
            sep_hop_size=config['sep_hop_size'], sep_num_blocks=config['sep_num_blocks'], sep_norm=config['sep_norm'],
            mask_nonlinear=config['mask_nonlinear'], causal=config['causal'], rnn_type=get('rnn_type') or 'lstm',
            n_sources=config['n_sources'], eps=config['eps'])
        if load_state_dict:
            model.load_state_dict(config['state_dict'])
        return model

    @property
    def num_parameters(self):
        return sum(p.numel() for p in self.parameters() if p.requires_grad)
