"""GALRNet behind the reference's class API (src/models/galrnet.py:13-250).

Same constructor, module tree, ``state_dict`` keys, ``get_config`` and ``num_parameters`` as the reference, so a checkpoint the
recipe's trainer saves (its ``get_config()`` plus ``'state_dict'``) loads with ``GALRNet(**config)`` and
``load_state_dict(strict=True)``.  Forward = encoder kernel -> pad + Segment1d (channels-last) + gLN over the segmented tensor
(``ctn_dpt_head_fwd`` without a bottleneck) -> N x GALRBlock (models/galr.py) -> OverlapAdd1d + crop -> PReLU + map 1x1 + GTU1d +
mask nonlinearity + w * mask + transposed-conv decoder (``ctn_dpt_tail_fwd`` with the bottleneck width equal to n_basis).
Envelope: trainable bases, monaural 3-D input, non-causal, sep_norm=True, low_dimension=True, mask 'relu' or 'sigmoid', the GALR
blocks' sizes (models/galr.py); forward only, dropout only in eval mode.
"""
import torch
import torch.nn as nn

from .. import _native as N
from ..utils.filterbank import choose_filterbank
from ..utils.model import choose_nonlinear
from ..utils.tasnet import choose_layer_norm
from ._dual_path import GTUTailModel, math_of, segment_geometry
from .galr import GALR
from .gtu import GTU1d
from .transform import Segment1d, OverlapAdd1d

EPS = 1e-12


class GALRNet(GTUTailModel):
    def __init__(self, n_basis, kernel_size, stride=None, enc_basis=None, dec_basis=None, sep_hidden_channels=128, sep_chunk_size=100,
                 sep_hop_size=50, sep_down_chunk_size=None, sep_num_blocks=6, sep_num_heads=8, sep_norm=True, sep_dropout=0.1,
                 mask_nonlinear='relu', causal=True, n_sources=2, low_dimension=True, eps=EPS, **kwargs):
        super().__init__()
        if stride is None:
            stride = kernel_size // 2
        assert kernel_size % stride == 0, "kernel_size is expected divisible by stride"
        if kwargs.get('in_channels', 1) != 1:
            raise NotImplementedError("multichannel GALRNet is outside the sm_90a path")
        if causal:
            raise NotImplementedError("causal GALRNet (cLN) is outside the sm_90a path: build it with causal=False (the reference's "
                                      "default is causal=True)")
        self.n_basis = n_basis
        self.kernel_size, self.stride = kernel_size, stride
        self.enc_basis, self.dec_basis = enc_basis, dec_basis
        self.enc_nonlinear = kwargs['enc_nonlinear'] if (enc_basis == 'trainable' and dec_basis != 'pinv') else None
        self.window_fn, self.enc_onesided, self.enc_return_complex = None, None, None
        self.sep_hidden_channels = sep_hidden_channels
        self.sep_chunk_size, self.sep_hop_size, self.sep_down_chunk_size = sep_chunk_size, sep_hop_size, sep_down_chunk_size
        self.sep_num_blocks, self.sep_num_heads = sep_num_blocks, sep_num_heads
        self.sep_norm, self.sep_dropout = sep_norm, sep_dropout
        self.low_dimension = low_dimension
        self.causal, self.mask_nonlinear = causal, mask_nonlinear
        self.n_sources, self.eps = n_sources, eps
        encoder, decoder = choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis, dec_basis=dec_basis, **kwargs)
        self.encoder = encoder
        self.separator = Separator(n_basis, hidden_channels=sep_hidden_channels, chunk_size=sep_chunk_size, hop_size=sep_hop_size,
                                   down_chunk_size=sep_down_chunk_size, num_blocks=sep_num_blocks, num_heads=sep_num_heads, norm=sep_norm,
                                   dropout=sep_dropout, mask_nonlinear=mask_nonlinear, low_dimension=low_dimension, causal=causal,
                                   n_sources=n_sources, eps=eps)
        self.decoder = decoder
        self.math = None

    def get_config(self):
        return {
            'n_basis': self.n_basis, 'kernel_size': self.kernel_size, 'stride': self.stride, 'enc_basis': self.enc_basis,
            'dec_basis': self.dec_basis, 'enc_nonlinear': self.enc_nonlinear, 'window_fn': self.window_fn,
            'enc_onesided': self.enc_onesided, 'enc_return_complex': self.enc_return_complex,
            'sep_hidden_channels': self.sep_hidden_channels, 'sep_chunk_size': self.sep_chunk_size, 'sep_hop_size': self.sep_hop_size,
            'sep_down_chunk_size': self.sep_down_chunk_size, 'sep_num_blocks': self.sep_num_blocks, 'sep_num_heads': self.sep_num_heads,
            'sep_norm': self.sep_norm, 'sep_dropout': self.sep_dropout, 'low_dimension': self.low_dimension,
            'mask_nonlinear': self.mask_nonlinear, 'causal': self.causal, 'n_sources': self.n_sources, 'eps': self.eps,
        }


class Separator(nn.Module):
    def __init__(self, num_features, hidden_channels=128, chunk_size=100, hop_size=50, down_chunk_size=None, num_blocks=6, num_heads=4,
                 norm=True, dropout=0.1, mask_nonlinear='relu', low_dimension=True, causal=True, n_sources=2, eps=EPS):
        super().__init__()
        if causal:
            raise NotImplementedError("causal GALRNet (cLN) is outside the sm_90a path")
        if not norm:
            raise NotImplementedError("sep_norm=False is outside the sm_90a path")
        if not low_dimension:
            raise NotImplementedError("low_dimension=False is outside the sm_90a path")
        if mask_nonlinear == 'softmax':
            raise NotImplementedError("mask_nonlinear='softmax' is outside the sm_90a path")
        if mask_nonlinear not in ('relu', 'sigmoid'):
            raise ValueError("Cannot support {}".format(mask_nonlinear))
        if down_chunk_size is None:
            raise ValueError("Specify down_chunk_size")
        self.num_features, self.n_sources = num_features, n_sources
        self.chunk_size, self.hop_size = chunk_size, hop_size
        self.eps = eps
        self.segment1d = Segment1d(chunk_size, hop_size)
        self.norm2d = choose_layer_norm('gLN', num_features, causal=False, eps=eps)
        self.galr = GALR(num_features, hidden_channels, chunk_size=chunk_size, down_chunk_size=down_chunk_size, num_blocks=num_blocks,
                         num_heads=num_heads, norm=norm, dropout=dropout, low_dimension=low_dimension, causal=causal, eps=eps)
        self.overlap_add1d = OverlapAdd1d(chunk_size, hop_size)
        self.prelu = nn.PReLU()
        self.map = nn.Conv1d(num_features, n_sources * num_features, kernel_size=1, stride=1)
        self.gtu = GTU1d(num_features, num_features, kernel_size=1, stride=1)
        self.mask_nonlinear = choose_nonlinear(mask_nonlinear)
        self.mask_relu = mask_nonlinear == 'relu'
        self.math = None

    folds_gln = False

    def check(self, B, n_frames):
        """the padding rule of galrnet.py:233-235, and every GALR block's launch limits"""
        S = segment_geometry(n_frames, self.chunk_size, self.hop_size)[2]
        for blk in self.galr.net:
            blk.inter_chunk_block.check_shape((B, S, self.chunk_size, self.num_features))

    def run_pitched(self, w, stats0, frames, pitch, dev):
        """w (B, N, pitch) pitched encoder output -> y (B, N, pitch): everything between the encoder and the PReLU of galrnet.py:243"""
        B = w.shape[0]
        Nf, K, P = self.num_features, self.chunk_size, self.hop_size
        pl, pr, S = segment_geometry(frames, K, P)
        st = N.stream_ptr(dev)
        z = torch.empty(B, S, K, Nf, dtype=torch.float32, device=dev)
        nws = N.ctn_dpt_head_workspace_bytes(B, Nf, Nf, pitch, S, K)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="galr_head"))
        g, b = self.norm2d.norm.weight, self.norm2d.norm.bias
        N.check(N.ctn_dpt_head_fwd(w.data_ptr(), None, None, g.data_ptr(), b.data_ptr(), z.data_ptr(), B, Nf, Nf, frames, pitch, K, P, pl, pr,
                                   float(self.eps), math_of(self.math), base, nbytes, st), "ctn_dpt_head_fwd")
        z = self.galr.forward_channels_last(z)
        y = torch.empty(B, Nf, pitch, dtype=torch.float32, device=dev)
        N.check(N.ctn_overlap_add_fwd(z.data_ptr(), y.data_ptr(), B, Nf, S, K, P, pl, frames, pitch, 1, st), "ctn_overlap_add_fwd")
        return y

    def forward(self, input):
        """input (batch_size, num_features, n_frames) -> mask (batch_size, n_sources, num_features, n_frames)"""
        raise NotImplementedError("the stand-alone GALRNet Separator.forward (materialised mask) is not built; use GALRNet")
