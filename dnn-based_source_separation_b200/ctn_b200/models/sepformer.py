"""SepFormer behind the reference's class API (src/models/sepformer.py:16-556).

Same constructors, module tree and ``state_dict`` keys as the reference (torch's own ``nn.TransformerEncoder`` /
``nn.TransformerEncoderLayer`` hold the layer parameters), so its checkpoints load with ``load_state_dict(strict=True)``.
Forward = encoder kernel (+ the gLN statistics of w) -> gLN + bottleneck_conv1d_in (``ctn_sep_head_fwd``) -> pad + Segment1d
into the pitched channel-first state (``ctn_segment_fwd`` with a row pitch) -> per SepFormerBlock one IntraTransformer and one
InterTransformer (``ctn_sfm_transformer_fwd`` each) -> OverlapAdd1d + crop (``ctn_overlap_add_fwd``) -> PReLU, map, GTU1d,
bottleneck_conv1d_out, mask nonlinearity, w * mask and the transposed-conv decoder (``ctn_dpt_tail_fwd`` with
bottleneck_conv1d_out).

The dual-path state stays (B, F, pitch) with token s*C + k for chunk s and frame k (csrc/ctn_sepformer.cu): the four Linear
layers of every encoder layer are ctn_pw contractions in the model's numeric mode, and the two paths differ only in the token
stride of their sequences.  As in the reference, each encoder's input is x + PositionalEncoding(x) = 2x + pe, and its outer
residual is the block input itself.
Envelope: trainable bases, monaural 3-D input, causal=False, sep_norm=True, sep_nonlinear='relu', mask 'relu' or 'sigmoid',
head dimensions F / heads in {8, 16, 32, 64} for the intra and the inter heads; forward only (sep_dropout acts as in eval()).
"""
import torch
import torch.nn as nn

from .. import _native as N
from ..utils.filterbank import choose_filterbank
from ..utils.model import choose_nonlinear
from ..utils.tasnet import choose_layer_norm
from ._dual_path import GTUTailModel, build_from_pretrained, eval_dropout, forward_only, math_of, segment_geometry
from .conv_tasnet import _load_checkpoint
from .gtu import GTU1d
from .transform import Segment1d, OverlapAdd1d
from .transformer import PositionalEncoding

EPS = 1e-12
PE_ROWS = 5000  # rows of PositionalEncoding's buffer (transformer.py:8): the longest sequence either path can take


class LayerNormWrapper(nn.Module):
    """the encoder's final norm (sepformer.py:522-556): gLN over each sequence; runs inside ctn_sfm_transformer_fwd"""

    def __init__(self, norm_name, num_features, causal=False, batch_first=False, eps=EPS):
        super().__init__()
        if norm_name != 'gLN':
            raise NotImplementedError("norm {!r} is outside the sm_90a SepFormer path ('gLN' only)".format(norm_name))
        self.batch_first = batch_first
        self.norm1d = choose_layer_norm(norm_name, num_features, causal=causal, eps=eps)

    def forward(self, input):
        raise NotImplementedError("the stand-alone LayerNormWrapper.forward is not built; it runs inside IntraTransformer / "
                                  "InterTransformer")


class _PathTransformer(nn.Module):
    """common body of IntraTransformer / InterTransformer (sepformer.py:438-520)"""
    intra = None

    def __init__(self, num_features, num_layers, num_heads, d_ff, norm, nonlinear, dropout, causal, norm_first, eps):
        super().__init__()
        if causal:
            raise NotImplementedError("causal SepFormer (cLN) is outside the sm_90a path: pass causal=False")
        if norm is not True and norm != 1:
            raise NotImplementedError("norm={!r} is outside the sm_90a path (sep_norm=True only)".format(norm))
        if norm_first:
            raise NotImplementedError("norm_first=True (pre-norm) is outside the sm_90a path")
        if nonlinear != 'relu':
            raise NotImplementedError("sep_nonlinear={!r} is outside the sm_90a path ('relu' only)".format(nonlinear))
        if not N.ctn_sfm_attn_supported(num_features, num_heads):
            raise NotImplementedError("num_features={} with num_heads={} is outside the attention kernel's envelope (head dimension "
                                      "in 8, 16, 32, 64)".format(num_features, num_heads))
        self.num_features = num_features
        self.num_layers, self.num_heads, self.d_ff, self.eps, self.dropout_p = num_layers, num_heads, d_ff, eps, dropout
        layer_norm = LayerNormWrapper('gLN', num_features, causal=False, batch_first=False, eps=eps)
        self.positional_encoding = PositionalEncoding(num_features, batch_first=False)
        encoder_layer = nn.TransformerEncoderLayer(num_features, num_heads, d_ff, dropout=dropout, activation=nonlinear,
                                                   layer_norm_eps=eps, batch_first=False, norm_first=norm_first)
        self.transformer = nn.TransformerEncoder(encoder_layer, num_layers=num_layers, norm=layer_norm, enable_nested_tensor=False)

    def weight_ptrs(self):
        """the host pointer array ctn_sfm_transformer_fwd takes: 12 per layer, then the encoding and the final gLN"""
        ts = []
        for layer in self.transformer.layers:
            a = layer.self_attn
            ts += [a.in_proj_weight, a.in_proj_bias, a.out_proj.weight, a.out_proj.bias, layer.linear1.weight, layer.linear1.bias,
                   layer.linear2.weight, layer.linear2.bias, layer.norm1.weight, layer.norm1.bias, layer.norm2.weight, layer.norm2.bias]
        g = self.transformer.norm.norm1d.norm
        ts += [self.positional_encoding.positional_encoding, g.weight, g.bias]
        for t in ts:
            if not t.is_contiguous():
                raise ValueError("SepFormer parameters must be contiguous")
        return (N._fp * len(ts))(*[t.data_ptr() for t in ts])

    def run_pitched(self, z, S, C, math):
        """z (B, F, pitch) pitched state, token s*C + k -> a new (B, F, pitch) tensor"""
        eval_dropout(self, self.dropout_p)
        B, F, pitch = z.shape
        dev = N.require_cuda(z)
        out = torch.empty_like(z)
        nws = N.ctn_sfm_transformer_workspace_bytes(B, F, self.d_ff, self.num_layers, pitch, math)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="sfm_transformer"))
        N.check(N.ctn_sfm_transformer_fwd(z.data_ptr(), out.data_ptr(), self.weight_ptrs(), B, F, self.num_heads, self.d_ff,
                                          self.num_layers, S, C, pitch, int(self.intra), float(self.eps), math, base, nbytes,
                                          N.stream_ptr(dev)), "ctn_sfm_transformer_fwd")
        return out

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return _on_pitched(lambda z, S, C: self.run_pitched(z, S, C, math_of(None)), input)


def _on_pitched(fn, input):
    """run fn on the pitched copy of a (B, F, S, C) tensor and return the (B, F, S, C) result"""
    B, F, S, C = input.shape
    _check_lengths(S, C)
    N.require_cuda(input)
    z = torch.zeros(B, F, N.ctn_pitch(S * C), dtype=torch.float32, device=input.device)
    z[:, :, :S * C] = input.reshape(B, F, S * C)
    return fn(z, S, C)[:, :, :S * C].reshape(B, F, S, C)


def _check_lengths(S, C):
    if S > PE_ROWS or C > PE_ROWS:
        raise ValueError("{} chunks of {} frames: the positional encoding has {} rows, so neither may exceed it".format(S, C, PE_ROWS))


class IntraTransformer(_PathTransformer):
    intra = True

    def __init__(self, num_features, num_layers=8, num_heads=8, d_ff=1024, norm=True, nonlinear='relu', dropout=1e-1, norm_first=False,
                 eps=EPS):
        super().__init__(num_features, num_layers, num_heads, d_ff, norm, nonlinear, dropout, False, norm_first, eps)


class InterTransformer(_PathTransformer):
    intra = False

    def __init__(self, num_features, num_layers=8, num_heads=8, d_ff=1024, norm=True, nonlinear='relu', dropout=1e-1, causal=False,
                 norm_first=False, eps=EPS):
        super().__init__(num_features, num_layers, num_heads, d_ff, norm, nonlinear, dropout, causal, norm_first, eps)


class SepFormerBlock(nn.Module):
    def __init__(self, num_layers_intra=8, num_layers_inter=8, num_heads_intra=8, num_heads_inter=8, d_intra=256, d_inter=256,
                 d_ff_intra=1024, d_ff_inter=1024, norm=True, dropout=1e-1, nonlinear='relu', causal=False, eps=EPS):
        super().__init__()
        if d_intra != d_inter:
            raise NotImplementedError("d_intra != d_inter is outside the sm_90a path")
        self.intra_transformer = IntraTransformer(d_intra, num_layers=num_layers_intra, num_heads=num_heads_intra, d_ff=d_ff_intra,
                                                  norm=norm, dropout=dropout, nonlinear=nonlinear, eps=eps)
        self.inter_transformer = InterTransformer(d_inter, num_layers=num_layers_inter, num_heads=num_heads_inter, d_ff=d_ff_inter,
                                                  norm=norm, dropout=dropout, nonlinear=nonlinear, causal=causal, eps=eps)

    def run_pitched(self, z, S, C, math):
        return self.inter_transformer.run_pitched(self.intra_transformer.run_pitched(z, S, C, math), S, C, math)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return _on_pitched(lambda z, S, C: self.run_pitched(z, S, C, math_of(None)), input)


class SepFormerBackbone(nn.Module):
    def __init__(self, num_blocks=2, num_layers_intra=8, num_layers_inter=8, num_heads_intra=8, num_heads_inter=8, d_intra=256,
                 d_inter=256, d_ff_intra=1024, d_ff_inter=1024, norm=True, dropout=1e-1, nonlinear='relu', causal=False, eps=EPS):
        super().__init__()
        self.net = nn.Sequential(*[SepFormerBlock(num_layers_intra=num_layers_intra, num_layers_inter=num_layers_inter,
                                                  num_heads_intra=num_heads_intra, num_heads_inter=num_heads_inter, d_intra=d_intra,
                                                  d_inter=d_inter, d_ff_intra=d_ff_intra, d_ff_inter=d_ff_inter, norm=norm,
                                                  dropout=dropout, nonlinear=nonlinear, causal=causal, eps=eps)
                                   for _ in range(num_blocks)])

    def run_pitched(self, z, S, C, math):
        for blk in self.net:
            z = blk.run_pitched(z, S, C, math)
        return z

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return _on_pitched(lambda z, S, C: self.run_pitched(z, S, C, math_of(None)), input)


class Separator(nn.Module):
    def __init__(self, num_features, bottleneck_channels, chunk_size=250, hop_size=125, num_blocks=2, num_layers_intra=8,
                 num_layers_inter=8, num_heads_intra=8, num_heads_inter=8, d_ff_intra=1024, d_ff_inter=1024, norm=True,
                 nonlinear='relu', dropout=1e-1, mask_nonlinear='relu', causal=False, n_sources=2, eps=EPS):
        super().__init__()
        if causal:
            raise NotImplementedError("causal SepFormer (cLN) is outside the sm_90a path: pass causal=False")
        if mask_nonlinear == 'softmax':
            raise NotImplementedError("mask_nonlinear='softmax' is outside the sm_90a path")
        if mask_nonlinear not in ('relu', 'sigmoid'):
            raise ValueError("Cannot support {}".format(mask_nonlinear))
        self.num_features, self.n_sources = num_features, n_sources
        self.bottleneck_channels = bottleneck_channels
        self.chunk_size, self.hop_size = chunk_size, hop_size
        self.norm = norm
        self.eps = eps
        self.norm1d = choose_layer_norm('gLN', num_features, causal=False, eps=eps)
        self.bottleneck_conv1d_in = nn.Conv1d(num_features, bottleneck_channels, kernel_size=1, stride=1)
        self.segment1d = Segment1d(chunk_size, hop_size)
        self.dptransformer = SepFormerBackbone(num_blocks=num_blocks, num_layers_intra=num_layers_intra, num_layers_inter=num_layers_inter,
                                               num_heads_intra=num_heads_intra, num_heads_inter=num_heads_inter, d_intra=bottleneck_channels,
                                               d_inter=bottleneck_channels, d_ff_intra=d_ff_intra, d_ff_inter=d_ff_inter, norm=norm,
                                               dropout=dropout, nonlinear=nonlinear, causal=causal, eps=eps)
        self.overlap_add1d = OverlapAdd1d(chunk_size, hop_size)
        self.prelu = nn.PReLU()
        self.map = nn.Conv1d(bottleneck_channels, n_sources * num_features, kernel_size=1, stride=1)
        self.gtu = GTU1d(num_features, num_features, kernel_size=1, stride=1)
        self.bottleneck_conv1d_out = nn.Conv1d(num_features, num_features, kernel_size=1, stride=1)
        self.mask_nonlinear = choose_nonlinear(mask_nonlinear)
        self.mask_relu = mask_nonlinear == 'relu'
        self.math = None

    folds_gln = True

    def check(self, B, n_frames):
        """the padding rule of sepformer.py:342-344, and sequences within the positional encoding's rows"""
        _check_lengths(segment_geometry(n_frames, self.chunk_size, self.hop_size)[2], self.chunk_size)

    def run_pitched(self, w, stats0, frames, pitch, dev):
        """w (B, N, pitch) pitched encoder output (+ its statistics) -> y (B, Bc, pitch): everything between the encoder and the
        PReLU of sepformer.py:353"""
        B = w.shape[0]
        Nf, Bc, K, P = self.num_features, self.bottleneck_channels, self.chunk_size, self.hop_size
        pl, pr, S = segment_geometry(frames, K, P)
        math = math_of(self.math)
        st = N.stream_ptr(dev)
        base, nbytes = N.aligned(N.workspace(dev, N.ctn_stage_workspace_bytes(Bc, Nf) + 256, tag="sfm_head"))
        x0 = torch.empty(B, Bc, pitch, dtype=torch.float32, device=dev)
        g0, b0 = self.norm1d.norm.weight, self.norm1d.norm.bias
        N.check(N.ctn_sep_head_fwd(w.data_ptr(), stats0.data_ptr(), g0.data_ptr(), b0.data_ptr(), self.bottleneck_conv1d_in.weight.data_ptr(),
                                   self.bottleneck_conv1d_in.bias.data_ptr(), x0.data_ptr(), B, Nf, Bc, frames, pitch, float(self.eps), math,
                                   base, nbytes, st), "ctn_sep_head_fwd")
        zp = N.ctn_pitch(S * K)
        z = torch.empty(B, Bc, zp, dtype=torch.float32, device=dev)
        N.check(N.ctn_segment_fwd(x0.data_ptr(), z.data_ptr(), B, Bc, frames, pitch, K, P, pl, pr, zp, st), "ctn_segment_fwd")
        z = self.dptransformer.run_pitched(z, S, K, math)
        y = torch.empty(B, Bc, pitch, dtype=torch.float32, device=dev)
        N.check(N.ctn_overlap_add_fwd(z.data_ptr(), y.data_ptr(), B, Bc, S, K, P, pl, frames, pitch, zp, st), "ctn_overlap_add_fwd")
        return y

    def forward(self, input):
        """input (batch_size, num_features, n_frames) -> mask (batch_size, n_sources, num_features, n_frames)"""
        raise NotImplementedError("the stand-alone SepFormer Separator.forward (materialised mask) is not built; use SepFormer")


class SepFormer(GTUTailModel):
    pretrained_model_ids = {
        "wsj0-mix": {
            8000: {
                2: "1-9pOv2B612IykvpA6kaGZSg4AUQPnoCg",
                3: "1-Rz31CGWVVzYVHXgIdp7Tuc0__K2SCPs"
            }
        }
    }

    def __init__(self, n_basis, kernel_size, stride=None, enc_basis=None, dec_basis=None, sep_bottleneck_channels=None, sep_chunk_size=250,
                 sep_hop_size=125, sep_num_blocks=2, sep_num_layers_intra=8, sep_num_layers_inter=8, sep_num_heads_intra=8,
                 sep_num_heads_inter=8, sep_d_ff_intra=1024, sep_d_ff_inter=1024, sep_norm=True, sep_nonlinear='relu', sep_dropout=1e-1,
                 mask_nonlinear='relu', causal=True, n_sources=2, eps=EPS, **kwargs):
        super().__init__()
        if stride is None:
            stride = kernel_size // 2
        assert kernel_size % stride == 0, "kernel_size is expected divisible by stride"
        if causal:
            raise NotImplementedError("causal=True (the reference's default: cLN in the inter path) is outside the sm_90a SepFormer "
                                      "path; construct with causal=False")
        self.in_channels = kwargs.get('in_channels', 1)
        if self.in_channels != 1:
            raise NotImplementedError("multichannel SepFormer is outside the sm_90a path")
        self.n_basis = n_basis
        self.kernel_size, self.stride = kernel_size, stride
        self.enc_basis, self.dec_basis = enc_basis, dec_basis
        self.enc_nonlinear = kwargs['enc_nonlinear'] if (enc_basis == 'trainable' and dec_basis != 'pinv') else None
        if enc_basis in ['Fourier', 'trainableFourier', 'trainableFourierTrainablePhase'] or \
                dec_basis in ['Fourier', 'trainableFourier', 'trainableFourierTrainablePhase']:
            self.window_fn = kwargs['window_fn']
            self.enc_onesided, self.enc_return_complex = kwargs['enc_onesided'], kwargs['enc_return_complex']
        else:
            self.window_fn = None
            self.enc_onesided, self.enc_return_complex = None, None
        if sep_bottleneck_channels is None:
            sep_bottleneck_channels = n_basis
        self.sep_bottleneck_channels = sep_bottleneck_channels
        self.sep_chunk_size, self.sep_hop_size = sep_chunk_size, sep_hop_size
        self.sep_num_blocks = sep_num_blocks
        self.sep_num_layers_intra, self.sep_num_layers_inter = sep_num_layers_intra, sep_num_layers_inter
        self.sep_num_heads_intra, self.sep_num_heads_inter = sep_num_heads_intra, sep_num_heads_inter
        self.sep_d_ff_intra, self.sep_d_ff_inter = sep_d_ff_intra, sep_d_ff_inter
        self.causal = causal
        self.sep_norm, self.sep_dropout = sep_norm, sep_dropout
        self.sep_nonlinear, self.mask_nonlinear = sep_nonlinear, mask_nonlinear
        self.n_sources = n_sources
        self.eps = eps
        encoder, decoder = choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis, dec_basis=dec_basis, **kwargs)
        self.encoder = encoder
        self.separator = Separator(n_basis, sep_bottleneck_channels, chunk_size=sep_chunk_size, hop_size=sep_hop_size,
                                   num_blocks=sep_num_blocks, num_layers_intra=sep_num_layers_intra, num_layers_inter=sep_num_layers_inter,
                                   num_heads_intra=sep_num_heads_intra, num_heads_inter=sep_num_heads_inter, d_ff_intra=sep_d_ff_intra,
                                   d_ff_inter=sep_d_ff_inter, norm=sep_norm, nonlinear=sep_nonlinear, dropout=sep_dropout,
                                   mask_nonlinear=mask_nonlinear, causal=causal, n_sources=n_sources, eps=eps)
        self.decoder = decoder
        self.math = None

    def get_config(self):
        return {
            'in_channels': self.in_channels, 'n_basis': self.n_basis, 'kernel_size': self.kernel_size, 'stride': self.stride,
            'enc_basis': self.enc_basis, 'dec_basis': self.dec_basis, 'enc_nonlinear': self.enc_nonlinear,
            'enc_onesided': self.enc_onesided, 'enc_return_complex': self.enc_return_complex, 'window_fn': self.window_fn,
            'sep_bottleneck_channels': self.sep_bottleneck_channels, 'sep_chunk_size': self.sep_chunk_size,
            'sep_hop_size': self.sep_hop_size, 'sep_num_blocks': self.sep_num_blocks,
            'sep_num_layers_intra': self.sep_num_layers_intra, 'sep_num_layers_inter': self.sep_num_layers_inter,
            'sep_num_heads_intra': self.sep_num_heads_intra, 'sep_num_heads_inter': self.sep_num_heads_inter,
            'sep_d_ff_intra': self.sep_d_ff_intra, 'sep_d_ff_inter': self.sep_d_ff_inter, 'sep_norm': self.sep_norm,
            'sep_nonlinear': self.sep_nonlinear, 'sep_dropout': self.sep_dropout, 'mask_nonlinear': self.mask_nonlinear,
            'causal': self.causal, 'n_sources': self.n_sources, 'eps': self.eps,
        }

    @classmethod
    def build_model(cls, model_path, load_state_dict=False):
        """sepformer.py:180-227"""
        c = _load_checkpoint(model_path)
        model = cls(
            c['n_basis'], in_channels=c['in_channels'], kernel_size=c['kernel_size'], stride=c['stride'], enc_basis=c['enc_basis'],
            dec_basis=c['dec_basis'], enc_nonlinear=c['enc_nonlinear'], window_fn=c['window_fn'], enc_onesided=c['enc_onesided'],
            enc_return_complex=c['enc_return_complex'], sep_bottleneck_channels=c['sep_bottleneck_channels'],
            sep_chunk_size=c['sep_chunk_size'], sep_hop_size=c['sep_hop_size'], sep_num_blocks=c['sep_num_blocks'],
            sep_num_layers_intra=c['sep_num_layers_intra'], sep_num_layers_inter=c['sep_num_layers_inter'],
            sep_num_heads_intra=c['sep_num_heads_intra'], sep_num_heads_inter=c['sep_num_heads_inter'],
            sep_d_ff_intra=c['sep_d_ff_intra'], sep_d_ff_inter=c['sep_d_ff_inter'], sep_norm=c['sep_norm'],
            sep_nonlinear=c['sep_nonlinear'], sep_dropout=c['sep_dropout'], mask_nonlinear=c['mask_nonlinear'], causal=c['causal'],
            n_sources=c['n_sources'], eps=c['eps'])
        if load_state_dict:
            model.load_state_dict(c['state_dict'])
        return model

    @classmethod
    def build_from_pretrained(cls, root="./pretrained", quiet=False, load_state_dict=True, **kwargs):
        """sepformer.py:229-269: <root>/SepFormer/wsj0-mix/sr<rate>/<n>speakers/model/<choice>.pth, loaded, never downloaded"""
        return build_from_pretrained(cls, root, load_state_dict, **kwargs)
