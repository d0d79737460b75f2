"""DPTNet (dual-path transformer network) behind the reference's class API (src/models/dptnet.py:15-572).

Same constructors, module tree and ``state_dict`` keys as the reference, so its checkpoints load with ``load_state_dict``.
Forward = encoder kernel -> bottleneck 1x1 + pad + Segment1d (channels-last) + gLN over the segmented tensor
(``ctn_dpt_head_fwd``) -> B x (intra, inter) ImprovedTransformer -> OverlapAdd1d + crop -> PReLU + map 1x1 + GTU1d + mask
nonlinearity + w * mask + transposed-conv decoder (``ctn_dpt_tail_fwd``).  Each ImprovedTransformer is
  * MultiheadAttentionBlock: ``ctn_mha_fwd`` (QKV projection, online-softmax attention, output projection), then
    ``ctn_seq_norm_fwd``: GroupNorm(1, F) per SEQUENCE of x + MHA(x);
  * FeedForwardBlock: ``ctn_bilstm_relu_proj_fwd`` (bi-LSTM on wgmma with the Linear fused, ReLU on its operand), then
    ``ctn_seq_norm_fwd`` of x + fc(ReLU(LSTM(x))), stored with the intra <-> inter swap.
The dual-path state stays channels-last, (batch, D1, D2, F), as on the DPRNN-TasNet path (csrc/ctn_dptnet.cu).
Envelope: trainable bases, monaural 3-D input, non-causal, sep_norm=True, sep_nonlinear='relu', mask 'relu' or 'sigmoid',
num_features and hidden_channels inside the native LSTM's sizes, head dimension F / heads in {8, 16, 32, 64}; forward only.
"""
import torch
import torch.nn as nn

from .. import _native as N
from ..utils.filterbank import choose_filterbank
from ..utils.model import choose_nonlinear
from ..utils.tasnet import choose_layer_norm
from ._dual_path import GTUTailModel, build_from_pretrained, eval_dropout, forward_only, math_of, segment_geometry
from .conv_tasnet import _load_checkpoint
from .dprnn import choose_rnn
from .gtu import GTU1d
from .transform import Segment1d, OverlapAdd1d

EPS = 1e-12


class MultiheadAttentionBlock(nn.Module):
    def __init__(self, embed_dim, num_heads, norm=True, dropout=0, causal=False, eps=EPS):
        super().__init__()
        if causal:
            raise NotImplementedError("causal DPTNet (cLN) is outside the sm_90a path")
        if not norm:
            raise NotImplementedError("norm=False is outside the sm_90a path")
        if not N.ctn_mha_supported(embed_dim, num_heads):
            raise NotImplementedError("embed_dim={} with num_heads={} is outside the attention kernel's envelope (embed_dim <= 128, "
                                      "head dimension in 8, 16, 32, 64)".format(embed_dim, num_heads))
        self.dropout = dropout != 0
        self.dropout_p = dropout
        self.norm = norm
        self.num_heads, self.eps = num_heads, eps
        self.multihead_attn = nn.MultiheadAttention(embed_dim, num_heads)
        if self.dropout:
            self.dropout1d = nn.Dropout(p=dropout)
        self.norm1d = choose_layer_norm('gLN', embed_dim, causal=False, eps=eps)

    def forward(self, input):
        """input, output (T, batch_size, embed_dim) (dptnet.py:502-525)"""
        forward_only(self, input)
        return self._step(input.permute(1, 0, 2).unsqueeze(0).contiguous(), False)[0].permute(1, 0, 2).contiguous()

    def _step(self, z, swap):
        """z (B, D1, D2, F) channels-last -> GroupNorm over each (b, d1) sequence of z + MHA(z), (B, D2, D1, F) when swap"""
        eval_dropout(self, self.dropout_p)
        B, D1, D2, F = z.shape
        dev = N.require_cuda(z)
        st = N.stream_ptr(dev)
        a = self.multihead_attn
        y = torch.empty_like(z)
        nws = N.ctn_mha_workspace_bytes(B * D1, D2, F)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="dpt_mha"))
        N.check(N.ctn_mha_fwd(z.data_ptr(), B * D1, D2, F, self.num_heads, a.in_proj_weight.data_ptr(), a.in_proj_bias.data_ptr(),
                              a.out_proj.weight.data_ptr(), a.out_proj.bias.data_ptr(), y.data_ptr(), base, nbytes, st), "ctn_mha_fwd")
        out = torch.empty((B, D2, D1, F) if swap else (B, D1, D2, F), dtype=torch.float32, device=dev)
        g, b = self.norm1d.norm.weight, self.norm1d.norm.bias
        N.check(N.ctn_seq_norm_fwd(y.data_ptr(), None, None, z.data_ptr(), g.data_ptr(), b.data_ptr(), out.data_ptr(), B, D1, D2, F,
                                   float(self.eps), int(swap), st), "ctn_seq_norm_fwd")
        return out


class FeedForwardBlock(nn.Module):
    def __init__(self, num_features, hidden_channels, norm=True, nonlinear='relu', causal=False, eps=EPS):
        super().__init__()
        if causal:
            raise NotImplementedError("causal DPTNet (uni-directional LSTM, cLN) is outside the sm_90a path")
        if not norm:
            raise NotImplementedError("norm=False is outside the sm_90a path")
        if nonlinear != 'relu':
            raise NotImplementedError("sep_nonlinear={!r} is outside the sm_90a path ('relu' only)".format(nonlinear))
        if not N.ctn_bilstm_supported(num_features, hidden_channels, num_features):
            raise NotImplementedError("num_features={}, hidden_channels={} are outside the native LSTM's envelope (32, 64, 128)"
                                      .format(num_features, hidden_channels))
        self.norm = norm
        self.hidden_channels, self.eps = hidden_channels, eps
        self.rnn = choose_rnn('lstm', input_size=num_features, hidden_size=hidden_channels, batch_first=False, bidirectional=True)
        self.nonlinear1d = choose_nonlinear(nonlinear)
        self.fc = nn.Linear(2 * hidden_channels, num_features)
        self.norm1d = choose_layer_norm('gLN', num_features, causal=False, eps=eps)

    def forward(self, input):
        """input, output (T, batch_size, num_features) (dptnet.py:548-572)"""
        forward_only(self, input)
        return self._step(input.permute(1, 0, 2).unsqueeze(0).contiguous(), False)[0].permute(1, 0, 2).contiguous()

    def _step(self, z, swap):
        """z (B, D1, D2, F) -> GroupNorm over each (b, d1) sequence of z + fc(ReLU(LSTM(z))), (B, D2, D1, F) when swap"""
        B, D1, D2, F = z.shape
        dev = N.require_cuda(z)
        st = N.stream_ptr(dev)
        r, H = self.rnn, self.hidden_channels
        ptrs = (N._fp * 8)(*[t.data_ptr() for t in (r.weight_ih_l0, r.weight_hh_l0, r.bias_ih_l0, r.bias_hh_l0, r.weight_ih_l0_reverse,
                                                     r.weight_hh_l0_reverse, r.bias_ih_l0_reverse, r.bias_hh_l0_reverse)])
        nws = N.ctn_bilstm_workspace_bytes(F, H, F)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="dpt_lstm"))
        P = torch.empty((2, B * D1, D2, F), dtype=torch.float32, device=dev)
        N.check(N.ctn_bilstm_relu_proj_fwd(z.data_ptr(), B * D1, D2, F, H, ptrs, self.fc.weight.data_ptr(), F, P.data_ptr(), None, base,
                                           nbytes, st), "ctn_bilstm_relu_proj_fwd")
        out = torch.empty((B, D2, D1, F) if swap else (B, D1, D2, F), dtype=torch.float32, device=dev)
        g, b = self.norm1d.norm.weight, self.norm1d.norm.bias
        N.check(N.ctn_seq_norm_fwd(P[0].data_ptr(), P[1].data_ptr(), self.fc.bias.data_ptr(), z.data_ptr(), g.data_ptr(), b.data_ptr(),
                                   out.data_ptr(), B, D1, D2, F, float(self.eps), int(swap), st), "ctn_seq_norm_fwd")
        return out


class ImprovedTransformer(nn.Module):
    def __init__(self, num_features, hidden_channels, num_heads=4, norm=True, nonlinear='relu', dropout=0, causal=False, eps=EPS):
        super().__init__()
        self.multihead_attn_block = MultiheadAttentionBlock(num_features, num_heads, norm=norm, dropout=dropout, causal=causal, eps=eps)
        self.subnet = FeedForwardBlock(num_features, hidden_channels, norm=norm, nonlinear=nonlinear, causal=causal, eps=eps)

    def forward(self, input):
        """input, output (T, batch_size, num_features)"""
        forward_only(self, input)
        return self._step(input.permute(1, 0, 2).unsqueeze(0).contiguous(), False)[0].permute(1, 0, 2).contiguous()

    def _step(self, z, swap):
        return self.subnet._step(self.multihead_attn_block._step(z, False), swap)


class IntraChunkTransformer(nn.Module):
    def __init__(self, num_features, hidden_channels, num_heads=4, norm=True, nonlinear='relu', dropout=0, eps=EPS):
        super().__init__()
        self.num_features = num_features
        self.transformer = ImprovedTransformer(num_features, hidden_channels, num_heads=num_heads, norm=norm, nonlinear=nonlinear,
                                               dropout=dropout, causal=False, eps=eps)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size) (dptnet.py:414-430)"""
        forward_only(self, input)
        return self.transformer._step(input.permute(0, 2, 3, 1).contiguous(), False).permute(0, 3, 1, 2).contiguous()


class InterChunkTransformer(nn.Module):
    def __init__(self, num_features, hidden_channels, num_heads=4, causal=False, norm=True, nonlinear='relu', dropout=0, eps=EPS):
        super().__init__()
        self.num_features = num_features
        self.transformer = ImprovedTransformer(num_features, hidden_channels, num_heads=num_heads, norm=norm, nonlinear=nonlinear,
                                               dropout=dropout, causal=causal, eps=eps)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size) (dptnet.py:445-461)"""
        forward_only(self, input)
        return self.transformer._step(input.permute(0, 3, 2, 1).contiguous(), False).permute(0, 3, 2, 1).contiguous()


class DualPathTransformerBlock(nn.Module):
    def __init__(self, num_features, hidden_channels, num_heads=4, norm=True, nonlinear='relu', dropout=0, causal=False, eps=EPS):
        super().__init__()
        self.intra_chunk_block = IntraChunkTransformer(num_features, hidden_channels, num_heads=num_heads, norm=norm, nonlinear=nonlinear,
                                                       dropout=dropout, eps=eps)
        self.inter_chunk_block = InterChunkTransformer(num_features, hidden_channels, num_heads=num_heads, norm=norm, nonlinear=nonlinear,
                                                       dropout=dropout, causal=causal, eps=eps)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return self.forward_channels_last(input.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2).contiguous()

    def forward_channels_last(self, z):
        """z (B, S, K, F) -> (B, S, K, F): intra over the K frames of each chunk (stored swapped to (B, K, S, F)), inter over the
        S chunks of each frame (swapped back)"""
        z = self.intra_chunk_block.transformer._step(z, True)
        return self.inter_chunk_block.transformer._step(z, True)


class DualPathTransformer(nn.Module):
    def __init__(self, num_features, hidden_channels, num_blocks=6, num_heads=4, norm=True, nonlinear='relu', dropout=0, causal=False,
                 eps=EPS):
        super().__init__()
        self.net = nn.Sequential(*[DualPathTransformerBlock(num_features, hidden_channels, num_heads=num_heads, norm=norm,
                                                            nonlinear=nonlinear, dropout=dropout, causal=causal, eps=eps)
                                   for _ in range(num_blocks)])

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return self.forward_channels_last(input.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2).contiguous()

    def forward_channels_last(self, z):
        for blk in self.net:
            z = blk.forward_channels_last(z)
        return z


class Separator(nn.Module):
    def __init__(self, num_features, bottleneck_channels=32, hidden_channels=128, chunk_size=100, hop_size=None, num_blocks=6,
                 num_heads=4, norm=True, nonlinear='relu', dropout=0, mask_nonlinear='relu', causal=True, n_sources=2, eps=EPS):
        super().__init__()
        if hop_size is None:
            hop_size = chunk_size // 2
        if causal:
            raise NotImplementedError("causal DPTNet (cLN, uni-directional inter-chunk LSTM) is outside the sm_90a path")
        if mask_nonlinear == 'softmax':
            raise NotImplementedError("mask_nonlinear='softmax' is outside the sm_90a path")
        if mask_nonlinear not in ('relu', 'sigmoid'):
            raise ValueError("Cannot support {}".format(mask_nonlinear))
        self.num_features, self.n_sources = num_features, n_sources
        self.bottleneck_channels = bottleneck_channels
        self.chunk_size, self.hop_size = chunk_size, hop_size
        self.eps = eps
        self.bottleneck_conv1d = nn.Conv1d(num_features, bottleneck_channels, kernel_size=1, stride=1)
        self.segment1d = Segment1d(chunk_size, hop_size)
        self.norm2d = choose_layer_norm('gLN', bottleneck_channels, causal=False, eps=eps)
        self.dptransformer = DualPathTransformer(bottleneck_channels, hidden_channels, num_blocks=num_blocks, num_heads=num_heads, norm=norm,
                                                 nonlinear=nonlinear, dropout=dropout, causal=causal, eps=eps)
        self.overlap_add1d = OverlapAdd1d(chunk_size, hop_size)
        self.prelu = nn.PReLU()
        self.map = nn.Conv1d(bottleneck_channels, n_sources * num_features, kernel_size=1, stride=1)
        self.gtu = GTU1d(num_features, num_features, kernel_size=1, stride=1)
        self.mask_nonlinear = choose_nonlinear(mask_nonlinear)
        self.mask_relu = mask_nonlinear == 'relu'
        self.math = None

    folds_gln = False

    def check(self, B, n_frames):
        segment_geometry(n_frames, self.chunk_size, self.hop_size)

    def run_pitched(self, w, stats0, frames, pitch, dev):
        """w (B, N, pitch) pitched encoder output -> y (B, Bc, pitch): everything between the encoder and the PReLU of dptnet.py:341"""
        B = w.shape[0]
        Nf, Bc, K, P = self.num_features, self.bottleneck_channels, self.chunk_size, self.hop_size
        pl, pr, S = segment_geometry(frames, K, P)
        st = N.stream_ptr(dev)
        z = torch.empty(B, S, K, Bc, dtype=torch.float32, device=dev)
        nws = N.ctn_dpt_head_workspace_bytes(B, Nf, Bc, pitch, S, K)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="dpt_head"))
        g, b = self.norm2d.norm.weight, self.norm2d.norm.bias
        N.check(N.ctn_dpt_head_fwd(w.data_ptr(), self.bottleneck_conv1d.weight.data_ptr(), self.bottleneck_conv1d.bias.data_ptr(),
                                   g.data_ptr(), b.data_ptr(), z.data_ptr(), B, Nf, Bc, frames, pitch, K, P, pl, pr, float(self.eps),
                                   math_of(self.math), base, nbytes, st), "ctn_dpt_head_fwd")
        z = self.dptransformer.forward_channels_last(z)
        y = torch.empty(B, Bc, pitch, dtype=torch.float32, device=dev)
        N.check(N.ctn_overlap_add_fwd(z.data_ptr(), y.data_ptr(), B, Bc, S, K, P, pl, frames, pitch, 1, st), "ctn_overlap_add_fwd")
        return y

    def forward(self, input):
        """input (batch_size, num_features, n_frames) -> mask (batch_size, n_sources, num_features, n_frames)"""
        raise NotImplementedError("the stand-alone DPTNet Separator.forward (materialised mask) is not built; use DPTNet")


class DPTNet(GTUTailModel):
    """Dual-path transformer based network"""
    pretrained_model_ids = {
        "wsj0-mix": {
            8000: {
                2: "1QJnJEK8aed7_ED07jD7buyGb37giEDUx",
                3: "1Rfb_vS8r2_Oqpg_zAV9y4WMzv106yrSP"
            },
            16000: {
                2: "",
                3: ""
            }
        }
    }

    def __init__(self, n_basis, kernel_size, stride=None, enc_basis=None, dec_basis=None, sep_bottleneck_channels=64,
                 sep_hidden_channels=256, sep_chunk_size=100, sep_hop_size=None, sep_num_blocks=6, sep_num_heads=4, sep_norm=True,
                 sep_nonlinear='relu', sep_dropout=0, mask_nonlinear='relu', causal=False, n_sources=2, eps=EPS, **kwargs):
        super().__init__()
        if stride is None:
            stride = kernel_size // 2
        if sep_hop_size is None:
            sep_hop_size = sep_chunk_size // 2
        assert kernel_size % stride == 0, "kernel_size is expected divisible by stride"
        assert n_basis % sep_num_heads == 0, "n_basis must be divisible by sep_num_heads"
        if kwargs.get('in_channels', 1) != 1:
            raise NotImplementedError("multichannel DPTNet is outside the sm_90a path")
        self.n_basis = n_basis
        self.kernel_size, self.stride = kernel_size, stride
        self.enc_basis, self.dec_basis = enc_basis, dec_basis
        self.enc_nonlinear = kwargs['enc_nonlinear'] if (enc_basis == 'trainable' and dec_basis != 'pinv') else None
        self.window_fn, self.enc_onesided, self.enc_return_complex = None, None, None
        self.sep_bottleneck_channels, self.sep_hidden_channels = sep_bottleneck_channels, sep_hidden_channels
        self.sep_chunk_size, self.sep_hop_size = sep_chunk_size, sep_hop_size
        self.sep_num_blocks, self.sep_num_heads = sep_num_blocks, sep_num_heads
        self.sep_norm, self.sep_nonlinear, self.sep_dropout = sep_norm, sep_nonlinear, sep_dropout
        self.causal, self.mask_nonlinear = causal, mask_nonlinear
        self.n_sources, self.eps = n_sources, eps
        encoder, decoder = choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis, dec_basis=dec_basis, **kwargs)
        self.encoder = encoder
        self.separator = Separator(n_basis, bottleneck_channels=sep_bottleneck_channels, hidden_channels=sep_hidden_channels,
                                   chunk_size=sep_chunk_size, hop_size=sep_hop_size, num_blocks=sep_num_blocks, num_heads=sep_num_heads,
                                   norm=sep_norm, nonlinear=sep_nonlinear, dropout=sep_dropout, mask_nonlinear=mask_nonlinear,
                                   causal=causal, n_sources=n_sources, eps=eps)
        self.decoder = decoder
        self.math = None

    def get_config(self):
        return {
            'n_basis': self.n_basis, 'kernel_size': self.kernel_size, 'stride': self.stride, 'enc_basis': self.enc_basis,
            'dec_basis': self.dec_basis, 'enc_nonlinear': self.enc_nonlinear, 'window_fn': self.window_fn,
            'enc_onesided': self.enc_onesided, 'enc_return_complex': self.enc_return_complex,
            'sep_hidden_channels': self.sep_hidden_channels, 'sep_bottleneck_channels': self.sep_bottleneck_channels,
            'sep_chunk_size': self.sep_chunk_size, 'sep_hop_size': self.sep_hop_size, 'sep_num_blocks': self.sep_num_blocks,
            'sep_num_heads': self.sep_num_heads, 'sep_norm': self.sep_norm, 'sep_nonlinear': self.sep_nonlinear,
            'sep_dropout': self.sep_dropout, 'mask_nonlinear': self.mask_nonlinear, 'causal': self.causal,
            'n_sources': self.n_sources, 'eps': self.eps,
        }

    @classmethod
    def build_model(cls, model_path, load_state_dict=False):
        """dptnet.py:175-217 (legacy keys n_bases / enc_bases / dec_bases tolerated)"""
        config = _load_checkpoint(model_path)
        get = config.get
        model = cls(
            get('n_bases') or config['n_basis'], config['kernel_size'], stride=config['stride'],
            enc_basis=get('enc_bases') or config['enc_basis'], dec_basis=get('dec_bases') or config['dec_basis'],
            enc_nonlinear=config['enc_nonlinear'], window_fn=config['window_fn'], enc_onesided=get('enc_onesided') or None,
            enc_return_complex=get('enc_return_complex') or None, sep_bottleneck_channels=config['sep_bottleneck_channels'],
            sep_hidden_channels=config['sep_hidden_channels'], sep_chunk_size=config['sep_chunk_size'],
            sep_hop_size=config['sep_hop_size'], sep_num_blocks=config['sep_num_blocks'], sep_num_heads=config['sep_num_heads'],
            sep_norm=config['sep_norm'], sep_nonlinear=config['sep_nonlinear'], sep_dropout=config['sep_dropout'],
            mask_nonlinear=config['mask_nonlinear'], causal=config['causal'], n_sources=config['n_sources'], eps=config['eps'])
        if load_state_dict:
            model.load_state_dict(config['state_dict'])
        return model

    @classmethod
    def build_from_pretrained(cls, root="./pretrained", quiet=False, load_state_dict=True, **kwargs):
        """dptnet.py:219-259: <root>/DPTNet/wsj0-mix/sr<rate>/<n>speakers/model/<choice>.pth, loaded, never downloaded"""
        return build_from_pretrained(cls, root, load_state_dict, **kwargs)
