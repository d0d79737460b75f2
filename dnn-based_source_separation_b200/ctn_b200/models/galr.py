"""GALR (globally attentive locally recurrent) blocks behind the reference's class API (src/models/galr.py:9-229).

Same constructors, module tree and ``state_dict`` keys as the reference.  The dual-path state stays channels-last,
(batch, S, chunk_size, F), end to end, as on the DPTNet path.  Each GALRBlock is
  * the intra-chunk block: the DPRNN ``IntraChunkRNN`` itself (``ctn_bilstm_proj_fwd`` + ``ctn_dprnn_norm_res2_fwd``, swap = 0);
  * the inter-chunk block, ``LowDimensionGloballyAttentiveBlock``: one ``ctn_galr_inter_fwd`` (csrc/ctn_galr.cu): fc_map along the
    chunk axis + LayerNorm over channels + positional encoding, multi-head attention over the S chunks of each down-sampled
    frame, gLN per sample of attention + residual, fc_inv back to the chunk axis, plus the block input.
The positional encoding's divisors 10000^(j / F) are formed once per F with the reference's fp32 expression on the host and kept
on the device in a cache that is not part of the ``state_dict``; the kernel divides and takes sin / cos in full precision.
Envelope: non-causal, norm=True, low_dimension=True, F in {32, 64, 128} with hidden_channels in the native LSTM's sizes,
1 <= down_chunk_size <= chunk_size, head dimension F / heads inside ``ctn_mha_supported``; forward only, dropout only in eval mode.
"""
import torch
import torch.nn as nn

from .. import _native as N
from ..utils.tasnet import choose_layer_norm
from ._dual_path import eval_dropout, forward_only
from .dprnn import IntraChunkRNN as LocallyRecurrentBlock

EPS = 1e-12


class GALR(nn.Module):
    def __init__(self, num_features, hidden_channels, num_blocks=6, num_heads=8, norm=True, dropout=1e-1, low_dimension=True, causal=False,
                 eps=EPS, **kwargs):
        super().__init__()
        self.net = nn.Sequential(*[GALRBlock(num_features, hidden_channels, num_heads=num_heads, norm=norm, dropout=dropout,
                                             low_dimension=low_dimension, causal=causal, eps=eps, **kwargs) for _ in range(num_blocks)])

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return self.forward_channels_last(input.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2).contiguous()

    def forward_channels_last(self, z):
        for blk in self.net:
            z = blk.forward_channels_last(z)
        return z


class GALRBlock(nn.Module):
    def __init__(self, num_features, hidden_channels, num_heads=8, causal=False, norm=True, dropout=1e-1, low_dimension=True, eps=EPS,
                 **kwargs):
        super().__init__()
        if causal:
            raise NotImplementedError("causal GALR (cLN) is outside the sm_90a path")
        if not low_dimension:
            raise NotImplementedError("low_dimension=False (GloballyAttentiveBlock) is outside the sm_90a path")
        if not N.ctn_bilstm_supported(num_features, hidden_channels, num_features):
            raise NotImplementedError("num_features={}, hidden_channels={} are outside the native LSTM's envelope (32, 64, 128)"
                                      .format(num_features, hidden_channels))
        self.intra_chunk_block = LocallyRecurrentBlock(num_features, hidden_channels=hidden_channels, norm=norm, eps=eps)
        self.inter_chunk_block = LowDimensionGloballyAttentiveBlock(num_features, chunk_size=kwargs['chunk_size'],
                                                                    down_chunk_size=kwargs['down_chunk_size'], num_heads=num_heads,
                                                                    causal=causal, norm=norm, dropout=dropout, eps=eps)

    def forward(self, input):
        """input, output (batch_size, num_features, S, chunk_size)"""
        forward_only(self, input)
        return self.forward_channels_last(input.permute(0, 2, 3, 1).contiguous()).permute(0, 3, 1, 2).contiguous()

    def forward_channels_last(self, z):
        """z (B, S, K, F) -> (B, S, K, F): the bi-LSTM over the K frames of each chunk, then the attention over the S chunks"""
        self.inter_chunk_block.check_shape(z.shape)
        eval_dropout(self.inter_chunk_block, self.inter_chunk_block.dropout_p)
        return self.inter_chunk_block._step(self.intra_chunk_block._step(z, swap=False))


class GloballyAttentiveBlockBase(nn.Module):
    def __init__(self):
        super().__init__()

    def positional_encoding(self, length: int, dimension: int, base=10000):
        """(length, dimension) encoding of galr.py:61-78, on the host in fp32: [sin | cos] of position / base^(j / dimension)"""
        assert dimension % 2 == 0, "dimension is expected even number but given odd number."
        indices = torch.arange(length).unsqueeze(dim=1) / self.pe_divisors(dimension, base).unsqueeze(dim=0)
        return torch.cat([torch.sin(indices), torch.cos(indices)], dim=1)

    @staticmethod
    def pe_divisors(dimension: int, base=10000):
        """the dimension // 2 fp32 divisors base^(j / dimension), by the reference's own expression (galr.py:73-75)"""
        return base ** (torch.arange(dimension // 2) / dimension)


class GloballyAttentiveBlock(GloballyAttentiveBlockBase):
    def __init__(self, num_features, num_heads=8, causal=False, norm=True, dropout=1e-1, eps=EPS):
        super().__init__()
        raise NotImplementedError("GloballyAttentiveBlock (low_dimension=False) is outside the sm_90a path")


class LowDimensionGloballyAttentiveBlock(GloballyAttentiveBlockBase):
    def __init__(self, num_features, chunk_size=100, down_chunk_size=32, num_heads=8, causal=False, norm=True, dropout=1e-1, eps=EPS):
        super().__init__()
        if causal:
            raise NotImplementedError("causal GALR (cLN) is outside the sm_90a path")
        if not norm:
            raise NotImplementedError("norm=False is outside the sm_90a path")
        if not N.ctn_galr_supported(num_features, chunk_size, down_chunk_size, num_heads):
            raise NotImplementedError("num_features={}, chunk_size={}, down_chunk_size={}, num_heads={} are outside the globally attentive "
                                      "block's envelope (num_features in 32, 64, 128; 1 <= down_chunk_size <= chunk_size; head dimension "
                                      "in 8, 16, 32, 64)".format(num_features, chunk_size, down_chunk_size, num_heads))
        self.down_chunk_size = down_chunk_size
        self.norm = norm
        self.chunk_size, self.num_heads, self.eps = chunk_size, num_heads, eps
        self.dropout_p = dropout
        self.fc_map = nn.Linear(chunk_size, down_chunk_size)
        self.norm2d_in = LayerNormAlongChannel(num_features, eps=eps)
        self.multihead_attn = nn.MultiheadAttention(num_features, num_heads)
        if dropout is not None:
            self.dropout = True
            self.dropout1d = nn.Dropout(p=dropout)
        else:
            self.dropout = False
        self.norm2d_out = choose_layer_norm('gLN', num_features, causal=False, eps=eps)
        self.fc_inv = nn.Linear(down_chunk_size, chunk_size)
        self._pe_div = {}  # (F, device) -> divisors; deliberately not a buffer: the state_dict keeps the reference's keys

    def forward(self, input):
        """input, output (batch_size, num_features, S, K) (galr.py:161-197)"""
        forward_only(self, input)
        eval_dropout(self, self.dropout_p)
        z = input.permute(0, 2, 3, 1).contiguous()
        self.check_shape(z.shape)
        return self._step(z).permute(0, 3, 1, 2).contiguous()

    def check_shape(self, shape):
        """refusals of ctn_galr_inter_fwd's launch limits for a state of shape (B, S, K, F), before anything runs"""
        if len(shape) != 4:
            raise ValueError("expected (batch_size, S, chunk_size, num_features), got {}".format(tuple(shape)))
        B, S, K, F = shape
        Q = self.down_chunk_size
        if K != self.chunk_size or F != self.norm2d_in.num_features:
            raise ValueError("chunk_size={}, num_features={} given to a block built for {}, {}".format(K, F, self.chunk_size,
                                                                                                   self.norm2d_in.num_features))
        if B > 65535 or S > 65535 or S * Q > 1 << 24:
            raise NotImplementedError("batch_size={}, S={} with down_chunk_size={} are outside the globally attentive block's launch "
                                      "limits (batch_size, S <= 65535; S * down_chunk_size <= 2^24)"
                                      .format(B, S, Q))

    def _divisors(self, F, dev):
        key = (F, dev)
        d = self._pe_div.get(key)
        if d is None:
            d = self.pe_divisors(F).to(device=dev, dtype=torch.float32)
            self._pe_div[key] = d
        return d

    def _step(self, z):
        """z (B, S, K, F) channels-last -> (B, S, K, F)"""
        B, S, K, F = z.shape
        dev = N.require_cuda(z)
        st = N.stream_ptr(dev)
        Q = self.down_chunk_size
        div = self._divisors(F, dev)
        a = self.multihead_attn
        ln, gn = self.norm2d_in.norm, self.norm2d_out.norm
        out = torch.empty_like(z)
        nws = N.ctn_galr_inter_workspace_bytes(B, S, K, Q, F)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="galr_inter"))
        N.check(N.ctn_galr_inter_fwd(z.data_ptr(), self.fc_map.weight.data_ptr(), self.fc_map.bias.data_ptr(), ln.weight.data_ptr(),
                                     ln.bias.data_ptr(), div.data_ptr(), self.num_heads, a.in_proj_weight.data_ptr(),
                                     a.in_proj_bias.data_ptr(), a.out_proj.weight.data_ptr(), a.out_proj.bias.data_ptr(),
                                     gn.weight.data_ptr(), gn.bias.data_ptr(), self.fc_inv.weight.data_ptr(), self.fc_inv.bias.data_ptr(),
                                     out.data_ptr(), B, S, K, Q, F, float(ln.eps), float(self.eps), base, nbytes, st), "ctn_galr_inter_fwd")
        return out


class LayerNormAlongChannel(nn.Module):
    def __init__(self, num_features, eps=EPS):
        super().__init__()
        self.num_features = num_features
        self.eps = eps
        self.norm = nn.LayerNorm(num_features, eps=eps)

    def forward(self, input):
        raise NotImplementedError("the stand-alone LayerNormAlongChannel.forward is not built; it runs inside "
                                  "LowDimensionGloballyAttentiveBlock")

    def __repr__(self):
        s = '{}'.format(self.__class__.__name__)
        s += '({num_features}, eps={eps})'
        return s.format(**self.__dict__)
