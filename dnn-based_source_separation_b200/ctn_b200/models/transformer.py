"""PositionalEncoding behind the reference's class API (src/models/transformer.py:7-43): the same (max_len, 1, F) buffer.

The buffer interleaves the two functions, [sin_0, cos_0, sin_1, cos_1, ...] along the features.  Inside SepFormer the native
path reads it from the module (``ctn_sfm_pos_enc_fwd``), so a checkpoint's buffer is used bit for bit; ``forward`` is the
reference's own addition for callers that use the module on its own.
"""
import torch
import torch.nn as nn


class PositionalEncoding(nn.Module):
    def __init__(self, num_features, dropout=0, max_len=5000, base=10000, batch_first=False):
        super().__init__()
        self.batch_first = batch_first
        position = torch.arange(max_len)
        index = torch.arange(0, num_features, 2) / num_features
        indices = position.unsqueeze(dim=1) / (base ** index.unsqueeze(dim=0))
        sin, cos = torch.sin(indices), torch.cos(indices)
        positional_encoding = torch.stack([sin, cos], dim=-1)  # (max_len, num_features // 2, 2): interleaved
        if batch_first:
            positional_encoding = positional_encoding.view(max_len, num_features)
        else:
            positional_encoding = positional_encoding.view(max_len, 1, num_features)
        self.register_buffer("positional_encoding", positional_encoding)
        self.dropout = nn.Dropout(p=dropout)

    def forward(self, input):
        """input (T, batch_size, num_features) or (batch_size, T, num_features) if batch_first -> input + encoding"""
        if self.batch_first:
            x = input + self.positional_encoding[:, :input.size(1)]
        else:
            x = input + self.positional_encoding[:input.size(0)]
        return self.dropout(x)
