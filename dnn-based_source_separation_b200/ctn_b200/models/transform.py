"""Segment1d / OverlapAdd1d on sm_90a gather / scatter kernels (csrc/ctn_dprnn.cu).

Mirrors src/models/transform.py:6-65 of the reference (same constructors, same shapes): ``Segment1d`` turns
(batch, features, frames) into (batch, features, S, chunk_size) with S = (frames - chunk_size) // hop_size + 1,
``OverlapAdd1d`` sums the overlapping chunks back into (batch, features, (S - 1) * hop_size + chunk_size).
The dual-path separators use the same entries with the padding / crop fused in: channels-last (``layout=1``: DPRNN, DPTNet,
GALRNet) or channel-first with padded rows (``layout`` = the row pitch: SepFormer).
"""
import torch
import torch.nn as nn

from .. import _native as N

ctn_segment_fwd, ctn_overlap_add_fwd, ctn_dprnn_norm_res_fwd = N.ctn_segment_fwd, N.ctn_overlap_add_fwd, N.ctn_dprnn_norm_res_fwd
ctn_stage_workspace_bytes, ctn_sep_head_fwd, ctn_sep_tail_fwd = N.ctn_stage_workspace_bytes, N.ctn_sep_head_fwd, N.ctn_sep_tail_fwd


class Segment1d(nn.Module):
    """Segmentation. Input tensor is 3-D (audio-like), but output tensor is 4-D (image-like)."""

    def __init__(self, chunk_size, hop_size):
        super().__init__()
        self.chunk_size, self.hop_size = chunk_size, hop_size

    def forward(self, input):
        """input (batch_size, num_features, n_frames) -> (batch_size, num_features, S, chunk_size)"""
        if input.dim() != 3:
            raise ValueError("input is expected 3-D (batch_size, num_features, n_frames), but given {}".format(tuple(input.size())))
        x = input.contiguous()
        dev = N.require_cuda(x)
        B, F, T = x.shape
        K, P = self.chunk_size, self.hop_size
        if T < K:
            raise ValueError("n_frames={} is shorter than chunk_size={}".format(T, K))
        S = (T - K) // P + 1
        out = torch.empty(B, F, S, K, dtype=torch.float32, device=dev)
        N.check(ctn_segment_fwd(x.data_ptr(), out.data_ptr(), B, F, T, T, K, P, 0, 0, 0, N.stream_ptr(dev)), "ctn_segment_fwd")
        return out

    def extra_repr(self):
        return "chunk_size={chunk_size}, hop_size={hop_size}".format(chunk_size=self.chunk_size, hop_size=self.hop_size)


class OverlapAdd1d(nn.Module):
    """Overlap-add operation. Input tensor is 4-D (image-like), but output tensor is 3-D (audio-like)."""

    def __init__(self, chunk_size, hop_size):
        super().__init__()
        self.chunk_size, self.hop_size = chunk_size, hop_size

    def forward(self, input):
        """input (batch_size, num_features, S, chunk_size) -> (batch_size, num_features, (S - 1) * hop_size + chunk_size)"""
        if input.dim() != 4:
            raise ValueError("input is expected 4-D (batch_size, num_features, S, chunk_size), but given {}".format(tuple(input.size())))
        x = input.contiguous()
        dev = N.require_cuda(x)
        B, F, S, K = x.shape
        P = self.hop_size
        T = (S - 1) * P + K
        out = torch.empty(B, F, T, dtype=torch.float32, device=dev)
        N.check(ctn_overlap_add_fwd(x.data_ptr(), out.data_ptr(), B, F, S, K, P, 0, T, T, 0, N.stream_ptr(dev)), "ctn_overlap_add_fwd")
        return out

    def extra_repr(self):
        return "chunk_size={chunk_size}, hop_size={hop_size}".format(chunk_size=self.chunk_size, hop_size=self.hop_size)
