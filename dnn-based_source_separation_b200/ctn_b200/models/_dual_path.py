"""Plumbing shared by the dual-path models (DPRNN-TasNet, DPTNet, SepFormer, GALRNet) and LSTM-TasNet.

* ``forward_only`` / ``eval_dropout``: the refusals of every native forward (no autograd graph, dropout only in eval mode);
* ``segment_geometry``: the reference's padding rule in front of Segment1d;
* ``math_of``: a model's numeric mode, or the package default;
* ``build_from_pretrained``: the checkpoint path the reference downloads to, loaded when it is there; nothing is downloaded;
* ``GTUTailModel``: forward / extract_latent of the models whose separator ends in PReLU -> map -> GTU1d -> mask
  (DPTNet, GALRNet, SepFormer): encoder, the separator's ``run_pitched`` and ``ctn_dpt_tail_fwd``.
"""
import os

import torch
import torch.nn as nn

from .. import _native as N
from . import tdcn as _tdcn
from .tdcn import resolve_math


def forward_only(module, *inputs):
    """refuse to run where autograd would record a graph: the native kernels have no backward, so the output would silently carry
    no gradient to the parameters or the inputs"""
    if torch.is_grad_enabled() and (any(p.requires_grad for p in module.parameters()) or any(t.requires_grad for t in inputs)):
        raise NotImplementedError("the {} path is forward-only: call under torch.no_grad()".format(type(module).__name__))


def eval_dropout(module, p):
    if module.training and p is not None and p > 0:
        raise NotImplementedError("dropout > 0 in training mode is outside the sm_90a path: call model.eval()")


def segment_geometry(n_frames, chunk_size, hop_size):
    """the padding rule of the reference's dual-path separators (e.g. dptnet.py:330-332) -> (pad_left, pad_right, S)"""
    K, P = chunk_size, hop_size
    padding = (P - (n_frames - K) % P) % P
    pl = padding // 2
    if n_frames + padding < K:
        raise ValueError("n_frames={} is too short for chunk_size={}".format(n_frames, K))
    return pl, padding - pl, (n_frames + padding - K) // P + 1


def math_of(math):
    return resolve_math(math if math is not None else _tdcn.DEFAULT_MATH)


def build_from_pretrained(cls, root, load_state_dict, **kwargs):
    """resolve <root>/<class>/wsj0-mix/sr<rate>/<n>speakers/model/<choice>.pth as the reference does and build the model from it.
    Nothing is downloaded: a missing file raises FileNotFoundError naming the expected path."""
    task = kwargs.get('task')
    if task not in cls.pretrained_model_ids:
        raise KeyError("Invalid task ({}) is specified.".format(task))
    if task not in ['wsj0-mix', 'wsj0']:
        raise NotImplementedError("Not support task={}.".format(task))
    sample_rate = kwargs.get('sample_rate') or 8000
    n_sources = kwargs.get('n_sources') or 2
    model_choice = kwargs.get('model_choice') or 'best'
    model_id = cls.pretrained_model_ids[task][sample_rate][n_sources]
    download_dir = os.path.join(root, cls.__name__, task, "sr{}/{}speakers".format(sample_rate, n_sources))
    model_path = os.path.join(download_dir, "model", "{}.pth".format(model_choice))
    if not os.path.exists(model_path):
        raise FileNotFoundError("{} not found (Google-Drive id {!r}); place the reference checkpoint there -- this path loads "
                                "checkpoints, it does not download them".format(model_path, model_id))
    model = cls.build_model(model_path, load_state_dict=load_state_dict)
    for key, value in {'n_sources': n_sources, 'sample_rate': sample_rate}.items():
        setattr(model, key, value)
    return model


class GTUTailModel(nn.Module):
    """forward of DPTNet, GALRNet and SepFormer.  The model holds encoder, separator, decoder and the attributes kernel_size,
    stride, n_basis, n_sources, sep_dropout and math; its Separator implements
      * check(B, n_frames): every refusal of the shape, before any device work;
      * folds_gln: whether its head folds the gLN of w (then the encoder also forms the statistics of w);
      * run_pitched(w, stats0, frames, pitch, dev) -> y (B, Bc, pitch), everything between the encoder and the tail's PReLU;
      * prelu, map, gtu, mask_relu, math and, for SepFormer, bottleneck_conv1d_out: the tail's parameters."""

    def forward(self, input):
        output, _ = self._run(input, want_latent=False)
        return output

    def extract_latent(self, input):
        """input (batch_size, 1, T) -> output (batch_size, n_sources, T), latent (batch_size, n_sources, n_basis, T')"""
        return self._run(input, want_latent=True)

    @property
    def num_parameters(self):
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def _run(self, input, want_latent):
        if input.dim() != 3:
            raise ValueError("input.size() is expected (?, 1, ?), but given {}".format(tuple(input.size())))
        assert input.size(1) == 1, "input.size() is expected (?, 1, ?), but given {}".format(input.size())
        forward_only(self, input)
        eval_dropout(self, self.sep_dropout)
        sep = self.separator
        B, _, T = input.shape
        frames, pl, pr = N.frames_of(T, self.kernel_size, self.stride)
        sep.check(B, frames)
        x = input.contiguous()
        dev = N.require_cuda(x)
        sep.math = self.math if self.math is not None else sep.math
        pitch = N.ctn_pitch(frames)
        st = N.stream_ptr(dev)
        Nb, S = self.n_basis, self.n_sources
        w = torch.empty(B, Nb, pitch, dtype=torch.float32, device=dev)
        stats0 = torch.zeros(2 * B, dtype=torch.float64, device=dev) if sep.folds_gln else None
        N.check(N.ctn_encoder_fwd(x.data_ptr(), self.encoder.conv1d.weight.data_ptr(), w.data_ptr(), B, T, pl, pr, Nb, self.kernel_size,
                                  self.stride, int(self.encoder.nonlinear), pitch, N.ptr(stats0), st), "ctn_encoder_fwd")
        y = sep.run_pitched(w, stats0, frames, pitch, dev)
        Bc = y.shape[1]
        out = torch.empty(B, S, T, dtype=torch.float32, device=dev)
        latent = torch.empty(B, S, Nb, frames, dtype=torch.float32, device=dev) if want_latent else None
        what = torch.empty(B, S * Nb, pitch, dtype=torch.float32, device=dev)
        bout = getattr(sep, "bottleneck_conv1d_out", None)
        bout_w, bout_b = (bout.weight, bout.bias) if bout is not None else (None, None)
        nws = N.ctn_dpt_tail_workspace_bytes(B, Nb, Bc, S, pitch, int(bout is not None))
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="gtu_tail"))
        N.check(N.ctn_dpt_tail_fwd(y.data_ptr(), w.data_ptr(), sep.prelu.weight.data_ptr(), sep.map.weight.data_ptr(), sep.map.bias.data_ptr(),
                                   sep.gtu.map.weight.data_ptr(), sep.gtu.map.bias.data_ptr(), sep.gtu.map_gate.weight.data_ptr(),
                                   sep.gtu.map_gate.bias.data_ptr(), N.ptr(bout_w), N.ptr(bout_b),
                                   self.decoder.conv_transpose1d.weight.data_ptr(), out.data_ptr(), N.ptr(latent), what.data_ptr(), B, Nb,
                                   Bc, S, frames, pitch, self.kernel_size, self.stride, pl, T, int(sep.mask_relu), math_of(sep.math), base,
                                   nbytes, st), "ctn_dpt_tail_fwd")
        return out, latent
