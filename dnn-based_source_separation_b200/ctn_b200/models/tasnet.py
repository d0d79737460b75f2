"""LSTM-TasNet behind the reference's class API (src/models/tasnet.py:66-381, ``TasNet``).

Same constructor, module tree and ``state_dict`` keys as the reference (torch's own ``nn.LSTM`` holds the recurrent parameters),
so its checkpoints load with ``load_state_dict(strict=True)``.  Forward:
  * encoder: ``GatedEncoder`` (enc_basis='trainableGated') -> ``ctn_tas_enc_gated_fwd``, which also forms the Separator's frame
    norm; the plain ``Encoder`` (enc_basis='trainable') -> ``ctn_encoder_fwd`` + ``ctn_tas_frame_norm_fwd``;
  * every LSTM layer -> ``ctn_tas_lstm_fwd`` (input projections as one contraction, then one cooperative recurrence launch); the last
    layer of each block after the first also forms skip = x + skip;
  * fc, the mask (sigmoid, or softmax over the sources), w * mask and the decoder -> ``ctn_tas_tail_fwd``.
Everything stays channel-first and pitched, (B, C, ctn_pitch(T')), between the stages.
Envelope: rnn_type='lstm', monaural 3-D input, sep_hidden_channels up to ``ctn_tas_lstm_max_hidden`` of the device; forward only.
A causal model with the plain encoder also streams: ``model.online(batch_size, max_chunk)`` (models/online.py).
"""
import torch
import torch.nn as nn

from .. import _native as N
from ..utils.filterbank import choose_filterbank
from ..utils.model import choose_nonlinear
from ._dual_path import build_from_pretrained, forward_only, math_of
from .conv_tasnet import _load_checkpoint
from .filterbank import GatedEncoder

EPS = 1e-12


def _choose_rnn(name, **kwargs):
    """src/utils/model.py:22-32"""
    if name == 'rnn':
        return nn.RNN(**kwargs)
    if name == 'lstm':
        return nn.LSTM(**kwargs)
    if name == 'gru':
        return nn.GRU(**kwargs)
    raise NotImplementedError("Invalid RNN is specified. Choose 'rnn', 'lstm', or 'gru' instead of {}.".format(name))


def _choose_tasnet_filterbank(n_basis, kernel_size, stride, enc_basis, dec_basis, **kwargs):
    """choose_filterbank for LSTM-TasNet: the gated encoder is built here (as src/utils/filterbank.py:24-26 builds it, with the
    default eps: TasNet's own eps never reaches it), every other basis goes through the shared choose_filterbank"""
    if enc_basis == 'trainableGated':
        in_channels = kwargs.get('in_channels') or 1
        encoder = GatedEncoder(in_channels, n_basis, kernel_size=kernel_size, stride=stride, eps=kwargs.get('eps') or EPS)
        _, decoder = choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis='trainable', dec_basis=dec_basis, **kwargs)
        return encoder, decoder
    return choose_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis, dec_basis=dec_basis, **kwargs)


class Separator(nn.Module):
    """Default separator of TasNet (tasnet.py:324-381): frame norm, X blocks of R-layer (bi-)LSTMs with a skip sum, fc, mask"""

    def __init__(self, n_basis, num_blocks, num_layers, hidden_channels, causal=False, mask_nonlinear='softmax', rnn_type='lstm',
                 n_sources=2, eps=EPS):
        super().__init__()
        self.num_blocks, self.num_layers = num_blocks, num_layers
        self.n_basis, self.n_sources = n_basis, n_sources
        self.hidden_channels = hidden_channels
        self.eps = eps
        self.num_directions = 1 if causal else 2
        self.gamma = nn.Parameter(torch.Tensor(1, n_basis, 1))
        self.beta = nn.Parameter(torch.Tensor(1, n_basis, 1))
        net = []
        for idx in range(num_blocks):
            in_channels = n_basis if idx == 0 else self.num_directions * hidden_channels
            net.append(_choose_rnn(rnn_type, input_size=in_channels, hidden_size=hidden_channels, num_layers=num_layers, batch_first=True,
                                   bidirectional=not causal))
        self.rnn = nn.Sequential(*net)
        self.fc = nn.Linear(self.num_directions * hidden_channels, n_sources * n_basis)
        if mask_nonlinear == 'sigmoid':
            kwargs = {}
        elif mask_nonlinear == 'softmax':
            kwargs = {"dim": 1}
        else:
            kwargs = {}
        self.mask_nonlinear = choose_nonlinear(mask_nonlinear, **kwargs)
        self.mask_softmax = mask_nonlinear == 'softmax'
        self.rnn_type = rnn_type
        self._reset_parameters()

    def _reset_parameters(self):
        self.gamma.data.fill_(1)
        self.beta.data.zero_()

    def check_envelope(self):
        if self.rnn_type != 'lstm':
            raise NotImplementedError("rnn_type={!r} is outside the sm_90a LSTM-TasNet path ('lstm' only)".format(self.rnn_type))
        if not isinstance(self.mask_nonlinear, (nn.Sigmoid, nn.Softmax)):
            raise NotImplementedError("mask_nonlinear must be 'sigmoid' or 'softmax' on the sm_90a LSTM-TasNet path")

    def check_hidden(self):
        dirs, H = self.num_directions, self.hidden_channels
        for rnn in self.rnn:
            if not N.ctn_tas_lstm_supported(rnn.input_size, H, dirs):
                raise NotImplementedError("sep_hidden_channels={} is outside the recurrence kernel's envelope: at most {} with {} "
                                          "direction(s) on this device".format(H, N.ctn_tas_lstm_max_hidden(dirs), dirs))

    def run_pitched(self, xn, frames, pitch, math, dev):
        """xn (B, N, pitch) frame-normalised encoder output -> skip sum (B, dirs H, pitch)"""
        B = xn.shape[0]
        dirs, H = self.num_directions, self.hidden_channels
        st = N.stream_ptr(dev)
        z, skip = xn, None
        for blk, rnn in enumerate(self.rnn):
            for layer in range(self.num_layers):
                F = rnn.input_size if layer == 0 else dirs * H
                out = torch.empty(B, dirs * H, pitch, dtype=torch.float32, device=dev)
                sfx = ["_l{}".format(layer)] + (["_l{}_reverse".format(layer)] if dirs == 2 else [])
                ts = [getattr(rnn, n + s) for s in sfx for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
                for t in ts:
                    if not t.is_contiguous() or t.device != dev or t.dtype != torch.float32:
                        raise ValueError("LSTM parameters must be contiguous float32 on {}".format(dev))
                wp = (N._fp * len(ts))(*[t.data_ptr() for t in ts])
                skip_in = skip_out = None
                if blk > 0 and layer == self.num_layers - 1:  # skip = x + skip (tasnet.py:369), formed by the block's last layer
                    skip_in, skip_out = skip, torch.empty(B, dirs * H, pitch, dtype=torch.float32, device=dev)
                nws = N.ctn_tas_lstm_workspace_bytes(B, F, H, dirs, pitch, math)
                base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="tas_lstm"))
                N.check(N.ctn_tas_lstm_fwd(z.data_ptr(), wp, out.data_ptr(), N.ptr(skip_in), N.ptr(skip_out), B, F, H, dirs, frames, pitch,
                                           math, base, nbytes, st), "ctn_tas_lstm_fwd")
                z = out
            skip = z if blk == 0 else skip_out
        return skip

    def forward(self, input):
        """input (batch_size, n_basis, n_frames) -> mask (batch_size, n_sources, n_basis, n_frames)"""
        raise NotImplementedError("the stand-alone LSTM-TasNet Separator.forward (materialised mask) is not built; use TasNet")


class TasNet(nn.Module):
    """
        LSTM-TasNet
    """
    pretrained_model_ids = {
        "wsj0-mix": {
            8000: {
                2: "1-Abh-BdiqfypKxfA9H2doS3ATK4D2fVT",
                3: "1-1geGVvj7ZJk9c5EEcmLBCrZazjHTqjS"
            }
        }
    }

    def __init__(self, n_basis, kernel_size=40, stride=None, enc_basis=None, dec_basis=None, sep_num_blocks=2, sep_num_layers=2,
                 sep_hidden_channels=500, mask_nonlinear='softmax', causal=False, rnn_type='lstm', n_sources=2, eps=EPS, **kwargs):
        super().__init__()
        if stride is None:
            stride = kernel_size // 2
        assert kernel_size % stride == 0, "kernel_size is expected divisible by stride"
        assert enc_basis in ['trainable', 'trainableGated'] and dec_basis == 'trainable', \
            "enc_basis is expected 'trainable' or 'trainableGated'. dec_basis is expected 'trainable'."
        self.in_channels = kwargs.get('in_channels', 1)
        self.n_basis = n_basis
        self.kernel_size, self.stride = kernel_size, stride
        self.enc_basis, self.dec_basis = enc_basis, dec_basis
        self.sep_num_blocks, self.sep_num_layers = sep_num_blocks, sep_num_layers
        self.sep_hidden_channels = sep_hidden_channels
        self.causal = causal
        self.mask_nonlinear = mask_nonlinear
        self.rnn_type = rnn_type
        self.n_sources = n_sources
        self.eps = eps
        encoder, decoder = _choose_tasnet_filterbank(n_basis, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis,
                                                     dec_basis=dec_basis, **kwargs)
        self.encoder = encoder
        self.separator = Separator(n_basis, num_blocks=sep_num_blocks, num_layers=sep_num_layers, hidden_channels=sep_hidden_channels,
                                   causal=causal, mask_nonlinear=mask_nonlinear, rnn_type=rnn_type, n_sources=n_sources, eps=eps)
        self.decoder = decoder
        self.math = None

    def forward(self, input):
        output, _ = self._run(input, want_latent=False)
        return output

    def extract_latent(self, input):
        """input (batch_size, 1, T) -> output (batch_size, n_sources, T), latent (batch_size, n_sources, n_basis, T')"""
        return self._run(input, want_latent=True)

    def _run(self, input, want_latent):
        n_dims = input.dim()
        if n_dims == 4:
            raise NotImplementedError("4-D (multichannel) input is outside the sm_90a LSTM-TasNet path")
        if n_dims != 3:
            raise ValueError("Not support {} dimension input".format(n_dims))
        assert input.size(1) == 1, "input.size() is expected (?, 1, ?), but given {}".format(input.size())
        if self.in_channels != 1:
            raise NotImplementedError("in_channels={} (multichannel) is outside the sm_90a LSTM-TasNet path".format(self.in_channels))
        sep = self.separator
        sep.check_envelope()
        forward_only(self, input)
        B, _, T = input.shape
        L, stride = self.kernel_size, self.stride
        padding = (stride - (T - L) % stride) % stride
        if T + padding < L:
            raise ValueError("the input ({} samples) is too short for one frame of kernel_size={}".format(T, L))
        x = input.contiguous()
        dev = N.require_cuda(x)
        sep.check_hidden()
        frames, pl, pr = N.frames_of(T, L, stride)
        pitch = N.ctn_pitch(frames)
        math = math_of(self.math)
        st = N.stream_ptr(dev)
        Nb, S = self.n_basis, self.n_sources
        w = torch.empty(B, Nb, pitch, dtype=torch.float32, device=dev)
        xn = torch.empty(B, Nb, pitch, dtype=torch.float32, device=dev)
        gamma, beta = sep.gamma.reshape(-1), sep.beta.reshape(-1)
        if isinstance(self.encoder, GatedEncoder):
            nrm = torch.empty(B, dtype=torch.float64, device=dev)
            N.check(N.ctn_tas_enc_gated_fwd(x.data_ptr(), self.encoder.conv1d_U.weight.data_ptr(), self.encoder.conv1d_V.weight.data_ptr(),
                                            gamma.data_ptr(), beta.data_ptr(), w.data_ptr(), xn.data_ptr(), nrm.data_ptr(), B, T, pl, pr, Nb,
                                            L, stride, pitch, float(self.encoder.eps), float(sep.eps), st), "ctn_tas_enc_gated_fwd")
        else:
            N.check(N.ctn_encoder_fwd(x.data_ptr(), self.encoder.conv1d.weight.data_ptr(), w.data_ptr(), B, T, pl, pr, Nb, L, stride,
                                      int(self.encoder.nonlinear), pitch, None, st), "ctn_encoder_fwd")
            N.check(N.ctn_tas_frame_norm_fwd(w.data_ptr(), gamma.data_ptr(), beta.data_ptr(), xn.data_ptr(), B, Nb, frames, pitch,
                                             float(sep.eps), st), "ctn_tas_frame_norm_fwd")
        skip = sep.run_pitched(xn, frames, pitch, math, dev)
        Hd = sep.num_directions * sep.hidden_channels
        out = torch.empty(B, S, T, dtype=torch.float32, device=dev)
        latent = torch.empty(B, S, Nb, frames, dtype=torch.float32, device=dev) if want_latent else None
        what = torch.empty(B, S * Nb, pitch, dtype=torch.float32, device=dev)
        nws = N.ctn_tas_tail_workspace_bytes(Nb, Hd, S, math)
        base, nbytes = N.aligned(N.workspace(dev, nws + 256, tag="tas_tail"))
        N.check(N.ctn_tas_tail_fwd(skip.data_ptr(), w.data_ptr(), sep.fc.weight.data_ptr(), sep.fc.bias.data_ptr(),
                                   self.decoder.conv_transpose1d.weight.data_ptr(), out.data_ptr(), N.ptr(latent), what.data_ptr(), B, Nb, Hd,
                                   S, frames, pitch, L, stride, pl, T, int(sep.mask_softmax), math, base, nbytes, st), "ctn_tas_tail_fwd")
        return out, latent

    def online(self, batch_size=1, max_chunk=320):
        """-> a streaming separator of a causal, plain-encoder model for ``batch_size`` streams and pushes of up to ``max_chunk``
        samples (a multiple of the stride): see ``ctn_b200.models.online.TasOnlineSeparator``.  The numeric mode is fixed here."""
        from .online import TasOnlineSeparator
        return TasOnlineSeparator(self, batch_size, max_chunk)

    @classmethod
    def build_model(cls, model_path, load_state_dict=False):
        """tasnet.py:191-225"""
        config = _load_checkpoint(model_path)
        in_channels = config.get('in_channels') or 1
        n_basis = config.get('n_bases') or config['n_basis']
        kernel_size, stride = config['kernel_size'], config['stride']
        enc_basis, dec_basis = config.get('enc_bases') or config['enc_basis'], config.get('dec_bases') or config['dec_basis']
        enc_nonlinear = config.get('enc_nonlinear')
        sep_num_blocks, sep_num_layers = config['sep_num_blocks'], config['sep_num_layers']
        sep_hidden_channels = config['sep_hidden_channels']
        causal = config['causal']
        mask_nonlinear = config['mask_nonlinear']
        rnn_type = config.get('rnn_type', 'lstm')
        n_sources = config['n_sources']
        eps = config.get('eps') or EPS
        model = cls(n_basis, in_channels=in_channels, kernel_size=kernel_size, stride=stride, enc_basis=enc_basis, dec_basis=dec_basis,
                    enc_nonlinear=enc_nonlinear, sep_num_blocks=sep_num_blocks, sep_num_layers=sep_num_layers,
                    sep_hidden_channels=sep_hidden_channels, mask_nonlinear=mask_nonlinear, causal=causal, rnn_type=rnn_type,
                    n_sources=n_sources, eps=eps)
        if load_state_dict:
            model.load_state_dict(config['state_dict'])
        return model

    @classmethod
    def build_from_pretrained(cls, root="./pretrained", quiet=False, load_state_dict=True, **kwargs):
        """tasnet.py:227-267: <root>/<class>/wsj0-mix/sr<rate>/<n>speakers/model/<choice>.pth, loaded, never downloaded"""
        return build_from_pretrained(cls, root, load_state_dict, **kwargs)

    @property
    def num_parameters(self):
        return sum(p.numel() for p in self.parameters() if p.requires_grad)

    def get_config(self):
        return {
            'in_channels': self.in_channels, 'n_basis': self.n_basis, 'kernel_size': self.kernel_size, 'stride': self.stride,
            'enc_basis': self.enc_basis, 'dec_basis': self.dec_basis, 'sep_num_blocks': self.sep_num_blocks,
            'sep_num_layers': self.sep_num_layers, 'sep_hidden_channels': self.sep_hidden_channels, 'causal': self.causal,
            'mask_nonlinear': self.mask_nonlinear, 'rnn_type': self.rnn_type, 'n_sources': self.n_sources, 'eps': self.eps,
        }
