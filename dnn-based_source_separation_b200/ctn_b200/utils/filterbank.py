"""choose_filterbank mirroring src/utils/filterbank.py:5-46: only the trainable encoder / decoder pair is in the
kernel envelope; Fourier / pinv / gated bases raise NotImplementedError (SURVEY.md 8b unsupported-config policy)."""
from ..models.filterbank import Encoder, Decoder

EPS = 1e-12


def choose_filterbank(hidden_channels, kernel_size, stride=None, enc_basis='trainable', dec_basis='trainable', **kwargs):
    in_channels = kwargs.get('in_channels') or 1
    if enc_basis != 'trainable':
        raise NotImplementedError("Not support {} for encoder (sm_90a path: 'trainable' only)".format(enc_basis))
    if dec_basis != 'trainable':
        raise NotImplementedError("Not support {} for decoder (sm_90a path: 'trainable' only)".format(dec_basis))
    encoder = Encoder(in_channels, hidden_channels, kernel_size, stride=stride, nonlinear=kwargs.get('enc_nonlinear'))
    decoder = Decoder(hidden_channels, in_channels, kernel_size, stride=stride)
    return encoder, decoder
