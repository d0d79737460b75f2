"""Factories mirroring src/utils/tasnet.py:14-31 of the reference."""
from ..modules.norm import GlobalLayerNorm, CumulativeLayerNorm1d

EPS = 1e-12


def choose_layer_norm(name, num_features, causal=False, eps=EPS, **kwargs):
    if name == 'cLN':
        return CumulativeLayerNorm1d(num_features, eps=eps)
    if name == 'gLN':
        if causal:
            raise ValueError("Global Layer Normalization is NOT causal.")
        return GlobalLayerNorm(num_features, eps=eps)
    if name in ('BN', 'batch', 'batch_norm'):
        raise NotImplementedError("BatchNorm is outside the sm_90a Conv-TasNet path (only 'gLN' / 'cLN').")
    raise NotImplementedError("Not support {} layer normalization.".format(name))
