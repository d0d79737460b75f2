"""ctn_b200 -- H100-native Conv-TasNet separation path (sm_90a CUDA behind the reference's class API).

    from ctn_b200.models.conv_tasnet import ConvTasNet
    from ctn_b200.criterion.sdr import NegSISDR
    from ctn_b200.criterion.pit import PIT1d

The parent directory also carries ``models/ modules/ criterion/ utils/`` shim packages so that putting it on
PYTHONPATH in place of the reference's ``src/`` makes ``from models.conv_tasnet import ConvTasNet`` resolve here
(the reference's own drop-in mechanism, egs/wsj0-mix/conv-tasnet/path.sh:3-4).
"""
from . import _native  # noqa: F401  (raises if the CUDA extension is not built: no CPU fallback)

__version__ = "0.1.0"


def set_default_math(mode: str) -> None:
    """'f16x3' (wgmma 3-pass fp16 split, fp32-parity; the default when the tensor-core family is built), 'tf32x3' (3-pass TF32 split),
    'tf32' (single pass, looser tolerance) or 'fp32' (CUDA-core FFMA).  One switch for every model class (ConvTasNet, DPRNNTasNet,
    stand-alone TimeDilatedConvNet / Separator): it lives in models.tdcn.DEFAULT_MATH."""
    from .models import tdcn
    if mode not in _native.MATH_NAMES:
        raise ValueError(f"unknown math mode {mode!r}; choose from {sorted(_native.MATH_NAMES)}")
    tdcn.DEFAULT_MATH = mode
