"""src/models/lstm_tasnet.py: LSTMTasNet is the reference's alias of TasNet."""
from .tasnet import TasNet

LSTMTasNet = TasNet  # for alias
