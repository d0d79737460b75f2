from ctn_b200.models.lstm_tasnet import *  # noqa: F401,F403
