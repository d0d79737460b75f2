from ctn_b200.models.transformer import *  # noqa: F401,F403
