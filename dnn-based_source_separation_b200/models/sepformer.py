from ctn_b200.models.sepformer import *  # noqa: F401,F403
