from ctn_b200.models.galrnet import *  # noqa: F401,F403
