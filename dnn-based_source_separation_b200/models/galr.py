from ctn_b200.models.galr import *  # noqa: F401,F403
