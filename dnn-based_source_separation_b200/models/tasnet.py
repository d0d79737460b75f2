from ctn_b200.models.tasnet import *  # noqa: F401,F403
