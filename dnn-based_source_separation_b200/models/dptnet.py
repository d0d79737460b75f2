from ctn_b200.models.dptnet import *  # noqa: F401,F403
