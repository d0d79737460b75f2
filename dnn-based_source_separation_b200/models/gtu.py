from ctn_b200.models.gtu import *  # noqa: F401,F403
