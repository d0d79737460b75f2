from ctn_b200.utils.bss import bss_eval_sources  # noqa: F401
