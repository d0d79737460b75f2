from ctn_b200.criterion.pit import pit, PIT, PIT1d, PIT2d, ORPIT, sinkpit, SinkPIT  # noqa: F401
