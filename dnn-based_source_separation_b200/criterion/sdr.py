from ctn_b200.criterion.sdr import sdr, SDR, NegSDR, sisdr, SISDR, NegSISDR, EPS  # noqa: F401
