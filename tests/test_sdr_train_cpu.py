"""The SDR training criterion without a GPU: the new C entries are exported and reject bad arguments before any CUDA call, the
PIT-over-SDR scratch is sized as documented, and the float64 restatements of tests/sdr_train_ref.py reproduce the reference's own
float64 answers in tests/golden/sdr_grad.pt (minted from the unmodified reference by tests/golden/make_golden_sdr_grad.py)."""
import math
import os

import pytest
import torch

import sdr_train_ref as R
from ctn_b200 import _native as N

NEW = ["ctn_sdr_bwd", "ctn_sdr_pit_scratch_bytes", "ctn_sdr_pit_fwd", "ctn_sdr_pit_bwd"]
FAKE = 1 << 20  # a non-null pointer that is never dereferenced: every call below is rejected before any CUDA call


def _golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "sdr_grad.pt"), weights_only=False)


def test_new_symbols_exported():
    for name in NEW:
        assert name in N.EXPORTED and hasattr(N.lib, name), name


def test_sdr_pit_scratch_bytes():
    for B in (1, 3, 40000, 70001):
        for S in range(1, 7):
            assert N.ctn_sdr_pit_scratch_bytes(B, S) == 8 * B * (S * S + S), (B, S)


def test_sdr_bwd_rejections():
    call = lambda **kw: N.ctn_sdr_bwd(*{**dict(est=FAKE, tgt=FAKE, rows=3, T=100, eps=1e-12, scratch=FAKE, g=None, coef=1.0, d=FAKE,
                                               stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(scratch=None), dict(d=None), dict(rows=0), dict(rows=-2), dict(T=0),
                dict(T=-1)):
        assert call(**bad) == N.CTN_EINVAL, bad


def test_sdr_pit_fwd_rejections():
    fwd = lambda **kw: N.ctn_sdr_pit_fwd(*{**dict(est=FAKE, tgt=FAKE, B=2, S=2, T=100, eps=1e-12, loss_b=FAKE, perm=FAKE, mean=None,
                                                  pair=None, scratch=FAKE, stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(loss_b=None), dict(perm=None), dict(scratch=None), dict(B=0), dict(B=-1),
                dict(T=0), dict(T=-4)):
        assert fwd(**bad) == N.CTN_EINVAL, bad
    for S in (0, -1, 7, 16):
        assert fwd(S=S) == N.CTN_EUNSUPPORTED, S


def test_sdr_pit_bwd_rejections():
    bwd = lambda **kw: N.ctn_sdr_pit_bwd(*{**dict(est=FAKE, tgt=FAKE, perm=FAKE, B=2, S=2, T=100, eps=1e-12, scratch=FAKE, g=None,
                                                  coef=-0.5, d=FAKE, stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(perm=None), dict(scratch=None), dict(d=None), dict(B=0), dict(T=0)):
        assert bwd(**bad) == N.CTN_EINVAL, bad
    for S in (0, 7):
        assert bwd(S=S) == N.CTN_EUNSUPPORTED, S


@pytest.mark.parametrize("S", [2, 3])
def test_pit_restatement_matches_golden(golden_dir, S):
    """PIT1d(NegSDR(), S): the reference's float64 loss, pattern and gradient from the float64 restatement"""
    r = _golden(golden_dir)["pit"][S]
    x, t = r["input"], r["target"]
    p = R.pit64(x, t)
    assert torch.equal(p["perm"], r["pattern64"]) and torch.equal(p["perm"], r["pattern"])
    assert bool(R.separated(p).all())
    torch.testing.assert_close(p["loss_b"], r["loss_b64"], rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(p["loss_b"].mean(), r["loss64"], rtol=1e-12, atol=1e-12)
    B = x.shape[0]
    g = R.pit_grad64(x, t, p["perm"], torch.full((B,), 1.0 / B, dtype=torch.float64))
    torch.testing.assert_close(g, r["grad64"], rtol=1e-10, atol=1e-15)
    # the reference's own fp32 run sits inside the kernels' bounds (a bound at least as loose as fp32 autograd's rounding)
    assert bool(((r["loss_b"].double() - p["loss_b"]).abs() <= p["bound"]).all())


def test_musdb_restatement_matches_golden(golden_dir):
    """NegSDR() on the standardised (B, S, C, T) batch: value and gradient of -mean over (B, S, C) of the row SDRs"""
    r = _golden(golden_dir)["musdb"]
    x, t = r["input"], r["target"]
    rows = x.shape[0] * x.shape[1] * x.shape[2]
    torch.testing.assert_close(-R.sdr64(x, t).mean(), r["loss64"], rtol=1e-12, atol=1e-12)
    g = R.sdr_grad64(x, t, torch.full(x.shape[:-1], -1.0 / rows, dtype=torch.float64))
    torch.testing.assert_close(g, r["grad64"], rtol=1e-10, atol=1e-15)


def test_bounds_catch_the_wrong_arithmetic():
    """each bound rejects what a broken kernel would produce: a transposed pair table, a residual by expansion, a dropped eps"""
    g = torch.Generator().manual_seed(5)
    t = torch.randn(3, 3, 4000, generator=g)
    x = t[:, [2, 0, 1]] + 1e-3 * torch.randn(3, 3, 4000, generator=g)   # ~60 dB on the matching pairs
    v, vb = R.pair_tables(x, t)
    assert bool(((v.transpose(1, 2) - v).abs() > vb + vb.transpose(1, 2)).any()), "transposed table within the bound"
    tp = t[:, [2, 0, 1]]
    xd, td = x.double(), tp.double()
    ee_exp = (td * td).sum(-1).float() - 2 * (xd * td).sum(-1).float() + (xd * xd).sum(-1).float()   # fp32 expansion
    v_exp = 10 * torch.log10(((td * td).sum(-1) + R.EPS) / (ee_exp.double().abs() + R.EPS))
    assert bool(((v_exp - R.sdr64(x, tp)).abs() > R.sdr_bound(x, tp)).all()), "expanded residual within the bound"
    same = t[0, :1]
    tt = float((same.double() ** 2).sum())
    v = float(R.sdr64(same, same))
    assert math.isfinite(v) and math.isclose(v, 10 * math.log10((tt + R.EPS) / R.EPS), rel_tol=1e-12), "x == t needs eps"
    assert float(R.sdr_grad64(same, same, torch.ones(1, dtype=torch.float64)).abs().max()) == 0.0
