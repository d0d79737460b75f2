"""The multichannel filter banks one kernel at a time against fp64 (``-m gpu``): ctn_encoder_mc_fwd, ctn_decoder_mc_fwd and the
channel weight gradient (ctn_probe_encdec_wgrad_mc) at every row of tests/mc_filterbank_ref.py, whose `reaches` text names the
kernel, branch and constant each row selects; then whole multichannel training steps at the geometries those rows single out.

Every output buffer starts as NaN, and sits between NaN guards that must stay NaN.  Every input sits inside a NaN-filled
allocation (x, sig) or carries NaN past `frames` in its pitch (w_hat, act): a cell never written, a write out of range or a read
past the valid range shows in the result.  dW accumulates, so it starts from a random base.  The bounds are derived in
mc_filterbank_ref.py from each kernel's summation order; every row prints its worst error as a share of its bound.
"""
import pytest
import torch

import convtasnet_oracle as O
import mc_filterbank_ref as R
from ctn_b200 import _native as N
from test_multichannel_train_gpu import _inputs, _run_case
from test_train_edges_gpu import MODES

pytestmark = pytest.mark.gpu

GUARD = 64  # NaN floats before and after every buffer (256 bytes: alignment is kept)
probe_wgrad_mc = N._sig("ctn_probe_encdec_wgrad_mc", N._i, N._fp, N._fp, N._fp, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i,
                        N._fp)


def _guarded(values, off=0):
    """a NaN-filled device allocation holding `values` (float32) `off` floats past a 256-byte boundary; -> (buffer, view)"""
    n = values.numel()
    buf = torch.full((2 * GUARD + off + n,), float("nan"), device="cuda")
    view = buf[GUARD + off:GUARD + off + n]
    view.copy_(values.reshape(-1).float())
    return buf, view.view(values.shape)


def _guards_intact(buf, off, n):
    return bool(torch.isnan(buf[:GUARD + off]).all()) and bool(torch.isnan(buf[GUARD + off + n:]).all())


def _pitched(v, pitch):
    """(..., frames) -> (..., pitch) with NaN in [frames, pitch)"""
    out = torch.full(v.shape[:-1] + (pitch,), float("nan"), dtype=torch.float64)
    out[..., :v.shape[-1]] = v
    return out


def _share(v, ref, bound):
    err = (v.double() - ref).abs()
    assert not bool(torch.isnan(err).any()), "NaN in the output: a cell never written, or a read past the valid range"
    return float((err / bound.clamp_min(1e-300)).max()), bool((err <= bound).all())


# ---- encoder -----------------------------------------------------------------------------------------------------------------
def _run_encoder(r, x, W, stats):
    pitch = R.enc_pitch(r)
    wbuf, w = _guarded(torch.full((r.B, r.N, pitch), float("nan")), r.w_off)
    st = torch.zeros(r.B, 2, dtype=torch.float64, device="cuda") if stats else None
    rc = N.ctn_encoder_mc_fwd(x.data_ptr(), W.data_ptr(), w.data_ptr(), r.B, r.C, R.enc_T(r), r.pl, r.pr, r.N, r.L, r.S, int(r.relu),
                              pitch, st.data_ptr() if stats else None, None)
    N.check(rc, "ctn_encoder_mc_fwd")
    launches = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert _guards_intact(wbuf, r.w_off, w.numel()), "a store outside w"
    return w.cpu(), (st.cpu() if stats else None), launches


@pytest.mark.parametrize("name", list(R.ENC))
def test_encoder_vs_fp64(name):
    r = R.ENC[name]
    kernel, _ = R.encoder_kernel(r)
    x64, W64 = R.enc_inputs(name, r)
    ref, mag = R.encoder(x64, W64, r.S, r.pl, r.pr, r.relu)
    bound = R.encoder_bound(r, mag)
    _, x = _guarded(x64)
    _, W = _guarded(W64)
    w, stats, launches = _run_encoder(r, x, W, r.stats)
    assert launches == 1, launches
    share, ok = _share(w[..., :r.frames], ref, bound)
    assert ok, "{} ({}): {:.2f}x the dot-product bound".format(name, kernel, share)
    assert bool((w[..., r.frames:] == 0).all()), "the padding columns [frames, w_pitch) must be exactly 0"
    worst_stats, n_cta = 0.0, -(-R.enc_pitch(r) // 128)
    if r.stats:
        own = w[..., :r.frames].double()
        for b in range(r.B):
            bs, bq = R.stats_bound(kernel != "k_encoder_mc", own[b], r.N, n_cta)
            es, eq = abs(float(stats[b, 0]) - float(own[b].sum())), abs(float(stats[b, 1]) - float((own[b] ** 2).sum()))
            assert es <= bs and eq <= bq, "{} sample {}: statistics {:.2f}x / {:.2f}x their bounds".format(name, b, es / bs, eq / bq)
            worst_stats = max(worst_stats, es / bs, eq / bq)
    w2, stats2, _ = _run_encoder(r, x, W, r.stats)
    assert torch.equal(w2, w), "a second call gave different bits"
    if r.stats:  # float atomics of the per-CTA partials land in any order
        for b in range(r.B):
            bs, bq = R.stats_bound(kernel != "k_encoder_mc", w[b, :, :r.frames].double(), r.N, n_cta)
            assert abs(float(stats2[b, 0] - stats[b, 0])) <= 2 * bs and abs(float(stats2[b, 1] - stats[b, 1])) <= 2 * bq
    print("[mc encoder {}] {:.3f} of the bound, statistics {:.3f} -- {}".format(name, share, worst_stats, r.reaches))


# ---- decoder -----------------------------------------------------------------------------------------------------------------
def _run_decoder(r, what, Wd, crop, T_out):
    ybuf, y = _guarded(torch.full((r.BS, r.C, T_out), float("nan")))
    N.check(N.ctn_decoder_mc_fwd(what.data_ptr(), Wd.data_ptr(), y.data_ptr(), r.BS, r.C, r.N, r.frames, r.pitch, r.S * r.R, r.S, crop,
                                 T_out, None), "ctn_decoder_mc_fwd")
    launches = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert _guards_intact(ybuf, 0, y.numel()), "a store outside y"
    return y.cpu(), launches


@pytest.mark.parametrize("name", list(R.DEC))
def test_decoder_vs_fp64(name):
    r = R.DEC[name]
    kernel, _ = R.decoder_kernel(r)
    what64, Wd64 = R.dec_inputs(name, r)
    crop, T_out = R.dec_geometry(r)
    ref, mag = R.decoder(what64, Wd64, r.S, crop, T_out)
    bound = R.decoder_bound(r, kernel, mag)
    _, what = _guarded(_pitched(what64, r.pitch))
    _, Wd = _guarded(Wd64)
    y, launches = _run_decoder(r, what, Wd, crop, T_out)
    assert launches == 1, launches
    share, ok = _share(y, ref, bound)
    assert ok, "{} ({}): {:.2f}x the dot-product bound".format(name, kernel, share)
    assert torch.equal(_run_decoder(r, what, Wd, crop, T_out)[0], y), "a second call gave different bits"
    print("[mc decoder {}] {:.3f} of the bound -- {}".format(name, share, r.reaches))


# ---- weight gradient ---------------------------------------------------------------------------------------------------------
def _run_wgrad(r, act, sig, base):
    dW = base.float().cuda()
    n0 = N.ctn_total_launch_count()
    rc = probe_wgrad_mc(act.data_ptr(), sig.data_ptr(), dW.data_ptr(), r.R, r.N, r.C, r.frames, R.pitch128(r.frames), R.wg_T(r), r.L,
                        r.S, r.pl, None)
    assert rc == 0, rc
    launches = N.ctn_total_launch_count() - n0
    torch.cuda.synchronize()
    return dW.cpu(), launches


@pytest.mark.parametrize("name", list(R.WG))
def test_wgrad_vs_fp64(name):
    r = R.WG[name]
    kernel, _ = R.wgrad_kernel(r)
    act64, sig64, base = R.wg_inputs(name, r)
    ref, mag = R.wgrad(act64, sig64, r.L, r.S, r.pl)
    bound = R.wgrad_bound(r, mag, base)
    _, act = _guarded(_pitched(act64, R.pitch128(r.frames)))
    _, sig = _guarded(sig64, r.sig_off)
    shares = []
    for _ in range(2):  # float atomics land in any order: the second call is held to the same bound, not to the same bits
        dW, launches = _run_wgrad(r, act, sig, base)
        assert launches == 1, launches
        share, ok = _share(dW.double() - base, ref, bound)
        assert ok, "{} ({}): {:.2f}x the summation bound".format(name, kernel, share)
        shares.append(share)
    print("[mc wgrad {}] {:.3f} / {:.3f} of the bound -- {}".format(name, shares[0], shares[1], r.reaches))


# ---- whole training steps ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(R.TRAIN))
def test_training_step_vs_fp64(case):
    """ConvTasNet(in_channels=C) with multichannel_training, driven by a seeded cotangent in the default mode: every gradient
    within 2e-4 of its role scale of fp64 autograd over the oracle (test_multichannel_train_gpu.py's criterion)"""
    e = R.TRAIN[case]
    cfg = O.OracleConfig(causal=False, in_channels=e.C, **e.shape)
    sd = O.synth_state_dict(cfg, seed=711)
    mixture, _, G = _inputs(cfg, e.batch, e.T, 712)
    _run_case(cfg, sd, mixture, G, ("mc-filterbank " + case, "G"), MODES[-1], e.reaches)
