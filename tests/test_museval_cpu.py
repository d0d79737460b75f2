"""BSS Eval v4 of source images without a GPU: the fp64 oracle against an independent QR formulation, museval's host logic
(padding and truncation, the (nsrc, nsampl, nchan) layout, the window count, eval_track's targets and its vocals / accompaniment
call, the median of the frames) and the C ABI's refusals, each returned before any CUDA call."""
import ctypes as C

import numpy as np
import pytest
import torch

import museval_ref as R
from ctn_b200 import _native as N
from ctn_b200.utils import museval as MV

FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced: every call below is refused before it would be


# (J, I, T, win, hop, coloured): M L <= 2048, windows with hop = win, hop < win, hop > win and win = T
@pytest.mark.parametrize("J,I,T,win,hop,coloured", [(1, 1, 2000, 700, 700, False), (2, 1, 2500, 900, 500, False),
                                                    (1, 2, 2600, 1000, 1300, False), (2, 2, 3000, 3000, 3000, False),
                                                    (2, 2, 3500, 800, 800, True)])
def test_oracle_matches_qr(J, I, T, win, hop, coloured):
    refs, ests = R.make_track(np.random.default_rng(J * 100 + I * 10 + T), J, I, T, coloured)
    a = R.metrics(refs, ests, win, hop, R.filters_fft)
    b = R.metrics(refs, ests, win, hop, R.filters_qr)
    tol = 1e-6 if coloured else 1e-8  # coloured references square a worse condition number in the normal equations
    assert a[0].shape == (J, R.nwin_of(T, win, hop))
    for x, y in zip(a, b):
        finite = np.isfinite(y)
        assert np.array_equal(finite, np.isfinite(x))
        assert np.all(np.abs(x[finite] - y[finite]) <= tol), np.max(np.abs(x[finite] - y[finite]))
    if J == 1:
        assert np.isposinf(a[2]).all()  # one source: P_all = P_j, no interference


def test_oracle_silence_rules():
    refs, ests = R.make_track(np.random.default_rng(4), 2, 2, 3000, False)
    refs[1, :, 1000:1500] = 0            # window 2 of 500 samples: a silent stem
    ests[0, :, 2000:2500] = 0            # window 4: a silent estimate
    refs[0, 1, 2500:3000] = -refs[0, 0, 2500:3000]  # window 5: an anti-phase stereo stem sums to zero
    sdr = R.metrics(refs, ests, 500, 500)[0]
    assert np.isnan(sdr[:, [2, 4, 5]]).all() and not np.isnan(sdr[:, [0, 1, 3]]).any()


def test_window_count():
    assert [R.nwin_of(*a) for a in ((44100 * 60, 44100, 44100), (1000, 1000, 1000), (1000, 400, 300), (1000, 300, 400),
                                    (999, 1000, 1000))] == [60, 1, 3, 2, 0]


def test_padding_and_layout(monkeypatch):
    seen = []

    def fake(ref, est, window, hop):
        seen.append((ref.clone(), est.clone(), window, hop))
        n = (ref.shape[2] - window + hop) // hop
        return tuple(torch.full((ref.shape[0], n), float(q)) for q in range(4))

    monkeypatch.setattr(MV, "bss_eval_images_v4", fake)
    ref = np.arange(2 * 10 * 2, dtype=np.float64).reshape(2, 10, 2)  # (nsrc, nsampl, nchan)
    long_est = np.ones((2, 13, 2))
    out = MV.evaluate(ref, long_est, win=4, hop=3)
    r, e, w, h = seen[-1]
    assert (w, h) == (4, 3) and r.shape == (2, 2, 10) and e.shape == (2, 2, 10)  # (J, I, T), estimates cut to T
    assert torch.equal(r[1, 0], torch.from_numpy(ref[1, :, 0]).float())
    assert [o.shape for o in out] == [(2, 3)] * 4 and all(isinstance(o, np.ndarray) for o in out)
    MV.evaluate(torch.from_numpy(ref), torch.ones(2, 7, 2), win=4, hop=3)
    e = seen[-1][1]
    assert torch.equal(e[:, :, :7], torch.ones(2, 2, 7)) and not e[:, :, 7:].any()  # zero-padded at the end
    with pytest.raises(ValueError):
        MV.evaluate(ref, long_est, padding=False)
    MV.evaluate(ref[..., 0], long_est[..., 0], win=4, hop=3)  # (nsrc, nsampl): one channel
    assert seen[-1][0].shape == (2, 1, 10)
    with pytest.raises(NotImplementedError):
        MV.evaluate(ref, ref, mode="v3")


def test_eval_track_targets(monkeypatch):
    calls = []

    def fake(references, estimates, win, hop, mode="v4", padding=True):
        calls.append(([float(np.asarray(r)[0, 0]) for r in references], win, hop))
        return tuple(np.array([[10.0 * i + q] for i in range(len(references))]) for q in range(4))

    monkeypatch.setattr(MV, "evaluate", fake)
    names = ["vocals", "drums", "bass", "other", "accompaniment", "linear_mixture"]
    refs = {k: np.full((8, 2), float(i)) for i, k in enumerate(names)}
    est = {k: np.zeros((8, 2)) for k in ("bass", "accompaniment", "vocals", "drums", "other")}
    s = MV.eval_track(refs, est, 44100, win=1.0, hop=0.5)
    # the track's order, linear_mixture dropped (no estimate), accompaniment left to the second call
    assert calls == [([0.0, 1.0, 2.0, 3.0], 44100, 22050), ([0.0, 4.0], 44100, 22050)]
    assert list(s) == ["drums", "bass", "other", "vocals", "accompaniment"]
    assert s["vocals"]["SDR"][0] == 0.0 and s["accompaniment"]["ISR"][0] == 11.0 and s["bass"]["SAR"][0] == 23.0
    calls.clear()
    s = MV.eval_track(refs, {k: est[k] for k in ("drums", "bass")}, 44100)
    assert calls == [([1.0, 2.0], 44100, 44100)] and list(s) == ["drums", "bass"]
    calls.clear()
    s = MV.eval_track(refs, {k: est[k] for k in ("vocals", "accompaniment")}, 44100)
    assert calls == [([0.0, 4.0], 44100, 44100)] and list(s) == ["vocals", "accompaniment"]
    calls.clear()
    with pytest.warns(UserWarning, match="at least two estimates"):
        assert MV.eval_track(refs, {"drums": est["drums"]}, 44100) == {}
    assert calls == []


def test_frames_median():
    s = {"drums": {"SDR": np.array([1.0, np.nan, 3.0, 10.0]), "ISR": np.array([np.nan, np.nan]), "SIR": np.array([np.inf, 0.0, 1.0]),
                   "SAR": np.array([2.0])}}
    m = MV.frames_median(s)["drums"]
    assert m["SDR"] == 3.0 and np.isnan(m["ISR"]) and m["SIR"] == 1.0 and m["SAR"] == 2.0


def _call(**kw):
    a = dict(ref=FAKE, est=FAKE, J=4, I=2, T=44100 * 4, win=44100, hop=44100, sdr=FAKE, isr=FAKE, sir=FAKE, sar=FAKE, status=FAKE,
             ws=FAKE, ws_bytes=1 << 40, stream=None)
    a.update(kw)
    return N.ctn_bss_eval_images(*a.values())


def test_abi_rejections():
    for name in ("ctn_bss_images_workspace_bytes", "ctn_bss_eval_images"):
        assert hasattr(N.lib, name) and name in N.EXPORTED
    for bad in (dict(ref=None), dict(est=None), dict(sdr=None), dict(isr=None), dict(sir=None), dict(sar=None), dict(status=None),
                dict(ws=None), dict(J=0), dict(I=0), dict(T=0), dict(J=-1), dict(win=0), dict(hop=0), dict(hop=-3),
                dict(win=44100 * 4 + 1), dict(T=44099)):
        assert _call(**bad) == N.CTN_EINVAL, bad
    for bad in (dict(J=5, I=2), dict(J=9, I=1), dict(J=1, I=9), dict(J=3, I=3), dict(J=1 << 16, I=1 << 16)):
        assert _call(**bad) == N.CTN_EUNSUPPORTED, bad
    assert _call(ws=FAKE + 8) == N.CTN_EALIGN
    assert _call(ws_bytes=1024) == N.CTN_EWORKSPACE
    n = C.c_size_t(0)
    assert N.ctn_bss_images_workspace_bytes(5, 2, 44100, 44100, 44100, C.byref(n)) == N.CTN_EUNSUPPORTED
    assert N.ctn_bss_images_workspace_bytes(4, 2, 100, 200, 100, C.byref(n)) == N.CTN_EINVAL  # nwin = 0
    assert N.ctn_bss_images_workspace_bytes(4, 2, 44100, 44100, 44100, None) == N.CTN_EINVAL


@pytest.mark.parametrize("J,I", [(1, 1), (2, 2), (4, 2), (8, 1)])
def test_workspace_depends_on_windows_not_samples(J, I):
    def size(T, win, hop):
        n = C.c_size_t(0)
        assert N.ctn_bss_images_workspace_bytes(J, I, T, win, hop, C.byref(n)) == N.CTN_OK
        return n.value
    # 60 windows either way: 1 s windows of a 60 s track, or 10 s windows hopping by 1 s over 69 s
    a, b = size(44100 * 60, 44100, 44100), size(44100 * 69, 441000, 44100)
    assert a == b
    assert size(44100 * 240, 44100, 44100) > a  # 240 windows keep more partial energies
    # G, its diagonal blocks and the correlation partial sums dominate
    M = J * I
    floor = 8 * ((M * 512) ** 2 + J * (I * 512) ** 2 + 2 * M * 128 * M * 512)
    assert floor < a < floor + (64 << 20)
