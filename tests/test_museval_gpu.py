"""BSS Eval v4 of source images on the GPU (ctn_bss_eval_images) against the fp64 oracle of tests/museval_ref.py: every SDR / ISR /
SIR / SAR within 1e-4 dB (the bound bss_eval_sources is held to), NaN and +inf where the oracle has them; the silence rules, a
perfect estimate, the rank-deficient refusal, repeat bits and a CUDA-graph replay, the launch count, the all-columns solve, and one
eval_track call at MUSDB shape."""
import ctypes as C

import numpy as np
import pytest
import torch

import museval_ref as R
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu

TOL_DB = 1e-4
SR = 44100


def _mv():
    from ctn_b200.utils import museval
    return museval


def _compare(tag, got, want):
    """got, want: SDR, ISR, SIR, SAR (J, nwin); NaN and +-inf at the same places, finite values within TOL_DB"""
    worst = []
    for name, g, o in zip(("SDR", "ISR", "SIR", "SAR"), got, want):
        g = np.asarray(g)
        assert g.shape == o.shape and g.dtype == np.float64, (name, g.shape, o.shape)
        assert np.array_equal(np.isnan(g), np.isnan(o)), (name, g, o)
        assert np.array_equal(g[np.isinf(o)], o[np.isinf(o)]) and np.array_equal(np.isinf(g), np.isinf(o)), (name, g, o)
        fin = np.isfinite(o)
        err = float(np.max(np.abs(g[fin] - o[fin]))) if fin.any() else 0.0
        worst.append(err)
        assert err <= TOL_DB, (name, err)
    print("museval {}: worst |dSDR| {:.2e} |dISR| {:.2e} |dSIR| {:.2e} |dSAR| {:.2e} dB".format(tag, *worst))


def _limit(J, I):
    """the shortest T at which the M L delayed references can be independent: T + L - 1 >= M L"""
    return J * I * 512 - 511


# (J, I, T, win, hop, coloured): every (J, I); T just above the rank limit, 5 s and 30 s; hop = win, hop < win, hop > win, win = T.
# Near the rank limit the references are white: low-pass ones make G so ill-conditioned there that the oracle's own LU solve and
# its QR route part by about the bound.
ROWS = [(1, 1, 1000, 400, 400, False), (2, 1, _limit(2, 1) + 100, 300, 150, False), (1, 2, 5 * SR, SR, SR, True),
        (2, 2, _limit(2, 2) + 100, _limit(2, 2) + 100, 1, False), (2, 2, 30 * SR, SR, SR // 2, False),
        (3, 2, 5 * SR, SR, 60000, True), (3, 2, _limit(3, 2) + 200, 1000, 700, False), (4, 2, _limit(4, 2) + 100, 1000, 900, False),
        (4, 2, 5 * SR, SR, SR, False), (4, 2, 30 * SR, SR, SR, True)]


@pytest.mark.parametrize("J,I,T,win,hop,coloured", ROWS)
def test_against_oracle(J, I, T, win, hop, coloured):
    mv = _mv()
    refs, ests = R.make_track(np.random.default_rng(J * 1000 + I * 100 + T % 997), J, I, T, coloured)
    got = mv.bss_eval_images_v4(torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda(), win, hop)
    assert all(t.is_cuda for t in got)
    _compare("J={} I={} T={} win={} hop={} {}".format(J, I, T, win, hop, "coloured" if coloured else "white"),
             [t.cpu().numpy() for t in got], R.metrics(refs, ests, win, hop))


def test_silent_windows():
    """a stem silent in one window, an estimate silent in another, an anti-phase stereo stem in a third: NaN for every source"""
    mv = _mv()
    win = SR // 2
    refs, ests = R.make_track(np.random.default_rng(31), 2, 2, 5 * SR, True)
    refs[1, :, 3 * win:4 * win] = 0
    ests[0, :, 5 * win:6 * win] = 0
    refs[0, 1, 7 * win:8 * win] = -refs[0, 0, 7 * win:8 * win]
    got = [t.numpy() for t in mv.bss_eval_images_v4(torch.from_numpy(refs), torch.from_numpy(ests), win, win)]  # CPU in, CPU out
    want = R.metrics(refs, ests, win, win)
    assert np.isnan(want[0][:, [3, 5, 7]]).all() and np.isfinite(np.delete(want[0], [3, 5, 7], axis=1)).all()
    _compare("silent windows", got, want)


def test_perfect_estimate():
    mv = _mv()
    refs, _ = R.make_track(np.random.default_rng(32), 2, 2, 3 * SR, False)
    sdr, isr, sir, sar = (t.numpy() for t in mv.bss_eval_images_v4(torch.from_numpy(refs), torch.from_numpy(refs)))
    print("museval e = r: SDR", sdr.min(), "ISR", isr.min(), "SIR", sir.min(), "SAR", sar.min())
    assert np.isposinf(sdr).all()
    assert np.all((isr > 150.0) | np.isposinf(isr))


def test_rank_deficient_is_refused():
    """M L > T + L - 1: G cannot be positive definite; museval would fall back to lstsq, this path says so"""
    mv = _mv()
    refs, ests = R.make_track(np.random.default_rng(33), 4, 2, _limit(4, 2) - 600, False)
    with pytest.raises(ValueError, match="positive definite"):
        mv.bss_eval_images_v4(torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda(), 1000, 1000)


def _raw(ref, est, win, hop, outs, status):
    J, I, T = ref.shape
    n = C.c_size_t(0)
    N.check(N.ctn_bss_images_workspace_bytes(J, I, T, win, hop, C.byref(n)))
    base, avail = N.aligned(N.workspace(ref.device, n.value + 256, "bss_images_test"))
    N.check(N.ctn_bss_eval_images(ref.data_ptr(), est.data_ptr(), J, I, T, win, hop, *(t.data_ptr() for t in outs), status.data_ptr(),
                                  base, avail, N.stream_ptr(ref.device)), "ctn_bss_eval_images")


@pytest.mark.parametrize("J,I", [(1, 1), (2, 1), (1, 2), (2, 2), (3, 2), (4, 2)])
def test_repeat_bits_graph_replay_and_launches(J, I):
    refs, ests = R.make_track(np.random.default_rng(40 + J * I), J, I, 3 * SR, True)
    ref, est = torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda()
    win, hop = SR, SR // 2
    nwin = R.nwin_of(3 * SR, win, hop)
    outs = [torch.empty((J, nwin), dtype=torch.float64, device="cuda") for _ in range(4)]
    status = torch.empty(1, dtype=torch.int32, device="cuda")
    _raw(ref, est, win, hop, outs, status)
    launches = N.ctn_last_launch_count()
    first = [t.clone() for t in outs]
    _raw(ref, est, win, hop, outs, status)
    assert all(torch.equal(a, b) for a, b in zip(first, outs)) and int(status) == 0
    # stages: silence, correlations, combine, build; Cholesky 3 nt - 2 per matrix set; solves 2 nt per set; projection, finish
    ntg, ntb = 8 * J * I, 8 * I
    assert launches == 4 + (3 * ntg - 2) + (3 * ntb - 2) + 2 * ntg + 2 * ntb + 2, launches
    for t in outs:
        t.zero_()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            _raw(ref, est, win, hop, outs, status)
    torch.cuda.current_stream().wait_stream(s)
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(first, outs))
    print("museval J={} I={}: {} launches, bit-identical repeat and graph replay".format(J, I, launches))


_p, _i = C.c_void_p, C.c_int
probe_factor = N._sig("ctn_probe_chol_factor", _i, _p, _p, _p, _i, _i, _p)
probe_solve = N._sig("ctn_probe_chol_solve", _i, _p, _p, _p, _p, _i, _i, _i, _i, _p)


@pytest.mark.parametrize("n,nmat,nrhs", [(512, 2, 1), (1024, 1, 8), (1536, 3, 2)])
def test_all_columns_solve(n, nmat, nrhs):
    """the all-columns solve against numpy and against the one-CTA-per-column solve on the same factor"""
    rng = np.random.default_rng(n + nrhs)
    A = np.stack([(lambda X: X.T @ X / n + 0.1 * np.eye(n))(rng.standard_normal((n + 64, n))) for _ in range(nmat)])
    B = rng.standard_normal((nmat, n, nrhs))
    dA = torch.from_numpy(A).cuda()
    W = torch.empty((nmat, n // 64, 64, 64), dtype=torch.float64, device="cuda")
    flag = torch.empty(nmat, dtype=torch.int32, device="cuda")
    N.check(probe_factor(dA.data_ptr(), W.data_ptr(), flag.data_ptr(), n, nmat, None))
    X = torch.from_numpy(B).cuda()
    tmp = torch.empty_like(X)
    N.check(probe_solve(dA.data_ptr(), W.data_ptr(), X.data_ptr(), tmp.data_ptr(), n, nmat, nrhs, 1, None))
    cols = torch.from_numpy(B.transpose(0, 2, 1).copy()).cuda()
    N.check(probe_solve(dA.data_ptr(), W.data_ptr(), cols.data_ptr(), None, n, nmat, nrhs, 0, None))
    torch.cuda.synchronize()
    assert not flag.any()
    want = np.linalg.solve(A, B)
    x = X.cpu().numpy()
    err = np.max(np.abs(x - want)) / np.max(np.abs(want))
    err_cols = np.max(np.abs(x - cols.cpu().numpy().transpose(0, 2, 1))) / np.max(np.abs(want))
    print("all-columns solve n={} nmat={} nrhs={}: rel err {:.1e} vs numpy, {:.1e} vs per-column".format(n, nmat, nrhs, err, err_cols))
    assert err < 1e-11 and err_cols < 1e-12


def test_eval_track_musdb_shape():
    """4 stems plus accompaniment, stereo, 60 s: both museval calls against the oracle"""
    mv = _mv()
    T = 60 * SR
    refs, ests = R.make_track(np.random.default_rng(50), 4, 2, T, True)
    names = ["vocals", "drums", "bass", "other"]
    acc_ref = (refs[1] + refs[2] + refs[3]).astype(np.float32)
    acc_est = (ests[1] + ests[2] + ests[3]).astype(np.float32)
    references = {k: refs[i].T for i, k in enumerate(names)}
    references["accompaniment"] = acc_ref.T
    estimates = {k: ests[i].T for i, k in enumerate(names)}
    estimates["accompaniment"] = acc_est.T
    scores = mv.eval_track(references, estimates, SR)
    assert list(scores) == ["drums", "bass", "other", "vocals", "accompaniment"]
    four = R.metrics(refs, ests, SR, SR)
    two = R.metrics(np.stack([refs[0], acc_ref]), np.stack([ests[0], acc_est]), SR, SR)
    for i, k in enumerate(names[1:], 1):
        _compare("eval_track " + k, [scores[k][m][None] for m in mv.METRICS], [x[i:i + 1] for x in four])
    for i, k in enumerate(["vocals", "accompaniment"]):
        _compare("eval_track " + k, [scores[k][m][None] for m in mv.METRICS], [x[i:i + 1] for x in two])
    med = mv.frames_median(scores)
    print("museval eval_track medians:", {k: {m: round(v, 3) for m, v in d.items()} for k, d in med.items()})
