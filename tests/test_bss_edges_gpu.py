"""Edge rows of BSS EVAL V4 (ctn_bss_eval_images), BSS_EVAL_SOURCES (ctn_bss_eval_sources) and their shared CHOLESKY (``-m gpu``)
against the fp64 oracles of tests/museval_ref.py and tests/bss_ref.py.  Rows, restated launch geometry and the extra oracles live
in tests/bss_edges_ref.py; each row's ``reaches`` names the branch and the constant that selects it, and every output is NaN-filled
before the call.

  A1. every k_mus_project<M, I> of mus_project_dispatch just above the rank limit, with its launch count and repeat bits.
  A2. window geometry: win = 1, win < L, ntile = 64 / 65 / 130 (per = 1, 2, 3), win = T over 5 minutes, hop > win, 3000 windows.
  A3. a 7-minute 4-stem stereo track and its vocals / accompaniment call, on a subset of windows, NaN pattern everywhere.
  A4. a stem whose right channel is its left + delta noise, and MUSDB18-style 16 kHz low-passed stems.  A5. an exactly mono stem.
  B1-B7. bss_eval_sources: T below the filter length, the exact rank limit, chunk and tile edges, wsj0-mix "max" mode, 8 kHz
  content at 16 kHz, rank-deficient references, a batch of 200 items.
  C. the shared Cholesky and both solves: sizes 2048 .. 4096, one non-PD matrix in a batch, NaN / inf entries, and the backward
  error of both solve routes at kappa 1e2 .. 1e13 and on the near-singular Gram matrix of A4.

Bounds: 1e-4 dB per finite value with NaN / +inf at the oracle's places.  Where the oracle's own LU (the normal equations, as
museval and mir_eval solve them) and its SVD projection part, the bound is 1e-4 dB + 4 |LU - SVD| per value; a rank-deficient
row must either be refused (ValueError naming the Gram matrix) or meet that bound against the SVD projection."""
import ctypes as C

import numpy as np
import pytest
import scipy.signal
import torch

import bss_edges_ref as E
import bss_ref as BR
import museval_ref as MR
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu

TOL = E.TOL_DB
SR = E.SR
NOISE_DB = 80.0  # a residual at rounding level: both oracle routes above 120 dB, the GPU must be above this


# ---- museval v4 --------------------------------------------------------------------------------------------------------------
def _images(ref, est, win, hop):
    """raw ctn_bss_eval_images on NaN-filled outputs -> (SDR, ISR, SIR, SAR numpy (J, nwin), status, launches)"""
    J, I, T = ref.shape
    nwin = (T - win + hop) // hop
    n = C.c_size_t(0)
    N.check(N.ctn_bss_images_workspace_bytes(J, I, T, win, hop, C.byref(n)))
    assert n.value == E.mus_workspace_bytes(J, I, T, win, hop)
    base, avail = N.aligned(N.workspace(ref.device, n.value + 256, "bss_edges"))
    outs = [torch.full((J, nwin), float("nan"), dtype=torch.float64, device=ref.device) for _ in range(4)]
    status = torch.full((1,), -1, dtype=torch.int32, device=ref.device)
    N.check(N.ctn_bss_eval_images(ref.data_ptr(), est.data_ptr(), J, I, T, win, hop, *(t.data_ptr() for t in outs), status.data_ptr(),
                                  base, avail, N.stream_ptr(ref.device)), "ctn_bss_eval_images")
    launches = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in outs], int(status.item()), launches


def _compare(tag, got, want, bound=TOL):
    """NaN and +inf where the oracle has them, finite values within ``bound`` (scalar or per value); prints worst error / bound"""
    ratio, worst = 0.0, []
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), np.shape(want))
    for q, (name, g, o) in enumerate(zip(("SDR", "ISR", "SIR", "SAR"), got, want)):
        g, o = np.asarray(g), np.asarray(o)
        assert g.shape == o.shape, (name, g.shape, o.shape)
        assert np.array_equal(np.isnan(g), np.isnan(o)), (tag, name, g, o)
        assert np.array_equal(np.isposinf(g), np.isposinf(o)), (tag, name, g, o)
        fin = np.isfinite(o)
        err = np.abs(g[fin] - o[fin])
        worst.append(float(err.max()) if fin.any() else 0.0)
        if fin.any():
            ratio = max(ratio, float(np.max(err / bound[q][fin])))
    print("{}: worst |dSDR| {:.1e} |dISR| {:.1e} |dSIR| {:.1e} |dSAR| {:.1e} dB, worst error / bound {:.2e}".format(tag, *worst, ratio))
    assert ratio <= 1.0, (tag, worst, ratio)
    return max(worst)


@pytest.mark.parametrize("row", E.A1, ids=lambda r: "J{}I{}".format(r["J"], r["I"]))
def test_a1_every_instantiation(row):
    J, I, T, win, hop = row["J"], row["I"], row["T"], row["win"], row["hop"]
    refs, ests = MR.make_track(np.random.default_rng(100 + 10 * J + I), J, I, T, False)
    ref, est = torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda()
    got, status, launches = _images(ref, est, win, hop)
    again, status2, _ = _images(ref, est, win, hop)
    assert status == status2 == 0 and launches == E.mus_launches(J, I), (status, launches)
    assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(got, again))
    _compare("A1 {} (T={} win={} hop={}, {} launches, repeat bit-identical)".format(row["reaches"], T, win, hop, launches), got,
             MR.metrics(refs, ests, win, hop))


@pytest.mark.parametrize("row", E.A2, ids=lambda r: r["name"])
def test_a2_window_geometry(row):
    J, I, T, win, hop = row["J"], row["I"], row["T"], row["win"], row["hop"]
    d = E.mus_dims(J, I, T, win, hop)
    assert all(d[k] == v for k, v in row["want"].items()), d
    refs, ests = MR.make_track(np.random.default_rng(200 + len(row["name"])), J, I, T, False)
    ref, est = torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda()
    got, status, _ = _images(ref, est, win, hop)
    assert status == 0
    if d["nwin"] * win > 5_000_000 or d["nwin"] > 100:
        # the oracle on a subset of windows, its whole-track filters from torch FFTs
        wins = sorted({w for w in [0, 1, d["nwin"] - 1] + list(range(0, d["nwin"], max(1, d["nwin"] // 60))) if w < d["nwin"]})
        conv = scipy.signal.oaconvolve if win > 1_000_000 else scipy.signal.fftconvolve
        want = E.metrics_windows(ref, est, win, hop, wins, E.filters_torch64(ref, est), conv=conv)
        got = [g[:, wins] for g in got]
    else:
        want = MR.metrics(refs, ests, win, hop)
    _compare("A2 {} (nwin {})".format(row["reaches"], d["nwin"]), got, want)


def _gpu_track(J, I, T, seed):
    """museval_ref.make_track's signals built on the GPU (low-pass stems, stereo mixes, estimates with a short FIR, cross-talk and
    noise): a 7-minute track is 1.2 GB of float32, too much to build with scipy in a test"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.float32)  # noqa: E731
    uni = lambda lo, hi: lo + (hi - lo) * float(torch.rand(1, generator=g, device="cuda"))  # noqa: E731
    h = torch.from_numpy(scipy.signal.firwin(129, 0.3)).float().cuda()
    src = torch.nn.functional.conv1d(rnd(J * I, 1, T), h.flip(0)[None, None], padding=128)[..., :T].reshape(J, I, T)
    refs = src.clone()
    for c in range(1, I):
        refs[:, c] = 0.7 * src[:, 0] + 0.5 * src[:, c]
    del src
    for j in range(J):
        refs[j] *= uni(0.3, 3.0)
    ests = torch.empty_like(refs)
    for j in range(J):
        fir = torch.zeros(24, device="cuda")
        fir[0] = 1.0
        fir[1:] = 0.3 * rnd(23) * torch.exp(-torch.arange(1, 24, device="cuda") / 5.0)
        ests[j] = torch.nn.functional.conv1d(refs[j][:, None], fir.flip(0)[None, None], padding=23)[:, 0, :T]
        for i in range(J):
            if i != j:
                ests[j] += uni(0.05, 0.3) * refs[i]
        ests[j] += uni(0.02, 0.2) * float(refs[j].std()) * rnd(I, T)
    return refs.contiguous(), ests.contiguous()


def _a3_call(tag, ref, est, silent_at):
    J, I, T = ref.shape
    d = E.mus_dims(J, I, T, SR, SR)
    assert (d["ntile"], d["per"], d["R"], d["last"]) == (88, 2, 44, 2) and T % SR
    got, status, launches = _images(ref, est, SR, SR)
    assert status == 0 and launches == E.mus_launches(J, I)
    nan = E.silent_windows(ref, est, SR, SR)
    assert nan[silent_at].all() and nan.sum() == len(silent_at)
    for g in got:
        assert np.array_equal(np.isnan(g).all(0), nan) and np.array_equal(np.isnan(g).any(0), nan)
    n = d["nwin"]
    wins = sorted(set([0, 1, 2, n - 3, n - 2, n - 1] + [int(x) for x in np.linspace(3, n - 4, 20)] + list(silent_at)))
    want = E.metrics_windows(ref, est, SR, SR, wins, E.filters_torch64(ref, est))
    return _compare("A3 {} ({} windows, {} compared, workspace {:.0f} MB)".format(tag, n, len(wins), E.mus_workspace_bytes(
        J, I, T, SR, SR) / 2 ** 20), [g[:, wins] for g in got], want)


def test_a3_whole_track():
    """4 low-pass stems in stereo, 7 min + 12345 samples at 44.1 kHz (T not a multiple of the 1 s window), eval_track's windows;
    one window with a silent stem and one with a silent estimate; then the vocals / accompaniment call"""
    T = 7 * 60 * SR + 12345
    refs, ests = _gpu_track(4, 2, T, 300)
    refs[1, :, 100 * SR:101 * SR] = 0
    ests[2, :, 250 * SR:251 * SR] = 0
    _a3_call("4 stems x stereo, 7 min", refs, ests, [100, 250])
    acc_r = (refs[1] + refs[2] + refs[3])[None]
    acc_e = (ests[1] + ests[2] + ests[3])[None]
    ref2, est2 = torch.cat([refs[:1], acc_r]).contiguous(), torch.cat([ests[:1], acc_e]).contiguous()
    del refs, ests
    _a3_call("vocals / accompaniment, 7 min", ref2, est2, [])


@pytest.mark.parametrize("delta", E.DELTAS + ("lowpass",))
def test_a4_conditioning(delta):
    """delta >= 1e-6: within 1e-4 dB + 4 |LU - SVD| per value.  delta = 1e-7 (-140 dB of channel difference): G's condition number
    is near 1 / eps, so any normal-equations answer is rounding noise along the near-null direction.  The Cholesky solve is
    backward stable there (test_c_backward_error_near_mono_gram), yet its answer lands up to 5.5x the LU's worst spread in the
    same metric from the projection (SIR: 3.4e-2 against 6.2e-3 dB); the row is held to 1e-4 dB + 8 x the LU's worst spread per
    metric.  The MUSDB18-style row is refused (CTN_BSS_NOT_PD: the steep low-pass leaves pivots at rounding level) or held to the
    per-value bound."""
    refs, ests, lu, svd = E.a4_oracle(delta, "cuda")
    got, status, _ = _images(torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda(), E.A4_WIN, E.A4_WIN)
    if delta == "lowpass" and status & N.BSS_NOT_PD:
        print("A4 MUSDB18-style low-pass stems: refused (CTN_BSS_NOT_PD); |LU - SVD| {:.1e} dB".format(float(np.max(np.abs(lu - svd)))))
        return
    assert status == 0
    gpu_lu = max(float(np.max(np.abs(g - o))) for g, o in zip(got, lu))
    gpu_svd = max(float(np.max(np.abs(g - o))) for g, o in zip(got, svd))
    print("A4 delta={}: |LU - SVD| {:.1e}, |GPU - LU| {:.1e}, |GPU - SVD| {:.1e} dB".format(
        delta, float(np.max(np.abs(lu - svd))), gpu_lu, gpu_svd))
    bound = E.a4_bound(lu, svd)
    if delta == 1e-7:
        bound = E.TOL_DB + 8 * np.abs(lu - svd).max(axis=(1, 2), keepdims=True)
    _compare("A4 delta={} (2 x 2, T = 20000, windows of {})".format(delta, E.A4_WIN), got, svd, bound)


def test_a5_exact_mono_stem():
    """R == L for stem 0: G is singular.  Refused with the Gram matrix named, or numbers within the A4 bound of the delta = 1e-7
    row against the SVD projection"""
    refs, ests, _, svd = E.a4_oracle(0.0, "cuda")
    _, _, lu7, svd7 = E.a4_oracle(1e-7, "cuda")
    got, status, _ = _images(torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda(), E.A4_WIN, E.A4_WIN)
    if status & N.BSS_NOT_PD:
        from ctn_b200.utils import museval
        with pytest.raises(ValueError, match="Gram matrix"):
            museval.bss_eval_images_v4(torch.from_numpy(refs).cuda(), torch.from_numpy(ests).cuda(), E.A4_WIN, E.A4_WIN)
        print("A5 exact mono stem: refused (CTN_BSS_NOT_PD)")
        return
    _compare("A5 exact mono stem: numbers", got, svd, E.TOL_DB + 4 * float(np.max(np.abs(lu7 - svd7))))


# ---- bss_eval_sources --------------------------------------------------------------------------------------------------------
def _sources(ref, est, perm_on=True):
    """raw ctn_bss_eval_sources on NaN-filled outputs: ref (B, S, T), est (B, K, S, T) -> sdr, sir, sar, perm (B, K, S), status (B,)"""
    B, S, T = ref.shape
    K = est.shape[1]
    ref, est = torch.as_tensor(ref).cuda().contiguous(), torch.as_tensor(est).cuda().contiguous()
    n = C.c_size_t(0)
    N.check(N.ctn_bss_workspace_bytes(B, K, S, T, C.byref(n)))
    base, avail = N.aligned(N.workspace(ref.device, n.value + 256, "bss_edges"))
    out = [torch.full((B, K, S), float("nan"), dtype=torch.float64, device="cuda") for _ in range(3)]
    perm = torch.full((B, K, S), -1, dtype=torch.int32, device="cuda")
    status = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    N.check(N.ctn_bss_eval_sources(ref.data_ptr(), est.data_ptr(), B, K, S, T, int(perm_on), *(t.data_ptr() for t in out),
                                   perm.data_ptr(), status.data_ptr(), base, avail, N.stream_ptr(ref.device)), "ctn_bss_eval_sources")
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in out], perm.cpu().numpy(), status.cpu().numpy()


def _check_set(tag, ref, est, got, perm, mixture, svd=True):
    """one estimate set of one item against the oracle's LU route and (svd) its SVD projection -> worst error / bound"""
    S = ref.shape[0]
    routes = E.bss_routes(ref, est, device="cuda") if svd else {"lu": BR.bss_eval_sources(ref, est, return_margin=True)}
    lu = routes["lu"]
    svd = routes.get("svd", lu)
    if isinstance(lu, Exception):
        lu = svd
    o_perm, margin = lu[3], lu[4]
    if margin > 1e-6 and np.array_equal(svd[3], o_perm):
        assert list(perm) == list(o_perm), (tag, perm, o_perm, margin)
    if not np.array_equal(perm, o_perm):  # a near-tie: score the oracle's assignment
        got, _, _ = _sources(ref[None], est[None, None, list(o_perm)], perm_on=False)
        got = [g[0, 0] for g in got]
    noise = ({"sar"} | ({"sdr"} if S == 1 else set())) if mixture else set()
    ratio = 0.0
    for q, name in enumerate(("sdr", "sir", "sar")):
        g, a, b = np.asarray(got[q]), np.asarray(lu[q]), np.asarray(svd[q])
        assert not np.isnan(g).any(), (tag, name, g)
        if name in noise:
            assert np.all(g >= NOISE_DB), (tag, name, g)
            continue
        for x, y, z in zip(g, a, b):
            if (not np.isfinite(y) or y > 120) and (not np.isfinite(z) or z > 120):
                assert x >= NOISE_DB, (tag, name, x, y, z)
                continue
            bound = TOL + (4 * abs(y - z) if np.isfinite(y) and np.isfinite(z) else 0.0)
            ratio = max(ratio, abs(x - y) / bound)
            assert abs(x - y) <= bound, (tag, name, x, y, z)
    return ratio


def _run_items(tag, refs, ests_sets, perm_on=True, items=None, svd=True, may_refuse=False):
    """refs (B, S, T), ests_sets (B, K, S, T) numpy; set 1 is the repeated mixture when K > 1"""
    got, perm, status = _sources(torch.from_numpy(refs), torch.from_numpy(ests_sets), perm_on)
    if may_refuse and (status & N.BSS_NOT_PD).any():
        print("{}: refused (CTN_BSS_NOT_PD)".format(tag))
        return
    assert (status == 0).all(), status
    ratio = 0.0
    for b in (range(refs.shape[0]) if items is None else items):
        for k in range(ests_sets.shape[1]):
            ratio = max(ratio, _check_set(tag, refs[b], ests_sets[b, k], [g[b, k] for g in got], perm[b, k], k == 1, svd))
    print("{}: worst error / bound {:.2e}".format(tag, ratio))


def _with_mixture(refs, ests):
    return np.stack([ests, np.repeat(refs.sum(0, keepdims=True), refs.shape[0], axis=0)])


@pytest.mark.parametrize("row", E.B1 + E.B2 + E.B3, ids=lambda r: r["name"])
def test_b1_b2_b3_shapes(row):
    S, T = row["S"], row["T"]
    refs, ests = BR.make_item(np.random.default_rng(500 + T + S), S, T)
    _run_items("B {} (S={} T={})".format(row["reaches"], S, T), refs[None], _with_mixture(refs, ests)[None], svd=row in E.B2)


@pytest.mark.parametrize("S", [2, 3])
def test_b4_max_mode(S):
    refs, ests = E.max_mode_item(600 + S, S, 32000)
    _run_items("B4 wsj0-mix max mode S={}".format(S), refs[None], _with_mixture(refs, ests)[None], svd=False)


@pytest.mark.parametrize("S", [2, 4])
def test_b5_band_limited(S):
    """the steep low-pass leaves the Gram matrix's trailing pivots at rounding level: refused (CTN_BSS_NOT_PD, where mir_eval's LU
    returns numbers), or within the A4 bound"""
    refs, ests = E.band_limited_item(70 + S, S, 16000)
    _run_items("B5 8 kHz content at 16 kHz S={}".format(S), refs[None], _with_mixture(refs, ests)[None], may_refuse=True)


@pytest.mark.parametrize("kind", ["scaled", "delayed"])
def test_b6_rank_deficient(kind):
    refs, ests = E.rank_deficient_item(kind)
    got, perm, status = _sources(torch.from_numpy(refs)[None], torch.from_numpy(ests)[None, None])
    if status[0] & N.BSS_NOT_PD:
        from ctn_b200.utils import bss
        with pytest.raises(ValueError, match="Gram matrix"):
            bss.bss_eval_sources(torch.from_numpy(refs), torch.from_numpy(ests))
        print("B6 {}: refused (CTN_BSS_NOT_PD)".format(kind))
        return
    assert status[0] == 0
    ratio = _check_set("B6 " + kind, refs, ests, [g[0, 0] for g in got], perm[0, 0], False)
    print("B6 {}: numbers, worst error / bound {:.2e}".format(kind, ratio))


def test_b7_batch_of_200():
    rng = np.random.default_rng(700)
    refs, ests = zip(*(BR.make_item(rng, 2, 8000) for _ in range(200)))
    refs = np.stack(refs)
    sets = np.stack([_with_mixture(r, e) for r, e in zip(refs, ests)])
    _run_items("B7 B = 200 (items 0, 199 and every 25th against the oracle)", refs, sets, items=sorted({0, 199, *range(12, 200, 25)}),
               svd=False)


# ---- the shared Cholesky -----------------------------------------------------------------------------------------------------
_p, _i = C.c_void_p, C.c_int
probe_factor = N._sig("ctn_probe_chol_factor", _i, _p, _p, _p, _i, _i, _p)
probe_solve = N._sig("ctn_probe_chol_solve", _i, _p, _p, _p, _p, _i, _i, _i, _i, _p)


def _spd(n, nmat, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    X = torch.randn(nmat, n + 64, n, generator=g, device="cuda", dtype=torch.float64)
    return X.transpose(1, 2) @ X / n + 0.1 * torch.eye(n, device="cuda", dtype=torch.float64)


def _factor(A):
    nmat, n, _ = A.shape
    A = A.clone()
    W = torch.full((nmat, n // 64, 64, 64), float("nan"), dtype=torch.float64, device="cuda")
    flag = torch.full((nmat,), -1, dtype=torch.int32, device="cuda")
    N.check(probe_factor(A.data_ptr(), W.data_ptr(), flag.data_ptr(), n, nmat, None))
    torch.cuda.synchronize()
    return A, W, flag.cpu().numpy()


@pytest.mark.parametrize("n,what", E.C_SIZES, ids=lambda x: str(x) if isinstance(x, int) else "")
def test_c_factor_and_solve_sizes(n, what):
    A = _spd(n, 2, n)
    F, W, flag = _factor(A)
    assert (flag == 0).all()
    Lg = torch.tril(F)
    want = torch.linalg.cholesky(A)
    err = float(((Lg - want).abs().amax((1, 2)) / want.abs().amax((1, 2))).max())
    B = torch.randn(2, n, 8, dtype=torch.float64, device="cuda")
    X = B.clone()
    N.check(probe_solve(F.data_ptr(), W.data_ptr(), X.data_ptr(), torch.empty_like(X).data_ptr(), n, 2, 8, 1, None))
    torch.cuda.synchronize()
    sol = torch.linalg.solve(A, B)
    serr = float((X - sol).abs().max() / sol.abs().max())
    print("C n={} ({}): factor rel {:.1e}, all-columns solve rel {:.1e}".format(n, what, err, serr))
    assert err < 1e-12 and serr < 1e-11


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_c_one_bad_matrix_in_a_batch(where):
    n = 1024
    A = _spd(n, 3, 7)
    p = {"first": 5, "middle": n // 2 + 3, "last": n - 1}[where]
    clean, Wc, fc = _factor(A)
    bad = A.clone()
    bad[1, p, p] = -1.0
    F, W, flag = _factor(bad)
    assert list(fc) == [0, 0, 0] and list(flag) == [0, 1, 0], flag
    for m in (0, 2):
        assert torch.equal(torch.tril(F[m]), torch.tril(clean[m])) and torch.equal(W[m], Wc[m])
    # the tiles before the bad pivot's are those of the clean factor
    t = p // 64
    assert torch.equal(torch.tril(F[1, :t * 64, :t * 64]), torch.tril(clean[1, :t * 64, :t * 64]))
    print("C non-PD pivot {} (tile {} of {}): only its matrix flagged, the others bit-identical".format(p, t, n // 64))


@pytest.mark.parametrize("poison", ["nan", "inf"])
def test_c_non_finite_entries_flag(poison):
    A = _spd(512, 2, 9)
    v = float(poison)
    A[0, 300, 200] = A[0, 200, 300] = v
    _, _, flag = _factor(A)
    assert list(flag) == [1, 0], flag


def _backward_error(A, x, b):
    """||A x - b||_inf / (||A||_inf ||x||_inf), the residual in float64 (its own rounding, about sqrt(n) eps, is far below the
    bound)"""
    r = A @ x - b
    return float(r.abs().max() / (A.abs().sum(1).max() * x.abs().max()))


def _both_routes(A, F, W, nrhs, g):
    """solve A x = b for nrhs random columns by route 1 (ctn_chol_solve_multi) and route 0 (k_chol_solve) on the factor F, W ->
    the worst backward error of the two.  The right-hand sides are copied into fresh buffers: both routes solve in place."""
    n = A.shape[-1]
    B = torch.randn(1, n, nrhs, generator=g, device="cuda", dtype=torch.float64)
    multi, tmp = B.clone(), torch.empty_like(B)
    cols = torch.empty(1, nrhs, n, dtype=torch.float64, device="cuda").copy_(B.transpose(1, 2))
    N.check(probe_solve(F.data_ptr(), W.data_ptr(), multi.data_ptr(), tmp.data_ptr(), n, 1, nrhs, 1, None))
    N.check(probe_solve(F.data_ptr(), W.data_ptr(), cols.data_ptr(), None, n, 1, nrhs, 0, None))
    torch.cuda.synchronize()
    return max(_backward_error(A[0], multi[0], B[0]), _backward_error(A[0], cols[0].T, B[0]))


@pytest.mark.parametrize("kappa", E.C_KAPPAS)
def test_c_backward_error(kappa):
    """A = Q diag(s) Q^T, s log-spaced from 1 to 1 / kappa: ||A x - b|| / (||A|| ||x||) <= 8 n 2^-53 for both routes, nrhs 1 .. 8.
    The solves apply the kept inverses of the 64 x 64 diagonal tiles; this is the check that they stay backward stable."""
    n = 1024
    g = torch.Generator(device="cuda").manual_seed(int(np.log10(kappa)))
    Q, _ = torch.linalg.qr(torch.randn(n, n, generator=g, device="cuda", dtype=torch.float64))
    s = torch.logspace(0, -np.log10(kappa), n, device="cuda", dtype=torch.float64)
    A = (Q * s) @ Q.T
    A = ((A + A.T) / 2)[None].contiguous()
    F, W, flag = _factor(A)
    assert flag[0] == 0
    bound = 8 * n * 2.0 ** -53
    worst = max(_both_routes(A, F, W, nrhs, g) for nrhs in range(1, 9))
    print("C kappa={:.0e}: worst backward error {:.1e} over both routes and nrhs 1..8 (bound {:.1e}, ratio {:.1e})".format(
        kappa, worst, bound, worst / bound))
    assert worst <= bound


def test_c_backward_error_near_mono_gram():
    """the G + eps I of the A4 delta = 1e-7 row (condition number near 1 / eps): the same backward-error bound"""
    refs, _ = E.near_mono_track(1e-7)
    A = torch.from_numpy(E.gram_fft(refs))[None].cuda()
    n = A.shape[-1]
    F, W, flag = _factor(A)
    assert flag[0] == 0
    g = torch.Generator(device="cuda").manual_seed(17)
    bound = 8 * n * 2.0 ** -53
    worst = max(_both_routes(A, F, W, nrhs, g) for nrhs in (1, 4, 8))
    print("C near-mono G (n = {}): worst backward error {:.1e} (bound {:.1e}, ratio {:.1e})".format(n, worst, bound, worst / bound))
    assert worst <= bound
