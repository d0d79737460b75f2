"""Shared pieces of the BSS Eval edge tests (tests/test_bss_edges_cpu.py and, with ``-m gpu``, tests/test_bss_edges_gpu.py).

- Restatements of the launch geometry of ctn_bss_images.cu (``mus_dims``, the workspace carve, the ``MUS_CASE`` dispatch list) and
  of ctn_bss.cu (the ``k_bss_corr`` time chunks and tiles, the ``k_bss_project`` ranges), so that each row can prove it reaches
  the branch its ``reaches`` text names.
- Oracles: ``metrics_windows`` (museval_ref.metrics on a subset of windows), ``filters_torch64`` (the whole-track filters from
  float64 torch FFTs, on any device), ``filters_svd`` / ``project_svd`` (the least-squares filters and projections from an SVD
  with a rank cut: the reference where the normal equations stop being trustworthy).
- Emulations of the kernels' summation geometry with named mutants (``mus_metrics_by_ranges``, ``bss_tables_chunked``): each mutant
  must move a named row by more than the bound, or the geometry the tests check would not matter.
- The row tables of sections A (museval v4), B (bss_eval_sources) and C (the shared Cholesky)."""
import functools
import re

import numpy as np
import scipy.linalg
import scipy.signal

import bss_ref as BR
import museval_ref as MR

L = 512
SR = 44100
TOL_DB = 1e-4

# ---- ctn_bss_images.cu geometry ----------------------------------------------------------------------------------------------
MUS_NCH, MUS_TU, MUS_PT, MUS_MAXR, MUS_NE = 128, 512, 512, 64, 7

# the (J, I) instantiations of k_mus_project<J I, I> in mus_project_dispatch, in source order
MUS_DISPATCH = [(1, 1), (2, 1), (3, 1), (4, 1), (5, 1), (6, 1), (7, 1), (8, 1), (1, 2), (2, 2), (3, 2), (4, 2), (1, 3), (2, 3), (1, 4),
                (2, 4), (1, 5), (1, 6), (1, 7), (1, 8)]


def dispatch_in_source(text):
    """the (J, I) pairs of the MUS_CASE lines of ctn_bss_images.cu, in order"""
    return [(int(a), int(b)) for a, b in re.findall(r"MUS_CASE\((\d+), (\d+)\)", text)]


def limit(J, I):
    """the shortest T at which the J I 512 delayed references can be independent: T + L - 1 >= J I L"""
    return J * I * L - (L - 1)


def mus_dims(J, I, T, win, hop):
    """mus_dims of ctn_bss_images.cu: windows, 512-sample output tiles per window (over win + L - 1 samples), tiles per range, ranges
    per window and the tiles of the last range"""
    nwin = (T - win + hop) // hop
    ntile = -(-(win + L - 1) // MUS_PT)
    per = -(-ntile // MUS_MAXR)
    R = -(-ntile // per)
    return dict(nwin=nwin, ntile=ntile, per=per, R=R, last=ntile - (R - 1) * per)


def _carve(sizes):
    off = 0
    for n in sizes:
        off = (off + 255) & ~255
        off += n
    return off


def mus_workspace_bytes(J, I, T, win, hop):
    """ctn_bss_images_workspace_bytes restated from carve_mus"""
    M, N, NB, nwin = J * I, J * I * L, I * L, mus_dims(J, I, T, win, hop)["nwin"]
    d = [2 * M * MUS_NCH * M * L, M * M * L, N * N, N * 64, J * NB * NB, J * NB * 64, N * M, N * M, N * I, N * I,
         nwin * MUS_MAXR * J * MUS_NE]
    return _carve([8 * n for n in d] + [4 * nwin * 2, 4, 4 * J]) + 256


def mus_launches(J, I):
    """silence, correlations, combine, build; 3 nt - 2 Cholesky launches per matrix set; 2 nt solve launches per set; projection
    and finish"""
    ntg, ntb = 8 * J * I, 8 * I
    return 4 + (3 * ntg - 2) + (3 * ntb - 2) + 2 * ntg + 2 * ntb + 2


# ---- ctn_bss.cu geometry -----------------------------------------------------------------------------------------------------
BSS_NCH, BSS_TU, BSS_NTT = 16, 1024, 64


def bss_chunks(T):
    """k_bss_corr: TC samples per chunk; per chunk the tile lengths it stages ([] for an empty chunk)"""
    TC = -(-T // BSS_NCH)
    tiles = []
    for c in range(BSS_NCH):
        lo, hi = min(T, c * TC), min(T, min(T, c * TC) + TC)
        tiles.append([min(BSS_TU, hi - u0) for u0 in range(lo, hi, BSS_TU)])
    return TC, tiles


def bss_ranges(T):
    """k_bss_project: the T + L - 1 outputs of an estimate in BSS_NTT ranges of ``span`` samples -> (span, range lengths)"""
    Tt = T + L - 1
    span = -(-Tt // BSS_NTT)
    return span, [max(0, min(Tt, min(Tt, r * span) + span) - min(Tt, r * span)) for r in range(BSS_NTT)]


# ---- oracles -----------------------------------------------------------------------------------------------------------------
def _np64(x):
    if hasattr(x, "detach"):
        x = x.detach().cpu().numpy()
    return np.asarray(x, dtype=np.float64)


def metrics_windows(refs, ests, win, hop, windows, filters=MR.filters_fft, conv=scipy.signal.fftconvolve):
    """museval_ref.metrics restricted to ``windows``: SDR, ISR, SIR, SAR (J, len(windows)).  A window's metrics depend on the
    whole-track filters and its own slice only.  ``filters`` is a function of (refs, ests) or its (C, Ct); refs / ests may be
    numpy or torch (only the filters and the chosen slices are read)."""
    J, I, T = refs.shape
    M = J * I
    C, Ct = filters(_np64(refs), _np64(ests)) if callable(filters) else filters
    Cm = C.reshape(M, L, M).transpose(0, 2, 1)
    out = np.full((4, J, len(windows)), np.nan)
    for n, w in enumerate(windows):
        sl = slice(w * hop, w * hop + win)
        r, e = _np64(refs[:, :, sl]), _np64(ests[:, :, sl])
        if MR._silent(r) or MR._silent(e):
            continue
        rw = r.reshape(M, win)
        p_all = conv(rw[:, None, :], Cm, axes=-1).sum(0)
        pad = lambda x: np.concatenate((x, np.zeros(x.shape[:-1] + (L - 1,))), axis=-1)  # noqa: E731
        s, ep = pad(r), pad(e)
        for j in range(J):
            ctj = Ct[j].reshape(I, L, I).transpose(0, 2, 1)
            p_j = conv(r[j][:, None, :], ctj, axes=-1).sum(0)
            pa = p_all[j * I:(j + 1) * I]
            q = [np.sum(s[j] ** 2), np.sum((ep[j] - s[j]) ** 2), np.sum((p_j - s[j]) ** 2), np.sum(p_j ** 2),
                 np.sum((pa - p_j) ** 2), np.sum(pa ** 2), np.sum((ep[j] - pa) ** 2)]
            out[:, j, n] = (MR._safe_db(q[0], q[1]), MR._safe_db(q[0], q[2]), MR._safe_db(q[3], q[4]), MR._safe_db(q[5], q[6]))
    return tuple(out)


def silent_windows(refs, ests, win, hop):
    """(nwin,) bool: museval's NaN rule for every window, from torch (any device) or numpy (J, I, T)"""
    import torch
    mask = None
    for x in (refs, ests):
        x = torch.as_tensor(x).double().sum(1)  # (J, T): the channel sum, in double as k_mus_silent forms it
        s = (x.unfold(-1, win, hop) == 0).all(-1).any(0)
        mask = s if mask is None else mask | s
    return mask.cpu().numpy()


def filters_torch64(refs, ests, device=None):
    """museval_ref.filters_fft with the whole-track correlations from float64 torch FFTs on ``device`` (the inputs' by default):
    seconds instead of minutes for a whole track on a GPU.  The dense solves run in numpy, as museval's do.  Independent of this
    project's kernels."""
    import torch
    refs, ests = torch.as_tensor(refs), torch.as_tensor(ests)
    if device is not None:
        refs, ests = refs.to(device), ests.to(device)
    J, I, T = refs.shape
    M = J * I
    nfft = 1 << int(np.ceil(np.log2(T + L - 1)))
    rf = torch.fft.rfft(refs.reshape(M, T).double(), n=nfft)
    G = np.zeros((M * L, M * L))
    D = np.zeros((M * L, M))
    idx = torch.arange(1 - L, L, device=rf.device) % nfft  # lags -(L-1) .. L-1
    for a in range(M):
        c = torch.fft.irfft(rf[a][None] * rf.conj(), n=nfft)[:, idx].cpu().numpy()  # c[b][k] = sum_u r_a(u + k) r_b(u)
        for b in range(M):
            cb = c[b]
            G[a * L:(a + 1) * L, b * L:(b + 1) * L] = scipy.linalg.toeplitz(cb[L - 1::-1], r=cb[L - 1:])
        del c
    ef = None
    for col in range(M):
        ef = torch.fft.rfft(ests.reshape(M, T)[col].double(), n=nfft)
        c = torch.fft.irfft(rf * ef.conj()[None], n=nfft)[:, idx[:L]].cpu().numpy()  # lags -(L-1) .. 0: sum_u r_a(u - k) e(u)
        D[:, col] = c[:, ::-1].reshape(-1)
    del rf, ef
    C = np.linalg.solve(G + MR.EPS * np.eye(M * L), D)
    Ct = np.zeros((J, I * L, I))
    for j in range(J):
        sl = slice(j * I * L, (j + 1) * I * L)
        Ct[j] = np.linalg.solve(G[sl, sl] + MR.EPS * np.eye(I * L), D[sl, j * I:(j + 1) * I])
    return C, Ct


RCOND = 1e-11  # singular values below RCOND x the largest count as zero: far below any signal, far above an exact copy's


def _delayed(rows, L=L):
    """(n, T) -> the (T + L - 1, n L) matrix of delayed rows"""
    n, T = rows.shape
    A = np.zeros((T + L - 1, n * L))
    for m in range(n):
        for k in range(L):
            A[k:k + T, m * L + k] = rows[m]
    return A


def _lstsq_svd(A, B, rcond=RCOND, device=None):
    """-> the minimum-norm solution of A X = B with singular values below rcond x the largest cut, and the kept left singular
    vectors.  The SVD runs in float64 torch on ``device`` (LAPACK on the CPU by default)."""
    import torch
    U, s, Vt = torch.linalg.svd(torch.from_numpy(A).to(device), full_matrices=False)
    U, s, Vt = U.cpu().numpy(), s.cpu().numpy(), Vt.cpu().numpy()
    keep = s > rcond * s[0]
    return Vt[keep].T @ ((U[:, keep].T @ B) / s[keep, None]), U[:, keep]


def filters_svd(refs, ests, rcond=RCOND, device=None):
    """museval_ref.filters_qr from an SVD with a rank cut: the minimum-norm least-squares filters.  Where the delayed references
    are rank deficient the filters are not unique, but every window's projection is (a null vector of the whole-track matrix of
    an exact copy is one of every window's too)."""
    refs, ests = _np64(refs), _np64(ests)
    J, I, T = refs.shape
    M = J * I
    A = _delayed(refs.reshape(M, T))
    e = np.hstack((ests.reshape(M, T), np.zeros((M, L - 1)))).T
    C = _lstsq_svd(A, e, rcond, device)[0]
    Ct = np.zeros((J, I * L, I))
    for j in range(J):
        Ct[j] = _lstsq_svd(np.ascontiguousarray(A[:, j * I * L:(j + 1) * I * L]), e[:, j * I:(j + 1) * I], rcond, device)[0]
    return C, Ct


def project_svd(refs, ests, rcond=RCOND, device=None):
    """bss_ref.project_qr from an SVD with a rank cut: the orthogonal projections onto the span of the delayed references, unique
    even when the filters are not"""
    refs, ests = _np64(refs), _np64(ests)
    S, T = refs.shape
    A = _delayed(refs)
    e = np.hstack((ests, np.zeros((ests.shape[0], L - 1))))
    U = _lstsq_svd(A, e.T, rcond, device)[1]
    P_all = (U @ (U.T @ e.T)).T
    P = np.zeros((ests.shape[0], S, T + L - 1))
    for i in range(S):
        Ui = _lstsq_svd(np.ascontiguousarray(A[:, i * L:(i + 1) * L]), e.T, rcond, device)[1]
        P[:, i] = (Ui @ (Ui.T @ e.T)).T
    return P_all, P


def bss_routes(refs, ests, compute_permutation=True, device=None):
    """bss_ref's answer by its LU route and by the SVD projection: {route: (sdr, sir, sar, perm, margin) or the LinAlgError}"""
    out = {}
    for name, proj in (("lu", BR.project_fft), ("svd", functools.partial(project_svd, device=device))):
        try:
            out[name] = BR.bss_eval_sources(refs, ests, compute_permutation, project=proj, return_margin=True)
        except np.linalg.LinAlgError as ex:
            out[name] = ex
    return out


# ---- emulations of the kernels' summation geometry, with mutants ----------------------------------------------------------------
MUS_MUTANTS = ("drop_last_range", "window_start_plus_one", "pj_wrong_source")


def filters_block_eps(refs, ests, block_eps=MR.EPS):
    """museval_ref.filters_fft, step for step, with ``block_eps`` on the diagonal of the per-source blocks (0: the mutant of DESIGN
    §10 point 3, which leaves the eps I off them)"""
    J, I, T = refs.shape
    M = J * I
    r = refs.reshape(M, T)
    e = ests.reshape(M, T)
    nfft = int(2 ** np.ceil(np.log2(T + L - 1)))
    rf = np.fft.rfft(r, n=nfft)
    ef = np.fft.rfft(e, n=nfft)
    G = np.zeros((M * L, M * L))
    for a in range(M):
        for b in range(M):
            c = np.fft.irfft(rf[a] * np.conj(rf[b]), n=nfft)
            G[a * L:(a + 1) * L, b * L:(b + 1) * L] = scipy.linalg.toeplitz(np.hstack((c[0], c[-1:-L:-1])), r=c[:L])
    D = np.zeros((M * L, M))
    for a in range(M):
        c = np.fft.irfft(rf[a][None] * np.conj(ef), n=nfft)
        D[a * L:(a + 1) * L] = np.hstack((c[:, :1], c[:, -1:-L:-1])).T
    C = np.linalg.solve(G + MR.EPS * np.eye(M * L), D)
    Ct = np.zeros((J, I * L, I))
    for j in range(J):
        sl = slice(j * I * L, (j + 1) * I * L)
        Ct[j] = np.linalg.solve(G[sl, sl] + block_eps * np.eye(I * L), D[sl, j * I:(j + 1) * I])
    return C, Ct


def mus_metrics_by_ranges(refs, ests, win, hop, windows, filters, mutant=None):
    """the energies of k_mus_project / k_mus_finish: per window, per-sample residuals over the win + L - 1 outputs, summed tile range
    by tile range as the kernel's grid covers them; ``mutant`` names one of MUS_MUTANTS"""
    refs, ests = _np64(refs), _np64(ests)
    J, I, T = refs.shape
    M = J * I
    d = mus_dims(J, I, T, win, hop)
    C, Ct = filters
    Cm = C.reshape(M, L, M).transpose(0, 2, 1)
    span = win + L - 1
    ranges = [(rg * d["per"] * MUS_PT, min(d["ntile"], rg * d["per"] + d["per"]) * MUS_PT) for rg in range(d["R"])]
    if mutant == "drop_last_range" and d["R"] > 1:
        ranges = ranges[:-1]
    out = np.full((4, J, len(windows)), np.nan)
    for n, w in enumerate(windows):
        s0 = w * hop + (1 if mutant == "window_start_plus_one" else 0)
        r = np.zeros((J, I, win))
        e = np.zeros((J, I, win))
        n_in = max(0, min(win, T - s0))
        r[:, :, :n_in], e[:, :, :n_in] = refs[:, :, s0:s0 + n_in], ests[:, :, s0:s0 + n_in]
        if MR._silent(r) or MR._silent(e):
            continue
        p_all = scipy.signal.fftconvolve(r.reshape(M, win)[:, None, :], Cm, axes=-1).sum(0)
        pad = lambda x: np.concatenate((x, np.zeros(x.shape[:-1] + (L - 1,))), axis=-1)  # noqa: E731
        s, ep = pad(r), pad(e)
        for j in range(J):
            src = (j + 1) % J if mutant == "pj_wrong_source" else j
            ctj = Ct[src].reshape(I, L, I).transpose(0, 2, 1)
            p_j = scipy.signal.fftconvolve(r[j][:, None, :], ctj, axes=-1).sum(0)
            pa = p_all[j * I:(j + 1) * I]
            per_t = [s[j] ** 2, (ep[j] - s[j]) ** 2, (p_j - s[j]) ** 2, p_j ** 2, (pa - p_j) ** 2, pa ** 2, (ep[j] - pa) ** 2]
            q = [sum(np.sum(x[:, lo:min(hi, span)]) for lo, hi in ranges) for x in per_t]
            out[:, j, n] = (MR._safe_db(q[0], q[1]), MR._safe_db(q[0], q[2]), MR._safe_db(q[3], q[4]), MR._safe_db(q[5], q[6]))
    return tuple(out)


def bss_corr_chunked(x, y, T, mutant=None):
    """k_bss_corr + k_bss_combine: corr(x, y)[m] = sum_u x(u) y(u + m), m < L, tile by tile of each time chunk; mutant
    'drop_last_tile' leaves the last tile of every chunk with more than one out"""
    TC, tiles = bss_chunks(T)
    yz = np.concatenate((y, np.zeros(L - 1)))
    acc = np.zeros(L)
    for c, lens in enumerate(tiles):
        if mutant == "drop_last_tile" and len(lens) > 1:
            lens = lens[:-1]
        u0 = c * TC
        for n in lens:
            acc += np.correlate(yz[u0:u0 + n + L - 1], x[u0:u0 + n], "valid")
            u0 += n
    return acc


def bss_tables_chunked(refs, ests, mutant=None):
    """bss_ref.tables with G and the right-hand sides from the chunked correlations"""
    refs, ests = _np64(refs), _np64(ests)
    S, T = refs.shape
    corr = [[bss_corr_chunked(refs[i], refs[j], T, mutant) for j in range(S)] for i in range(S)]
    G = np.zeros((S * L, S * L))
    for i in range(S):
        for j in range(S):
            # G[iL+k, jL+l] = corr(r_i, r_j)[k - l] for k >= l, corr(r_j, r_i)[l - k] otherwise
            G[i * L:(i + 1) * L, j * L:(j + 1) * L] = scipy.linalg.toeplitz(corr[i][j], r=corr[j][i])
    D = np.stack([np.concatenate([bss_corr_chunked(refs[i], ests[a], T, mutant) for i in range(S)]) for a in range(S)], 1)

    def project(refs, ests):
        C_all = np.linalg.solve(G, D)
        P_all = np.zeros((S, T + L - 1))
        P = np.zeros((S, S, T + L - 1))
        for i in range(S):
            C_i = np.linalg.solve(G[i * L:(i + 1) * L, i * L:(i + 1) * L], D[i * L:(i + 1) * L])
            for a in range(S):
                P_all[a] += scipy.signal.fftconvolve(C_all[i * L:(i + 1) * L, a], refs[i])
                P[a, i] = scipy.signal.fftconvolve(C_i[:, a], refs[i])
        return P_all, P

    return BR.tables(refs, ests, project)


# ---- test signals ------------------------------------------------------------------------------------------------------------
def steep_lowpass(cutoff, numtaps=511):
    """a steep linear-phase FIR low-pass (cutoff as a fraction of Nyquist), about 120 dB of stop band"""
    return scipy.signal.firwin(numtaps, cutoff, window=("kaiser", 12.0))


def near_mono_track(delta, seed=2, J=2, I=2, T=20000):
    """museval_ref.make_track with stem 0's right channel = its left + delta std noise (delta = 0: an exact copy)"""
    rng = np.random.default_rng(seed)
    refs, ests = MR.make_track(rng, J, I, T, False)
    refs[0, 1] = (refs[0, 0] + delta * np.std(refs[0, 0]) * rng.standard_normal(T)).astype(np.float32)
    return refs, ests


def lowpass_track(seed=3, J=2, I=2, T=20000, cutoff=16.0 / 22.05):
    """MUSDB18-style stems: references low-passed at 16 of 22.05 kHz (the AAC cutoff of the non-HQ release) by a steep FIR"""
    rng = np.random.default_rng(seed)
    refs, ests = MR.make_track(rng, J, I, T, False)
    h = steep_lowpass(cutoff)
    refs = scipy.signal.lfilter(h, [1.0], refs.astype(np.float64), axis=-1).astype(np.float32)
    return refs, ests


def max_mode_item(seed, S, T):
    """wsj0-mix "max" mode: references zero-padded at the start and the end, reference 1 silent over its last 35 %, and estimates
    that leak cross-talk and noise into every silence"""
    rng = np.random.default_rng(seed)
    refs, ests = BR.make_item(rng, S, T, coloured=True)
    refs = refs.astype(np.float64)
    for j in range(S):
        refs[j, :int(rng.integers(200, 3000))] = 0
        refs[j, T - int(rng.integers(200, 3000)):] = 0
    refs[1, int(0.65 * T):] = 0
    leak = np.stack([sum(rng.uniform(0.05, 0.2) * refs[i] for i in range(S) if i != j) for j in range(S)])
    ests = refs + leak + 0.02 * np.std(refs) * rng.standard_normal((S, T))
    return refs.astype(np.float32), ests.astype(np.float32)


def band_limited_item(seed, S, T):
    """16 kHz references with 8 kHz content (the cfg5 recipe): white noise low-passed at 0.5 of the band by a steep FIR"""
    rng = np.random.default_rng(seed)
    refs, ests = BR.make_item(rng, S, T)
    refs = scipy.signal.lfilter(steep_lowpass(0.5), [1.0], refs.astype(np.float64), axis=1)
    ests = ests.astype(np.float64)
    for j in range(S):
        ests[j] += 0.5 * refs[j]
    return refs.astype(np.float32), ests.astype(np.float32)


def rank_deficient_item(kind, seed=61, T=8000):
    """reference 1 = 0.5 reference 0 ('scaled'), or reference 0 delayed by 100 samples with reference 0 silent over its last 100
    ('delayed', so that the delayed copy lies exactly in the span)"""
    rng = np.random.default_rng(seed)
    refs, ests = BR.make_item(rng, 2, T)
    if kind == "scaled":
        refs[1] = refs[0] * np.float32(0.5)
    else:
        refs[0, T - 100:] = 0
        refs[1] = 0
        refs[1, 100:] = refs[0, :T - 100]
    return refs, ests


# ---- rows --------------------------------------------------------------------------------------------------------------------
def _a1_row(J, I):
    M = J * I
    T = limit(J, I) + 300
    win, hop = max(1, T // 3), max(1, T // 5)
    return dict(J=J, I=I, T=T, win=win, hop=hop,
                reaches="k_mus_project<{M}, {I}>, k_mus_corr<{M}>, G {N} x {N} ({nt} tiles), blocks {B} x {B} ({J} of them), "
                        "ctn_chol_solve_multi nrhs = {M} (G) and {I} (blocks)".format(M=M, I=I, J=J, N=M * L, nt=M * 8, B=I * L))


A1 = [_a1_row(J, I) for J, I in MUS_DISPATCH]

# (name, J, I, T, win, hop, windows or None for all, expected dims)
A2 = [
    dict(name="win1", J=2, I=2, T=limit(2, 2) + 300, win=1, hop=300, want=dict(ntile=1, per=1, R=1),
         reaches="win = 1: one output tile, 511 of its 512 outputs the filter tail"),
    dict(name="win100", J=2, I=2, T=limit(2, 2) + 300, win=100, hop=97, want=dict(ntile=2, per=1, R=2),
         reaches="win = 100 < L: ntile = 2, the second tile partly beyond span"),
    dict(name="win32257", J=2, I=2, T=40000, win=32257, hop=7000, want=dict(ntile=64, per=1, R=64, last=1),
         reaches="win = 32257: ntile = 64 = MUS_MAXR, per = 1, R = 64"),
    dict(name="win32258", J=2, I=2, T=40000, win=32258, hop=7000, want=dict(ntile=65, per=2, R=33, last=1),
         reaches="win = 32258: ntile = 65, per = 2, ragged last range of 1 tile"),
    dict(name="win66049", J=2, I=2, T=80000, win=66049, hop=6000, want=dict(ntile=130, per=3, R=44, last=1),
         reaches="win = 66049: ntile = 130, per = 3, R = 44, ragged last range of 1 tile"),
    dict(name="win_eq_T_5min", J=1, I=2, T=300 * SR, win=300 * SR, hop=300 * SR, want=dict(ntile=25841, per=404, R=64, last=389),
         reaches="win = T = 5 min: ntile = 25841, per = 404, R = 64, last range 389 tiles"),
    dict(name="hop_gt_win", J=2, I=2, T=100000, win=30000, hop=45000, want=dict(nwin=2, ntile=60, per=1, R=60),
         reaches="hop > win: nwin = 2, samples 75000 .. 99999 never scored"),
    dict(name="3000_windows", J=2, I=2, T=30 * SR, win=441, hop=441, want=dict(nwin=3000, ntile=2, per=1, R=2),
         reaches="win = hop = 441 over 30 s: nwin = 3000, 6000 projection CTAs"),
]

DELTAS = (1e-3, 1e-5, 1e-6, 1e-7)
A4_WIN = 5000

# B: (name, S, T, K, kind)
# want: TC, empty chunks, the last non-empty chunk's tile lengths, the projection span and the non-empty ranges
B1 = [dict(name="S1_T{}".format(T), S=1, T=T, reaches=r, want=w) for T, r, w in (
    (1, "T = 1 < BSS_NCH: TC = 1, 15 empty chunks; 64 projection ranges of 8 outputs",
     dict(TC=1, empty=15, last_tiles=[1], span=8, ranges=[8] * 64)),
    (7, "T = 7 < BSS_NCH: TC = 1, 9 empty chunks; ranges of 9, the 58th of 5, 6 empty",
     dict(TC=1, empty=9, last_tiles=[1], span=9, ranges=[9] * 57 + [5])),
    (100, "T = 100: TC = 7, a 2-sample chunk and an empty one; ranges of 10, the 62nd of 1",
     dict(TC=7, empty=1, last_tiles=[2], span=10, ranges=[10] * 61 + [1])),
    (511, "T = 511: TC = 32, the last chunk 31; ranges of 16, the last 14",
     dict(TC=32, empty=0, last_tiles=[31], span=16, ranges=[16] * 63 + [14])),
    (512, "T = 512 = L: TC = 32, whole chunks; ranges of 16, the last 15",
     dict(TC=32, empty=0, last_tiles=[32], span=16, ranges=[16] * 63 + [15])),
    (513, "T = 513: TC = 33, the last chunk 18; 64 whole ranges of 16",
     dict(TC=33, empty=0, last_tiles=[18], span=16, ranges=[16] * 64)),
    (1023, "T = 1023: TC = 64, the last chunk 63; ranges of 24, the last 22",
     dict(TC=64, empty=0, last_tiles=[63], span=24, ranges=[24] * 63 + [22])))]
B2 = [dict(name="S{}_T{}".format(S, T), S=S, T=T, reaches="S L = T + L - 1 = {}: the delayed references square".format(S * L))
      for S, T in ((2, 513), (3, 1025), (4, 1537))]
B3 = [dict(name="T{}".format(T), S=2, T=T, reaches=r, want=w) for T, r, w in (
    (16383, "T = 16383: TC = 1024 = BSS_TU, the last chunk 1023",
     dict(TC=1024, empty=0, last_tiles=[1023], tiles_per_chunk=1)),
    (16384, "T = 16384: TC = 1024 = BSS_TU, 16 whole one-tile chunks",
     dict(TC=1024, empty=0, last_tiles=[1024], tiles_per_chunk=1)),
    (16385, "T = 16385: TC = 1025, a 1-sample second tile per chunk, the last chunk 1010",
     dict(TC=1025, empty=0, last_tiles=[1010], tiles_per_chunk=2)),
    (3 * 16384 + 17, "T = 49169: TC = 3074, tiles of 1024 x 3 + 2, the last chunk 3059 (1024 x 2 + 1011)",
     dict(TC=3074, empty=0, last_tiles=[1024, 1024, 1011], tiles_per_chunk=4)))]

# C: Cholesky sizes (n, what it stands for)
C_SIZES = [(2048, "G at S = 4, museval's block at I = 4"), (2560, "G at M = 5, block at I = 5"), (3072, "G at M = 6, block at I = 6"),
           (3584, "G at M = 7, block at I = 7"), (4096, "G at M = 8, block at I = 8")]
C_KAPPAS = (1e2, 1e6, 1e10, 1e13)


def gram_fft(refs):
    """G + eps I of museval_ref.filters_fft (M L square) for references (J, I, T)"""
    J, I, T = refs.shape
    M = J * I
    r = refs.reshape(M, T).astype(np.float64)
    nfft = int(2 ** np.ceil(np.log2(T + L - 1)))
    rf = np.fft.rfft(r, n=nfft)
    G = np.zeros((M * L, M * L))
    for a in range(M):
        for b in range(M):
            c = np.fft.irfft(rf[a] * np.conj(rf[b]), n=nfft)
            G[a * L:(a + 1) * L, b * L:(b + 1) * L] = scipy.linalg.toeplitz(np.hstack((c[0], c[-1:-L:-1])), r=c[:L])
    return G + MR.EPS * np.eye(M * L)


@functools.lru_cache(maxsize=None)
def a4_oracle(delta, device=None):
    """(refs, ests, LU metrics or None where numpy's LU finds G + eps I singular, SVD metrics) of the near-mono row (delta = 0: an
    exact copy); delta = 'lowpass' for the MUSDB18-style row"""
    refs, ests = lowpass_track() if delta == "lowpass" else near_mono_track(delta)
    try:
        lu = np.array(MR.metrics(refs, ests, A4_WIN, A4_WIN, MR.filters_fft))
    except np.linalg.LinAlgError:
        lu = None
    svd = np.array(MR.metrics(refs, ests, A4_WIN, A4_WIN, functools.partial(filters_svd, device=device)))
    return refs, ests, lu, svd


def a4_bound(lu, svd):
    """per metric and window: TOL_DB + 4 |LU - SVD|, the oracle's own spread where the normal equations part from the projection"""
    return TOL_DB + 4.0 * np.abs(np.asarray(lu) - np.asarray(svd))
