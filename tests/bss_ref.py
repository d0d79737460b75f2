"""Float64 oracle of BSS Eval (mir_eval 0.7 ``bss_eval_sources``, filter length 512) in numpy / scipy, restated from its
definition along mir_eval's own route: FFT correlations, the dense block-Toeplitz Gram matrix, a dense solve, projections by FFT
convolution and explicit residual signals.  Nothing here calls the library.  ``project_qr`` is a second, independent route (QR of
the explicit matrix of delayed references), and ``make_item`` builds the test signals the CPU and GPU tests share."""
import itertools

import numpy as np
import scipy.linalg
import scipy.signal

L = 512


def _validate(refs, ests):
    if refs.shape != ests.shape:
        raise ValueError("shape mismatch: {} vs {}".format(refs.shape, ests.shape))
    if np.any(np.all(refs == 0, axis=1)):
        raise ValueError("a reference source is silent")
    if np.any(np.all(ests == 0, axis=1)):
        raise ValueError("an estimated source is silent")


def _safe_db(num, den):
    return np.inf if den == 0 else 10 * np.log10(num / den)


def project_fft(refs, ests):
    """refs (S, T), ests (n, T) -> P_all (n, T+L-1) and P (n, S, T+L-1): the projections of every estimate on all delayed
    references and on those of reference j alone"""
    S, T = refs.shape
    nfft = int(2 ** np.ceil(np.log2(T + L - 1)))
    sf = np.fft.rfft(refs, n=nfft)
    ef = np.fft.rfft(ests, n=nfft)
    G = np.zeros((S * L, S * L))
    for i in range(S):
        for j in range(S):
            ssf = np.fft.irfft(sf[i] * np.conj(sf[j]), n=nfft)  # ssf[m] = sum_u r_i(u + m) r_j(u)
            G[i * L:(i + 1) * L, j * L:(j + 1) * L] = scipy.linalg.toeplitz(np.hstack((ssf[0], ssf[-1:-L:-1])), r=ssf[:L])
    D = np.zeros((S * L, ests.shape[0]))
    for i in range(S):
        ssef = np.fft.irfft(sf[i][None] * np.conj(ef), n=nfft)  # (n, nfft): sum_u r_i(u + m) e(u)
        D[i * L:(i + 1) * L] = np.hstack((ssef[:, :1], ssef[:, -1:-L:-1])).T
    n = ests.shape[0]
    C_all = np.linalg.solve(G, D)
    P_all = np.zeros((n, T + L - 1))
    P = np.zeros((n, S, T + L - 1))
    for i in range(S):
        C_i = np.linalg.solve(G[i * L:(i + 1) * L, i * L:(i + 1) * L], D[i * L:(i + 1) * L])
        for a in range(n):
            P_all[a] += scipy.signal.fftconvolve(C_all[i * L:(i + 1) * L, a], refs[i])
            P[a, i] = scipy.signal.fftconvolve(C_i[:, a], refs[i])
    return P_all, P


def project_qr(refs, ests):
    """project_fft by an independent route: QR of the explicit (T+L-1) x (S L) matrix of delayed references"""
    S, T = refs.shape
    A = np.zeros((T + L - 1, S * L))
    for i in range(S):
        for k in range(L):
            A[k:k + T, i * L + k] = refs[i]
    e = np.hstack((ests, np.zeros((ests.shape[0], L - 1))))
    Q = np.linalg.qr(A)[0]
    P_all = (Q @ (Q.T @ e.T)).T
    P = np.zeros((ests.shape[0], S, T + L - 1))
    for i in range(S):
        Qi = np.linalg.qr(A[:, i * L:(i + 1) * L])[0]
        P[:, i] = (Qi @ (Qi.T @ e.T)).T
    return P_all, P


def tables(refs, ests, project=project_fft):
    """-> SDR, SIR, SAR (S, S) over (estimate a, reference j), from explicit residual signals"""
    S, T = refs.shape
    P_all, P = project(refs, ests)
    e = np.hstack((ests, np.zeros((S, L - 1))))
    sdr, sir, sar = (np.empty((S, S)) for _ in range(3))
    for a in range(S):
        for j in range(S):
            sdr[a, j] = _safe_db(np.sum(P[a, j] ** 2), np.sum((e[a] - P[a, j]) ** 2))
            sir[a, j] = _safe_db(np.sum(P[a, j] ** 2), np.sum((P_all[a] - P[a, j]) ** 2))
            sar[a, j] = _safe_db(np.sum(P_all[a] ** 2), np.sum((e[a] - P_all[a]) ** 2))
    return sdr, sir, sar


def bss_eval_sources(refs, ests, compute_permutation=True, project=project_fft, return_margin=False):
    """refs, ests (S, T) -> sdr, sir, sar (S,), perm (S,), as mir_eval returns them; return_margin adds the gap in dB between the
    best and the second-best mean SIR (inf for S = 1 or without permutation)"""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    ests = np.atleast_2d(np.asarray(ests, dtype=np.float64))
    _validate(refs, ests)
    S = refs.shape[0]
    sdr, sir, sar = tables(refs, ests, project)
    dum = np.arange(S)
    margin = np.inf
    if compute_permutation:
        perms = list(itertools.permutations(range(S)))
        mean_sir = np.array([np.mean(sir[list(p), dum]) for p in perms])
        popt = perms[int(np.argmax(mean_sir))]
        if len(perms) > 1:
            top = np.sort(mean_sir)[::-1]
            margin = top[0] - top[1]
    else:
        popt = tuple(range(S))
    idx = (list(popt), dum)
    out = (sdr[idx], sir[idx], sar[idx], np.asarray(popt))
    return out + (margin,) if return_margin else out


def make_item(rng, S, T, coloured=False):
    """references (S, T) and a shuffled set of estimates (S, T), float32: each estimate is its reference through a short random
    FIR plus cross-talk from the others and white noise.  coloured: the references are low-pass filtered noise (most of their
    energy below 0.4 of the band, like 8 kHz speech), which makes the Gram matrix far worse conditioned than white ones"""
    refs = rng.standard_normal((S, T))
    if coloured:
        refs = scipy.signal.lfilter(scipy.signal.firwin(129, 0.4), [1.0], refs, axis=1)
    refs = refs * rng.uniform(0.3, 3.0, (S, 1))
    ests = np.empty_like(refs)
    for j in range(S):
        h = np.zeros(24)
        h[0] = 1.0
        h[1:] = 0.3 * rng.standard_normal(23) * np.exp(-np.arange(1, 24) / 5.0)
        ests[j] = scipy.signal.lfilter(h, [1.0], refs[j])
        for i in range(S):
            if i != j:
                ests[j] += rng.uniform(0.05, 0.3) * refs[i]
        ests[j] += rng.uniform(0.02, 0.2) * np.std(refs[j]) * rng.standard_normal(T)
    ests = ests[rng.permutation(S)]
    return refs.astype(np.float32), ests.astype(np.float32)
