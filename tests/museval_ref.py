"""Float64 oracle of BSS Eval v4 for multichannel source images (museval 0.4 ``evaluate(..., mode='v4')``), in numpy / scipy,
restated from the definition along museval's route: FFT correlations over the whole track, a dense solve of G + eps I and of its
per-source diagonal blocks, projections of each window's zero-padded slice by FFT convolution, and energies of explicit residual
signals.  Nothing here calls museval.  ``filters_qr`` is a second, independent route to the filters (a QR least-squares fit on the
explicit matrix of delayed references), and ``make_track`` builds the test signals the CPU and GPU tests share."""
import numpy as np
import scipy.linalg
import scipy.signal

L = 512
EPS = np.finfo(np.float64).eps


def _safe_db(num, den):
    return np.inf if den == 0 else 10 * np.log10(num / den)


def nwin_of(T, win, hop):
    return (T - win + hop) // hop


def filters_fft(refs, ests):
    """refs, ests (J, I, T) -> C (M L, M) and Ct (J, I L, I): the distortion filters of every estimate row on all M = J I delayed
    reference rows, and on the rows of its own source alone, from G + eps I and its diagonal blocks"""
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
            c = np.fft.irfft(rf[a] * np.conj(rf[b]), n=nfft)  # c[k] = sum_u r_a(u + k) r_b(u)
            G[a * L:(a + 1) * L, b * L:(b + 1) * L] = scipy.linalg.toeplitz(np.hstack((c[0], c[-1:-L:-1])), r=c[:L])
    D = np.zeros((M * L, M))
    for a in range(M):
        c = np.fft.irfft(rf[a][None] * np.conj(ef), n=nfft)  # (M, nfft): sum_u r_a(u + k) e(u)
        D[a * L:(a + 1) * L] = np.hstack((c[:, :1], c[:, -1:-L:-1])).T
    C = np.linalg.solve(G + EPS * np.eye(M * L), D)
    Ct = np.zeros((J, I * L, I))
    for j in range(J):
        sl = slice(j * I * L, (j + 1) * I * L)
        Ct[j] = np.linalg.solve(G[sl, sl] + EPS * np.eye(I * L), D[sl, j * I:(j + 1) * I])
    return C, Ct


def filters_qr(refs, ests):
    """filters_fft by an independent route: least squares of each estimate row (zero-padded by L - 1) on the explicit
    (T + L - 1) x (M L) matrix of delayed references, by QR (no eps: it is far below the bound at these sizes)"""
    J, I, T = refs.shape
    M = J * I
    r = refs.reshape(M, T)
    A = np.zeros((T + L - 1, M * L))
    for m in range(M):
        for k in range(L):
            A[k:k + T, m * L + k] = r[m]
    e = np.hstack((ests.reshape(M, T), np.zeros((M, L - 1)))).T
    Q, R = np.linalg.qr(A)
    C = scipy.linalg.solve_triangular(R, Q.T @ e)
    Ct = np.zeros((J, I * L, I))
    for j in range(J):
        Qj, Rj = np.linalg.qr(A[:, j * I * L:(j + 1) * I * L])
        Ct[j] = scipy.linalg.solve_triangular(Rj, Qj.T @ e[:, j * I:(j + 1) * I])
    return C, Ct


def _silent(x):
    """museval._any_source_silent on one window of (J, I, n): the channel sum of some source is zero throughout"""
    return bool(np.any(np.all(np.sum(x, axis=1) == 0, axis=1)))


def metrics(refs, ests, win, hop, filters=filters_fft):
    """refs, ests (J, I, T) -> SDR, ISR, SIR, SAR (J, nwin) float64"""
    refs = np.asarray(refs, dtype=np.float64)
    ests = np.asarray(ests, dtype=np.float64)
    J, I, T = refs.shape
    M = J * I
    nwin = nwin_of(T, win, hop)
    C, Ct = filters(refs, ests)
    Cm = C.reshape(M, L, M).transpose(0, 2, 1)  # [m][col][k]
    out = np.full((4, J, nwin), np.nan)
    for w in range(nwin):
        sl = slice(w * hop, w * hop + win)
        r, e = refs[:, :, sl], ests[:, :, sl]
        if _silent(r) or _silent(e):
            continue
        rw = r.reshape(M, win)
        p_all = scipy.signal.fftconvolve(rw[:, None, :], Cm, axes=-1).sum(0)  # (col, win + L - 1)
        pad = lambda x: np.concatenate((x, np.zeros(x.shape[:-1] + (L - 1,))), axis=-1)  # noqa: E731
        s, ep = pad(r), pad(e)
        for j in range(J):
            ctj = Ct[j].reshape(I, L, I).transpose(0, 2, 1)  # [c'][c][k]
            p_j = scipy.signal.fftconvolve(r[j][:, None, :], ctj, axes=-1).sum(0)  # (c, win + L - 1)
            pa = p_all[j * I:(j + 1) * I]
            q = [np.sum(s[j] ** 2), np.sum((ep[j] - s[j]) ** 2), np.sum((p_j - s[j]) ** 2), np.sum(p_j ** 2),
                 np.sum((pa - p_j) ** 2), np.sum(pa ** 2), np.sum((ep[j] - pa) ** 2)]
            out[:, j, w] = (_safe_db(q[0], q[1]), _safe_db(q[0], q[2]), _safe_db(q[3], q[4]), _safe_db(q[5], q[6]))
    return tuple(out)


def make_track(rng, J, I, T, coloured=False):
    """references and estimates (J, I, T) float32.  Each stem is noise (low-pass filtered when coloured, like music), its second
    channel a mix of the first and fresh noise; each estimate channel is its reference through a short random FIR plus
    cross-talk from the other stems and white noise"""
    src = rng.standard_normal((J, I, T))
    if coloured:
        src = scipy.signal.lfilter(scipy.signal.firwin(129, 0.3), [1.0], src, axis=-1)
    refs = src.copy()
    for c in range(1, I):
        refs[:, c] = 0.7 * src[:, 0] + 0.5 * src[:, c]
    refs *= rng.uniform(0.3, 3.0, (J, 1, 1))
    ests = np.empty_like(refs)
    for j in range(J):
        for c in range(I):
            h = np.zeros(24)
            h[0] = 1.0
            h[1:] = 0.3 * rng.standard_normal(23) * np.exp(-np.arange(1, 24) / 5.0)
            ests[j, c] = scipy.signal.lfilter(h, [1.0], refs[j, c])
            for i in range(J):
                if i != j:
                    ests[j, c] += rng.uniform(0.05, 0.3) * refs[i, c]
            ests[j, c] += rng.uniform(0.02, 0.2) * np.std(refs[j, c]) * rng.standard_normal(T)
    return refs.astype(np.float32), ests.astype(np.float32)
