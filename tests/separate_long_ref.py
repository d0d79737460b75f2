"""Float64 restatement of ConvTasNet.separate_long's post-processing in plain torch / Python, written from DESIGN.md: the chunk
plan, the permutation alignment of neighbouring chunks and the windowed overlap-add.  Nothing here calls the library; the
per-chunk estimates are an input."""
import itertools
import math

import torch


def plan(T, chunk, hop):
    """-> (starts, Lc): chunk k covers [starts[k], starts[k] + Lc)"""
    if T <= chunk:
        return [0], T
    starts = []
    s = 0
    while s + chunk < T:
        starts.append(s)
        s += hop
    starts.append(T - chunk)
    return starts, chunk


def align(est, starts, Lc):
    """est (K, S, Lc) of ONE recording -> list of K tuples: perms[k][s] = row of chunk k that carries source s"""
    K, S, _ = est.shape
    e = est.double()
    perms = [tuple(range(S))]
    for k in range(K - 1):
        ov = starts[k] + Lc - starts[k + 1]
        a = e[k, :, Lc - ov:]
        b = e[k + 1, :, :ov]
        c = a @ b.t()                                       # c[i][j] = <e_k[i], e_{k+1}[j]>
        best, best_v = None, None
        for pi in itertools.permutations(range(S)):
            v = sum(float(c[i, pi[i]]) for i in range(S))
            if best is None or v > best_v:
                best, best_v = pi, v
        perms.append(tuple(best[perms[k][s]] for s in range(S)))
    return perms


def weights(starts, Lc, T):
    """(K, T) float64: w_k(t), zero outside chunk k"""
    K = len(starts)
    w = torch.zeros(K, T, dtype=torch.float64)
    for k, s0 in enumerate(starts):
        wk = torch.ones(Lc, dtype=torch.float64)
        if k > 0:
            a = max(starts[k - 1] + Lc - s0, 0)
            if a > 0:
                wk[:a] *= torch.sin(0.5 * math.pi * (torch.arange(a, dtype=torch.float64) + 0.5) / a) ** 2
        if k < K - 1:
            n = max(s0 + Lc - starts[k + 1], 0)
            if n > 0:
                wk[Lc - n:] *= torch.cos(0.5 * math.pi * (torch.arange(n, dtype=torch.float64) + 0.5) / n) ** 2
        w[k, s0:s0 + Lc] = wk
    return w


def overlap_add(est, perms, starts, Lc, T):
    """est (K, S, Lc), perms: K tuples (None: identity) -> (S, T) float64"""
    K, S, _ = est.shape
    w = weights(starts, Lc, T)
    num = torch.zeros(S, T, dtype=torch.float64)
    for k, s0 in enumerate(starts):
        rows = list(perms[k]) if perms is not None else list(range(S))
        num[:, s0:s0 + Lc] += w[k, s0:s0 + Lc] * est[k, rows].double()
    return num / w.sum(0)


def separate(est, B, T, chunk, hop, do_align=True):
    """est (B*K, S, Lc), chunk index b*K + k -> (out (B, S, T) float64, perms (B, K, S) int64)"""
    starts, Lc = plan(T, chunk, hop)
    K, S = len(starts), est.shape[1]
    outs, allp = [], []
    for b in range(B):
        e = est[b * K:(b + 1) * K]
        p = align(e, starts, Lc) if (do_align and S > 1) else [tuple(range(S))] * K
        outs.append(overlap_add(e, p, starts, Lc, T))
        allp.append(p)
    return torch.stack(outs), torch.tensor(allp, dtype=torch.int64).reshape(B, K, S)
