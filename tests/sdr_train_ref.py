"""Float64 restatements of the SDR criterion the recipes train with (src/criterion/sdr.py:6-20 ``sdr``, :72-110 ``NegSDR``,
src/criterion/pit.py:9-44 ``pit``) and per-row error bounds derived from the arithmetic of csrc/ctn_loss.cu (k_sdr_partial /
k_sdr_pit_pass, SdrPair, k_sdr_bwd / k_sdr_pit_bwd).  Every reference is computed in float64 from the same fp32 inputs.

Value of a pair, v = 10 log10f((|t|^2 + eps) / (|t - x|^2 + eps)), u = 2^-24:
  * |t|^2: fp32 squares summed in runs of at most four, then double: relative error <= 4u;
  * |t - x|^2 accumulated as an explicit residual: the difference t - x rounds once (2u on its square), the run of four adds 3u:
    relative error <= 6u (a residual formed as |t|^2 - 2<x,t> + |x|^2 would instead be off by ~u |t|^2 / |t - x|^2, a whole
    decibel at 60 dB);
  * both sums are cast to fp32 (u), eps is added (u), the quotient rounds (u), log10f (2u |v|);
  |v - v64| <= 2 [K10 (5u tt / (tt + eps) + 7u ee / (ee + eps) + 3u) + 2u |v64|], K10 = 10 / ln 10; the factor 2 covers the
  double sums and second-order terms.  Dropping eps makes a row with x == t infinite, which no finite bound accepts.
Gradient of a pair, d = g c (t - x), c = 20 / (ln 10 (|t - x|^2 + eps)), formed in double from the residual sum and cast to fp32:
  |d - d64| <= 2 (6u ee / (ee + eps) + 4u + g_rel) |d64| per element: the residual's relative error, the cast of c, the fp32
  difference and the product, plus g_rel, the relative error of the upstream weight g when fp32 arithmetic formed it (a mean's
  1/n).  A transposed residual table scores pair (j, i) in place of (i, j), which moves the value by far more than this.
PIT: loss_b = -(1/S) sum_i v[i][perm i] summed in fp32 in source order: its bound is the mean of the pair bounds plus S u mean |v|.
"""
import itertools
import math

import torch

U = 2.0 ** -24
EPS = 1e-12
K10 = 10.0 / math.log(10.0)


def stats(x, t):
    """x, t (..., T) -> (tt, ee) in float64"""
    x, t = x.double(), t.double()
    return (t * t).sum(-1), ((t - x) ** 2).sum(-1)


def sdr64(x, t, eps=EPS):
    tt, ee = stats(x, t)
    return 10.0 * torch.log10((tt + eps) / (ee + eps))


def sdr_bound(x, t, eps=EPS):
    tt, ee = stats(x, t)
    v = 10.0 * torch.log10((tt + eps) / (ee + eps))
    return 2.0 * (K10 * (5 * U * tt / (tt + eps) + 7 * U * ee / (ee + eps) + 3 * U) + 2 * U * v.abs())


def grad_coef64(x, t, eps=EPS):
    """dSDR / dx = c (t - x): c (...) in float64"""
    _, ee = stats(x, t)
    return 2.0 * K10 / (ee + eps)


def sdr_grad64(x, t, g, eps=EPS):
    """g (...) float64 weights per row -> g dSDR/dx (..., T) in float64"""
    return (g * grad_coef64(x, t, eps)).unsqueeze(-1) * (t.double() - x.double())


def sdr_grad_bound(x, t, g, eps=EPS, g_rel=0.0):
    """per-element bound on |d - d64|; g_rel = the relative error of the fp32 upstream weight"""
    _, ee = stats(x, t)
    rel = 2.0 * (6 * U * ee / (ee + eps) + 4 * U + g_rel)
    return rel.unsqueeze(-1) * sdr_grad64(x, t, g, eps).abs() + 1e-30


def pair_tables(x, t, eps=EPS):
    """x, t (B, S, T) -> v64 (B, S, S) = SDR(x_i, t_j) and its bound, both float64"""
    xe, te = x.unsqueeze(2), t.unsqueeze(1)
    return sdr64(xe, te, eps), sdr_bound(xe, te, eps)


def perms(S):
    return list(itertools.permutations(range(S)))


def pit64(x, t, eps=EPS):
    """PIT(NegSDR) in float64: -> dict(loss_b (B), perm (B, S) int64 (first minimum in itertools order), bound (B), all (B, P) losses,
    all_bound (B, P), v (B, S, S), v_bound (B, S, S))"""
    v, vb = pair_tables(x, t, eps)
    B, S, _ = v.shape
    P = torch.tensor(perms(S), dtype=torch.long)
    idx = torch.arange(S)
    vals = torch.stack([-v[:, idx, p].mean(-1) for p in P], dim=1)
    bnds = torch.stack([vb[:, idx, p].mean(-1) + S * U * v[:, idx, p].abs().mean(-1) for p in P], dim=1)
    best = torch.argmin(vals, dim=1)  # first minimum
    ar = torch.arange(B)
    return dict(loss_b=vals[ar, best], perm=P[best], bound=bnds[ar, best], all=vals, all_bound=bnds, v=v, v_bound=vb)


def separated(r):
    """(B,) bool: the best permutation beats every other one by more than the two bounds together"""
    vals, bnds = r["all"], r["all_bound"]
    if vals.shape[1] == 1:
        return torch.ones(vals.shape[0], dtype=torch.bool)
    best = vals.min(dim=1, keepdim=True).values
    best_b = torch.gather(bnds, 1, torch.argmin(vals, dim=1, keepdim=True))
    margin = vals - best - best_b - bnds
    is_best = vals == best
    return torch.where(is_best, torch.ones_like(margin, dtype=torch.bool), margin > 0).all(dim=1)


def pit_grad64(x, t, perm, g, eps=EPS):
    """gradient of sum_b g[b] loss_b w.r.t. x through `perm`: loss_b = -(1/S) sum_i SDR(x_i, t_perm(i)) -> (B, S, T) float64"""
    B, S, _ = x.shape
    tp = torch.gather(t, 1, perm.unsqueeze(-1).expand(t.shape))
    return sdr_grad64(x, tp, (-g.double() / S).unsqueeze(-1).expand(B, S), eps)


def pit_grad_bound(x, t, perm, g, eps=EPS, g_rel=0.0):
    B, S, _ = x.shape
    tp = torch.gather(t, 1, perm.unsqueeze(-1).expand(t.shape))
    return sdr_grad_bound(x, tp, (-g.double() / S).unsqueeze(-1).expand(B, S), eps, g_rel)


# ---- differentiable float64 restatements (torch autograd), for the end-to-end gradients --------------------------------------

def sdr_autograd(x, t, eps=EPS):
    """src/criterion/sdr.py:6-20 on any dtype, differentiable"""
    return 10.0 * torch.log10(((t * t).sum(-1) + eps) / (((t - x) ** 2).sum(-1) + eps))


def pit_neg_sdr_autograd(x, t, eps=EPS):
    """PIT1d(NegSDR(), S)(x, t) (batch mean) on (B, S, T), differentiable -> (loss, perm)"""
    S = x.shape[1]
    P = torch.tensor(perms(S), dtype=torch.long)
    losses = torch.stack([-sdr_autograd(x, t[:, p], eps).mean(-1) for p in P], dim=1)
    loss, idx = torch.min(losses, dim=1)
    return loss.mean(), P[idx]


def orpit_neg_sdr(x, t, rest, eps=EPS):
    """ORPIT(NegSDR()) on x (B, 2, T), t (B, n, T), with rest[b, i] (B, n, T) = the sum of the other targets as the caller formed it
    -> (loss_b (B), indices (B), and the candidates' values (B, n)), differentiable"""
    n = t.shape[1]
    cand = -sdr_autograd(x[:, :1], t, eps) - sdr_autograd(x[:, 1:], rest, eps) / (n - 1)
    loss_b, idx = torch.min(cand, dim=1)
    return loss_b, idx, cand


def sinkpit_neg_sdr(x, t, coldness=1.0, iteration=10, eps=EPS):
    """sinkpit(NegSDR()) on (B, S, T) without the batch mean (src/criterion/pit.py:162-194), differentiable -> (loss_b, P)"""
    B, S, T = x.shape
    L = -sdr_autograd(x.unsqueeze(2).expand(B, S, S, T), t.unsqueeze(1).expand(B, S, S, T), eps)
    Z = -coldness * L
    for _ in range(iteration):
        Z = Z - torch.logsumexp(Z, dim=1, keepdim=True)
        Z = Z - torch.logsumexp(Z, dim=2, keepdim=True)
    P = torch.exp(Z)
    return torch.sum((L + Z / coldness) * P, dim=(1, 2)), P
