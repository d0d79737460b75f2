"""fp64 references of the causal training path's kernels: the closed form of the cLN backward (with an optional PReLU in front)
and the causal depthwise backward, each with the magnitude its fp32 evaluation is judged against.

Closed form (DESIGN.md, "Causal training"), per sample, n_t = C (t + 1), S_t / Q_t the inclusive prefix sums over frames of
sum_c x / sum_c x^2, m_t = S_t / n_t, v_t = Q_t / n_t - m_t^2, s_t = sqrt(max(v_t, 0)), r_t = 1 / (s_t + eps):
    g = dy gamma_c ; a_t = sum_c g ; b_t = sum_c g (x - m_t) ; e_t = -r_t^2 b_t / (2 s_t)  (0 where v_t <= 0)
    dS_t = (-r_t a_t - 2 m_t e_t) / n_t ; dQ_t = e_t / n_t ; U, V = their suffix sums over frames
    dx = g r + U + 2 x V ; dgamma_c = sum dy (x - m) r ; dbeta_c = sum dy
"""
import torch

U24 = 2.0 ** -24


def prelu(x, a):
    return torch.where(x >= 0, x, a * x)


def cln_stats(x):
    """x (B, C, T) fp64 -> (S, Q, n) each (B, T)"""
    B, C, T = x.shape
    S = torch.cumsum(x.sum(1), 1)
    Q = torch.cumsum((x * x).sum(1), 1)
    n = (C * torch.arange(1, T + 1, dtype=x.dtype)).expand(B, T)
    return S, Q, n


def cln_fwd(x, gamma, beta, eps):
    S, Q, n = cln_stats(x)
    m = S / n
    sd = (Q / n - m * m).clamp_min(0).sqrt()
    return (x - m[:, None]) / (sd[:, None] + eps) * gamma.view(1, -1, 1) + beta.view(1, -1, 1)


def cln_bwd(dy, pre, gamma, eps, slope=None):
    """-> dict of fp64 results (dpre, dgamma, dbeta, dslope, dbias) and `mag`, the same sums over absolute values of their terms.
    All of dy, pre (B, C, T), gamma (C) in fp64; slope: python float or None."""
    x = pre if slope is None else prelu(pre, slope)
    S, Q, n = cln_stats(x)
    m = S / n
    v = Q / n - m * m
    pos = v > 0
    sd = torch.where(pos, v.clamp_min(0).sqrt(), torch.zeros_like(v))
    r = 1.0 / (sd + eps)
    g = dy * gamma.view(1, -1, 1)
    a = g.sum(1)
    b = (g * (x - m[:, None])).sum(1)
    e = torch.where(pos, -r * r * b / (2 * torch.where(pos, sd, torch.ones_like(sd))), torch.zeros_like(v))
    dS = (-r * a - 2 * m * e) / n
    dQ = e / n
    U = torch.flip(torch.cumsum(torch.flip(dS, [1]), 1), [1])
    V = torch.flip(torch.cumsum(torch.flip(dQ, [1]), 1), [1])
    dx = g * r[:, None] + U[:, None] + 2 * x * V[:, None]
    # U and V are sums over every later frame and every channel of terms that carry the rounding of g = dy gamma and of PReLU(pre):
    # their error scales with the sums of the terms' absolute values (Um, Vm), not with |U|, |V|, which cancel
    A = g.abs().sum(1)
    E = torch.where(pos, r * r * (g.abs() * (x.abs() + m.abs()[:, None])).sum(1) / (2 * torch.where(pos, sd, torch.ones_like(sd))),
                    torch.zeros_like(v))
    Um = torch.flip(torch.cumsum(torch.flip((r * A + 2 * m.abs() * E) / n, [1]), 1), [1])
    Vm = torch.flip(torch.cumsum(torch.flip(E / n, [1]), 1), [1])
    dx_mag = (g * r[:, None]).abs() + Um[:, None] + 2 * x.abs() * Vm[:, None]
    xc, xc_mag = (x - m[:, None]) * r[:, None], (x.abs() + m.abs()[:, None]) * r[:, None]
    out = dict(dgamma=(dy * xc).sum((0, 2)), dbeta=dy.sum((0, 2)))
    mag = dict(dgamma=(dy.abs() * xc_mag).sum((0, 2)), dbeta=dy.abs().sum((0, 2)))
    if slope is None:
        out["dpre"], mag["dpre"] = dx, dx_mag
    else:
        neg = ~(pre > 0)
        k = torch.where(neg, torch.full_like(pre, slope), torch.ones_like(pre))
        out["dpre"], mag["dpre"] = dx * k, dx_mag * k.abs()
        out["dslope"] = (dx * pre * neg).sum().reshape(1)
        mag["dslope"] = (dx_mag * pre.abs() * neg).sum().reshape(1)
        out["dbias"], mag["dbias"] = out["dpre"].sum((0, 2)), mag["dpre"].sum((0, 2))
    out["mag"] = mag
    return out


def cdw_fwd(hn, wd, bd, dil):
    """causal depthwise conv: u[c][t] = bd[c] + sum_k wd[c][k] hn[c][t - (P - 1 - k) dil]"""
    B, C, T = hn.shape
    P = wd.shape[1]
    u = bd.view(1, C, 1).expand(B, C, T).clone()
    for k in range(P):
        off = (P - 1 - k) * dil
        if off < T:
            u[:, :, off:] += wd[:, k].view(1, C, 1) * hn[:, :, :T - off]
    return u


def cdw_bwd(du, hn, wd, dil):
    """-> (dhn, dwd, mag_dhn, mag_dwd) of cdw_fwd"""
    B, C, T = hn.shape
    P = wd.shape[1]
    dhn, mhn = torch.zeros_like(hn), torch.zeros_like(hn)
    dwd, mwd = torch.zeros_like(wd), torch.zeros_like(wd)
    for k in range(P):
        off = (P - 1 - k) * dil
        if off < T:
            dhn[:, :, :T - off] += wd[:, k].view(1, C, 1) * du[:, :, off:]
            mhn[:, :, :T - off] += (wd[:, k].view(1, C, 1) * du[:, :, off:]).abs()
            dwd[:, k] = (du[:, :, off:] * hn[:, :, :T - off]).sum((0, 2))
            mwd[:, k] = (du[:, :, off:] * hn[:, :, :T - off]).abs().sum((0, 2))
    return dhn, dwd, mhn, mwd
