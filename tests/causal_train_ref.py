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


def cln_conv(x, gamma, beta, eps=1e-12):
    """The oracle's cLN (convtasnet_oracle.cln, the same expressions in the same order, so the forward is bit-identical wherever
    v_t >= 0) with the kernels' convention at v_t <= 0: the root is taken of 1 there and masked to 0, so autograd sees a
    constant variance and gives e_t = 0 instead of the inf / NaN of d sqrt(v) / dv at v = 0."""
    B, C, T = x.shape
    cum_sum = torch.cumsum(x.sum(dim=1), dim=1)
    cum_sq = torch.cumsum((x ** 2).sum(dim=1), dim=1)
    cum_num = torch.arange(C, C * (T + 1), C, dtype=x.dtype, device=x.device)
    cum_mean = cum_sum / cum_num
    cum_var = cum_sq / cum_num - cum_mean ** 2
    pos = cum_var > 0
    sd = torch.where(pos, torch.sqrt(torch.where(pos, cum_var, torch.ones_like(cum_var))), torch.zeros_like(cum_var))
    return (x - cum_mean.unsqueeze(1)) / (sd.unsqueeze(1) + eps) * gamma.view(1, C, 1) + beta.view(1, C, 1)


def silent_onset_(x, zero, fade):
    """in place on (..., T): the first `zero` samples exactly 0, then a linear fade-in over `fade` samples"""
    x[..., :zero] = 0
    x[..., zero:zero + fade] *= torch.arange(1, fade + 1, dtype=x.dtype) / fade
    return x


# cLN backward mutants (a plausible bug of k_cln_bwd_sums / k_cln_bwd_scan each), for tests/test_causal_train_edges_cpu.py:
#   "exclusive"  U, V summed over t > tau instead of t >= tau
#   "seg_first"  the first frame of each per-thread segment of the 1024-thread reverse scan left out of U, V
#   "slices8"    channels >= CLN_BWD_SLICES = 8 left out of (a_t, b_t)
#   "unclamped"  e_t = -r_t^2 b_t / (2 s_t) also where v_t <= 0
CLN_MUTANTS = ("exclusive", "seg_first", "slices8", "unclamped")


def cln_bwd(dy, pre, gamma, eps, slope=None, mut=None):
    """-> dict of fp64 results (dpre, dgamma, dbeta, dslope, dbias) and `mag`, the same sums over absolute values of their terms.
    All of dy, pre (B, C, T), gamma (C) in fp64; slope: python float or None; mut: None or one of CLN_MUTANTS."""
    x = pre if slope is None else prelu(pre, slope)
    S, Q, n = cln_stats(x)
    m = S / n
    v = Q / n - m * m
    pos = v > 0
    sd = torch.where(pos, v.clamp_min(0).sqrt(), torch.zeros_like(v))
    r = 1.0 / (sd + eps)
    g = dy * gamma.view(1, -1, 1)
    gs = g[:, :8] if mut == "slices8" else g
    a = gs.sum(1)
    b = (gs * (x[:, :gs.shape[1]] - m[:, None])).sum(1)
    if mut == "unclamped":
        e = -r * r * b / (2 * sd)
    else:
        e = torch.where(pos, -r * r * b / (2 * torch.where(pos, sd, torch.ones_like(sd))), torch.zeros_like(v))
    dS = (-r * a - 2 * m * e) / n
    dQ = e / n
    if mut == "seg_first":
        T = x.shape[-1]
        per = (T + 1023) // 1024
        keep = ((T - 1 - torch.arange(T)) % per != 0).to(x.dtype)  # reversed frame index j = T - 1 - t, segments start at j % per == 0
        dS, dQ = dS * keep, dQ * keep
    U = torch.flip(torch.cumsum(torch.flip(dS, [1]), 1), [1])
    V = torch.flip(torch.cumsum(torch.flip(dQ, [1]), 1), [1])
    if mut == "exclusive":
        U, V = U - dS, V - dQ
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


def _taps(P, mut):
    """mut "drop_last": tap P - 1 (the one at offset 0, the only one inside when the dilation passes the frame count) left out"""
    return range(P - 1) if mut == "drop_last" else range(P)


def cdw_fwd(hn, wd, bd, dil, mut=None):
    """causal depthwise conv: u[c][t] = bd[c] + sum_k wd[c][k] hn[c][t - (P - 1 - k) dil]"""
    B, C, T = hn.shape
    P = wd.shape[1]
    u = bd.view(1, C, 1).expand(B, C, T).clone()
    for k in _taps(P, mut):
        off = (P - 1 - k) * dil
        if off < T:
            u[:, :, off:] += wd[:, k].view(1, C, 1) * hn[:, :, :T - off]
    return u


def cdw_bwd(du, hn, wd, dil, mut=None):
    """-> (dhn, dwd, mag_dhn, mag_dwd) of cdw_fwd"""
    B, C, T = hn.shape
    P = wd.shape[1]
    dhn, mhn = torch.zeros_like(hn), torch.zeros_like(hn)
    dwd, mwd = torch.zeros_like(wd), torch.zeros_like(wd)
    for k in _taps(P, mut):
        off = (P - 1 - k) * dil
        if off < T:
            dhn[:, :, :T - off] += wd[:, k].view(1, C, 1) * du[:, :, off:]
            mhn[:, :, :T - off] += (wd[:, k].view(1, C, 1) * du[:, :, off:]).abs()
            dwd[:, k] = (du[:, :, off:] * hn[:, :, :T - off]).sum((0, 2))
            mwd[:, k] = (du[:, :, off:] * hn[:, :, :T - off]).abs().sum((0, 2))
    return dhn, dwd, mhn, mwd


# ---- the probe rows of tests/test_causal_train_edges_gpu.py and the bounds they are held to ------------------------------------
# cLN backward: frame counts around the 1024-thread scan (1, 2 and 16 frames per thread), channel counts below, just past and far
# past CLN_BWD_SLICES = 8; inputs "randn" (randn + 0.3), "silent" (sample 0 starts with 5/8 of its frames at exactly 0, then a
# 1/32 fade-in, as the silent-onset model row; sample 1 as "randn") and "dc" (100 + randn: the mean dominates Q_t / n_t - m_t^2)
CLN_FRAMES, CLN_CHANNELS, CLN_INPUTS, CLN_B = (1024, 1025, 2049, 15999), (3, 9, 512), ("randn", "silent", "dc"), 2
EPS_PROBE = 1e-8


def cln_row(frames, C, slope, kind):
    """-> (dy, pre, gamma) in fp32 for one cLN backward row"""
    g = torch.Generator().manual_seed(frames * 7 + C + (0 if slope is None else 1) + 10 * CLN_INPUTS.index(kind))
    pre = torch.randn(CLN_B, C, frames, generator=g) + (100.0 if kind == "dc" else 0.3)
    if kind == "silent":
        silent_onset_(pre[0], 5 * frames // 8, max(1, frames // 32))
    dy = torch.randn(CLN_B, C, frames, generator=g)
    gamma = 1.0 + 0.3 * torch.randn(C, generator=g)
    return dy, pre, gamma


def cln_bwd_bounds(want, frames, slope):
    """{output: bound} of the kernels' fp32 evaluation: dpre 24 ulps of its magnitude, the per-row sums 4 ulps more for every
    1024-frame stretch a thread adds before the block's double reduction (the bounds of tests/test_causal_train_gpu.py)"""
    mag, n_seq = want["mag"], 4 * ((frames + 1023) // 1024)
    b = dict(dpre=24 * U24 * mag["dpre"], dgamma=(16 + n_seq) * U24 * mag["dgamma"], dbeta=(8 + n_seq) * U24 * mag["dbeta"])
    if slope is not None:  # with no pre <= 0 (the "dc" input) dslope is exactly 0 and its magnitude too
        b["dslope"] = (32 + n_seq) * U24 * mag["dslope"]
        b["dbias"] = (32 + n_seq) * U24 * mag["dbias"]
    return {k: v + 1e-30 for k, v in b.items()}


# causal depthwise: widths 4, 6, 7 and 8 = CTN_MAX_P (k_cdw_bwd's w / acc / part arrays full), dilations inside and far past the
# frame count, one frame, one past a 32-frame warp, 1003 and 15999 frames
CDW_P, CDW_DIL, CDW_FRAMES, CDW_BC = (4, 6, 7, 8), (1, 16, 512), (1, 33, 1003, 15999), ((1, 1), (3, 136))
SLOPE_PROBE = 0.25


def cdw_row(P, dil, frames, B, C):
    """-> (hpre, du, g1, b1, wd, bd) in fp32 for one causal depthwise row"""
    g = torch.Generator().manual_seed(P * 100 + dil + frames + C)
    hpre = torch.randn(B, C, frames, generator=g) + 0.3
    du = torch.randn(B, C, frames, generator=g)
    g1, b1 = 1.0 + 0.3 * torch.randn(C, generator=g), 0.2 * torch.randn(C, generator=g)
    wd, bd = torch.randn(C, P, generator=g), torch.randn(C, generator=g)
    return hpre, du, g1, b1, wd, bd


def cdw_expect(hpre, du, g1, b1, wd, bd, dil, mut=None):
    """fp64 (u_pre, d_hn, d_wd) of the row and their bounds (those of tests/test_causal_train_gpu.py): -> {output: (value, bound)}.
    hn carries the error of (x - m) r: 2^-24 (|x| + |m|) r |gamma| per element, folded in through |hn| + that term."""
    h64 = prelu(hpre.double(), SLOPE_PROBE)
    g1, b1, wd, bd, du = g1.double(), b1.double(), wd.double(), bd.double(), du.double()
    hn = cln_fwd(h64, g1, b1, EPS_PROBE)
    u = cdw_fwd(hn, wd, bd, dil, mut)
    dhn, dwd, mhn, _ = cdw_bwd(du, hn, wd, dil, mut)
    S, Q, n = cln_stats(h64)
    m = S / n
    r = 1.0 / ((Q / n - m * m).clamp_min(0).sqrt() + EPS_PROBE)
    hn_mag = (h64.abs() + m.abs()[:, None]) * r[:, None] * g1.abs().view(1, -1, 1) + b1.abs().view(1, -1, 1)
    _, _, _, mwd_h = cdw_bwd(du, hn_mag, wd.abs(), dil)
    u_mag = cdw_fwd(hn_mag, wd.abs(), bd.abs(), dil)
    P, frames = wd.shape[1], hpre.shape[-1]
    n_seq = (frames + 255) // 256
    return dict(upre=(u, (8 + 2 * P) * U24 * u_mag + 1e-30), dhn=(dhn, (2 + P) * U24 * mhn + 1e-12),
                dwd=(dwd, (16 + n_seq) * U24 * mwd_h + 1e-12))
