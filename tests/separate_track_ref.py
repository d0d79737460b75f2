"""Float64 restatement of ConvTasNet.separate_track around the forward, in plain torch / Python, written from DESIGN.md §12: the
two segment plans, the per-(segment, channel) statistics, the standardised chunks, and the de-standardising overlap-add.
Nothing here calls the library; the per-chunk estimates are an input.  Also the error bounds the GPU tests hold the kernels to."""
import math

import torch

import separate_long_ref as SL

U64 = 2.0 ** -53   # unit roundoff of double
U32 = 2.0 ** -24   # unit roundoff of float


def plan(T, segment, hop=None):
    """-> (starts, Lc).  hop None / 0: the tester's layout (K = ceil(T / segment) segments of `segment` samples, zeros past T);
    otherwise the cross-faded chunk plan of separate_long"""
    if not hop:
        K = -(-T // segment)
        return [k * segment for k in range(K)], segment
    return SL.plan(T, segment, hop)


def chunks(x, starts, Lc):
    """x (B, C, T) float64 -> (B*K, C, Lc), chunk index b*K + k, zeros past T"""
    B, Cn, T = x.shape
    out = torch.zeros(B * len(starts), Cn, Lc, dtype=torch.float64)
    for b in range(B):
        for k, s0 in enumerate(starts):
            n = min(Lc, T - s0)
            out[b * len(starts) + k, :, :n] = x[b, :, s0:s0 + n].double()
    return out


def stats(xc):
    """xc (G, C, Lc) -> (G, C, 2) float64: mean and unbiased std of every row, each sum taken exactly (math.fsum)"""
    G, Cn, Lc = xc.shape
    out = torch.empty(G, Cn, 2, dtype=torch.float64)
    for g in range(G):
        for c in range(Cn):
            v = xc[g, c].tolist()
            m = math.fsum(v) / Lc
            out[g, c, 0] = m
            out[g, c, 1] = math.sqrt(math.fsum((a - m) ** 2 for a in v) / (Lc - 1))
    return out


def standardise(xc, st, eps=1e-12):
    """(G, C, Lc), (G, C, 2) -> (x - mean) / (std + eps) in float64"""
    return (xc - st[..., :1]) / (st[..., 1:] + eps)


def weights(starts, Lc, cross_faded):
    """(K, Tp) float64 over the padded extent Tp = starts[-1] + Lc: the sin^2 / cos^2 ramps of separate_long, or 1 inside each
    segment of the tester's layout"""
    Tp = starts[-1] + Lc
    if cross_faded:
        return SL.weights(starts, Lc, Tp)
    w = torch.zeros(len(starts), Tp, dtype=torch.float64)
    for k, s0 in enumerate(starts):
        w[k, s0:s0 + Lc] = 1.0
    return w


def overlap_add(est, st, starts, Lc, T, cross_faded, magnitude=False):
    """est (K, S, C, Lc) standardised estimates of ONE track, st (K, C, 2) -> (S, C, T) float64:
    sum_k w_k (std_kc est_k + mean_kc) / sum_k w_k over the chunks covering each sample.  magnitude: also the same weighted
    mean of |std_kc est_k| + |mean_kc|, the scale the rounding errors of the sum are relative to"""
    S, Cn = est.shape[1], est.shape[2]
    w = weights(starts, Lc, cross_faded)
    Tp = w.shape[1]
    num = torch.zeros(S, Cn, Tp, dtype=torch.float64)
    mag = torch.zeros(S, Cn, Tp, dtype=torch.float64)
    for k, s0 in enumerate(starts):
        sd, mu = st[k, :, 1][None, :, None], st[k, :, 0][None, :, None]
        e = est[k].double()
        num[:, :, s0:s0 + Lc] += w[k, s0:s0 + Lc] * (sd * e + mu)
        mag[:, :, s0:s0 + Lc] += w[k, s0:s0 + Lc] * ((sd * e).abs() + mu.abs())
    den = w.sum(0)
    out = (num / den)[:, :, :T]
    return (out, (mag / den)[:, :, :T]) if magnitude else out


def separate(x, est, segment, hop=None):
    """x (B, C, T), est (B*K, S, C, Lc) standardised chunk estimates -> (B, S, C, T) float64"""
    B, Cn, T = x.shape
    starts, Lc = plan(T, segment, hop)
    K = len(starts)
    st = stats(chunks(x, starts, Lc)).reshape(B, K, Cn, 2)
    return torch.stack([overlap_add(est[b * K:(b + 1) * K], st[b], starts, Lc, T, bool(hop)) for b in range(B)])


# ---- error bounds of the kernels ------------------------------------------------------------------------------------------------
# k_track_stats sums d = x - s (s = the row's first sample) and d^2 in double in some fixed order, then
#   mean = s + S1 / n,  var = (S2 - S1 (S1 / n)) / (n - 1),  std = sqrt(var).
# d is exact (two floats); a recursive or tree sum of n terms errs by at most (n - 1) u sum|terms| (Higham, eq. 4.4), so
#   |dS1| <= n u A1,  A1 = sum |d|;   |dS2| <= (n + 1) u A2,  A2 = sum d^2  (the square adds one rounding).
# mean: |dmean| <= |dS1| / n + 2 u (|s| + |S1| / n)                      (division and add)
# var : |dvar| <= (|dS2| + 2 |S1| |dS1| / n + 4 u (A2 + S1^2 / n)) / (n - 1)   (first order; the 4 u covers the product,
#        divisions and subtraction);  |dstd| <= |dvar| / (2 std) + u std, and never more than sqrt(|dvar|) + u std.
# The fsum reference adds a few u of its own; the bounds below carry a factor of 2 for it and for second-order terms.
def stats_bounds(xc):
    """xc (G, C, Lc) float64 -> (G, C, 2) bounds of |mean - ref|, |std - ref|"""
    n = xc.shape[-1]
    s = xc[..., :1]
    d = xc - s
    A1, A2, S1 = d.abs().sum(-1), (d * d).sum(-1), d.sum(-1)
    dS1, dS2 = n * U64 * A1, (n + 1) * U64 * A2
    dmean = dS1 / n + 2 * U64 * (s[..., 0].abs() + S1.abs() / n)
    dvar = (dS2 + 2 * S1.abs() * dS1 / n + 4 * U64 * (A2 + S1 * S1 / n)) / (n - 1)
    var = (A2 - S1 * S1 / n).clamp_min(0) / (n - 1)
    std = var.sqrt()
    dstd = torch.minimum(dvar / (2 * std.clamp_min(1e-300)), dvar.sqrt()) + U64 * std
    return 2 * torch.stack([dmean, dstd], -1) + 1e-300


def gather_bound(xc, st, eps=1e-12):
    """bound of |kernel - fp64| of the standardised chunks, given the kernel's own statistics st: one fp32 rounding of the value
    plus the double rounding of the subtraction and division (3 u64 relative)"""
    y = standardise(xc, st, eps)
    return U32 * y.abs() + 4 * U64 * y.abs() + 1e-45


def ola_bound(ref, mag):
    """one fp32 rounding of the fp64 value, plus the double arithmetic: two fused roundings per chunk, the sum over at most four
    chunks, the reciprocal of the weights' sum and the product (a few u64 of the weighted magnitude mag)"""
    return U32 * ref.abs() + 32 * U64 * mag + 1e-45
