"""fp64 references, error bounds and rows of the training path's streaming and filter-bank gradient kernels (ctn_train.cu).

Plain torch, no import of the native library: test_train_kernels_cpu.py shows here that the bounds reject plausible bugs,
test_train_kernels_gpu.py holds each kernel to them through the verification hook (include/ctn_b200_probe.h).

Every reference is written from the operation's definition in float64 and takes the kernel's inputs as given: fp32 values
held in float64, the float mask, the slope as a float, and the float (mean, rstd) that gln_mean_rstd (ctn_common.cuh)
derives from the double statistics.  Phase 2 of the gLN backward takes the per-sample sums the kernel itself produced, and
the statistics side outputs are judged against the kernel's own main output, so each kernel answers for its own arithmetic.

Bounds (u = 2^-24; every bound is per output element):
  * element-wise outputs: c u M, where M is the formula's magnitude (every term's absolute value, subtractions turned into
    additions) and c counts the fp32 roundings on the way:
      y + bias (k_bias_prelu_stats)                           c = 1,  M = |y| + |bias|
      hn = fma(g rstd, act(x), b - mean rstd g)               c = 5,  M_hn = |g| rstd (|act(x)| + |mean|) + |b|
                                                              (k_act_norm's output; act = PReLU adds one rounding)
      u_pre = bd + sum_k wd_k hn[t + k d - pl] (P fmas)       c = P + 5,  M = |bd| + sum_k |wd_k| M_hn[t + k d - pl]
      d_hn = sum_k wd_k dU[t - k d + pl] (P fmas)             c = P + 1,  V = sum_k |wd_k dU[t - k d + pl]|
      da = rstd (g dy - mg - xh mgx), xh = (act(x)-mean) rstd c = 6,  M_da = rstd (|g dy| + |mg| + |mgx| rstd (|act(x)| + |mean|))
        d_pre = da or a da                                    c = 7 with the PReLU (times |a| on its slope branch)
      d_mpre = d w m (1 - m)                                  c = 5,  M = |d w m (1 - m)|
      d_wprod = sum_s d_s m_s (S fmas)                        c = S + 1
      PReLU and its backward (one product)                    c = 1,  M = |a x|, |a dy| (exact on the identity branch)
      dw + dwprod (k_dw_combine)                              c = 1
    xh is computed in fp32 from the fp32 mean / rstd, so M carries |act(x)| + |mean|, not |xh|: the bound still holds under a
    DC offset, the same shape as the stand-alone norm bound in test_forward_edges_gpu.py.
  * reductions: (k + L + p + c) u sum|terms|, plus the first-order error the terms themselves carry.  k is the length of one
    thread's fp32 chain, read off the launch shape: nq = ceil(frames / 1024) quads per thread in the 4-wide kernels (plus the
    2 or 4 roundings of sum4 / dot4 inside a quad), ceil(frames / 256) elements in the scalar ones, 4 nq in the per-element
    loop of k_gln_prelu_bwd_apply, upc * 32 in k_wgrad.  L = ceil(log2 p') for a shuffle tree of p' lanes (5 for a warp).
    Float atomics onto one address add their p partials one after another in no fixed order, so they count p, not log2 p:
    B for the per-channel gradients (one CTA per (c, b)), C * B for a slope, 8 warps + gy CTAs in k_encdec_wgrad, the split
    count in k_wgrad.  Stages in double (block sums, per-sample sums, statistics) count as exact.  c counts the roundings that
    produce one term and the final cast to float.
  * accumulators: every "+=" output starts from a random nonzero base; the check is on out - base with p u |base| added,
    p the float atomics onto that address (each rounds relative to the running total, which carries the base).

Inputs the kernels assume zero-padded (columns [frames, pitch)): none of the loads of a (B, C, pitch) row past frames reach an
output except through a product with a masked zero.  k_gln_bwd_reduce and k_dw_bwd multiply the masked-zero dy by the
pad-lane xhat of pre / h, and k_mask_bwd multiplies the masked d by the pad lanes of mask: those pads must be finite (a NaN
pad poisons the sums), any finite value is harmless.  The tests fill every input pad with finite garbage (1e6 randn) and
require the element-wise outputs to be bit-identical to a call with zero pads.
"""
import torch

U = 2.0 ** -24
SCALES = (1e-3, 1.0, 1e3)  # per-sample scale of B = 3 rows: a statistic read from the wrong sample is off by 1e3
EPS = 1e-8
WARP_TREE = 5


def pitch_of(frames, extra=0):
    return -(-frames // 128) * 128 + extra


def nq(frames, step=1024):
    """fp32 chain steps of one thread that walks t = tid * (step / 256 * ...) in strides of `step`"""
    return -(-frames // step)


def f32(x):
    return x.float().double()


def prelu(x, a):
    return torch.where(x >= 0, x, a * x)


def act(x, a):
    return x if a is None else prelu(x, a)


def stats_of(x):
    return torch.stack([x.sum((1, 2)), (x * x).sum((1, 2))], 1)


def mean_rstd_f(stats, n, eps):
    """gln_mean_rstd: (mean, rstd) computed in double from the double stats, then rounded to float; each (B, 1, 1)"""
    mean = stats[:, 0] / n
    var = (stats[:, 1] / n - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))
    return f32(mean)[:, None, None], f32(rstd)[:, None, None]


def shift(x, s):
    """y[..., t] = x[..., t + s] inside [0, F), 0 outside"""
    F = x.shape[-1]
    y = torch.zeros_like(x)
    if abs(s) >= F:
        return y
    if s >= 0:
        y[..., :F - s] = x[..., s:]
    else:
        y[..., -s:] = x[..., :F + s]
    return y


def pad_left_of(P, d):
    return (P - 1) * d // 2


def col(v):
    return v[None, :, None]


# ---- forward kernels ------------------------------------------------------------------------------------------------------
def stats_from_output(v, a, frames):
    """stats[b] of PReLU(v; a) judged against the kernel's own output v: (k_bias_prelu_stats, k_dw_train_fwd)"""
    p = prelu(v, a)
    k = nq(frames)
    val = stats_of(p)
    bnd = torch.stack([(k + 3) * U * p.abs().sum((1, 2)), (k + 6) * U * (p * p).sum((1, 2))], 1)
    return val, bnd


def bias_prelu_stats(y, bias, a):
    return {"y": (y + col(bias), U * (y.abs() + col(bias).abs()))}


def norm_terms(x, a, g, b, stats, n, eps):
    """(gLN(act(x)), M_hn, mean, rstd, act(x))"""
    mean, rstd = mean_rstd_f(stats, n, eps)
    q = act(x, a)
    hn = col(g) * (q - mean) * rstd + col(b)
    mag = col(g).abs() * rstd * (q.abs() + mean.abs()) + col(b).abs()
    return hn, mag, mean, rstd, q


def act_norm(pre, a, g, bt, stats, n, eps):
    y, mag, *_ = norm_terms(pre, a, g, bt, stats, n, eps)
    return {"y": (y, 5 * U * mag)}


def dw_train_fwd(h, g1, b1, wd, bd, a1, stats1, n1, eps, P, d, pl):
    hn, mag, *_ = norm_terms(h, a1, g1, b1, stats1, n1, eps)
    u, um = col(bd).expand_as(h).clone(), col(bd).abs().expand_as(h).clone()
    for k in range(P):
        u = u + col(wd[:, k]) * shift(hn, k * d - pl)
        um = um + col(wd[:, k]).abs() * shift(mag, k * d - pl)
    return {"upre": (u, (P + 5) * U * um)}


# ---- gLN (+ PReLU) backward -------------------------------------------------------------------------------------------------
def gln_reduce(dy, pre, a, g, stats, n, eps, mut=None):
    """phase 1: dbeta, dgamma (C), sums (B, 2)"""
    B, C, F = dy.shape
    if mut == "n_pitch":
        n = n // F * pitch_of(F)
    if mut == "sample0":
        stats = stats[:1].expand(B, 2)
    mean, rstd = mean_rstd_f(stats, n, eps)
    x = act(pre, a)
    xh = (x - mean) * rstd
    t0, t1 = dy.abs(), dy.abs() * rstd * (x.abs() + mean.abs())
    k = nq(F)
    gc = col(g)
    out = {
        "dbeta": (dy.sum((0, 2)), (k + 3 + B) * U * t0.sum((0, 2))),
        "dgamma": (dy.mul(xh).sum((0, 2)), (k + 8 + B) * U * t1.sum((0, 2))),
        "sums": (torch.stack([(gc * dy).sum((1, 2)), (gc * dy * xh).sum((1, 2))], 1),
                 torch.stack([(k + 2) * U * (gc.abs() * t0).sum((1, 2)), (k + 7) * U * (gc.abs() * t1).sum((1, 2))], 1)),
    }
    return out


def gln_apply(dy, pre, a, g, stats, n, eps, sums, mut=None):
    """phase 2 from the given (B, 2) sums: dpre, dslope (scalar, a given), dbias (C)"""
    B, C, F = dy.shape
    if mut == "n_pitch":
        n = n // F * pitch_of(F)
    if mut == "sample0":
        stats, sums = stats[:1].expand(B, 2), sums[:1].expand(B, 2)
    mean, rstd = mean_rstd_f(stats, n, eps)
    mg, mgx = f32(sums[:, 0] / n)[:, None, None], f32(sums[:, 1] / n)[:, None, None]
    x = act(pre, a)
    xh = (x - mean) * rstd
    gc = col(g)
    da = rstd * (gc * dy - mg - (0.0 if mut == "no_mgx" else xh * mgx))
    M = rstd * ((gc * dy).abs() + mg.abs() + mgx.abs() * rstd * (x.abs() + mean.abs()))
    k4 = 4 * nq(F)
    out = {}
    if a is None:
        dpre, fac, c = da, torch.ones_like(da), 6
    else:
        neg = ~(pre > 0)
        dpre = torch.where(neg, a * da, da)
        fac = torch.where(neg, torch.full_like(da, abs(a)), torch.ones_like(da))
        c = 7
        out["dslope"] = ((da * pre * neg).sum(), (k4 + C * B + 8) * U * (pre.abs() * M * neg).sum())
    out["dpre"] = (dpre, c * U * M * fac)
    out["dbias"] = (dpre.sum((0, 2)), (k4 + B + 8) * U * (M * fac).sum((0, 2)))
    return out


def gln_bwd(dy, pre, a, g, stats, n, eps, mut=None):
    """both phases with exact sums (the composition the mutants of the CPU test act on)"""
    r = gln_reduce(dy, pre, a, g, stats, n, eps, mut)
    out = gln_apply(dy, pre, a, g, stats, n, eps, r["sums"][0], mut)
    out.update(r)
    return out


# ---- depthwise backward -----------------------------------------------------------------------------------------------------
def dw_bwd(dU, h, a1, g1, b1, stats1, n1, eps, wd, P, d, pl, mut=None):
    """d_hn, dwd (C, P), and phase 1 of the gLN1 backward on the reference d_hn: dbeta, dgamma (C), sums (B, 2)"""
    B, C, F = dU.shape
    if mut == "pl_up":
        pl = -(-(P - 1) * d // 2)
    hn, mag, mean, rstd, x = norm_terms(h, a1, g1, b1, stats1, n1, eps)
    v, V = torch.zeros_like(dU), torch.zeros_like(dU)
    dwd, dwdb = [], []
    keep = torch.ones(F, dtype=dU.dtype, device=dU.device)
    if mut == "drop_quad" and F % 4:
        keep[F - F % 4:] = 0.0
    k = nq(F)
    for j in range(P):
        s = (j * d - pl) if mut == "fwd_tap" else (pl - j * d)
        v = v + col(wd[:, j]) * shift(dU, s)
        V = V + col(wd[:, j]).abs() * shift(dU, s).abs()
        dwd.append((dU * shift(hn, j * d - pl) * keep).sum((0, 2)))
        dwdb.append((k + 15 + B) * U * (dU.abs() * shift(mag, j * d - pl)).sum((0, 2)))
    xh = (x - mean) * rstd
    t1 = V * rstd * (x.abs() + mean.abs())
    gc = col(g1)
    return {
        "dhn": (v, (P + 1) * U * V),
        "dwd": (torch.stack(dwd, 1), torch.stack(dwdb, 1)),
        "dbeta": (v.sum((0, 2)), (k + B + P + 9) * U * V.sum((0, 2))),
        "dgamma": ((v * xh).sum((0, 2)), (k + B + P + 14) * U * t1.sum((0, 2))),
        "sums": (torch.stack([(gc * v).sum((1, 2)), (gc * v * xh).sum((1, 2))], 1),
                 torch.stack([(k + B + P + 9) * U * (gc.abs() * V).sum((1, 2)),
                              (k + B + P + 14) * U * (gc.abs() * t1).sum((1, 2))], 1)),
    }


# ---- mask head, PReLU, combine ----------------------------------------------------------------------------------------------
def mask_bwd(dwhat, w, m, mut=None):
    """dwhat, m: (B, S, N, F); w: (B, N, F) -> d_mpre (B, S, N, F), d_wprod (B, N, F)"""
    S = dwhat.shape[1]
    mm = m if mut == "m_only" else m * (1 - m)
    dm = dwhat * w[:, None] * mm
    src = dwhat[:, :S - 1] * m[:, :S - 1] if mut == "drop_src" else dwhat * m
    return {"dmpre": (dm, 5 * U * (dwhat * w[:, None] * m * (1 - m)).abs()),
            "dwprod": (src.sum(1), (S + 1) * U * (dwhat * m).abs().sum(1))}


def prelu_apply(x, a):
    return {"y": (prelu(x, a), U * (a * x).abs() * (x < 0))}


def prelu_bwd(dy, pre, a, mut=None):
    B, C, F = dy.shape
    neg = (pre < 0) | ((pre == 0) & (mut != "ident0"))
    return {"dpre": (torch.where(neg, a * dy, dy), U * (a * dy).abs() * ~(pre > 0)),
            "dslope": ((dy * pre * ~(pre > 0)).sum(), (nq(F, 256) + C * B + 2) * U * (dy * pre).abs().sum())}


def dw_combine(dw, dwprod, w, relu):
    v = dw + dwprod
    if relu:
        v = v * (w > 0)
    return {"dw": (v, U * (dw.abs() + dwprod.abs()))}


def rowsum(dy):
    B, C, F = dy.shape
    return {"out": (dy.sum((0, 2)), (nq(F) + 3 + B) * U * dy.abs().sum((0, 2)))}


# ---- filter-bank and 1x1 weight gradients -----------------------------------------------------------------------------------
def encdec_gy(R, N):
    """grid rows of k_encdec_wgrad (ctn_encdec_wgrad)"""
    return max(1, min(R, -(-4 * 148 // N)))


def encdec_wgrad(act_, sig, L, stride, pl, mut=None):
    """act_ (R, N, F), sig (R, T) -> dW (N, L) = sum_{r,f} act[r][n][f] sig[r][f stride + k - pl] (0 outside [0, T))"""
    R, N, F = act_.shape
    T = sig.shape[1]
    if mut == "no_pl":
        pl = 0
    idx = torch.arange(F, device=sig.device)[:, None] * stride + torch.arange(L, device=sig.device)[None, :] - pl
    ok = (idx >= 0) & (idx < T)
    if mut == "skip_partial":
        ok = ok & ok.all(1, keepdim=True)
    win = sig[:, idx.clamp(0, T - 1)] * ok  # (R, F, L)
    full = sig[:, idx.clamp(0, T - 1)].abs() * ((idx >= 0) & (idx < T))
    val = torch.einsum("rnf,rfl->nl", act_, win)
    mag = torch.einsum("rnf,rfl->nl", act_.abs(), full)
    if L <= 32:
        gy = encdec_gy(R, N)
        k = nq(F, 256) * -(-R // gy) + WARP_TREE + 8 + gy + 2
    else:
        k = nq(F, 256) + 3
    return {"dW": (val, k * U * mag)}


def wgrad_fp32_chain(M, K, B, frames, split=None):
    """the fp32 (FFMA) k_wgrad's reduction length per output: 32 units_per_cta + splits (+ 2), as ctn_wgrad splits the work"""
    worst = 0
    for Mp in ([split, M - split] if split else [M]):
        tiles = -(-Mp // 64) * -(-K // 64)
        total = B * -(-frames // 32)
        splits = max(1, min(total, -(-4 * 148 // tiles)))
        upc = -(-total // splits)
        splits = -(-total // upc)
        worst = max(worst, 32 * upc + splits + 2)
    return worst


def wgrad_fp32(dy, x, split=None, mut=None):
    """reference of the (mutated) fp32 weight gradient: dy (B, M, F), x (B, K, F) -> (M, K)"""
    B, M, F = dy.shape
    if mut == "drop_chunk":
        keep = torch.ones(F, dtype=dy.dtype, device=dy.device)
        keep[(F - 1) // 32 * 32:] = 0.0
        dy = dy * keep
    out = torch.einsum("bmt,bkt->mk", dy, x)
    if mut == "split_off" and split:
        out = torch.cat([out[:split], out[split + 1:], torch.zeros_like(out[:1])])
    return out


# ---- rows ------------------------------------------------------------------------------------------------------------------
def _r(reaches, **kw):
    d = dict(B=3, C=3, F=129, extra=0, reaches=reaches)
    d.update(kw)
    return d


FRAMES = [1, 3, 5, 127, 128, 129, 1023, 1024, 1025, 4095, 4096, 4097]
_FR_WHY = {1: "one frame", 3: "3 frames: one partial quad", 5: "5 frames: a full quad and a partial one",
           127: "127: partial last quad", 128: "128 = pitch", 129: "129: one lane into the next quad",
           1023: "1023: one block's 1024-frame stride, partial", 1024: "1024: exactly one block stride",
           1025: "1025: second trip of the 1024-frame stride", 4095: "4095: the 4096-frame load batch, partial",
           4096: "4096: exactly one load batch", 4097: "4097: second load batch, one lane"}


def _frame_rows(**kw):
    rows = {f"F{F}": _r(_FR_WHY[F], F=F, **kw) for F in FRAMES}
    rows["C1"] = _r("C = 1: one channel", C=1, **kw)
    rows["C1025"] = _r("C = 1025: the channel loop's second trip at the 1024-CTA cap (grid_cb)", C=1025, F=33, **kw)
    rows["wide"] = _r("pitch = ctn_pitch(frames) + 256", F=129, extra=256, **kw)
    rows["paper"] = _r("paper length: 4 s at 8 kHz = 3999 frames, H = 512, B = 4", B=4, C=512, F=3999, **kw)
    return rows


ROWS = {
    "bias_prelu_stats": _frame_rows(),
    "act_norm": {**_frame_rows(), "noact": _r("act off (slope null, the gLN0 recompute)", act=False),
                 "dc": _r("DC offset 100x the spread in pre", dc=True, F=1025)},
    "gln_bwd": {**_frame_rows(),
                "noact": _r("act off (gLN0 backward: slope, dslope, dbias null)", act=False),
                "nulls": _r("dslope and dbias null with act on", nulls=True),
                "alias": _r("dpre aliasing dy, as the pipeline calls it", alias=True, F=4097),
                "alias_C1025": _r("dpre aliasing dy at C = 1025", alias=True, C=1025, F=129),
                "dc": _r("DC offset 100x the spread in pre", dc=True, F=1025),
                "zeros": _r("pre with exact +0.0 / -0.0: the slope branch at 0", zeros=True)},
    "prelu": {**_frame_rows(), "zeros": _r("exact +0.0 / -0.0 in pre: the slope branch at 0, no dslope term", zeros=True)},
    "dw_combine": {**_frame_rows(), "relu": _r("encoder ReLU on: zero where !(w > 0), w with exact zeros", relu=True, zeros=True),
                   "relu_C1025": _r("ReLU at C = 1025", relu=True, C=1025, F=33)},
    "rows": {"F1": _r("one frame", F=1), "F129": _r("M K not a multiple of 256", F=129, C=5),
             "acc": _r("accumulate", F=1025, acc=True),
             "strides": _r("both batch strides wider than C pitch", F=129, C=5, strides=True),
             "strides_acc": _r("strided accumulate at C = 1025", F=33, C=1025, strides=True, acc=True)},
    "transpose": {"1x1": _r("M = K = 1", M=1, K=1), "7x37": _r("M K = 259: one CTA past 256", M=7, K=37),
                  "300x100": _r("300 x 100", M=300, K=100), "2560x1024": _r("S N = 2560 by 1024", M=2560, K=1024)},
    "rowsum": {**{k: v for k, v in _frame_rows().items() if k != "C1025"},
               "SN2560": _r("C = S N = 2560 (one CTA per channel)", C=2560, F=129),
               "stride": _r("batch stride wider than C pitch (rows of dcat)", F=129, stride=True)},
    "mask_bwd": {"S1_F5": _r("S = 1, partial quad", S=1, N=7, F=5), "S2_F129": _r("S = 2", S=2, N=7, F=129),
                 "S5_F1025": _r("S = 5, 1025 frames", S=5, N=3, F=1025),
                 "S2_N1280": _r("S N = 2560: N = 1280 > 1024-CTA cap", S=2, N=1280, F=33),
                 "S2_edges": _r("mask exactly 0, 1 and 1 - 2^-24", S=2, N=7, F=129, edges=True),
                 "wide": _r("pitch + 256", S=2, N=7, F=129, extra=256),
                 "C1": _r("N = 1, S = 2", S=2, N=1, F=4097)},
}

# depthwise rows: P, dilation, frames, channels
_DW = {}
for _P in (1, 2, 3, 4, 7, 8):
    _DW[f"P{_P}_d1"] = _r(f"P = {_P}, d = 1" + (": even P, pad_left (P-1)/2 rounds down" if _P % 2 == 0 else ""), P=_P, d=1)
for _P in (2, 3, 4, 8):
    for _d, _why in ((2, "d = 2"), (64, "d = 64"), (128, "d = frames - 1"), (129, "d = frames"),
                     (264, "d = pitch + 8: every off-centre tap is padding")):
        _DW[f"P{_P}_d{_d}"] = _r(f"P = {_P}, {_why}", P=_P, d=_d)
_DW["P3_d1_F1"] = _r("P = 3, one frame", P=3, d=1, F=1)
_DW["P4_d3_F5"] = _r("P = 4, d = 3, 5 frames: partial quad, odd (P-1) d", P=4, d=3, F=5)
_DW["P3_d2_F1025"] = _r("P = 3, d = 2, 1025 frames", P=3, d=2, F=1025)
_DW["P3_d1_F4097"] = _r("P = 3, d = 1, 4097 frames", P=3, d=1, F=4097)
_DW["P3_d4_C1"] = _r("P = 3, d = 4, C = 1", P=3, d=4, C=1)
_DW["P3_d2_C1025"] = _r("P = 3, d = 2, C = 1025: channel loop's second trip (forward)", P=3, d=2, C=1025, F=33)
_DW["P3_d1_wide"] = _r("P = 3, pitch + 256", P=3, d=1, extra=256)
_DW["P3_dc"] = _r("P = 3, DC offset 100x the spread in h", P=3, d=2, dc=True, F=1025)
_DW["P3_paper"] = _r("paper length: P = 3, d = 8, H = 512, B = 4, 3999 frames", P=3, d=8, B=4, C=512, F=3999)
ROWS["dw"] = _DW

# filter-bank weight gradient rows: (L, stride), frames from T, R, N
_ED = {}
for _L, _S in ((4, 2), (16, 8), (20, 10), (32, 16), (33, 11), (40, 20), (64, 32)):
    _ED[f"L{_L}_s{_S}"] = _r(f"L / stride = {_L} / {_S}" + (" (fast path)" if _L <= 32 else " (generic)"), L=_L, stride=_S,
                             T=1003, R=3, N=24)
_ED["L16_T1000_vec"] = _r("float4 branch on: T % 4 == 0, pad_left % 4 == 0, aligned base", L=16, stride=8, T=1000, R=3, N=24,
                          pl=4)
_ED["L16_T1001"] = _r("float4 off: T % 4 != 0", L=16, stride=8, T=1001, R=3, N=24, pl=4)
_ED["L16_off1"] = _r("float4 off: signal base offset by one float", L=16, stride=8, T=1000, R=3, N=24, pl=4, off=1)
_ED["L16_pl2"] = _r("float4 off: pad_left % 4 != 0; first and last windows partial", L=16, stride=8, T=1000, R=3, N=24, pl=2)
_ED["L16_R1"] = _r("R = 1", L=16, stride=8, T=1003, R=1, N=24)
_ED["L16_R64_N24"] = _r("R = 64, N = 24: gy = 25 < R, several rows per CTA", L=16, stride=8, T=403, R=64, N=24)
_ED["L16_R64_N1024"] = _r("R = 64, N = 1024: gy = 1", L=16, stride=8, T=203, R=64, N=1024)
_ED["L40_R64_N24"] = _r("generic, R = 64", L=40, stride=20, T=403, R=64, N=24)
_ED["L4_T5"] = _r("L = 4 over 5 samples: every window partial or edge", L=4, stride=2, T=5, R=3, N=5)
ROWS["encdec"] = _ED

# composed chain (gLN2/PReLU2 backward -> k_dw_bwd -> gLN1/PReLU1 apply), one per depthwise shape class
COMPOSED = {k: ROWS["dw"][k] for k in ("P1_d1", "P2_d1", "P3_d1", "P4_d3_F5", "P8_d1", "P3_d64", "P3_d129", "P4_d128",
                                       "P3_d1_F4097", "P3_d2_C1025")}


def encdec_geometry(r):
    """(frames, pad_left) of an encdec row: frames windows of L at `stride` over T samples padded by pl on the left"""
    L, S, T = r["L"], r["stride"], r["T"]
    pl = r.get("pl")
    if pl is None:
        rem = (T - L) % S
        padding = (S - rem) % S
        pl = padding // 2
        return (T + padding - L) // S + 1, pl
    return (T + 2 * pl - L) // S + 1, pl


# ---- inputs --------------------------------------------------------------------------------------------------------------
def gen(name):
    return torch.Generator().manual_seed(sum(map(ord, name)) * 7 + len(name))


def rnd(g, *shape, scale=1.0, shift_=0.0):
    return f32(torch.randn(*shape, generator=g, dtype=torch.float64) * scale + shift_)


def sample_scale(B):
    s = torch.tensor([SCALES[b % 3] for b in range(B)], dtype=torch.float64)
    return s[:, None, None]


def with_zeros(x, g):
    """sprinkle exact +0.0 and -0.0 into x"""
    z = torch.rand(x.shape, generator=g) < 0.1
    nz = torch.rand(x.shape, generator=g) < 0.5
    x = torch.where(z, torch.zeros_like(x), x)
    return torch.where(z & nz, -torch.zeros_like(x), x)


def activation(g, r, spread=1.0):
    """(B, C, F) per-sample scaled, optional DC offset / exact zeros"""
    B, C, F = r["B"], r["C"], r["F"]
    x = rnd(g, B, C, F, scale=spread, shift_=0.1)
    if r.get("dc"):
        x = f32(x + 100.0 * spread)
    x = f32(x * sample_scale(B))
    if r.get("zeros"):
        x = with_zeros(x, g)
    return x


def norm_params(g, C):
    return rnd(g, C, scale=0.3, shift_=1.0), rnd(g, C, scale=0.2)


A1, A2 = float(f32(torch.tensor(0.3))), float(f32(torch.tensor(-0.2)))  # PReLU slopes, as the kernels read them


def dw_inputs(name, r):
    """generator, h, g1, b1, wd, bd, dU, stats1 of a depthwise row"""
    g = gen("dw" + name)
    B, C, F, P = r["B"], r["C"], r["F"], r["P"]
    h = activation(g, r)
    g1, b1 = norm_params(g, C)
    wd, bd = rnd(g, C, P, scale=0.5), rnd(g, C, scale=0.1)
    dU = rnd(g, B, C, F)
    return g, h, g1, b1, wd, bd, dU, stats_of(prelu(h, A1))


def gln_inputs(name, r):
    """generator, slope (None: act off), pre, dy, gamma, stats of a gLN backward row"""
    g = gen("gln" + name)
    B, C, F = r["B"], r["C"], r["F"]
    sl = None if r.get("act") is False else A1
    pre = activation(g, r)
    dy = rnd(g, B, C, F)
    gm, _ = norm_params(g, C)
    return g, sl, pre, dy, gm, stats_of(act(pre, sl))
