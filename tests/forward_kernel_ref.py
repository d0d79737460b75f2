"""fp64 references, error bounds and rows of the inference forward's streaming kernels: the gLN folds (k_fold_batch), the
depthwise stage (k_dw<3> / k_dw<0>), the residual update (k_finish), the skip sum (k_skip_reduce), the separator's gLN0
statistics (k_stats_pitch), the filter banks (k_encoder, k_encoder_v4, k_decoder, k_decoder_generic) and the causal pipeline's
per-frame kernels (k_dw_plain, k_res_skip, k_bias_rows, the pitched cLN).

Plain torch, no import of the native library: test_forward_kernels_cpu.py shows here that the bounds reject plausible bugs,
test_forward_kernels_gpu.py holds each kernel to them through the verification hook (include/ctn_b200_probe.h) or the public
ctn_encoder_fwd / ctn_decoder_fwd.  Helpers and conventions are those of train_kernel_ref.py.

Every reference is written from the operation's definition in float64 and takes the kernel's inputs as given: fp32 values held
in float64, and the float (mean, rstd) that gln_mean_rstd derives from the double statistics.  Statistics side outputs are
judged against the fp64 sums of the kernel's own main output.

Bounds (u = 2^-24, d = 2^-53; per output element; M is the formula's magnitude, every term's absolute value):
  * fold, one warp per row, lane l walks k = l, l + 32, ...: k = ceil(K / 32) chain steps, then a 5-level warp tree.
      Wf = fl(w gamma)                            a single product: bit-exact
      v1 = sum_k w beta + bias                    (k + 5 + 1) u (sum_k |w beta| + |bias|)       (fmaf chain, tree, + bias)
      v2 = sum_k Wf                               (k + 5 + 1) u sum_k |Wf|      (the sum of the rounded Wf; one more rounding
                                                  covers nvcc contracting w gamma into the chain's add)
      vb = sum_k |w| (|gamma| R + |beta|) + |bias|   (k + 5 + 3) u vb64, both ways: every term is >= 0, so each rounding is
                                                  relative to the result.  The fp16 scales need vb >= the true row bound up
                                                  to this budget, and a vb far above it would waste their headroom.
  * k_dw: g = fl(gamma rstd) and sh = fl(beta - fl(mean rstd) gamma) (3 roundings, 2 if contracted), hn = fma(h, g, sh),
    then P fmas from bd, then PReLU (|a| < 1 on the negative branch).  hn carries 5 u M_hn (g: 1, sh: 3, the fma: 1) with
    M_hn = |gamma| rstd (|h| + |mean|) + |beta| (|mean| in M: the bound survives a DC offset), so
      u = PReLU(bd + sum_k wd_k hn[t + k d - pl])  (P + 6) u (|bd| + sum_k |wd_k| M_hn[t + k d - pl])
    stats2: each thread adds its 4 fp32 values (3 roundings; sumsq 4 with the squares) before double: 3 u sum|u|, 4 u sum u^2,
    plus (n_cta + 8) d of the double stage (block tree, one atomic per CTA).
  * skip reduce over n blocks: c_i = fl(v1 - fl(mean rstd) v2) (3 roundings, fewer if contracted), term = fma(rstd, r, c_i),
    n fp32 adds from 0:  (n + 4) u sum_i M_i,  M_i = rstd |r| + |v1| + |mean| rstd |v2|.
  * finish: x = fl(x0 + fma(rstd, r, c)):  5 u (|x0| + M).
  * k_stats_pitch: every element in double: k = ceil(frames / 256) ceil(C / gx) chain steps per thread, an 8-level block tree
    and gx atomics (gx = min(C, 64) CTAs per sample):  (k + 8 + gx + 1) d sum|x| (sum x^2).  A DC offset of 1e3 moves
    neither bound relative to the sums it is judged against; fp32 partials would fail it.
  * encoder: an L-term fmaf chain, |w - w64| <= L u sum_k |W x|; ReLU is exact.
    stats: k_encoder adds 4 channels pairwise (2 roundings) into an fp32 partial that spills to double after 16 groups
    (64 values): (2 + G) u sum|w|, (3 + G) u sum w^2, G = min(16, ceil(N / 4)).  k_encoder_v4 adds each channel's 4 frames
    pairwise (2) into a partial spilled after 4 channel groups (16 channels): (2 + 16) u sum|w|; its sumsq is one fmaf chain
    over those 64 values: 65 u sum w^2.  Plus (N / 64 + 8 + n_cta) d.
  * decoder: k_decoder splits the channels over DEC_SPLIT = 4 thread groups; each runs a chain of ceil(N / 4) R fmas and the 3
    partials meet in 3 shared-memory adds: (ceil(N / 4) R + 3) u sum |what Wd|.  k_decoder_generic: one R N chain.
  * k_dw_plain: bd + P fmas, PReLU:  (P + 1) u (|bd| + sum_k |wd_k h|).
  * k_res_skip: (base + r) + b: 2 u (|base| + |r| + |b|) (fresh skip rows: 1 u).  k_bias_rows: u (|y| + |bias|).
  * pitched cLN: 8 u ((|x| + |mean|) rstd |gamma| + |beta|) from fp64 statistics, the stand-alone norm bound of
    test_forward_edges_gpu.py.
A rounding-order change alone (say, a longer fp32 chain before a spill) moves a result by less than 4x these worst-case
bounds; the mutants of test_forward_kernels_cpu.py are the wrong-value bugs a bound can catch.
"""
import torch

from train_kernel_ref import (A2, EPS, U, WARP_TREE, col, f32, gen, mean_rstd_f, norm_params, pitch_of, prelu, rnd,
                              sample_scale, shift, stats_of)

DU = 2.0 ** -53
DEC_SPLIT = 4


def _z(x):
    return torch.zeros_like(x)


# ---- fold ------------------------------------------------------------------------------------------------------------------
def fold(W, bias, gamma, beta, R, mut=None):
    """W (M, K), bias (M) or None, gamma / beta (K), R float -> Wf, v1, v2, vb"""
    M, K = W.shape
    k = -(-K // 32) + WARP_TREE
    Wf = f32(W * gamma[None])
    bias_ = _z(W[:, 0]) if bias is None else bias
    v1 = (W * (gamma if mut == "v1_gamma" else beta)[None]).sum(1) + (0.0 if mut == "no_bias" else bias_)
    v2 = (W if mut == "v2_w" else Wf).sum(1)
    vb = (W.abs() * (gamma.abs() * R + beta.abs())[None]).sum(1) + bias_.abs()
    return {"Wf": (Wf, _z(Wf)),
            "v1": (v1, (k + 1) * U * ((W * beta[None]).abs().sum(1) + bias_.abs())),
            "v2": (v2, (k + 1) * U * Wf.abs().sum(1)),
            "vb": (vb, (k + 3) * U * vb)}


# ---- depthwise (k_dw) ------------------------------------------------------------------------------------------------------
def dw_fwd(h, g1, b1, wd, bd, a2, stats1, n1, eps, P, d, mut=None):
    B, C, F = h.shape
    pl = (P - 1) * d // 2
    if mut == "pl_off":
        pl += 1
    if mut == "dil_half":
        d = d // 2
    if mut == "n_pitch":
        n1 = n1 // F * pitch_of(F)
    if mut == "sample0":
        stats1 = stats1[:1].expand(B, 2)
    mean, rstd = mean_rstd_f(stats1, n1, eps)
    hn = col(g1) * rstd * (h - mean) + col(b1)
    mag = col(g1).abs() * rstd * (h.abs() + mean.abs()) + col(b1).abs()
    u, um = col(bd).expand_as(h).clone(), col(bd).abs().expand_as(h).clone()
    for k in range(P):
        u = u + col(wd[:, k]) * shift(hn, k * d - pl)
        um = um + col(wd[:, k]).abs() * shift(mag, k * d - pl)
    return {"u": (prelu(u, a2), (P + 6) * U * um)}


def dw_cta(C, pitch):
    return C * -(-pitch // 512)


def stats_fp32_quads(v, n_cta):
    """stats[b] of v (B, C, F) as k_dw forms them (4 fp32 values per thread, then double), judged against v itself"""
    a, s = v.abs().sum((1, 2)), (v * v).sum((1, 2))
    dd = (n_cta + 8) * DU
    return stats_of(v), torch.stack([(3 * U + dd) * a, (4 * U + dd) * s], 1)


# ---- skip reduce / finish --------------------------------------------------------------------------------------------------
def skip_reduce(jobs, Sc, n2, eps, mut=None):
    """jobs: list of dict(r (B, Mt, F), v1 (Mt), v2 (Mt), stats (B, 2), off) -> skip (B, Sc, F)"""
    acc = mag = 0.0
    for i, jb in enumerate(jobs):
        st, off = jb["stats"], jb["off"]
        if mut == "prev_stats" and i > 0:
            st = jobs[i - 1]["stats"]
        if mut == "sample0":
            st = st[:1].expand_as(st)
        if mut == "off0":
            off = 0
        mean, rstd = mean_rstd_f(st, n2, eps)
        r, a, b = jb["r"][:, off:off + Sc], col(jb["v1"][off:off + Sc]), col(jb["v2"][off:off + Sc])
        acc = acc + rstd * r + a - mean * rstd * b
        mag = mag + rstd * r.abs() + a.abs() + mean.abs() * rstd * b.abs()
    return {"skip": (acc, (len(jobs) + 4) * U * mag)}


def finish(x0, r, v1, v2, stats, n2, eps, Bc, mut=None):
    if mut == "sample0":
        stats = stats[:1].expand_as(stats)
    mean, rstd = mean_rstd_f(stats, n2, eps)
    r = r[:, :Bc]
    a, b = col(v1[:Bc]), col(v2[:Bc])
    return {"x": (x0 + rstd * r + a - mean * rstd * b,
                  5 * U * (x0.abs() + rstd * r.abs() + a.abs() + mean.abs() * rstd * b.abs()))}


# ---- gLN0 statistics in double (k_stats_pitch) -----------------------------------------------------------------------------
def stats_pitch(x, mut=None):
    B, C, F = x.shape
    gx = min(C, 64)
    k = -(-F // 256) * -(-C // gx) + 8 + gx + 1
    if mut == "fp32_partials":  # each thread's chain in fp32 before double (what the kernel's comment warns against)
        y = x.float()
        s = y.sum(2).double().sum(1)
        ss = (y * y).sum(2).double().sum(1)
        val = torch.stack([s, ss], 1)
    else:
        val = stats_of(x)
    return {"stats": (val, torch.stack([k * DU * x.abs().sum((1, 2)), k * DU * (x * x).sum((1, 2))], 1))}


# ---- filter banks ----------------------------------------------------------------------------------------------------------
def enc_geometry(T, L, stride, pl):
    """(pad_right, frames) of a row whose padded length is a whole number of strides past L"""
    Tp = T + pl
    pr = (stride - (Tp - L) % stride) % stride if Tp >= L else L - Tp
    return pr, (Tp + pr - L) // stride + 1


def encoder(x, W, stride, pl, pr, relu):
    """x (B, T), W (N, L) -> w (B, N, frames)"""
    xp = torch.nn.functional.pad(x, (pl, pr))[:, None]
    w = torch.nn.functional.conv1d(xp, W[:, None], stride=stride)
    mag = torch.nn.functional.conv1d(xp.abs(), W.abs()[:, None], stride=stride)
    L = W.shape[1]
    return {"w": (w.clamp_min(0.0) if relu else w, L * U * mag)}


def encoder_stats(w, v4, n_cta, mut=None):
    """stats[b] of the kernel's own output w (B, N, F), as k_encoder / k_encoder_v4 form them"""
    B, N, F = w.shape
    if v4:
        ca, cs = 2 + 16, 65
    else:
        G = min(16, -(-N // 4))
        ca, cs = 2 + G, 3 + G
    dd = (N / 64 + 8 + n_cta) * DU
    val = stats_of(w)
    if mut == "spill_lost":
        # a spill that resets the fp32 partial without carrying it: only the channels after the last spill point survive
        # (k_encoder spills after channel 64 j + 63, k_encoder_v4 after 16 channels of each warp's quarter)
        keep = torch.zeros(N, dtype=w.dtype, device=w.device)
        if v4:
            nq = (((N + 3) // 4 + 3) // 4) * 4
            for wb in range(4):
                lo, hi = wb * nq, min(N, wb * nq + nq)
                if hi > lo:
                    last = lo + ((hi - lo) // 16) * 16 if (hi - lo) % 16 else hi
                    keep[last:hi] = 1.0
        else:
            keep[((N + 3) // 4 * 4) // 64 * 64:] = 1.0
        val = stats_of(w * keep[None, :, None])
    return {"stats": (val, torch.stack([(ca * U + dd) * w.abs().sum((1, 2)), (cs * U + dd) * (w * w).sum((1, 2))], 1))}


def decoder(what, Wd, stride, crop, T_out, mut=None):
    """what (BS, N, F), Wd (N, L) -> y (BS, T_out) = conv_transpose1d(what, Wd, stride)[crop : crop + T_out]"""
    BS, N, F = what.shape
    L = Wd.shape[1]
    R = L // stride
    generic = (stride, R) not in ((8, 2), (1, 2), (10, 2), (2, 2))
    if mut == "drop_part" and not generic:
        nper = -(-N // DEC_SPLIT)
        what = what.clone()
        what[:, 3 * nper:] = 0.0
    full = torch.nn.functional.conv_transpose1d(what, Wd[:, None], stride=stride)[:, 0]
    mag = torch.nn.functional.conv_transpose1d(what.abs(), Wd.abs()[:, None], stride=stride)[:, 0]
    c = R * N if generic else -(-N // DEC_SPLIT) * R + DEC_SPLIT - 1
    at = crop + 1 if mut == "crop_off" else crop
    full = torch.nn.functional.pad(full, (0, 1))  # a crop one past the end reads 0
    return {"y": (full[:, at:at + T_out], c * U * mag[:, crop:crop + T_out])}


# ---- causal per-frame kernels ----------------------------------------------------------------------------------------------
def dw_plain(h, wd, bd, a, P, d, mut=None):
    pl = (P - 1) * d
    if mut == "causal_sym":
        pl = (P - 1) * d // 2
    if mut == "dil_half":
        d = d // 2
    u, um = col(bd).expand_as(h).clone(), col(bd).abs().expand_as(h).clone()
    for k in range(P):
        s = shift(h, k * d - pl)
        u = u + col(wd[:, k]) * s
        um = um + col(wd[:, k]).abs() * s.abs()
    return {"u": (prelu(u, a), (P + 1) * U * um)}


def res_skip(r, xin, skip0, bo, bs, Bc, has_out, skip_init, mut=None):
    """r (B, Mt, F); xin (B, Bc, F); skip0 (B, Sc, F) -> x, skip"""
    out = {}
    if has_out:
        q = r[:, :Bc]
        out["x"] = (xin + q + col(bo), 2 * U * (xin.abs() + q.abs() + col(bo).abs()))
        q = r[:, Bc:]
    else:
        q = r
    fresh = skip_init and mut != "no_skip_init"
    base = _z(skip0) if fresh else skip0
    out["skip"] = (base + q + col(bs), 2 * U * (base.abs() + q.abs() + col(bs).abs()))
    return out


def bias_rows(y, bias):
    return {"y": (y + col(bias), U * (y.abs() + col(bias).abs()))}


def cln(x, g, b, eps):
    B, C, F = x.shape
    n = torch.arange(1, F + 1, dtype=torch.float64, device=x.device) * C
    mean = (x.sum(1).cumsum(1) / n)[:, None]
    var = ((x * x).sum(1).cumsum(1) / n)[:, None] - mean ** 2
    rstd = 1.0 / (torch.sqrt(var.clamp_min(0.0)) + eps)
    return {"y": (col(g) * (x - mean) * rstd + col(b),
                  8 * U * ((x.abs() + mean.abs()) * rstd * col(g).abs() + col(b).abs()))}


# ---- rows ------------------------------------------------------------------------------------------------------------------
def _r(reaches, **kw):
    d = dict(B=3, C=5, F=129, extra=0, reaches=reaches)
    d.update(kw)
    return d


def _pairs(n, M, K):
    """n fold jobs laid out as the pipelines' preparation lays them out: [out; skip] pairs sharing one FoldedConv (the skip job
    at row_offset = Bc), an odd one last (the skip-only block)"""
    return [dict(M=M, K=K, off=M if j % 2 else 0, grp=j // 2) for j in range(n)]


FOLD = {
    "n47_paper": _r("47 jobs at paper size (23 [out; skip] pairs + the last block's skip): one launch, one short of 48",
                    jobs=_pairs(47, 128, 512)),
    "n48": _r("48 jobs: exactly one full launch", jobs=_pairs(48, 16, 96)),
    "n49": _r("49 jobs: a second launch of one job", jobs=_pairs(49, 16, 96)),
    "n128": _r("128 jobs: three launches (48 + 48 + 32)", jobs=_pairs(128, 8, 64)),
    "M128_M256": _r("M = 128 and M = 256 in one launch: the short job's warps past its rows return early",
                    jobs=[dict(M=128, K=512, off=0, grp=0), dict(M=256, K=512, off=0, grp=1), dict(M=128, K=64, off=0, grp=2)]),
    "M1_3_5": _r("M in {1, 3, 5}: a partial 4-warp CTA", jobs=[dict(M=1, K=33, off=0, grp=0), dict(M=3, K=31, off=0, grp=1),
                                                            dict(M=5, K=512, off=0, grp=2)]),
    "K_edges": _r("K in {1, 31, 33, 512, 1056}: lanes without work, one trip, a second partial trip, 33 trips",
                  jobs=[dict(M=7, K=K, off=0, grp=i) for i, K in enumerate((1, 31, 33, 512, 1056))]),
    "nobias": _r("bias null (v1 = W beta, vb without |bias|)", jobs=_pairs(3, 24, 96), nobias=True),
    "novb": _r("vb null: the DPRNN stage path (ctn_sep_head_fwd, R = 0)", jobs=[dict(M=64, K=512, off=0, grp=0)], novb=True),
}

DW = {}
for _d, _why in ((1, "offsets -1 0 1: the scalar branch for the outer taps"), (3, "d = 3: scalar branch"),
                 (4, "d = 4: every tap 128-bit"), (6, "d = 6: pl = 6, scalar outer taps"), (8, "d = 8: 128-bit taps"),
                 (2048, "d = 2048 > frames: the outer taps read only padding")):
    DW[f"P3_d{_d}"] = _r(f"k_dw<3>, {_why}", P=3, d=_d)
for _P in (1, 2, 4, 7):
    DW[f"P{_P}_d1"] = _r(f"k_dw<0>, P = {_P}" + (": even P, pad_left rounds down" if _P % 2 == 0 else ""), P=_P, d=1)
    DW[f"P{_P}_d2"] = _r(f"k_dw<0>, P = {_P}, d = 2", P=_P, d=2)
for _F in (1, 3, 5, 3999):
    DW[f"P3_d2_F{_F}"] = _r(f"{_F} frame(s)", P=3, d=2, F=_F)
DW["P3_d1_wide"] = _r("pitch + 256: whole CTAs past frames add zero statistics", P=3, d=1, extra=256)
DW["P4_d4_wide"] = _r("k_dw<0>, pitch + 256", P=4, d=4, extra=256)
DW["P3_dc"] = _r("DC offset 100x the spread in h", P=3, d=4, dc=True, F=1025)
DW["P3_H512"] = _r("H = 512, B = 3, 3999 frames, d = 8", P=3, d=8, C=512, F=3999)

SKIP = {
    "n1_Sc13": _r("n = 1: one skip-only block", n=1, Sc=13, Bc=5),
    "n3_Sc13_F129": _r("n = 3, Sc = 13, frames % 4 = 1", n=3, Sc=13, Bc=5),
    "n24_Sc128_F1001": _r("n = 24 (paper depth), Sc = 128, frames % 4 = 1", n=24, Sc=128, Bc=16, F=1001),
    "n64_Sc1_F5": _r("n = 64 = CTN_MAX_BLOCKS, Sc = 1, 5 frames", n=64, Sc=1, Bc=3, F=5),
    "n24_Sc13_F3999": _r("n = 24, paper length 3999 frames (% 4 = 3)", n=24, Sc=13, Bc=5, F=3999),
    "n3_wide": _r("pitch + 256", n=3, Sc=13, Bc=5, F=130, extra=256),
}

FINISH = {
    "Bc1_F1": _r("Bc = 1, one frame", Bc=1, Sc=3, F=1),
    "Bc5_F129": _r("Bc = 5, Sc = 13", Bc=5, Sc=13, F=129),
    "Bc128_F3999": _r("Bc = 128, paper length", Bc=128, Sc=128, F=3999),
    "wide": _r("pitch + 256", Bc=5, Sc=3, F=130, extra=256),
}

STATS = {
    "C1_F1": _r("C = 1, one frame", C=1, F=1),
    "C24_F255": _r("C = 24, 255 frames: one thread short of a full 256-stride", C=24, F=255),
    "C64_F257": _r("C = 64 = the CTA grid, 257 frames: a second stride trip", C=64, F=257),
    "C65_F4000": _r("C = 65 > 64: the channel loop's second trip", C=65, F=4000),
    "C512_F4000_dc": _r("C = 512, DC offset 1e3", C=512, F=4000, dc=True),
    "C65_F257_dc": _r("C = 65, DC offset 1e3", C=65, F=257, dc=True),
    "wide": _r("pitch + 256", C=24, F=130, extra=256),
}

ENC = {}
for _L in (2, 4, 8, 16, 20):
    ENC[f"v4_L{_L}"] = _r(f"k_encoder_v4<{_L},{_L // 2}>", L=_L, S=_L // 2, N=33, T=2003)
    ENC[f"L{_L}_pitch4"] = _r(f"k_encoder<{_L}>: w_pitch % 128 != 0", L=_L, S=_L // 2, N=33, T=2003, wpad=4)
    ENC[f"L{_L}_off4"] = _r(f"k_encoder<{_L}>: w offset by 4 bytes", L=_L, S=_L // 2, N=33, T=2003, woff=1)
for _L in (32, 40, 64):
    ENC[f"L{_L}"] = _r(f"k_encoder<{_L}>, stride {_L // 2}", L=_L, S=_L // 2, N=24, T=4001)
ENC["L16_s4"] = _r("k_encoder<16>, stride 4", L=16, S=4, N=24, T=2003)
for _N in (1, 3, 512):
    ENC[f"v4_N{_N}"] = _r(f"v4, N = {_N}", L=16, S=8, N=_N, T=2003)
    ENC[f"L16_pitch4_N{_N}"] = _r(f"k_encoder<16>, N = {_N}", L=16, S=8, N=_N, T=2003, wpad=4)
ENC["v4_N700"] = _r("v4, N = 700: 48 928 B dynamic, over 48 KB only with the static red[64]: the opt-in", L=16, S=8, N=700, T=2003)
ENC["L16_pitch4_N700"] = _r("k_encoder<16>, N = 700: the opt-in for its static red[64]", L=16, S=8, N=700, T=2003, wpad=4)
ENC["v4_relu"] = _r("v4, ReLU", L=16, S=8, N=33, T=2003, relu=True)
ENC["L16_pitch4_relu"] = _r("k_encoder<16>, ReLU", L=16, S=8, N=33, T=2003, relu=True, wpad=4)
ENC["v4_pl"] = _r("v4, pad_left = 8: the first window reads padding", L=16, S=8, N=33, T=2001, pl=8)
ENC["v4_tile"] = _r("v4, a partial last 128-frame tile (frames % 128 = 1)", L=16, S=8, N=33, T=129 * 8 + 8)
ENC["v4_paper"] = _r("v4, paper encoder: N = 512, 4 s at 8 kHz", L=16, S=8, N=512, T=32000, B=2)

DEC = {}
for (_S, _R) in ((8, 2), (1, 2), (10, 2), (2, 2)):
    for _N in (1, 3, 5, 512):
        DEC[f"S{_S}_R{_R}_N{_N}"] = _r(f"k_decoder<{_S},{_R}>, N = {_N}", S=_S, L=_S * _R, N=_N, F=129, crop=0)
    DEC[f"S{_S}_R{_R}_crop7"] = _r(f"k_decoder<{_S},{_R}>, crop 7, T_out short of the full length", S=_S, L=_S * _R, N=24,
                                   F=129, crop=7, short=5)
DEC["gen_R1"] = _r("k_decoder_generic, R = 1 (L = stride = 8)", S=8, L=8, N=24, F=129, crop=0)
DEC["gen_R4"] = _r("k_decoder_generic, R = 4 (L = 16, stride 4)", S=4, L=16, N=24, F=129, crop=0)
DEC["gen_R4_crop7"] = _r("k_decoder_generic, R = 4, crop 7, short", S=4, L=16, N=5, F=129, crop=7, short=3)
DEC["gen_R2_N512"] = _r("k_decoder_generic, L = 6, stride 3, N = 512", S=3, L=6, N=512, F=129, crop=0)
DEC["S8_R2_paper"] = _r("k_decoder<8,2>, N = 512, 3999 frames", S=8, L=16, N=512, F=3999, crop=4, short=4)
for _r_ in DEC.values():
    _r_["B"] = 6  # BS: 3 samples x 2 sources

PLAIN = {}
for _P, _d in ((1, 1), (3, 1), (3, 2), (3, 4), (5, 2), (3, 64), (3, 2048), (5, 2048)):
    PLAIN[f"P{_P}_d{_d}"] = _r(f"P = {_P}, d = {_d}" + (" > frames" if _d > 129 else ""), P=_P, d=_d)
PLAIN["P3_d2_F1"] = _r("one frame", P=3, d=2, F=1)
PLAIN["P3_d4_C1025"] = _r("C = 1025 > the 1024-CTA grid", P=3, d=4, C=1025, F=33)
PLAIN["P3_d8_wide"] = _r("pitch + 256", P=3, d=8, extra=256)

RES = {
    "inplace_first": _r("in place (causal / online block 0): has_out, skip_init = 1", Bc=5, Sc=3, has_out=1, init=1, inplace=1),
    "inplace_acc": _r("in place, skip accumulated (skip_init = 0)", Bc=5, Sc=3, has_out=1, init=0, inplace=1),
    "outofplace": _r("out of place (un-fused training forward)", Bc=5, Sc=3, has_out=1, init=0, inplace=0),
    "outofplace_first": _r("out of place, skip_init = 1", Bc=5, Sc=3, has_out=1, init=1, inplace=0),
    "skip_only": _r("has_out = 0 (last block), skip accumulated", Bc=5, Sc=3, has_out=0, init=0, inplace=1),
    "skip_only_init": _r("has_out = 0 and skip_init = 1 (a one-block stack)", Bc=5, Sc=3, has_out=0, init=1, inplace=1),
    "C1025": _r("Mt = 1030 > the 1024-CTA grid", Bc=1000, Sc=30, has_out=1, init=0, inplace=1, F=33),
    "F1_wide": _r("one frame, pitch + 256", Bc=5, Sc=3, has_out=1, init=1, inplace=1, F=1, extra=256),
}

BIAS = {"F129": _r("129 frames"), "F1": _r("one frame", F=1), "C1025": _r("C = 1025 > the 1024-CTA grid", C=1025, F=33),
        "wide": _r("pitch + 256", extra=256)}

CLN = {"F1": _r("one frame", F=1), "F129_C65": _r("C = 65 > 64: the apply kernel's channel loop", C=65),
       "F1025": _r("1025 frames: 2 per scan thread", F=1025), "wide": _r("pitch + 256", F=130, extra=256)}


# ---- inputs ----------------------------------------------------------------------------------------------------------------
def fold_inputs(name, r):
    """per job (W, bias | None, gamma, beta); R"""
    g = gen("fold" + name)
    out = []
    for jb in r["jobs"]:
        M, K = jb["M"], jb["K"]
        W = rnd(g, M, K, scale=K ** -0.5)
        gamma, beta = rnd(g, K, scale=0.3, shift_=1.0), rnd(g, K, scale=0.2)
        bias = None if r.get("nobias") else rnd(g, M, scale=0.1)
        out.append((W, bias, gamma, beta))
    return out, float(f32(torch.tensor(0.0 if r.get("novb") else 1131.4)))


def shared_norm(inputs, r):
    """the jobs of one [out; skip] pair fold the same gLN: give the pair's second job its first job's gamma / beta"""
    out = list(inputs)
    for i, jb in enumerate(r["jobs"]):
        if jb["off"]:
            W, bias, _, _ = out[i]
            out[i] = (W, bias, out[i - 1][2], out[i - 1][3])
    return out


def dw_inputs(name, r):
    g = gen("fdw" + name)
    B, C, F, P = r["B"], r["C"], r["F"], r["P"]
    h = rnd(g, B, C, F, shift_=0.1)
    if r.get("dc"):
        h = f32(h + 100.0)
    h = f32(h * sample_scale(B))
    g1, b1 = norm_params(g, C)
    wd, bd = rnd(g, C, P, scale=0.5), rnd(g, C, scale=0.1)
    return h, g1, b1, wd, bd, stats_of(h)


def block_stats(g, B, n, i):
    """(B, 2) statistics of a synthetic u over n elements: sample b scaled by SCALES[b % 3], block i its own mean / spread"""
    s = sample_scale(B)[:, 0, 0]
    mean = s * (0.3 + 0.07 * i)
    var = (s * (1.0 + 0.11 * i)) ** 2
    return torch.stack([n * mean, n * (var + mean * mean)], 1)


def skip_inputs(name, r):
    g = gen("skip" + name)
    B, F, n, Sc, Bc = r["B"], r["F"], r["n"], r["Sc"], r["Bc"]
    jobs = []
    for i in range(n):
        last = i == n - 1
        Mt = Sc if last else Bc + Sc
        jobs.append(dict(r=f32(rnd(g, B, Mt, F, scale=3.0) * sample_scale(B)), v1=rnd(g, Mt), v2=rnd(g, Mt, scale=0.5),
                         stats=block_stats(g, B, 7.0 * F, i), off=0 if last else Bc, Mt=Mt))
    return jobs, 7.0 * F


def finish_inputs(name, r):
    g = gen("fin" + name)
    B, F, Bc, Sc = r["B"], r["F"], r["Bc"], r["Sc"]
    return (rnd(g, B, Bc, F, shift_=2.0), f32(rnd(g, B, Bc + Sc, F, scale=3.0) * sample_scale(B)), rnd(g, Bc + Sc),
            rnd(g, Bc + Sc, scale=0.5), block_stats(g, B, 7.0 * F, 1), 7.0 * F)


def stats_inputs(name, r):
    g = gen("stp" + name)
    x = rnd(g, r["B"], r["C"], r["F"], shift_=0.2)
    if r.get("dc"):
        x = f32(x + 1e3)
    return f32(x * sample_scale(r["B"]))


def enc_inputs(name, r):
    g = gen("enc" + name)
    B, T = r["B"], r["T"]
    x = f32(rnd(g, B, T) * sample_scale(B)[:, :, 0])
    W = rnd(g, r["N"], r["L"], scale=r["L"] ** -0.5)
    pl = r.get("pl", 0)
    pr, F = enc_geometry(T, r["L"], r["S"], pl)
    return x, W, pl, pr, F


def dec_inputs(name, r):
    g = gen("dec" + name)
    BS, N, F, L = r["B"], r["N"], r["F"], r["L"]
    what = f32(rnd(g, BS, N, F).abs() * sample_scale(BS))
    Wd = rnd(g, N, L, scale=N ** -0.5)
    full = (F - 1) * r["S"] + L
    T_out = full - r["crop"] - r.get("short", 0)
    return what, Wd, T_out


def plain_inputs(name, r):
    g = gen("plain" + name)
    B, C, F, P = r["B"], r["C"], r["F"], r["P"]
    return f32(rnd(g, B, C, F) * sample_scale(B)), rnd(g, C, P, scale=0.5), rnd(g, C, scale=0.1)


def res_inputs(name, r):
    g = gen("res" + name)
    B, F, Bc, Sc = r["B"], r["F"], r["Bc"], r["Sc"]
    Mt = Bc + Sc if r["has_out"] else Sc
    return (rnd(g, B, Mt, F), rnd(g, B, Bc, F, shift_=1.0), rnd(g, B, Sc, F, shift_=-1.0), rnd(g, Bc, scale=0.1),
            rnd(g, Sc, scale=0.1))
