"""Rows, dispatch predicates, launch counts, fp64 references and bounds of tests/test_stage_entries_gpu.py (test infrastructure
only): the C entries that run one stage each -- the separator head and tail (ctn_sep_head_fwd, ctn_sep_tail_fwd: DPRNN-TasNet's
stages around its dual-path blocks) and the plain depthwise-separable convolution (ctn_depthwise_conv1d_fwd,
ctn_pointwise_conv1d_fwd: modules.conv.DepthwiseSeparableConv1d).

Plain torch, no import of the native library: test_stage_entries_cpu.py shows without a GPU that every row reaches the branch its
`reaches` text names, that the restatements agree with the oracle and F.conv1d, and that each bound rejects planted defects.

What each entry runs (csrc/ctn_api.cu, ctn_conv.cu):
  * head: k_fold_batch (Wf = W diag(gamma), v1 = b + W beta, v2 = W gamma; no vb), the weight image (tensor-core modes), one
    EPI_HEAD contraction x0 = rstd (Wf w) + (v1 - mean rstd v2) with (mean, rstd) from the caller's stats0 over n = N frames.
  * tail: the weight image (tensor-core modes), one PRO_PRELU + EPI_MASK contraction what = w[n % N] sigmoid(Wm PReLU(y) + bm),
    ctn_decoder_fwd (k_decoder<stride, 2> for stride in {8, 1, 10, 2} with L = 2 stride, k_decoder_generic otherwise), and the
    latent copy when asked for.  Neither operand carries an operand scale, so f16x3 runs both stages on the tf32 pieces: the same
    kernel and the same image as tf32x3, bit for bit, and never k_maskdec.
  * depthwise: one k_depthwise1d, a bias and K fmas per output, a 64-CTA grid-stride loop over y_pitch (> 16384 columns loop).
  * pointwise: the weight image (tensor-core modes), one contraction (EPI_RAW; with a bias EPI_H with a PReLU slope of 1, its
    statistics into workspace scratch), then ctn_copy_from_pitch (one launch per 65535 rows).

Pad columns [frames, pitch) of the pitched inputs (w and y of the head / tail, x of the pointwise stage): the contraction kernels
load them (whole 128-frame tiles), but a 1x1 contraction's column t only reaches output column t, every epilogue writes 0 there,
EPI_MASK reads w only at valid columns, and the decoder reads only valid frames.  So the pads may hold anything, NaN included: the
GPU file fills them with NaN and requires the bits of a call with zero pads.

Bounds (u = 2^-24; per output element; pw_criterion.py's gate for the contractions):
  * head: e <= bound(mode) of pw_criterion (fp32: (K + 8) u; tf32x3 / f16x3: E_drop / 8; tf32: 2 E_onepass) on the folded form,
    plus the fold's own rounding (forward_kernel_ref.fold: (ceil(K / 32) + 6) u on v1 and v2) carried by the epilogue:
    (ceil(K / 32) + 7) u (sum |W beta| + |b| + |mean| rstd sum |W gamma|).  The folded form's cancellation under a DC offset is
    inherent: |mean| rstd sum |W gamma| is in every term's magnitude.
  * tail: the mask contraction's allowance A = SLACK u |what| + bound(mode) den per element of what (= the latent), pushed
    through the decoder's |Wd|, plus the decoder's own bound (forward_kernel_ref.decoder).  Where the fp64 mask is below 2^-120
    (logits under about -83, which the 1e3-scaled samples reach) A also takes |what| itself: the kernel's fp32 sigmoid
    (__expf, __fdividef) returns 0 there, an absolute error below 1e-36 |w| that no relative bound can hold.
  * depthwise: (K + 1) u (|bias| + sum_k |w_k x|).
  * pointwise: the pw_criterion gate on EPI_RAW or EPI_H(bias, slope 1), with SLACK u |y|.
"""
import collections
import math

import torch
import torch.nn.functional as F

import forward_kernel_ref as FK
import pw_criterion as PC
from train_kernel_ref import f32, gen, rnd, sample_scale

U = PC.U
TILE = 128
MODES = ("fp32", "tf32x3", "f16x3", "tf32")
COPY_ROWS = 65535
DEC_SPECIAL = ((8, 2), (1, 2), (10, 2), (2, 2))   # (stride, L / stride) of the k_decoder<S, 2> instantiations
REJECT = 4.0                                      # a planted defect must land this many times past the bound
SIGMOID_FLOOR = 2.0 ** -120                       # a mask below this may come out as 0 (fp32 range, not accuracy)


def ceil_div(a, b):
    return -(-a // b)


def pitch(frames):
    return ceil_div(frames, TILE) * TILE


def frames_of(T, L, stride):
    """ctn_frames: (frames, pl, pr)"""
    padding = (stride - (T - L) % stride) % stride
    pl = padding // 2
    return (T + padding - L) // stride + 1, pl, padding - pl


def dw_out_len(T, K, stride, padding, dilation):
    return (T + 2 * padding - dilation * (K - 1) - 1) // stride + 1


# ---- dispatch predicates and launch counts --------------------------------------------------------------------------------
def decoder_kernel(L, stride):
    R = L // stride
    return "k_decoder<{},{}>".format(stride, R) if (stride, R) in DEC_SPECIAL else "k_decoder_generic"


def head_launches(mode):
    """k_fold_batch, the weight image (tensor-core modes), the EPI_HEAD contraction"""
    return 1 + (mode != "fp32") + 1


def tail_launches(mode, B, S, N, latent):
    """the weight image (tensor-core modes), the EPI_MASK contraction, the decoder, the latent copy"""
    return (mode != "fp32") + 1 + 1 + (ceil_div(B * S * N, COPY_ROWS) if latent else 0)


def pw_launches(mode, B, M):
    return (mode != "fp32") + 1 + ceil_div(B * M, COPY_ROWS)


DW_LAUNCHES = 1
DW_GRID_COLS = 64 * 256   # k_depthwise1d: at most 64 CTAs of 256 threads along the columns


# ---- rows ------------------------------------------------------------------------------------------------------------------
Head = collections.namedtuple("Head", "B N Bc frames dc eps enc reaches")
Tail = collections.namedtuple("Tail", "B N Bc S L stride T latent reaches")
Dw = collections.namedtuple("Dw", "B C T K stride padding dilation bias extra reaches")
Pw = collections.namedtuple("Pw", "B M K frames bias reaches")

EPS = 1e-8


def _head(B, N, Bc, frames, reaches, dc=0.0, eps=EPS, enc=None):
    return Head(B, N, Bc, frames, dc, eps, enc, reaches)


HEAD = {
    "bc1_n1_f1_b1": _head(1, 1, 1, 1, "Bc = N = 1, one frame: a 1-row n-tile, a 1-channel K slab, one column of 128"),
    "bc129_n513_f129_b37": _head(37, 513, 129, 129, "Bc = 129 (a 1-row second n-tile), N = 513 (a 1-channel last slab), "
                                 "frames = 129 (pitch 256), B = 37 at scales 1e-3 / 1 / 1e3"),
    "bc128_n64_f3999": _head(1, 64, 128, 3999, "Bc = 128: one whole n-tile; 3999 frames (pitch 4096)"),
    "bc129_n64_f127_b37": _head(37, 64, 129, 127, "127 frames: one short of a tile; B = 37"),
    "bc1_n513_f128": _head(2, 513, 1, 128, "128 frames: exactly one tile, pitch == frames"),
    "dc": _head(3, 64, 128, 129, "w = 1e3 + N(0, 1): the folded gLN's cancellation", dc=1e3),
    "eps_var": _head(2, 64, 64, 200, "eps = 1e-3 against var(w) ~ 1e-3: eps inside the sqrt matters", eps=1e-3),
    "enc_stats": _head(2, 64, 128, 0, "w and stats0 from ctn_encoder_fwd (L = 16, stride 8, T = 4003), as DPRNN-TasNet passes them",
                       enc=(16, 8, 4003)),
}


def _tail(B, N, Bc, S, L, stride, T, latent, reaches):
    return Tail(B, N, Bc, S, L, stride, T, latent, reaches)


TAIL = {
    "s2_l16s8_n128": _tail(2, 128, 64, 2, 16, 8, 4003, False, "k_decoder<8,2>; the shape on which the model path fuses k_maskdec "
                                                               "in f16x3: this entry must not"),
    "s2_l16s8_n128_lat": _tail(2, 128, 64, 2, 16, 8, 1001, True, "k_decoder<8,2>, latent; T = 1001 = 1 mod 8"),
    "s1_l2s1_n5": _tail(3, 5, 7, 1, 2, 1, 300, True, "k_decoder<1,2>, S = 1, N = 5, Bc = 7, latent"),
    "s4_l20s10_n129": _tail(2, 129, 33, 4, 20, 10, 2001, True, "k_decoder<10,2>, S = 4, N = 129 (a 1-row last n-tile of S N = "
                                                                "516), T = 2001 = 1 mod 10"),
    "s2_l4s2_n33_b37": _tail(37, 33, 16, 2, 4, 2, 257, False, "k_decoder<2,2>, B = 37, T = 257 = 1 mod 2"),
    "s2_l16s4_n7": _tail(2, 7, 20, 2, 16, 4, 513, True, "k_decoder_generic (R = 4), T = 513 = 1 mod 4, latent"),
    "s1_l40s20_n64": _tail(2, 64, 64, 1, 40, 20, 4001, False, "k_decoder_generic at L / stride = 40 / 20, T = 4001 = 1 mod 20"),
    "s4_l16s8_n1_f1": _tail(1, 1, 1, 4, 16, 8, 16, True, "N = Bc = 1, one frame (T = L), S = 4, latent"),
}


def _dw(B, C, T, K, reaches, stride=None, padding=0, dilation=1, bias=True, extra=0):
    return Dw(B, C, T, K, K if stride is None else stride, padding, dilation, bias, extra, reaches)


DW = {
    "to1": _dw(2, 5, 3, 3, "To = 1: T + 2 padding == span", stride=1, padding=1, dilation=2),
    "stride_gt_k": _dw(2, 5, 1000, 3, "stride 5 > K = 3: skipped samples", stride=5, padding=1),
    "stride_default": _dw(2, 5, 1001, 4, "stride defaulting to K = 4 (the module's default)"),
    "dil_span_gt_t": _dw(2, 5, 60, 3, "dilation (K - 1) = 100 > T = 60, padding 25: outer taps read padding", stride=1,
                         padding=25, dilation=50),
    "to_gt_16384": _dw(2, 3, 40000, 3, "To = 40000 > 64 x 256: the grid-stride loop", stride=1, padding=1),
    "c1_nobias": _dw(2, 1, 777, 5, "C = 1, no bias", stride=2, padding=2, dilation=3, bias=False),
    "b37_pitch": _dw(37, 5, 300, 3, "B = 37, y_pitch = pitch + 128 > To", stride=1, padding=1, extra=128),
    "nobias_pitch": _dw(3, 7, 129, 3, "no bias, y_pitch = pitch + 256", stride=1, padding=1, dilation=2, bias=False, extra=256),
}


def _pw(B, M, K, frames, reaches, bias=True):
    return Pw(B, M, K, frames, bias, reaches)


PW = {
    "m1_k33": _pw(2, 1, 33, 129, "M = 1: a 1-row n-tile; K = 33: a 1-channel second slab"),
    "m129_k64_b37": _pw(37, 129, 64, 129, "M = 129, B = 37"),
    "k1056": _pw(2, 64, 1056, 300, "K = 1056: 33 slabs"),
    "k1_nobias": _pw(2, 16, 1, 257, "K = 1 (C = 1), no bias: EPI_RAW", bias=False),
    "m129_nobias_f1": _pw(3, 129, 40, 1, "one frame, no bias", bias=False),
}


# ---- branches --------------------------------------------------------------------------------------------------------------
BRANCHES = {
    "head_partial_ntile": "head: Bc % 128 != 0 (a partial last n-tile)",
    "head_full_ntile": "head: Bc % 128 == 0 (whole n-tiles)",
    "head_ragged_k": "head: N % 32 != 0 (a partial last K slab)",
    "head_tile_edge": "head: frames within one of a multiple of 128",
    "head_dc": "head: a DC offset large against the spread",
    "head_eps": "head: eps comparable to the variance",
    "head_enc_stats": "head: stats0 from ctn_encoder_fwd",
    "head_b37": "head: B = 37",
    "dec_8_2": "tail: k_decoder<8,2>", "dec_1_2": "tail: k_decoder<1,2>", "dec_10_2": "tail: k_decoder<10,2>",
    "dec_2_2": "tail: k_decoder<2,2>", "dec_generic": "tail: k_decoder_generic",
    "tail_S1": "tail: S = 1", "tail_S2": "tail: S = 2", "tail_S4": "tail: S = 4",
    "tail_ragged_n": "tail: N not a multiple of 4 or 128",
    "tail_t1_mod_stride": "tail: T = 1 mod stride",
    "tail_latent": "tail: a latent", "tail_no_latent": "tail: no latent",
    "tail_maskdec_shape": "tail: L / stride 16 / 8, N % 128 == 0, Bc <= 128 (k_maskdec's shape)",
    "dw_to1": "depthwise: To = 1", "dw_stride_gt_k": "depthwise: stride > K", "dw_stride_default": "depthwise: stride == K",
    "dw_span_gt_t": "depthwise: dilation (K - 1) > T", "dw_grid_stride": "depthwise: To > 16384 (grid-stride loop)",
    "dw_c1": "depthwise: C = 1", "dw_nobias": "depthwise: no bias", "dw_bias": "depthwise: a bias", "dw_b37": "depthwise: B = 37",
    "dw_wide_pitch": "depthwise: y_pitch > pitch(To)",
    "pw_m1": "pointwise: M = 1", "pw_m129": "pointwise: M = 129", "pw_k1056": "pointwise: K = 1056", "pw_k1": "pointwise: K = 1",
    "pw_bias": "pointwise: a bias (EPI_H, slope 1)", "pw_nobias": "pointwise: no bias (EPI_RAW)", "pw_b37": "pointwise: B = 37",
}


def head_frames(r):
    return frames_of(r.enc[2], r.enc[0], r.enc[1])[0] if r.enc else r.frames


def head_branches(r):
    f, got = head_frames(r), set()
    got.add("head_partial_ntile" if r.Bc % TILE else "head_full_ntile")
    if r.N % 32:
        got.add("head_ragged_k")
    if min(f % TILE, TILE - f % TILE) <= 1:
        got.add("head_tile_edge")
    if r.dc:
        got.add("head_dc")
    if r.eps > 1e-6:
        got.add("head_eps")
    if r.enc:
        got.add("head_enc_stats")
    if r.B == 37:
        got.add("head_b37")
    return got


def tail_branches(r):
    got = {"dec_generic" if decoder_kernel(r.L, r.stride) == "k_decoder_generic" else "dec_{}_{}".format(r.stride, r.L // r.stride),
           "tail_S{}".format(r.S), "tail_latent" if r.latent else "tail_no_latent"}
    if r.N % 4 and r.N % 128:
        got.add("tail_ragged_n")
    if r.T % r.stride == 1 % r.stride:
        got.add("tail_t1_mod_stride")
    if r.L == 16 and r.stride == 8 and r.N % 128 == 0 and r.Bc <= 128:
        got.add("tail_maskdec_shape")
    return got


def dw_branches(r):
    To, got = dw_out_len(r.T, r.K, r.stride, r.padding, r.dilation), set()
    if To == 1:
        got.add("dw_to1")
    if r.stride > r.K:
        got.add("dw_stride_gt_k")
    if r.stride == r.K:
        got.add("dw_stride_default")
    if r.dilation * (r.K - 1) > r.T:
        got.add("dw_span_gt_t")
    if pitch(To) + r.extra > DW_GRID_COLS:
        got.add("dw_grid_stride")
    if r.C == 1:
        got.add("dw_c1")
    got.add("dw_bias" if r.bias else "dw_nobias")
    if r.B == 37:
        got.add("dw_b37")
    if r.extra:
        got.add("dw_wide_pitch")
    return got


def pw_branches(r):
    got = {"pw_bias" if r.bias else "pw_nobias"}
    for k, ok in (("pw_m1", r.M == 1), ("pw_m129", r.M == 129), ("pw_k1056", r.K == 1056), ("pw_k1", r.K == 1), ("pw_b37", r.B == 37)):
        if ok:
            got.add(k)
    return got


# the branches each row names in its `reaches` text
EXPECT = {
    ("head", "bc1_n1_f1_b1"): {"head_partial_ntile", "head_ragged_k", "head_tile_edge"},
    ("head", "bc129_n513_f129_b37"): {"head_partial_ntile", "head_ragged_k", "head_tile_edge", "head_b37"},
    ("head", "bc128_n64_f3999"): {"head_full_ntile"},
    ("head", "bc129_n64_f127_b37"): {"head_partial_ntile", "head_tile_edge", "head_b37"},
    ("head", "bc1_n513_f128"): {"head_partial_ntile", "head_ragged_k", "head_tile_edge"},
    ("head", "dc"): {"head_dc", "head_full_ntile", "head_tile_edge"},
    ("head", "eps_var"): {"head_eps"},
    ("head", "enc_stats"): {"head_enc_stats", "head_full_ntile"},
    ("tail", "s2_l16s8_n128"): {"dec_8_2", "tail_S2", "tail_maskdec_shape", "tail_no_latent"},
    ("tail", "s2_l16s8_n128_lat"): {"dec_8_2", "tail_latent", "tail_t1_mod_stride", "tail_maskdec_shape"},
    ("tail", "s1_l2s1_n5"): {"dec_1_2", "tail_S1", "tail_ragged_n", "tail_latent"},
    ("tail", "s4_l20s10_n129"): {"dec_10_2", "tail_S4", "tail_ragged_n", "tail_t1_mod_stride", "tail_latent"},
    ("tail", "s2_l4s2_n33_b37"): {"dec_2_2", "tail_ragged_n", "tail_t1_mod_stride", "tail_no_latent"},
    ("tail", "s2_l16s4_n7"): {"dec_generic", "tail_ragged_n", "tail_t1_mod_stride", "tail_latent"},
    ("tail", "s1_l40s20_n64"): {"dec_generic", "tail_S1", "tail_t1_mod_stride", "tail_no_latent"},
    ("tail", "s4_l16s8_n1_f1"): {"dec_8_2", "tail_S4", "tail_ragged_n", "tail_latent"},
    ("dw", "to1"): {"dw_to1"},
    ("dw", "stride_gt_k"): {"dw_stride_gt_k"},
    ("dw", "stride_default"): {"dw_stride_default"},
    ("dw", "dil_span_gt_t"): {"dw_span_gt_t"},
    ("dw", "to_gt_16384"): {"dw_grid_stride"},
    ("dw", "c1_nobias"): {"dw_c1", "dw_nobias"},
    ("dw", "b37_pitch"): {"dw_b37", "dw_wide_pitch", "dw_bias"},
    ("dw", "nobias_pitch"): {"dw_nobias", "dw_wide_pitch"},
    ("pw", "m1_k33"): {"pw_m1", "pw_bias"},
    ("pw", "m129_k64_b37"): {"pw_m129", "pw_b37"},
    ("pw", "k1056"): {"pw_k1056"},
    ("pw", "k1_nobias"): {"pw_k1", "pw_nobias"},
    ("pw", "m129_nobias_f1"): {"pw_m129", "pw_nobias"},
}


def all_rows():
    """(group, name, row, branches it names, branches reached)"""
    out = []
    for grp, rows, fn in (("head", HEAD, head_branches), ("tail", TAIL, tail_branches), ("dw", DW, dw_branches),
                          ("pw", PW, pw_branches)):
        out += [(grp, n, r, EXPECT[(grp, n)], fn(r)) for n, r in rows.items()]
    return out


# ---- inputs ----------------------------------------------------------------------------------------------------------------
def head_inputs(name, r):
    """float32-valued float64 tensors: w (B, N, F) (None for the encoder row: the GPU file encodes x), x (B, 1, T) or None,
    enc_w (N, L) or None, gamma, beta (N), W (Bc, N), bias (Bc)"""
    g = gen("head" + name)
    B, N, Bc = r.B, r.N, r.Bc
    w = x = enc_w = None
    if r.enc:
        L, stride, T = r.enc
        x = f32(rnd(g, B, 1, T) * sample_scale(B))
        enc_w = rnd(g, N, L, scale=L ** -0.5)
    else:
        spread = 0.03 if r.eps > 1e-6 else 1.0
        w = f32((rnd(g, B, N, r.frames, scale=spread, shift_=0.1 * spread) + r.dc) * sample_scale(B))
    gamma, beta = rnd(g, N, scale=0.3, shift_=1.0), rnd(g, N, scale=0.2)
    W, bias = rnd(g, Bc, N, scale=N ** -0.5), rnd(g, Bc, scale=0.1)
    return dict(w=w, x=x, enc_w=enc_w, gamma=gamma, beta=beta, W=W, bias=bias)


def tail_inputs(name, r):
    g = gen("tail" + name)
    B, N, Bc, S = r.B, r.N, r.Bc, r.S
    frames = frames_of(r.T, r.L, r.stride)[0]
    # y is the separator body's normalised output: O(1) in every sample (scaled like w, the 1e3 samples' logits would sit in
    # sigmoid's flat tails, where the gate's E_drop is not defined); w, the encoder output, takes the per-sample scales
    y = rnd(g, B, Bc, frames)
    w = f32(rnd(g, B, N, frames).abs() * sample_scale(B))
    a = float(f32(torch.tensor(0.25)))
    Wm, bm = rnd(g, S * N, Bc, scale=Bc ** -0.5), rnd(g, S * N, scale=0.5)
    Wd = rnd(g, N, r.L, scale=N ** -0.5)
    return dict(y=y, w=w, a=a, Wm=Wm, bm=bm, Wd=Wd)


def dw_inputs(name, r):
    g = gen("dw" + name)
    x = f32(rnd(g, r.B, r.C, r.T) * sample_scale(r.B))
    return dict(x=x, w=rnd(g, r.C, r.K, scale=0.5), bias=rnd(g, r.C, scale=0.1) if r.bias else None)


def pw_inputs(name, r):
    g = gen("pw" + name)
    x = f32(rnd(g, r.B, r.K, r.frames) * sample_scale(r.B))
    return dict(x=x, W=rnd(g, r.M, r.K, scale=r.K ** -0.5), bias=rnd(g, r.M, scale=0.1) if r.bias else None)


# ---- fp64 restatements -----------------------------------------------------------------------------------------------------
def gln_frames(w, stats, gamma, beta, eps, n, mut=None):
    """gLN of w (B, N, F) from (sum, sumsq) statistics over n elements: biased variance, eps inside the sqrt"""
    mean = stats[:, 0] / n
    var = (stats[:, 1] / n - mean * mean).clamp_min(0.0)
    rstd = 1.0 / (torch.sqrt(var) + eps) if mut == "eps_outside" else 1.0 / torch.sqrt(var + eps)
    return (w - mean[:, None, None]) * rstd[:, None, None] * gamma[None, :, None] + beta[None, :, None]


def stats_frames(w):
    return torch.stack([w.sum((1, 2)), (w * w).sum((1, 2))], 1)


def head64(w, stats, gamma, beta, W, bias, eps, mut=None):
    """x0 = W gLN(w) + b, the gLN over the valid frames (w holds only those).  mut: 'eps_outside' (1 / (std + eps)), 'n_pitch'
    (the element count and sums over the whole pitch, zero pads)"""
    B, N, Fr = w.shape
    n = N * Fr
    if mut == "n_pitch":
        n = N * pitch(Fr)
    x = gln_frames(w, stats, gamma, beta, eps, n, mut)
    return torch.einsum("mk,bkt->bmt", W, x) + bias[None, :, None]


def head_reference(w, stats, gamma, beta, W, bias, eps):
    """pw_criterion.Reference of the folded form x0 = rstd (W diag(gamma) w) + (v1 - mean rstd v2), and the fold's allowance"""
    N, Fr = w.shape[1], w.shape[2]
    Wf, v1, v2 = W * gamma[None], bias + W @ beta, W @ gamma
    ref = PC.Reference(Wf, w, w.abs(), PC.epi_head(v1, v2, stats, N * Fr, eps))
    mean, rstd = PC.mean_rstd(stats, N * Fr, eps)
    kf = ceil_div(N, 32) + 7
    fold = kf * U * ((W * beta[None]).abs().sum(1) + bias.abs() + mean.abs().view(-1, 1) * rstd.view(-1, 1) * Wf.abs().sum(1))
    return ref, fold[:, :, None]


def tail64(y, w, a, Wm, bm, Wd, S, stride, crop, T, mut=None):
    """-> out (B, S, T), latent (B, S, N, F).  mut: 'no_bias', 'prelu_pos' (the slope on positive values too), 'crop_off' (one
    sample late), 'latent_pitch' (rows read at a stride of frames from the pitched w_hat)"""
    B, N, Fr = w.shape
    p = a * y if mut == "prelu_pos" else PC.prelu(y, a)
    logit = torch.einsum("mk,bkt->bmt", Wm, p) + (0.0 if mut == "no_bias" else bm[None, :, None])
    what = torch.sigmoid(logit) * w.repeat(1, S, 1)
    full = F.conv_transpose1d(what.reshape(B * S, N, Fr), Wd[:, None], stride=stride)[:, 0]
    at = crop + 1 if mut == "crop_off" else crop
    full = F.pad(full, (0, 1))
    out = full[:, at:at + T].reshape(B, S, T)
    lat = what.reshape(B, S, N, Fr)
    if mut == "latent_pitch":
        P = pitch(Fr)
        flat = F.pad(what, (0, P - Fr)).reshape(-1)
        lat = flat[:B * S * N * Fr].reshape(B, S, N, Fr)
    return out, lat


def tail_reference(y, w, a, Wm, bm, Wd, S, stride, crop, T):
    """the mask contraction's pw_criterion.Reference (its D is w_hat = the latent) and a function mode -> (latent allowance,
    output allowance)"""
    B, N, Fr = w.shape
    P = PC.prelu(y, a)
    ref = PC.Reference(Wm, P, P.abs(), PC.epi_mask(bm, w, N))
    what, den, smag = ref.out["D"]
    # sigmoid(logit) below fp32's normal range (logit < -87: __expf overflows, the quotient flushes): the kernel's mask is 0 there
    under = torch.sigmoid(torch.einsum("mk,bkt->bmt", Wm, P) + bm[None, :, None]) < SIGMOID_FLOOR

    def allowance(mode):
        lat = PC.SLACK_ULPS * U * smag + ref.bound(mode) * den + torch.where(under, smag, 0.0)
        dec = FK.decoder(what.reshape(B * S, N, Fr), Wd, stride, crop, T)["y"][1]
        prop = F.conv_transpose1d(lat.reshape(B * S, N, Fr), Wd.abs()[:, None], stride=stride)[:, 0, crop:crop + T]
        return lat.reshape(B, S, N, Fr), (prop + dec).reshape(B, S, T)
    return ref, allowance


def depthwise64(x, w, bias, stride, padding, dilation, mut=None):
    """y[b][c][to] = bias[c] + sum_k w[c][k] x[b][c][to stride + k dilation - padding] (zero outside [0, T)), with its magnitude.
    mut: 'dil_off' (dilation + 1), 'one_side' (all the padding on the right), 'stride_ignored' (stride 1); To is kept."""
    B, C, T = x.shape
    K = w.shape[1]
    To = dw_out_len(T, K, stride, padding, dilation)
    d = dilation + 1 if mut == "dil_off" else dilation
    s = 1 if mut == "stride_ignored" else stride
    off = 0 if mut == "one_side" else padding
    b = torch.zeros(C, dtype=x.dtype) if bias is None else bias
    y = b[None, :, None].expand(B, C, To).clone()
    m = b.abs()[None, :, None].expand(B, C, To).clone()
    to = torch.arange(To)
    for k in range(K):
        t = to * s + k * d - off
        ok = (t >= 0) & (t < T)
        xv = torch.zeros(B, C, To, dtype=x.dtype)
        xv[..., ok] = x[..., t[ok]]
        y = y + w[None, :, k, None] * xv
        m = m + (w[None, :, k, None] * xv).abs()
    return y, m


def depthwise_bound(m, K):
    return (K + 1) * U * m


def pointwise64(x, W, bias):
    y = torch.einsum("mk,bkt->bmt", W, x)
    return y if bias is None else y + bias[None, :, None]


def pointwise_reference(x, W, bias):
    epi = PC.epi_raw() if bias is None else PC.epi_h(bias, 1.0)
    return PC.Reference(W, x, x.abs(), epi)


def share(got, ref64, allowance):
    """max |got - ref64| / allowance (inf on a non-finite value or an error where the allowance is 0)"""
    got = got.double()
    if not bool(torch.isfinite(got).all()):
        return math.inf
    err = (got - ref64).abs()
    r = torch.where(allowance > 0, err / allowance.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def gate_allowance(ref, mode, key="D"):
    """pw_criterion's gate as a per-element allowance: SLACK u smag + bound(mode) den"""
    _, den, smag = ref.out[key]
    return PC.SLACK_ULPS * U * smag + ref.bound(mode, key) * den
