"""Rows, fp64 references, error bounds and kernel-selection rules of the multichannel filter banks (in_channels = C): the encoder
ctn_encoder_mc_fwd (k_encoder_v4_mc<L, L/2> / k_encoder_mc), the decoder ctn_decoder_mc_fwd (k_decoder_mc_v<S, 2> / k_decoder_mc)
and the filter-bank weight gradient ctn_encdec_wgrad (k_encdec_wgrad / k_encdec_wgrad_generic) over C channels.

Plain torch, no import of the native library: test_mc_filterbank_cpu.py checks here that the references agree with torch, that
every row reaches the kernel its `reaches` text names, that every instantiation and every fallback reason has a row, and that the
bounds reject plausible bugs; test_mc_filterbank_gpu.py holds the kernels to them.

Every reference is written from the operation's definition in float64 over the kernel's fp32 inputs, and returns the value with
its magnitude M (the same sum over |terms|).  Bounds, u = 2^-24, d = 2^-53, per output element (fmaf rounds once per step, so a
chain of k fmaf from 0 is within k u M of the exact sum, whatever the order):
  * encoder  w[b][n][f] = sum_c sum_k W[n][c][k] xpad[b][c][f S + k]: both kernels run one fmaf chain over the C L terms (the
    fast one channel by channel in registers, the fallback skipping the zero padding), ReLU is exact:  C L u M.
  * decoder  y[bs][c][t] = sum_n sum_{f, k: f S + k = t + crop} what[bs][n][f] Wd[n][c][k], R = L / S frames per sample:
    k_decoder_mc_v splits the N bases over DEC_SPLIT = 4 thread groups, each a chain of ceil(N / 4) R fmaf, and adds the other 3
    partials:  (ceil(N / 4) R + 3) u M.  k_decoder_mc is one chain of N R fmaf:  N R u M.
  Shared memory: the fast encoder needs the 48 KB opt-in once its dynamic size plus its static red[64] (512 B) passes 48 KB.
  * statistics (sum w, sum w^2 per sample, atomically added onto a double pair): k_encoder_v4_mc adds a base's 4 frames pairwise
    (2 roundings) into an fp32 partial that spills to double after 4 groups of 4 bases (16 additions); its sum of squares is one
    fmaf chain over those 64 values:  18 u sum|w|, 64 u sum w^2.  k_encoder_mc accumulates in double.  Both add the double
    stage: (N + 8 + n_cta + 2) d of the same sums (thread chain, block tree, one atomic per CTA), and 64 d for the fp64
    reference's own summation.
  * weight gradient  dW[n][c][k] += sum_{r, f} act[r][n][f] sig[r C + c][f S + k - pl] (0 outside [0, T)):
      k_encdec_wgrad (L <= 32), grid (N C, gy), gy = clamp(ceil(592 / (N C)), 1, R): a thread walks its frames f = tid,
      tid + 256, ... of rows r = y, y + gy, ...: a chain of m = ceil(frames / 256) ceil(R / gy) fmaf.  Then a 5-level warp tree,
      8 warps' float atomics onto a shared slot (in no fixed order: 8 additions) and gy CTAs' float atomics onto dW:
        (m + 5 + 8 + gy + 1) u M + gy u |base|         (+1: the second-order term of the chain; base: dW's value on entry)
      k_encdec_wgrad_generic (any L), one CTA per (n, c, k): ceil(frames / 256) fmaf per row and thread in fp32, each row's
      partial added in double, a double block tree, one rounding to float and one float atomic onto dW:
        (ceil(frames / 256) + 2) u M + u |base| + (R + 8) d M
A kernel that drops a channel, shifts a tap, loses the last frame, reads a column past the valid range or swaps the weight's
channel and basis strides moves some output by far more than these bounds: MUTANTS below, checked by test_mc_filterbank_cpu.py.
"""
import collections
import math

import torch

U = 2.0 ** -24
DU = 2.0 ** -53
DEC_SPLIT = 4           # ctn_encdec.cu
ENCDEC_MAX_L = 32       # ctn_train.cu
SMEM_OPT_IN = 48 * 1024
ENC_STATIC_SMEM = 8 * 64  # the encoder kernels' static red[64] doubles count against the 48 KB too
SMEM_MAX = 200 * 1024
GRID_X_MAX = 0x7fffffff
SCALES = (1e-3, 1.0, 1e3)  # per-sample input scale: statistics read from the wrong sample are off by 1e3
MUTANTS = ("drop_channel", "shift_tap", "drop_last_frame", "read_past", "swap_strides")


def pitch128(frames):
    return -(-frames // 128) * 128


def gen(name):
    return torch.Generator().manual_seed(sum(map(ord, name)) * 7 + len(name))


def f32(x):
    return x.float().double()


# ---- rows ------------------------------------------------------------------------------------------------------------------
# T = (frames - 1) S + L - pl - pr.  pitch None: ctn_pitch(frames) (a multiple of 128); w_off: w starts that many floats past a
# 16-byte boundary.
Enc = collections.namedtuple("Enc", "C N L S B frames pl pr pitch w_off relu stats reaches")
# what (BS, N, pitch) with NaN past frames; the output is full[crop : full_len - tail], full_len = (frames - 1) S + R S.
Dec = collections.namedtuple("Dec", "C N S R BS frames pitch crop tail reaches")
# act (R, N, pitch) with NaN past frames, sig (R C, T) placed sig_off floats past a 16-byte boundary.
Wg = collections.namedtuple("Wg", "C N L S R frames pl pr sig_off reaches")


def enc_T(r):
    return (r.frames - 1) * r.S + r.L - r.pl - r.pr


def enc_pitch(r):
    return pitch128(r.frames) if r.pitch is None else r.pitch


ENC = {
    "L2-C1-N1-f1": Enc(1, 1, 2, 1, 1, 1, 0, 0, None, 0, False, False,
                       "k_encoder_v4_mc<2,1>: C = 1 through the multichannel entry; N = 1, so 3 of 4 warps own no basis; one frame"),
    "L4-C2-N3-f3": Enc(2, 3, 4, 2, 3, 3, 1, 1, None, 0, True, True,
                       "k_encoder_v4_mc<4,2>: N = 3 < 4 (the padded N4 column and the store loop's break); 3 frames in one 4-frame "
                       "group; pad 1 / 1; ReLU; statistics of B = 3"),
    "L8-C3-N13-f129": Enc(3, 13, 8, 4, 3, 129, 2, 2, None, 0, False, True,
                          "k_encoder_v4_mc<8,4>: N = 13; 129 frames, one past a 128-frame CTA; pad 2 / 2; statistics"),
    "L8-C2-N16-pitch256": Enc(2, 16, 8, 4, 2, 128, 2, 2, 256, 0, True, False,
                              "k_encoder_v4_mc<8,4>: w_pitch = 256 for 128 frames: the second CTA stores only zero padding"),
    "L16-C2-N292-48KB": Enc(2, 292, 16, 8, 1, 4, 4, 4, None, 0, False, False,
                            "k_encoder_v4_mc<16,8>: 48 640 B, with the static 512 B exactly 48 KB, the default limit; 4 frames"),
    "L16-C2-N296-opt-in": Enc(2, 296, 16, 8, 1, 4, 4, 4, None, 0, False, False,
                              "k_encoder_v4_mc<16,8> [opt-in]: 49 152 B dynamic, over 48 KB only with the static 512 B; 4 frames"),
    "L16-C2-N297-opt-in": Enc(2, 297, 16, 8, 3, 129, 4, 4, None, 0, True, True,
                              "k_encoder_v4_mc<16,8> [opt-in]: 49 664 B, N % 4 = 1; ReLU; statistics"),
    "L16-C8-N256-176KB": Enc(8, 256, 16, 8, 3, 128, 4, 4, None, 0, False, True,
                             "k_encoder_v4_mc<16,8> [opt-in]: C = 8, N = 256, 176 128 B; 128 frames; statistics"),
    "L16-C8-N312-200KB": Enc(8, 312, 16, 8, 1, 5, 4, 4, None, 0, False, False,
                             "k_encoder_v4_mc<16,8> [opt-in]: shared memory exactly 200 KB, the largest the fast path takes; 5 frames"),
    "L20-C2-N42-ragged": Enc(2, 42, 20, 10, 3, 127, 3, 4, None, 0, True, True,
                             "k_encoder_v4_mc<20,10>: N = 42; pad 3 / 4 (ragged T); 127 frames; ReLU; statistics"),
    "L2-C64-N42": Enc(64, 42, 2, 1, 2, 5, 0, 0, None, 0, False, True,
                      "k_encoder_v4_mc<2,1> [opt-in]: C = 64, 120 832 B; 5 frames; statistics of B = 2"),
    "L4-C64-N4-long": Enc(64, 4, 4, 2, 2, 4000, 1, 1, None, 0, True, True,
                          "k_encoder_v4_mc<4,2> [opt-in]: C = 64, N = 4, 102 400 B; 4000 frames over 32 CTAs; ReLU; statistics"),
    "L16S4": Enc(2, 13, 16, 4, 1, 5, 2, 2, None, 0, False, False, "k_encoder_mc [L != 2 stride]: 16 / 4; 5 frames"),
    "L16S16": Enc(3, 4, 16, 16, 3, 3, 0, 0, None, 0, True, True,
                  "k_encoder_mc [L != 2 stride]: 16 / 16, no overlap; N = 4; ReLU; statistics"),
    "L12S6": Enc(2, 42, 12, 6, 1, 128, 3, 3, None, 0, False, False, "k_encoder_mc [L outside the switch]: 12 / 6; 128 frames"),
    "L40S20": Enc(3, 1, 40, 20, 3, 129, 3, 4, None, 0, True, True,
                  "k_encoder_mc [L outside the switch]: 40 / 20; N = 1; 129 frames; ReLU; statistics"),
    "pitch129": Enc(2, 42, 16, 8, 3, 129, 4, 4, 129, 0, False, True,
                    "k_encoder_mc [w_pitch % 128]: w_pitch = frames = 129, as the Encoder module passes; statistics"),
    "w+1": Enc(2, 13, 16, 8, 1, 127, 4, 4, None, 1, False, False, "k_encoder_mc [w misaligned]: w one float past a 16-byte boundary"),
    "L16-C10-N256-220KB": Enc(10, 256, 16, 8, 3, 128, 4, 4, None, 0, False, True,
                              "k_encoder_mc [shared memory > 200 KB]: C = 10, N = 256 would need 220 160 B; statistics"),
    "L16-C8-N313": Enc(8, 313, 16, 8, 1, 4, 4, 4, None, 0, False, False,
                       "k_encoder_mc [shared memory > 200 KB]: 206 848 B, the first N past 200 KB at C = 8"),
}

DEC = {
    "S1-N1-C2-BS12": Dec(2, 1, 1, 2, 12, 126, 131, 0, 0, "k_decoder_mc_v<1,2>: N = 1 < DEC_SPLIT; 127 segments; BS = 12"),
    "S2-N3-C3": Dec(3, 3, 2, 2, 1, 127, 133, 1, 2, "k_decoder_mc_v<2,2>: N = 3; 128 segments; crop 1 / 2"),
    "S8-N5-C64": Dec(64, 5, 8, 2, 1, 128, 130, 3, 5, "k_decoder_mc_v<8,2>: C = 64, N = 5 (not a multiple of DEC_SPLIT); 129 segments; crop 3 / 5"),
    "S10-N512-opt-in": Dec(2, 512, 10, 2, 12, 128, 256, 5, 5,
                           "k_decoder_mc_v<10,2> [opt-in]: N = 512, 56 320 B; 129 segments; crop 5 / 5; BS = 12"),
    "S10-N2368-200KB": Dec(2, 2368, 10, 2, 1, 3, 8, 0, 0,
                           "k_decoder_mc_v<10,2> [opt-in]: shared memory exactly 200 KB, the largest the fast path takes"),
    "S10-N2369": Dec(2, 2369, 10, 2, 1, 3, 8, 0, 0, "k_decoder_mc [shared memory > 200 KB]: 204 880 B"),
    "S8-f1": Dec(3, 3, 8, 2, 12, 1, 4, 2, 3, "k_decoder_mc_v<8,2>: one frame, two segments; crop 2 / 3"),
    "R1-S16": Dec(3, 5, 16, 1, 1, 127, 130, 0, 0, "k_decoder_mc [R != 2]: stride = L = 16, no overlap"),
    "R4-S4": Dec(2, 3, 4, 4, 12, 128, 131, 1, 1, "k_decoder_mc [R != 2]: 16 / 4; crop 1 / 1; BS = 12"),
    "S20R2-C64": Dec(64, 42, 20, 2, 1, 127, 131, 7, 9, "k_decoder_mc [stride outside the list]: 40 / 20, C = 64; crop 7 / 9"),
}

WG = {
    "vec-gyR": Wg(2, 4, 16, 8, 3, 300, 8, 8, 0,
                  "k_encdec_wgrad [gy = R] [vector] [boundary]: N C = 8, gy = R = 3; 300 frames (2 per thread for the first 44)"),
    "L6-scalar": Wg(3, 5, 6, 4, 2, 200, 4, 2, 0, "k_encdec_wgrad [gy = R] [scalar: L % 4] [boundary]: L = 6, everything else aligned"),
    "S2-scalar": Wg(2, 3, 16, 2, 2, 301, 8, 8, 0, "k_encdec_wgrad [gy = R] [scalar: stride % 4] [boundary]: stride 2"),
    "pl2-scalar": Wg(2, 3, 16, 8, 2, 100, 2, 6, 0, "k_encdec_wgrad [gy = R] [scalar: pad_left % 4] [boundary]: pad 2 / 6"),
    "T799-scalar": Wg(2, 3, 16, 8, 2, 100, 4, 5, 0, "k_encdec_wgrad [gy = R] [scalar: T % 4] [boundary]: T = 799"),
    "sig+1-scalar": Wg(2, 3, 16, 8, 2, 100, 8, 8, 1, "k_encdec_wgrad [gy = R] [scalar: sig misaligned] [boundary]: sig one float past 16 B"),
    "gy1-vec": Wg(2, 296, 8, 4, 4, 129, 4, 4, 0, "k_encdec_wgrad [gy = 1] [vector] [boundary]: N C = 592"),
    "gy3-R12": Wg(2, 100, 20, 10, 12, 50, 5, 5, 0, "k_encdec_wgrad [gy = 3] [scalar: stride % 4, pad_left % 4] [boundary]: N C = 200, R = 12"),
    "boundary-only": Wg(3, 7, 32, 16, 2, 1, 10, 10, 0, "k_encdec_wgrad [gy = R] [boundary]: L = 32 = ENCDEC_MAX_L, one frame wider than T = 12"),
    "vec-C64": Wg(64, 3, 4, 4, 5, 257, 0, 0, 0, "k_encdec_wgrad [gy = 4] [vector]: C = 64, no padding; 257 frames"),
    "L33": Wg(2, 5, 33, 11, 2, 300, 11, 11, 0, "k_encdec_wgrad_generic: L = 33 = ENCDEC_MAX_L + 1; 300 frames"),
    "L40-C3": Wg(3, 13, 40, 20, 3, 129, 3, 4, 0, "k_encdec_wgrad_generic: L = 40; pad 3 / 4"),
    "L64-C64": Wg(64, 4, 64, 32, 2, 40, 16, 16, 0, "k_encdec_wgrad_generic: L = 64, C = 64"),
    "NC65536": Wg(64, 1024, 40, 20, 2, 30, 10, 10, 0,
                  "k_encdec_wgrad_generic: N C = 65 536, one past the gridDim.y limit the (L, N C) grid had"),
}

# Whole multichannel training steps (test_mc_filterbank_gpu.py, cotangent-driven, default mode): (C, shape, batch, T, reaches)
McTrain = collections.namedtuple("McTrain", "C shape batch T reaches")
_SEP = dict(sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16, sep_kernel_size=3, sep_num_blocks=1,
            sep_num_layers=2, n_sources=2)
TRAIN = {
    "C2-L4S2": McTrain(2, dict(_SEP, n_basis=32, kernel_size=4, stride=2), 2, 301,
                       "k_encoder_v4_mc<4,2> (encoder and decoder adjoint), k_decoder_mc_v<2,2>"),
    "C3-L8S4": McTrain(3, dict(_SEP, n_basis=24, kernel_size=8, stride=4), 2, 517, "k_encoder_v4_mc<8,4>, k_decoder_mc"),
    "C8-L16S8-N256": McTrain(8, dict(_SEP, n_basis=256, kernel_size=16, stride=8), 1, 1037,
                             "k_encoder_v4_mc<16,8> with the opt-in near 176 KB (encoder and adjoint)"),
    "C10-L16S8-N256": McTrain(10, dict(_SEP, n_basis=256, kernel_size=16, stride=8), 1, 1037,
                              "k_encoder_mc: shared memory > 200 KB (encoder and adjoint)"),
    "C2-N42": McTrain(2, dict(_SEP, n_basis=42, kernel_size=16, stride=8), 2, 1037, "N = 42, N % 4 != 0, through k_encoder_v4_mc<16,8>"),
    "C64-L40-N1024": McTrain(64, dict(_SEP, n_basis=1024, kernel_size=40, stride=20), 1, 600,
                             "k_encdec_wgrad_generic at N C = 65 536 (both filter banks)"),
}


# ---- selection rules ---------------------------------------------------------------------------------------------------------
ENC_FAST_L = (2, 4, 8, 16, 20)   # ctn_encoder_mc_fwd: switch (L) { ENC_MC_CASE(2) ... ENC_MC_CASE(20) }
DEC_FAST_S = (8, 1, 10, 2)       # ctn_decoder_mc_fwd: the launch_decoder_mc_v<S, 2> if-chain


def encoder_smem(C, N, L):
    """encoder_v4_mc_smem<L> (ctn_encdec.cu): C L N4 filter floats + C 32 XWP window floats"""
    xw4 = (3 * (L // 2) + L + 3) // 4 * 4
    xwp = xw4 if (xw4 // 4) % 2 else xw4 + 4
    return 4 * (C * L * ((N + 3) & ~3) + C * 32 * xwp)


def decoder_smem(N, S, R):
    """launch_decoder_mc_v (ctn_encdec.cu): N S R filter floats + (DEC_SPLIT - 1) S 128 partial sums"""
    return 4 * (N * S * R + (DEC_SPLIT - 1) * S * 128)


def encoder_kernel(r):
    """(kernel, tags) that ctn_encoder_mc_fwd launches for an Enc row (ctn_encdec.cu, ctn_encoder_mc_fwd and launch_encoder_v4_mc)"""
    if r.L != 2 * r.S:
        return "k_encoder_mc", ("L != 2 stride",)
    if enc_pitch(r) % 128:
        return "k_encoder_mc", ("w_pitch % 128",)
    if r.w_off % 4:
        return "k_encoder_mc", ("w misaligned",)
    if r.L not in ENC_FAST_L:
        return "k_encoder_mc", ("L outside the switch",)
    smem = encoder_smem(r.C, r.N, r.L)
    if smem > SMEM_MAX:
        return "k_encoder_mc", ("shared memory > 200 KB",)
    return "k_encoder_v4_mc<{},{}>".format(r.L, r.S), (("opt-in",) if smem + ENC_STATIC_SMEM > SMEM_OPT_IN else ())


def decoder_kernel(r):
    """(kernel, tags) that ctn_decoder_mc_fwd launches for a Dec row (ctn_decoder_mc_fwd and launch_decoder_mc_v)"""
    if r.R != 2:
        return "k_decoder_mc", ("R != 2",)
    if r.S not in DEC_FAST_S:
        return "k_decoder_mc", ("stride outside the list",)
    smem = decoder_smem(r.N, r.S, r.R)
    if smem > SMEM_MAX:
        return "k_decoder_mc", ("shared memory > 200 KB",)
    if r.C * ((r.frames + r.R - 1 + 127) // 128) > GRID_X_MAX:
        return "k_decoder_mc", ("C tiles > gridDim.x",)
    return "k_decoder_mc_v<{},{}>".format(r.S, r.R), (("opt-in",) if smem > SMEM_OPT_IN else ())


def wgrad_gy(R, NC):
    """ctn_encdec_wgrad: gy = ceil(4 * 148 / NC), at most R, at least 1"""
    return max(1, min(R, -(-4 * 148 // NC)))


def wg_T(r):
    return (r.frames - 1) * r.S + r.L - r.pl - r.pr


def wgrad_kernel(r):
    """(kernel, tags) of ctn_encdec_wgrad for a Wg row, with the branches of k_encdec_wgrad its frames take"""
    if r.L > ENCDEC_MAX_L:
        return "k_encdec_wgrad_generic", ()
    T, gy = wg_T(r), wgrad_gy(r.R, r.N * r.C)
    tags = ["gy = R" if gy == r.R else "gy = 1" if gy == 1 else "gy = {}".format(gy)]
    fails = [name for name, bad in (("L % 4", r.L % 4), ("stride % 4", r.S % 4), ("pad_left % 4", r.pl % 4), ("T % 4", T % 4),
                                    ("sig misaligned", r.sig_off % 4)) if bad]
    t0 = torch.arange(r.frames) * r.S - r.pl
    interior = (t0 >= 0) & (t0 + r.L <= T)
    if bool(interior.any()):
        tags.append("vector" if not fails else "scalar: " + ", ".join(fails))
    if not bool(interior.all()):
        tags.append("boundary")
    return "k_encdec_wgrad", tuple(tags)


def label(kernel, tags):
    """the head every row's `reaches` text starts with: the kernel, then each tag in brackets, then ':'"""
    return kernel + "".join(" [{}]".format(t) for t in tags) + ":"


# ---- inputs ------------------------------------------------------------------------------------------------------------------
def enc_inputs(name, r):
    """x (B, C, T) scaled per sample, W (N, C, L), both fp32 values in float64"""
    g = gen("enc" + name)
    scale = torch.tensor([SCALES[b % 3] for b in range(r.B)], dtype=torch.float64)[:, None, None]
    x = f32(torch.randn(r.B, r.C, enc_T(r), generator=g, dtype=torch.float64) * scale)
    W = f32((torch.rand(r.N, r.C, r.L, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(r.C * r.L))
    return x, W


def dec_inputs(name, r):
    g = gen("dec" + name)
    what = f32(torch.randn(r.BS, r.N, r.frames, generator=g, dtype=torch.float64))
    Wd = f32((torch.rand(r.N, r.C, r.S * r.R, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(r.S * r.R))
    return what, Wd


def wg_inputs(name, r):
    """act (R, N, frames), sig (R, C, T), base (N, C, L): dW's value on entry"""
    g = gen("wg" + name)
    act = f32(torch.randn(r.R, r.N, r.frames, generator=g, dtype=torch.float64))
    sig = f32(torch.randn(r.R, r.C, wg_T(r), generator=g, dtype=torch.float64))
    base = f32(torch.randn(r.N, r.C, r.L, generator=g, dtype=torch.float64))
    return act, sig, base


# ---- fp64 references, (value, magnitude) -----------------------------------------------------------------------------------
def _shift_tap(W):
    """tap 0's weight applied one sample later (on top of tap 1)"""
    W = W.clone()
    W[..., 1] += W[..., 0]
    W[..., 0] = 0
    return W


def _swap(W):
    """W (N, C, L) read with its channel and basis strides swapped: the memory taken as (C, N, L)"""
    N_, C_, L_ = W.shape
    return W.reshape(C_, N_, L_).transpose(0, 1)


def encoder(x, W, S, pl, pr, relu, mut=None):
    """w[b][n][f] = sum_c sum_k W[n][c][k] xpad[b][c][f S + k]; -> (w, M) with M = sum |W| |xpad| (before ReLU)"""
    if mut == "drop_channel":
        x = torch.cat([x[:, :-1], torch.zeros_like(x[:, -1:])], 1)
    if mut == "shift_tap":
        W = _shift_tap(W)
    if mut == "swap_strides":
        W = _swap(W)
    xp = torch.nn.functional.pad(x, (pl, pr))
    if mut == "read_past" and pr > 0:
        xp = xp.clone()
        xp[..., pl + x.shape[-1]] = 1.0 + xp.abs().max()  # the first right-pad sample read as data
    win = xp.unfold(2, W.shape[-1], S)  # (B, C, F, L)
    w = torch.einsum("bcfk,nck->bnf", win, W)
    mag = torch.einsum("bcfk,nck->bnf", win.abs(), W.abs())
    if relu:
        w = torch.relu(w)
    if mut == "drop_last_frame":
        w = w.clone()
        w[..., -1] = 0
    return w, mag


def encoder_bound(r, mag):
    return r.C * r.L * U * mag


def decoder(what, Wd, S, crop, T_out, mut=None):
    """y[bs][c][t] = sum_n sum_{f, k: f S + k = t + crop} what[bs][n][f] Wd[n][c][k]; -> (y, M)"""
    if mut == "drop_channel":
        what = torch.cat([what[:, :-1], torch.zeros_like(what[:, -1:])], 1)
    if mut == "shift_tap":
        Wd = _shift_tap(Wd)
    if mut == "swap_strides":
        Wd = _swap(Wd)
    if mut == "drop_last_frame":
        what = what.clone()
        what[..., -1] = 0
    if mut == "read_past":  # the column past frames read as one more frame
        what = torch.cat([what, 1.0 + what.abs().amax(-1, keepdim=True)], -1)
    BS, N_, F = what.shape
    L = Wd.shape[-1]
    full_len = (F - 1) * S + L
    out, mag = [], []
    for v, wd in ((what, Wd), (what.abs(), Wd.abs())):
        contrib = torch.einsum("bnf,nck->bcfk", v, wd)  # (BS, C, F, L): frame f's tap k lands on sample f S + k
        idx = (torch.arange(F)[:, None] * S + torch.arange(L)[None, :]).reshape(-1)
        y = torch.zeros(BS, Wd.shape[1], full_len, dtype=torch.float64).index_add_(2, idx, contrib.reshape(BS, Wd.shape[1], -1))
        out.append(y[..., crop:crop + T_out])
    return out[0], out[1]


def decoder_bound(r, kernel, mag):
    k = r.N * r.R if kernel == "k_decoder_mc" else -(-r.N // DEC_SPLIT) * r.R + DEC_SPLIT - 1
    return k * U * mag


def dec_geometry(r):
    """(crop_left, T_out)"""
    full_len = (r.frames - 1) * r.S + r.S * r.R
    return r.crop, full_len - r.crop - r.tail


def stats_bound(fast, w, n, n_cta):
    """bounds of (sum w, sum w^2) of one sample's outputs w (the kernel's own, in float64) over n bases"""
    a, q = float(w.abs().sum()), float((w * w).sum())
    dbl = (n + 8 + n_cta + 2 + 64) * DU  # + 64: the fp64 reference's own sum
    return ((18 * U if fast else 0.0) + dbl) * a, ((64 * U if fast else 0.0) + dbl) * q


def wgrad(act, sig, L, S, pl, mut=None):
    """dW[n][c][k] = sum_{r, f} act[r][n][f] sig[r][c][f S + k - pl] (0 outside [0, T)); -> (dW, M)"""
    if mut == "drop_last_frame":
        act = act.clone()
        act[..., -1] = 0
    if mut == "read_past":  # the column past frames read as one more frame
        act = torch.cat([act, 1.0 + act.abs().amax(-1, keepdim=True)], -1)
    R, N_, F = act.shape
    T = sig.shape[-1]
    idx = torch.arange(F)[:, None] * S + torch.arange(L)[None, :] - pl
    if mut == "shift_tap":
        idx = idx.clone()
        idx[:, 0] += 1
    ok = (idx >= 0) & (idx < T)
    win = sig[:, :, idx.clamp(0, T - 1)] * ok  # (R, C, F, L)
    dW = torch.einsum("rnf,rcfk->nck", act, win)
    mag = torch.einsum("rnf,rcfk->nck", act.abs(), win.abs())
    if mut == "drop_channel":
        dW = dW.clone()
        dW[:, -1] = 0
    if mut == "swap_strides":  # the (C, N, L)-ordered result stored into (N, C, L) memory
        dW = dW.transpose(0, 1).reshape(dW.shape)
    return dW, mag


def wgrad_bound(r, mag, base):
    chain = -(-r.frames // 256)
    if r.L > ENCDEC_MAX_L:
        return (chain + 2) * U * mag + U * base.abs() + (r.R + 8) * DU * mag
    gy = wgrad_gy(r.R, r.N * r.C)
    return (chain * -(-r.R // gy) + 5 + 8 + gy + 1) * U * mag + gy * U * base.abs()
