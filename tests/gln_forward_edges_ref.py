"""Rows, dispatch predicates, launch counts and fp64 references of tests/test_gln_forward_edges_gpu.py (test infrastructure only):
the non-causal (gLN), sigmoid-mask Conv-TasNet inference forward -- ctn_convtasnet_fwd, ctn_separator_fwd, ctn_tcn_fwd and
ctn_tcn_blocks_fwd -- at the shapes where run_tcn / run_separator (csrc/ctn_api.cu) change branch.

The predicates below restate the host's dispatch in plain Python, so that tests/test_gln_forward_edges_cpu.py can show without a
GPU that each row reaches the branch its `reaches` text names, and the GPU file can pin each call's launch count: a row that
silently took another branch would launch a different number of kernels.
  * depthwise stage (run_tcn): the fused producer PRO_DW runs in the tensor-core modes when P = 3 and d in {1, 2, 4k}
    (dw_fusable); otherwise ctn_dw_fwd (k_dw) + a PRO_NONE pw2, one launch more.  pad_left = (P - 1) d // 2.
  * residual update: deferred into the next block's PRO_RES producer in the tensor-core modes (the last block's only when x_out is
    asked for, one k_finish); k_finish inside the loop in fp32 for every block with an out head.
  * n-tiles of 128 output channels: pw2 of a block with an out head has M = Bc + Sc, the last block's M = Sc.
  * fused mask + decoder (k_maskdec): f16x3, N % 128 == 0, L = 16 / stride 8, Sc <= 128 (MD_MAX_K), padded S N <= 2048
    (F16_MAX_ROWS), monaural, no latent; otherwise EPI_MASK + ctn_decoder_fwd.
  * encoder crop: T pads by (stride - (T - L) % stride) % stride, pl = padding // 2 on the left; the decoder crops pl.

The fp64 references: O.conv_tasnet_fwd / O.separator_fwd / O.tdcn_fwd for the 2^l dilations, and chain() -- O.residual_block
block by block with explicit dilations -- for ctn_tcn_blocks_fwd.  model64() restates O.conv_tasnet_fwd with the mutants of the
CPU file; unmutated it equals the oracle.
"""
import collections
import math

import torch
import torch.nn.functional as F

import convtasnet_oracle as O

OUT_RTOL, OUT_ATOL = 1e-4, 2e-5      # fp32, tf32x3, f16x3 against fp64 (test_forward_edges_gpu.py's model bound)
TF32_RTOL, TF32_ATOL = 2e-2, 5e-3    # tf32
EPS = O.EPS
TILE = 128            # CTN_TILE_T: pitch granularity; also the n-tile width (NT) and the time tile of k_maskdec
MD_MAX_K = 128        # k_maskdec keeps the Sc-channel operand resident
F16_MAX_ROWS = 2048   # padded output channels of an fp16-piece contraction
MAX_JOBS = 48         # jobs per k_fold_batch / weight-image launch
MAX_BLOCKS = 64       # CTN_MAX_BLOCKS: skip-reduction and operand-scale tables
MODES = ("fp32", "tf32x3", "f16x3", "tf32")


def tol(mode):
    return (TF32_RTOL, TF32_ATOL) if mode == "tf32" else (OUT_RTOL, OUT_ATOL)


def share(y, ref, rtol, atol):
    """max |y - ref| / (atol + rtol |ref|): <= 1 passes torch.testing.assert_close(rtol, atol)"""
    return float(((y.double() - ref.double()).abs() / (atol + rtol * ref.double().abs())).max())


# ---- dispatch predicates (ctn_api.cu, ctn_wgmma.cu) -----------------------------------------------------------------------
def ceil_div(a, b):
    return -(-a // b)


def pitch(frames):
    return ceil_div(frames, TILE) * TILE


def n_tiles(M):
    return ceil_div(M, TILE)


def pad_left(P, d):
    return (P - 1) * d // 2


def dw_fusable(P, d):
    return P == 3 and (d == 1 or d == 2 or d % 4 == 0)


def frames_of(T, L, stride):
    """ctn_frames: (frames, pl, pr)"""
    padding = (stride - (T - L) % stride) % stride
    pl = padding // 2
    return (T + padding - L) // stride + 1, pl, padding - pl


def eff_math(M, mode):
    return "tf32x3" if mode == "f16x3" and n_tiles(M) * TILE > F16_MAX_ROWS else mode


def maskdec(cfg, mode, latent=False, in_channels=1):
    """run_separator takes k_maskdec (the fused mask + decoder)"""
    return (mode == "f16x3" and not latent and in_channels == 1 and cfg.mask_nonlinear == "sigmoid" and cfg.kernel_size == 16
            and cfg.stride == 8 and cfg.n_basis % TILE == 0 and cfg.sep_skip_channels <= MD_MAX_K
            and eff_math(cfg.n_sources * cfg.n_basis, mode) == "f16x3")


def default_dils(cfg):
    return [2 ** l for _ in range(cfg.sep_num_blocks) for l in range(cfg.sep_num_layers)]


# ---- launch counts ---------------------------------------------------------------------------------------------------------
def tcn_launches(Bc, H, Sc, P, dils, mode, last_out=False, x_final=False):
    """run_tcn: preparation (folds, weight images, operand scales), per block pw1 + (PRO_DW pw2 | k_dw + pw2) [+ k_finish in
    fp32], the skip reduction, and the last block's finish when x_out is asked for in a tensor-core mode"""
    n, tc = len(dils), mode != "fp32"
    outs = [True] * (n - 1) + [last_out]
    folds = sum(2 if o else 1 for o in outs)
    k = ceil_div(folds, MAX_JOBS)
    if tc:
        Ms = [H] * n + [Bc + Sc if o else Sc for o in outs]
        uniform = all(eff_math(M, mode) == mode for M in Ms)
        k += ceil_div(2 * n, MAX_JOBS) if uniform else 2 * n
    if mode == "f16x3":
        k += 2                                   # k_scale_partials, k_scale_chain
    for d, o in zip(dils, outs):
        k += 1                                   # pw1
        k += 1 if tc and dw_fusable(P, d) else 2
        k += 1 if (not tc and o) else 0          # k_finish
    k += 1                                       # k_skip_reduce
    if x_final and tc and last_out:
        k += 1
    return k


def _rows_launches(rows):
    return ceil_div(rows, 65535)


def separator_core_launches(cfg, B, mode, dils=None):
    """run_separator without the mask tail: head fold (+ head and mask weight images), head contraction, the TCN"""
    dils = dils or default_dils(cfg)
    k = 1 + (2 if mode != "fp32" else 0) + 1
    return k + tcn_launches(cfg.sep_bottleneck_channels, cfg.sep_hidden_channels, cfg.sep_skip_channels, cfg.sep_kernel_size,
                            dils, mode)


def model_launches(cfg, B, mode, latent):
    k = 1 + separator_core_launches(cfg, B, mode) + 1      # encoder, separator, mask (k_maskdec or EPI_MASK)
    if not maskdec(cfg, mode, latent):
        k += 1                                             # ctn_decoder_fwd
    if latent:
        k += _rows_launches(B * cfg.n_sources * cfg.n_basis)
    return k


def separator_launches(cfg, B, mode):
    return (_rows_launches(B * cfg.n_basis) + 1 + separator_core_launches(cfg, B, mode) + 1
            + _rows_launches(B * cfg.n_sources * cfg.n_basis))


def tcn_fwd_launches(Bc, H, Sc, P, dils, mode, B, last_out=False, x_out=False):
    """ctn_tcn_fwd / ctn_tcn_blocks_fwd: copy in, the measured x_0 bound (f16x3), the stack, copies out"""
    k = _rows_launches(B * Bc) + (1 if mode == "f16x3" else 0)
    k += tcn_launches(Bc, H, Sc, P, dils, mode, last_out, x_out)
    k += _rows_launches(B * Sc) + (_rows_launches(B * Bc) if x_out else 0)
    return k


# ---- branches --------------------------------------------------------------------------------------------------------------
BRANCHES = {
    "pro_dw": "the fused depthwise producer PRO_DW (P = 3, d in {1, 2, 4k})",
    "dw_standalone": "k_dw + a PRO_NONE pw2 (P != 3, or d not in {1, 2, 4k})",
    "res_after_fused": "PRO_RES reading a residual whose r came from a PRO_DW pw2",
    "res_after_standalone": "PRO_RES reading a residual whose r came from a PRO_NONE pw2",
    "lone_block": "one block: no out head, no PRO_RES",
    "pw2_ntiles_odd": "a pw2 with an odd n-tile count (the channel split's idle second warpgroup)",
    "pw2_ntiles_even": "a pw2 with an even n-tile count (M = 256 at paper size)",
    "even_P": "even P: pad_left rounds down, the pad is asymmetric",
    "dil_ge_frames": "a dilation >= frames: every outer tap reads padding",
    "skip_jobs_64": "64 blocks: the full skip-reduction and operand-scale tables, two k_fold_batch launches",
    "ragged_K": "Bc, H or Sc not a multiple of 32: no interior K slab",
    "tile_edge_64": "frames within one of a multiple of 64 (the channel-split kernels' frame tile)",
    "tile_edge_128": "frames within one of a multiple of 128 (pitch, k_maskdec's frame tile)",
    "maskdec": "k_maskdec (the fused mask + decoder)",
    "maskdec_short": "k_maskdec over a single frame tile with T shorter than one tile's samples",
    "maskdec_multi_ntile": "k_maskdec with three n-tiles per source",
    "maskdec_S1": "k_maskdec at S = 1",
    "maskdec_off_N": "no k_maskdec: N % 128 != 0",
    "maskdec_off_K": "no k_maskdec: Sc > 128 (EPI_MASK + k_decoder<8,2>)",
    "maskdec_off_L": "no k_maskdec: L / stride != 16 / 8 (EPI_MASK + k_decoder<10,2>)",
    "x_final": "ctn_tcn_blocks_fwd with x_out: the last block's update after the loop (tensor-core modes)",
}


def branches(cfg, frames_list, dils=None, last_out=False, x_out=False, model=True):
    """the BRANCHES a forward of cfg at these frame counts reaches (tensor-core modes for the TCN, f16x3 for the mask tail)"""
    dils = dils or default_dils(cfg)
    Bc, H, Sc, P = cfg.sep_bottleneck_channels, cfg.sep_hidden_channels, cfg.sep_skip_channels, cfg.sep_kernel_size
    n = len(dils)
    outs = [True] * (n - 1) + [last_out]
    got = set()
    fus = [dw_fusable(P, d) for d in dils]
    got |= {"pro_dw"} if any(fus) else set()
    got |= {"dw_standalone"} if not all(fus) else set()
    for i in range(1, n):
        got.add("res_after_fused" if fus[i - 1] else "res_after_standalone")
    if n == 1 and not last_out:
        got.add("lone_block")
    for o in outs:
        got.add("pw2_ntiles_odd" if n_tiles(Bc + Sc if o else Sc) % 2 else "pw2_ntiles_even")
    if P % 2 == 0:
        got.add("even_P")
    if any(d >= f for d in dils for f in frames_list):
        got.add("dil_ge_frames")
    if n == MAX_BLOCKS:
        got.add("skip_jobs_64")
    if any(c % 32 for c in (Bc, H, Sc)):
        got.add("ragged_K")
    for f in frames_list:
        if min(f % 64, 64 - f % 64) <= 1 and f > 1:
            got.add("tile_edge_64")
        if min(f % 128, 128 - f % 128) <= 1 and f > 1:
            got.add("tile_edge_128")
    if x_out and last_out:
        got.add("x_final")
    if model:
        if maskdec(cfg, "f16x3"):
            got.add("maskdec")
            if cfg.n_basis // TILE == 3:
                got.add("maskdec_multi_ntile")
            if cfg.n_sources == 1:
                got.add("maskdec_S1")
            if any(f <= TILE for f in frames_list) and any((f - 1) * cfg.stride + cfg.kernel_size < TILE * cfg.stride
                                                           for f in frames_list):
                got.add("maskdec_short")
        else:
            if cfg.n_basis % TILE:
                got.add("maskdec_off_N")
            if cfg.sep_skip_channels > MD_MAX_K:
                got.add("maskdec_off_K")
            if (cfg.kernel_size, cfg.stride) != (16, 8):
                got.add("maskdec_off_L")
    return got


# ---- rows ------------------------------------------------------------------------------------------------------------------
def cfg_of(N=128, L=16, stride=8, Bc=32, H=64, Sc=32, P=3, R=1, X=4, S=2, relu=False):
    return O.OracleConfig(n_basis=N, kernel_size=L, stride=stride, sep_bottleneck_channels=Bc, sep_hidden_channels=H,
                          sep_skip_channels=Sc, sep_kernel_size=P, sep_num_blocks=R, sep_num_layers=X, n_sources=S,
                          enc_nonlinear="relu" if relu else None, causal=False)


PAPER = dict(N=512, L=16, stride=8, Bc=128, H=512, Sc=128, P=3, R=3, X=8, S=2)
SMALL = dict(N=128, L=16, stride=8, Bc=32, H=64, Sc=32, P=3, R=1, X=4, S=2)

Row = collections.namedtuple("Row", "cfg B Ts seed inputs expect reaches")


def _row(widths, B, Ts, seed, expect, reaches, inputs="synth", **kw):
    return Row(cfg_of(**dict(widths, **kw)), B, tuple(Ts), seed, inputs, frozenset(expect), reaches)


def _T(frames, L=16, stride=8, extra=3):
    """a signal length of `frames` frames whose pad is `extra` samples (pl = extra // 2)"""
    T = (frames - 1) * stride + L - extra
    assert frames_of(T, L, stride)[0] == frames
    return T


TILE_FRAMES = (1, 63, 64, 65, 127, 128, 129, 255, 257)

ROWS = {
    "paper": _row(PAPER, 2, [32000], 701, {"pro_dw", "res_after_fused", "pw2_ntiles_even", "pw2_ntiles_odd", "maskdec"},
                  "cfg2: channel-split pw2 (M = 256, 2 n-tiles), last block M = Sc = 128 (1 n-tile), k_maskdec over 32 frame tiles"),
    "paper-short": _row(PAPER, 2, [17, 24], 702, {"maskdec", "maskdec_short", "dil_ge_frames"},
                        "2 frames: one frame tile, T_out = 17 / 24 < 128 stride samples: k_maskdec's crop (pl = 3 / 0) and its "
                        "tile seams inside one tile; every d >= 2 reads only padding"),
    "tile-edges": _row(SMALL, 2, [_T(f) for f in TILE_FRAMES], 703, {"tile_edge_64", "tile_edge_128", "maskdec", "pro_dw"},
                       "frames in {1, 63, 64, 65, 127, 128, 129, 255, 257}: the 64-frame tiles of PRO_DW / PRO_RES and the 128-frame "
                       "tiles of k_maskdec and the pitch, pl = 1"),
    "sc129": _row(SMALL, 2, [1037], 704, {"maskdec_off_K", "pw2_ntiles_even", "ragged_K"},
                  "Sc = 129 > MD_MAX_K: EPI_MASK + k_decoder<8,2>; pw2 M = Mt = Bc + Sc = 161, not a multiple of 128 (2 n-tiles, the "
                  "second 33 rows deep), last M = 129 (2 n-tiles, 1 row)",
                  Sc=129),
    "n384-s3": _row(SMALL, 2, [1037], 705, {"maskdec", "maskdec_multi_ntile"},
                    "N = 384, S = 3: k_maskdec with three n-tiles per source (S N = 1152)", N=384, S=3),
    "n200": _row(SMALL, 2, [1037], 706, {"maskdec_off_N"}, "N = 200: N % 128 != 0, EPI_MASK + k_decoder<8,2>", N=200),
    "l20": _row(SMALL, 2, [1283], 707, {"maskdec_off_L"}, "L = 20 / stride 10: no k_maskdec; EPI_MASK + k_decoder<10,2>, pl = 1",
                L=20, stride=10),
    "s1": _row(SMALL, 2, [1037], 708, {"maskdec", "maskdec_S1"}, "S = 1 (enhancement): k_maskdec with M = N", S=1),
    "ragged-widths": _row(SMALL, 2, [1037], 709, {"ragged_K", "pw2_ntiles_odd"},
                          "Bc = 33, H = 100, Sc = 24: K % 32 != 0 in every contraction, Hp = 112, pw2 M = 57 and 24 (1 n-tile)",
                          Bc=33, H=100, Sc=24),
    "deep-dilation": _row(SMALL, 2, [_T(500)], 710, {"dil_ge_frames", "pro_dw"},
                          "P = 3, X = 12 at 500 frames: d = 512 .. 2048 >= frames, every outer tap reads padding (all fused)", X=12),
    "p1": _row(SMALL, 2, [1037], 711, {"dw_standalone", "res_after_standalone"}, "P = 1: k_dw<0> + PRO_NONE pw2 in every block",
               P=1),
    "p2": _row(SMALL, 2, [1037], 712, {"dw_standalone", "res_after_standalone", "even_P"},
               "P = 2: k_dw<0>, pad_left = d // 2 (asymmetric)", P=2),
    "p4": _row(SMALL, 2, [1037], 713, {"dw_standalone", "res_after_standalone", "even_P"},
               "P = 4: k_dw<0>, pad_left = 3 d // 2", P=4),
    "p8": _row(SMALL, 2, [1037], 714, {"dw_standalone", "res_after_standalone", "even_P"},
               "P = 8: k_dw<0>, pad_left = 7 d // 2", P=8),
    "rx1": _row(SMALL, 2, [1037], 715, {"lone_block"}, "R X = 1 x 1: a lone block, no out head, no PRO_RES", R=1, X=1),
    "rx64": _row(SMALL, 2, [1037], 716, {"skip_jobs_64"}, "R X = 8 x 8 = 64 = CTN_MAX_BLOCKS: 64 skip jobs, 64 scale jobs, "
                                                          "127 fold jobs in 3 launches", R=8, X=8),
    "silence": _row(SMALL, 5, [4000], 717, {"maskdec"}, "ReLU encoder: an ordinary, an exact-zero, a silent-onset, a near-silent "
                    "(gLN0 variance ~4 eps) and a 1e4-amplitude sample in one batch; k_maskdec and k_decoder", inputs="silence",
                    relu=True),
    "b37": _row(dict(SMALL, N=64, Bc=16, H=32, Sc=16, X=3), 37, [1037], 718, {"maskdec_off_N"},
                "B = 37: each sample alone equals its row of the batch"),
    "long": _row(dict(SMALL, X=8), 1, [480000], 719, {"maskdec", "pro_dw"},
                 "60 s at 8 kHz (59999 frames): the f16x3 operand scales at the DESIGN section 2 headroom point"),
}


def frames_list(row):
    return [frames_of(T, row.cfg.kernel_size, row.cfg.stride)[0] for T in row.Ts]


# ---- inputs ----------------------------------------------------------------------------------------------------------------
NEAR_SILENT_VAR = 4.0 * EPS


def state_dict(row):
    return O.synth_state_dict(row.cfg, seed=row.seed)


def mixture(row, T, sd=None):
    """(B, 1, T) float32"""
    x, _ = O.synth_batch(row.B, row.cfg.n_sources, T, seed=row.seed + 1)
    if row.inputs != "silence":
        return x
    ref = x[0:1].double()
    # the near-silent sample: the ordinary one scaled so that its encoder output's variance (the gLN0 statistic) is a few eps
    w = O.encoder_fwd(F.pad(ref, frames_of(T, row.cfg.kernel_size, row.cfg.stride)[1:]), sd["encoder.conv1d.weight"].double(),
                      row.cfg.stride, relu=True)
    a = math.sqrt(NEAR_SILENT_VAR / float(w.var(unbiased=False)))
    out = torch.stack([x[0], torch.zeros_like(x[0]), x[1], (ref[0] * a).float(), x[2] * 1e4])
    out[2, :, : T // 2] = 0.0   # silent onset
    return out


# ---- fp64 references -------------------------------------------------------------------------------------------------------
def blocks_state_dict(n, Bc, H, Sc, P, last_out, seed):
    """(sd, prefixes) of n blocks: with last_out every block has an out head (the first n of n + 1)"""
    cfg = cfg_of(Bc=Bc, H=H, Sc=Sc, P=P, R=1, X=n + (1 if last_out else 0))
    sd = O.synth_state_dict(cfg, seed=seed)
    return sd, [f"separator.tdcn.net.0.net.{i}." for i in range(n)]


def chain(x, sd, prefixes, dils, P, last_out, eps=EPS, mut=None, mut_block=None):
    """ctn_tcn_blocks_fwd in fp64: O.residual_block per block with its own dilation -> (x after the last block, skip sum).
    mut: 'drop_last_update' (x_out without the last block's residual), 'pow2' (2^l dilations), 'drop_skip' (block mut_block's
    skip head left out of the sum)"""
    n = len(prefixes)
    skip = 0
    for i, (pf, d) in enumerate(zip(prefixes, dils)):
        if mut == "pow2":
            d = 2 ** i
        dual = i < n - 1 or last_out
        out, s = O.residual_block(x, sd, pf, kernel_size=P, dilation=d, causal=False, dual_head=dual, nonlinear=True, norm=True,
                                  eps=eps)
        if out is not None and not (mut == "drop_last_update" and i == n - 1):
            x = out
        if not (mut == "drop_skip" and i == mut_block):
            skip = skip + s
    return x, skip


def _dw_block(x, sd, pf, P, d, dual, eps, pl):
    """O.residual_block (non-causal) with the depthwise stage's left pad given: the pad mutant's block"""
    T = x.shape[-1]
    h = O.gln(O.prelu(F.conv1d(x, sd[pf + "bottleneck_conv1d.weight"], sd[pf + "bottleneck_conv1d.bias"]),
                      sd[pf + "nonlinear1d.weight"]), sd[pf + "norm1d.norm.weight"], sd[pf + "norm1d.norm.bias"], eps)
    p2 = pf + "separable_conv1d."
    h = F.pad(h, (pl, (P - 1) * d - pl))
    u = F.conv1d(h, sd[p2 + "depthwise_conv1d.weight"], sd[p2 + "depthwise_conv1d.bias"], dilation=d, groups=h.shape[1])
    assert u.shape[-1] == T
    u = O.gln(O.prelu(u, sd[p2 + "nonlinear1d.weight"]), sd[p2 + "norm1d.norm.weight"], sd[p2 + "norm1d.norm.bias"], eps)
    out = F.conv1d(u, sd[p2 + "output_pointwise_conv1d.weight"], sd[p2 + "output_pointwise_conv1d.bias"]) + x if dual else None
    return out, F.conv1d(u, sd[p2 + "skip_pointwise_conv1d.weight"], sd[p2 + "skip_pointwise_conv1d.bias"])


def _gln_eps_outside(x, gamma, beta, eps):
    """gLN with eps added to the standard deviation instead of the variance (the cLN convention, norm.py:90)"""
    B = x.shape[0]
    flat = x.reshape(B, -1)
    mean = flat.mean(1).view(B, 1, 1)
    std = flat.var(1, unbiased=False).sqrt().view(B, 1, 1)
    return (x - mean) / (std + eps) * gamma.view(1, -1, 1) + beta.view(1, -1, 1)


def model64(x, sd, cfg, mut=None, mut_block=None):
    """O.conv_tasnet_fwd (3-D input, gLN, sigmoid) restated over the blocks, with the mutants:
    'pad_up' (even P: the depthwise pad_left rounded up), 'drop_skip' (block mut_block's skip head left out), 'crop_off' (the
    decoder crop one sample right), 'eps_outside' (gLN0's eps outside the sqrt)"""
    B, _, T = x.shape
    L, S = cfg.kernel_size, cfg.stride
    _, pl, pr = frames_of(T, L, S)
    w = O.encoder_fwd(F.pad(x, (pl, pr)), sd["encoder.conv1d.weight"], S, relu=cfg.enc_nonlinear == "relu")
    g0, b0 = sd["separator.norm1d.norm.weight"], sd["separator.norm1d.norm.bias"]
    y = _gln_eps_outside(w, g0, b0, cfg.eps) if mut == "eps_outside" else O.gln(w, g0, b0, cfg.eps)
    y = F.conv1d(y, sd["separator.bottleneck_conv1d.weight"], sd["separator.bottleneck_conv1d.bias"])
    n = cfg.sep_num_blocks * cfg.sep_num_layers
    skip = 0
    for i, d in enumerate(default_dils(cfg)):
        pf = f"separator.tdcn.net.{i // cfg.sep_num_layers}.net.{i % cfg.sep_num_layers}."
        P = cfg.sep_kernel_size
        pad = pad_left(P, d) + (1 if mut == "pad_up" and ((P - 1) * d) % 2 else 0)
        out, s = _dw_block(y, sd, pf, P, d, i < n - 1, EPS, pad)
        if out is not None:
            y = out
        if not (mut == "drop_skip" and i == mut_block):
            skip = skip + s
    m = torch.sigmoid(F.conv1d(O.prelu(skip, sd["separator.prelu.weight"]), sd["separator.mask_conv1d.weight"],
                               sd["separator.mask_conv1d.bias"]))
    w_hat = w.unsqueeze(1) * m.view(B, cfg.n_sources, cfg.n_basis, -1)
    full = O.decoder_fwd(w_hat.reshape(B * cfg.n_sources, cfg.n_basis, -1), sd["decoder.conv_transpose1d.weight"], S)
    full = F.pad(full.view(B, cfg.n_sources, -1), (0, 1))
    at = pl + (1 if mut == "crop_off" else 0)
    return full[..., at:at + T], w_hat


# ---- stand-alone entries -----------------------------------------------------------------------------------------------------
# ctn_separator_fwd at the sc129 and paper-short widths (the head's row bounds come from w itself), ctn_tcn_fwd at |x| ~ 1e3 and
# 1e-3 (the x_0 bound ctn_absmax_pitch measures), ctn_tcn_blocks_fwd with explicit dilations.
SEPARATORS = {
    "sc129": (ROWS["sc129"].cfg, 2, 129, "Sc = 129 widths, 129 frames: k_stats_pitch, EPI_MASK with the mask written out"),
    "paper-short": (ROWS["paper"].cfg, 2, 3, "paper widths, 3 frames"),
}
TCN_AMPS = {"amp1e3": 1e3, "amp1e-3": 1e-3}
TCN_CFG = cfg_of(R=2, X=4)
TCN_FRAMES = 1000

BlocksRow = collections.namedtuple("BlocksRow", "dils last_out x_out Bc H Sc P B frames seed expect reaches")
MIXED_DILS = (1, 3, 2, 5, 4, 6, 7, 12)
BLOCKS = {
    "mixed": BlocksRow(MIXED_DILS, False, False, 32, 64, 32, 3, 2, 517, 801, {"pro_dw", "dw_standalone", "res_after_fused",
                                                                              "res_after_standalone"},
                       "dilations 1 3 2 5 4 6 7 12: fused (1, 2, 4, 12) and stand-alone (3, 5, 6, 7) depthwise blocks alternate, so "
                       "PRO_RES reads residuals of both kinds; the last block skip-only"),
    "mixed-xout": BlocksRow(MIXED_DILS, True, True, 32, 64, 32, 3, 2, 517, 802, {"x_final", "res_after_standalone"},
                            "the same run with an out head on the last block and x_out: its update after the loop (k_finish) in the "
                            "tensor-core modes, inside the loop in fp32"),
    "n64": BlocksRow(tuple((i % 13) + 1 for i in range(64)), False, False, 16, 48, 16, 3, 2, 300, 803,
                     {"skip_jobs_64", "dw_standalone", "pro_dw"},
                     "64 blocks = CTN_MAX_BLOCKS, dilations 1 .. 13 repeating: full skip and scale tables"),
}


def blocks_cfg(r):
    return cfg_of(Bc=r.Bc, H=r.H, Sc=r.Sc, P=r.P, R=1, X=len(r.dils))


def all_expected():
    """every row's declared branches: (id, expect, branches reached)"""
    out = []
    for k, r in ROWS.items():
        out.append((k, r.expect, branches(r.cfg, frames_list(r))))
    for k, r in BLOCKS.items():
        out.append(("blocks-" + k, r.expect, branches(blocks_cfg(r), [r.frames], list(r.dils), r.last_out, r.x_out, model=False)))
    return out
