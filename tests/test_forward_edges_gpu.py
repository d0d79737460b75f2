"""Edge shapes of the FORWARD-ONLY paths (``-m gpu``) against the CPU oracle (oracle/convtasnet_oracle.py) run in FLOAT64.

test_parity_gpu.py checks these kernels at one or two toy shapes each.  Here each runs at the shapes that select its
branches, and every row's `reaches` field names the branch and the constant that selects it:
  A. cLN (k_cln_step / k_cln_scan / k_cln_apply) at one and several frames per scan thread, with C past the 64-CTA channel
     grid and a leading run of exact-zero frames; the causal Conv-TasNet (ctn_causal.cu) through extract_latent and forward,
     its separator() and TimeDilatedConvNet past 1024 frames, and the causality of separator().
  B. The softmax mask (k_softmax_mask) over S*N channels below, at and above F16_MAX_ROWS, and with logits beyond +-100.
  C. The multichannel filter banks as modules and inside ConvTasNet(in_channels=C): the fast k_encoder_v4_mc / k_decoder_mc_v
     and the fallback k_encoder_mc / k_decoder_mc, as each row's `reaches` names.  The modules pass w_pitch = frames, so their
     encoder is fast only at a multiple of 128 frames; the model passes a 128-frame pitch.  test_mc_filterbank_gpu.py tests each
     of these kernels alone at its edges.
  D. Stand-alone gLN (k_gln_stats / k_gln_apply) past both grid-stride limits, both stand-alone norms under a DC offset, and
     the gLN statistics of stand-alone separator() (k_stats_pitch) under the same offsets.

Norm outputs start as NaN, so a cell a kernel never writes shows up.  The float64 answer and the fp32 oracle's own distance
to it are computed once per case (_CACHE).  That distance goes into failure messages and the printed summary; it is not a
bound: for long T the fp32 oracle's cumsum-based cLN is itself the inaccurate party.

Bounds:
  models, separator(), TimeDilatedConvNet: rtol 1e-4 / atol 2e-5 of fp64 ('fp32', 'tf32x3', 'f16x3'); the stated rtol 2e-2 /
    atol 5e-3 ('tf32').  The softmax masks of section B take atol x max|mask|.
  stand-alone norms: |y - y64| <= 8 u ((|x| + |mean|) rstd |gamma| + |beta|), u = 2^-24, mean / rstd in fp64 -- the forward
    error of (x - mean) * rstd * gamma + beta evaluated in fp32 from accurate statistics.  A flat bound cannot hold once a DC
    offset makes |x| >> the spread.
  filter banks: |y - y64| <= K u (|W| * |x|), K = the terms of one output (C L encoder, N L / stride decoder): the error bound
    of an fp32 dot product.
  causality: separator(w[..., :F1]) == separator(w)[..., :F1] within rtol 1e-6.
  separator() under a DC offset: the model bound (atol x max|mask|) plus the mask's response to the folded head's rounding
    budget, derived from the norm bound (see test_separator_dc_offset_vs_fp64).
"""
import collections
import ctypes as C

import pytest
import torch
import torch.nn.functional as F_

import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet
from ctn_b200.models.filterbank import Decoder, Encoder
from ctn_b200.models.tdcn import TimeDilatedConvNet
from ctn_b200.modules.norm import CumulativeLayerNorm1d, GlobalLayerNorm
from test_parity_gpu import MODES as PARITY_MODES

pytestmark = pytest.mark.gpu

MODES = PARITY_MODES + (["tf32"] if N.ctn_has_tcgen05() else [])
OUT_RTOL, OUT_ATOL = 1e-4, 2e-5
TF32_RTOL, TF32_ATOL = 2e-2, 5e-3
U, NORM_C = 2.0 ** -24, 8.0
CAUSAL_RTOL, CAUSAL_ATOL = 1e-6, 1e-7   # masks lie in [0, 1]
EPS = O.EPS

_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def _tol(mode):
    return (TF32_RTOL, TF32_ATOL) if mode == "tf32" else (OUT_RTOL, OUT_ATOL)


def _ratio(x, ref, rtol, atol):
    """max over elements of |x - ref| / (atol + rtol |ref|): <= 1 passes torch.testing.assert_close(rtol, atol)"""
    return float(((x.double() - ref.double()).abs() / (atol + rtol * ref.double().abs())).max())


def _cfg(**kw):
    base = dict(n_basis=40, kernel_size=16, sep_bottleneck_channels=24, sep_hidden_channels=48, sep_skip_channels=20,
                sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=3, n_sources=2)
    base.update(kw)
    return O.OracleConfig(**base)


def _build(cfg, sd, mode):
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, stride=cfg.stride, enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg.enc_nonlinear, sep_hidden_channels=cfg.sep_hidden_channels,
                   sep_bottleneck_channels=cfg.sep_bottleneck_channels, sep_skip_channels=cfg.sep_skip_channels,
                   sep_kernel_size=cfg.sep_kernel_size, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers,
                   mask_nonlinear=cfg.mask_nonlinear, causal=cfg.causal, n_sources=cfg.n_sources, eps=cfg.eps,
                   in_channels=cfg.in_channels)
    m.load_state_dict(sd, strict=True)
    m.math = mode
    return m.cuda().eval()


def _model_reference(key, cfg, sd, x):
    """fp64 (out, latent) of O.conv_tasnet_fwd and the fp32 oracle's distance to it, as a share of the fp32-parity bound"""
    def fn():
        sd64 = {k: v.double() for k, v in sd.items()}
        out64, lat64 = O.conv_tasnet_fwd(x.double(), sd64, cfg)
        out32, lat32 = O.conv_tasnet_fwd(x, sd, cfg)
        r32 = max(_ratio(out32, out64, OUT_RTOL, OUT_ATOL), _ratio(lat32, lat64, OUT_RTOL, OUT_ATOL))
        return out64, lat64, r32
    return _cached(("model",) + key, fn)


def _check_model(model, x, out64, lat64, r32, mode, what):
    """extract_latent (output, latent) and forward (output) against fp64; returns the worst share of the bound"""
    rtol, atol = _tol(mode)
    with torch.no_grad():
        out, latent = model.extract_latent(x.cuda())
        fwd = model(x.cuda())
    worst = 0.0
    for name, y, ref in (("extract_latent output", out, out64), ("latent", latent, lat64), ("forward output", fwd, out64)):
        y = y.cpu()
        assert y.shape == ref.shape, (what, name, tuple(y.shape), tuple(ref.shape))
        torch.testing.assert_close(y.double(), ref, rtol=rtol, atol=atol,
                                   msg=lambda m: "{} {}: {} (fp32 oracle: {:.3f} of the fp32-parity bound)".format(what, name, m, r32))
        worst = max(worst, _ratio(y, ref, rtol, atol))
    return worst


# ---- stand-alone norms ------------------------------------------------------------------------------------------------------
def _norm_inputs(B, Cc, T, seed, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cc, T, generator=g) * 0.8 + 0.3 + offset
    gamma = 1.0 + 0.2 * (torch.rand(Cc, generator=g) - 0.5)
    beta = 0.1 * (torch.rand(Cc, generator=g) - 0.5)
    return x, gamma, beta


def _run_norm(kind, x, gamma, beta):
    """ctn_gln_fwd / ctn_cln_fwd on a (B, C, T) tensor into a NaN-filled output"""
    dev = torch.device("cuda")
    B, Cc, T = x.shape
    xd, gd, bd = (t.to(dev).contiguous() for t in (x, gamma, beta))
    y = torch.full_like(xd, float("nan"))
    if kind == "gLN":
        scratch = torch.empty(2 * B, dtype=torch.float64, device=dev)
        N.check(N.ctn_gln_fwd(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), y.data_ptr(), B, Cc, T, EPS, scratch.data_ptr(),
                              N.stream_ptr(dev)), "ctn_gln_fwd")
    else:
        scratch = torch.full((2 * B * T,), float("nan"), dtype=torch.float64, device=dev)
        N.check(N.ctn_cln_fwd(xd.data_ptr(), gd.data_ptr(), bd.data_ptr(), y.data_ptr(), B, Cc, T, EPS, scratch.data_ptr(),
                              N.stream_ptr(dev)), "ctn_cln_fwd")
    return y.cpu()


def _norm_reference(key, kind, x, gamma, beta):
    """(y64, scale, fp32 oracle's worst share of the bound); scale = (|x| + |mean|) rstd |gamma| + |beta| per element"""
    def fn():
        B, Cc, T = x.shape
        x64, g64, b64 = x.double(), gamma.double(), beta.double()
        if kind == "gLN":
            y64, y32 = O.gln(x64, g64, b64, EPS), O.gln(x, gamma, beta, EPS)
            flat = x64.reshape(B, -1)
            mean = flat.mean(1).view(B, 1, 1)
            rstd = 1.0 / torch.sqrt(flat.var(1, unbiased=False).view(B, 1, 1) + EPS)
        else:
            y64, y32 = O.cln(x64, g64, b64, EPS), O.cln(x, gamma, beta, EPS)
            n = torch.arange(1, T + 1, dtype=torch.float64) * Cc
            mean = (x64.sum(1).cumsum(1) / n).unsqueeze(1)
            var = ((x64 * x64).sum(1).cumsum(1) / n).unsqueeze(1) - mean ** 2
            rstd = 1.0 / (torch.sqrt(var.clamp_min(0.0)) + EPS)
        scale = (x64.abs() + mean.abs()) * rstd * g64.abs().view(1, Cc, 1) + b64.abs().view(1, Cc, 1)
        r32 = float(((y32.double() - y64).abs() / (NORM_C * U * scale)).max())
        return y64, scale, r32
    return _cached(("norm",) + key, fn)


def _check_norm(y, y64, scale, r32, what):
    """every cell finite and within the per-element bound; returns the worst share of the bound"""
    assert torch.isfinite(y).all(), "{}: {} non-finite / unwritten cells".format(what, int((~torch.isfinite(y)).sum()))
    share = (y.double() - y64).abs() / (NORM_C * U * scale)
    worst = float(share.max())
    at = tuple(int(i) for i in torch.nonzero(share == share.max())[0])
    assert worst <= 1.0, "{}: |y - y64| = {:.3e} at {} is {:.2f}x the bound {:.3e} (fp32 oracle: {:.2f}x)".format(
        what, float((y.double() - y64).abs()[at]), at, worst, float(NORM_C * U * scale[at]), r32)
    return worst


# ---- A. cLN and the causal pipeline ------------------------------------------------------------------------------------------
def _scan_text(T):
    per = -(-T // 1024)
    busy = -(-T // per)
    return "k_cln_scan: {} frame(s) per thread, {} of 1024 threads busy".format(per, busy)


Cln = collections.namedtuple("Cln", "B C T shape4 reaches")

CLNS = {
    "T1-C1": Cln(2, 1, 1, None, "one frame, one channel: n = 1, var exactly 0, y = beta; " + _scan_text(1)),
    "T1023-C63": Cln(2, 63, 1023, None, "C=63 < 64: one k_cln_apply CTA row per channel; " + _scan_text(1023)),
    "T1024-C64": Cln(2, 64, 1024, None, "C=64: gridDim.y = C; " + _scan_text(1024)),
    "T1025-C65": Cln(3, 65, 1025, None, "C=65 > 64: the channel loop of k_cln_apply; " + _scan_text(1025)),
    "T4097-C512": Cln(2, 512, 4097, None, "C=512: 8 channels per k_cln_apply thread; " + _scan_text(4097)),
    "T100000-C65": Cln(2, 65, 100000, None, "100000 frames: " + _scan_text(100000)),
    "T100000-C1": Cln(1, 1, 100000, None, "one channel over 100000 frames: " + _scan_text(100000)),
    "4D-T1025-C64": Cln(2, 64, 1025, (25, 41), "the 4-D input (B, C, S, K) of CumulativeLayerNorm1d, S*K = 1025; " + _scan_text(1025)),
}


@pytest.mark.parametrize("case", list(CLNS))
def test_cln_vs_fp64(case):
    """Each CLNS row through ctn_cln_fwd (3-D rows, NaN-filled output) or CumulativeLayerNorm1d (4-D row): every cell finite
    and within the per-element norm bound of fp64."""
    e = CLNS[case]
    x, gamma, beta = _norm_inputs(e.B, e.C, e.T, seed=e.C * 100003 + e.T)
    y64, scale, r32 = _norm_reference(("cLN", case), "cLN", x, gamma, beta)
    if e.shape4 is None:
        y = _run_norm("cLN", x, gamma, beta)
    else:
        m = CumulativeLayerNorm1d(e.C)
        m.load_state_dict({"gamma": gamma.view(1, e.C, 1), "beta": beta.view(1, e.C, 1)})
        with torch.no_grad():
            y4 = m.cuda()(x.reshape(e.B, e.C, *e.shape4).cuda())
        assert y4.shape == (e.B, e.C) + e.shape4
        y = y4.cpu().reshape(e.B, e.C, e.T)
    worst = _check_norm(y, y64, scale, r32, case)
    print("[cLN {}] {:.3f} of bound; fp32 oracle {:.3f} -- {}".format(case, worst, r32, e.reaches))


def test_cln_leading_zero_frames():
    """A leading run of 1500 exact-zero frames (more than one scan segment): mean 0, var 0, so those frames equal beta
    bit for bit (0 * 1/eps = 0); every frame finite and the rest within the norm bound."""
    B, Cc, T, Z = 2, 64, 3000, 1500
    x, gamma, beta = _norm_inputs(B, Cc, T, seed=7)
    x[..., :Z] = 0.0
    y = _run_norm("cLN", x, gamma, beta)
    assert torch.isfinite(y).all()
    assert torch.equal(y[..., :Z], beta.view(1, Cc, 1).expand(B, Cc, Z)), "zero frames are not exactly beta"
    y64, scale, r32 = _norm_reference(("cLN", "zeros"), "cLN", x, gamma, beta)
    worst = _check_norm(y, y64, scale, r32, "zeros")
    print("[cLN zeros] {:.3f} of bound; fp32 oracle {:.3f}".format(worst, r32))


Causal = collections.namedtuple("Causal", "shape batch T frames reaches")

CAUSAL = {
    "F1-P3": Causal(dict(sep_kernel_size=3, sep_num_layers=4), 2, 16, 1,
                    "one frame: every dilated tap (d = 1 .. 8 > frames) reads padding; " + _scan_text(1)),
    "F128-P1-R2": Causal(dict(n_basis=33, sep_bottleneck_channels=16, sep_hidden_channels=40, sep_skip_channels=13, sep_kernel_size=1,
                              sep_num_blocks=2), 2, 1032, 128,
                         "128 frames = one 128-column tile; P=1: no padding; R=2: the last layer of block 1 has no output head; "
                         "N=33, Sc=13"),
    "F129-P2-relu": Causal(dict(sep_kernel_size=2, sep_num_blocks=2, enc_nonlinear="relu"), 2, 1037, 129,
                           "129 frames: one frame past a tile; ragged T (pad 1 / 2); P=2; encoder ReLU"),
    "F1999-P5": Causal(dict(sep_kernel_size=5, sep_num_blocks=2, sep_num_layers=4, n_sources=3), 2, 15995, 1999,
                       "P=5, pad_left = 4d; 3 sources; " + _scan_text(1999)),
    "F4001-P8": Causal(dict(n_basis=24, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16, sep_kernel_size=8,
                            sep_num_layers=13), 1, 32016, 4001,
                       "P=8; dilation 4096 > 4001 frames on the last layer; " + _scan_text(4001)),
    "wide": Causal(dict(n_basis=32, sep_bottleneck_channels=1040, sep_hidden_channels=1056, sep_skip_channels=24, sep_num_layers=2),
                   2, 168, 20, "Bc=1040, H=1056, Bc+Sc=1064: more rows than the 1024 CTAs of grid_cb, so the row loops of "
                               "k_bias_rows, k_dw_plain and k_res_skip_inplace run; 20 frames"),
}


def _causal_case(case):
    e = CAUSAL[case]
    cfg = _cfg(causal=True, **e.shape)
    sd = O.synth_state_dict(cfg, seed=601)
    mixture, _ = O.synth_batch(e.batch, cfg.n_sources, e.T, seed=602)
    return cfg, sd, mixture


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(CAUSAL))
def test_causal_model_vs_fp64(case, mode):
    """Each CAUSAL row through the causal ConvTasNet's extract_latent (output, latent) and forward (output) against the fp64
    oracle."""
    e = CAUSAL[case]
    cfg, sd, mixture = _causal_case(case)
    assert N.frames_of(e.T, cfg.kernel_size, cfg.stride)[0] == e.frames
    out64, lat64, r32 = _model_reference(("causal", case), cfg, sd, mixture)
    worst = _check_model(_build(cfg, sd, mode), mixture, out64, lat64, r32, mode, case)
    print("[causal {} {}] {:.3f} of bound; fp32 oracle {:.3f} -- {}".format(case, mode, worst, r32, e.reaches))


LONG = _cfg(sep_num_blocks=2, causal=True)


def _long_inputs():
    g = torch.Generator().manual_seed(611)
    w = 0.3 * torch.randn(2, LONG.n_basis, 2500, generator=g) + 0.05
    x = torch.randn(2, LONG.sep_bottleneck_channels, 3000, generator=g)
    return O.synth_state_dict(LONG, seed=612), w, x


def _separator(cfg, sd, mode):
    model = _build(cfg, sd, mode)
    model.separator.math = mode
    return model.separator


@pytest.mark.parametrize("mode", MODES)
def test_causal_separator_long_vs_fp64(mode):
    """Causal separator() (ctn_separator_fwd: the mask-out path) at 2500 frames against O.separator_fwd in fp64"""
    sd, w, _ = _long_inputs()

    def fn():
        ref = O.separator_fwd(w.double(), {k: v.double() for k, v in sd.items()}, LONG)
        return ref, _ratio(O.separator_fwd(w, sd, LONG), ref, OUT_RTOL, OUT_ATOL)
    ref, r32 = _cached(("sep", "long"), fn)
    with torch.no_grad():
        mask = _separator(LONG, sd, mode)(w.cuda()).cpu()
    rtol, atol = _tol(mode)
    torch.testing.assert_close(mask.double(), ref, rtol=rtol, atol=atol, msg=lambda m: "{} (fp32 oracle: {:.3f})".format(m, r32))
    print("[causal separator 2500 frames {}] {:.3f} of bound; fp32 oracle {:.3f} -- {}".format(
        mode, _ratio(mask, ref, rtol, atol), r32, _scan_text(2500)))


@pytest.mark.parametrize("mode", MODES)
def test_causal_tdcn_long_vs_fp64(mode):
    """Causal TimeDilatedConvNet (ctn_tcn_fwd -> ctn_causal_tcn) at 3000 frames against O.tdcn_fwd in fp64"""
    sd, _, x = _long_inputs()
    kw = dict(kernel_size=LONG.sep_kernel_size, num_blocks=LONG.sep_num_blocks, num_layers=LONG.sep_num_layers, dilated=True,
              causal=True, nonlinear=True, norm=True, eps=EPS)

    def fn():
        ref = O.tdcn_fwd(x.double(), {k: v.double() for k, v in sd.items()}, "separator.tdcn.", **kw)
        return ref, _ratio(O.tdcn_fwd(x, sd, "separator.tdcn.", **kw), ref, OUT_RTOL, OUT_ATOL)
    ref, r32 = _cached(("tdcn", "long"), fn)
    net = TimeDilatedConvNet(LONG.sep_bottleneck_channels, hidden_channels=LONG.sep_hidden_channels, skip_channels=LONG.sep_skip_channels,
                             kernel_size=LONG.sep_kernel_size, num_blocks=LONG.sep_num_blocks, num_layers=LONG.sep_num_layers,
                             dilated=True, separable=True, causal=True, nonlinear="prelu", norm=True)
    net.load_state_dict({k[len("separator.tdcn."):]: v for k, v in sd.items() if k.startswith("separator.tdcn.")}, strict=True)
    net.math = mode
    with torch.no_grad():
        y = net.cuda()(x.cuda()).cpu()
    rtol, atol = _tol(mode)
    torch.testing.assert_close(y.double(), ref, rtol=rtol, atol=atol, msg=lambda m: "{} (fp32 oracle: {:.3f})".format(m, r32))
    print("[causal tdcn 3000 frames {}] {:.3f} of bound; fp32 oracle {:.3f} -- {}".format(
        mode, _ratio(y, ref, rtol, atol), r32, _scan_text(3000)))


@pytest.mark.parametrize("mode", MODES)
def test_causal_separator_is_causal(mode):
    """separator(w[..., :F1]) == separator(w)[..., :F1] within rtol 1e-6 for F1 < F = 2500: frame t of a causal model depends
    on frames <= t only.  A scan that reaches one frame too far, or any other look-ahead, breaks it."""
    sd, w, _ = _long_inputs()
    sep = _separator(LONG, sd, mode)
    with torch.no_grad():
        full = sep(w.cuda()).cpu()
        for F1 in (1, 1023, 1024, 1025, 1999):
            part = sep(w[..., :F1].contiguous().cuda()).cpu()
            torch.testing.assert_close(part, full[..., :F1], rtol=CAUSAL_RTOL, atol=CAUSAL_ATOL,
                                       msg=lambda m: "F1={}: {}".format(F1, m))


# ---- B. softmax mask ---------------------------------------------------------------------------------------------------------
Soft = collections.namedtuple("Soft", "N S T frames causal big reaches")

SOFTS = {
    "S1-N40": Soft(40, 1, 1032, 128, False, False, "S=1: softmax over the N=40 channels of one source; 128 frames"),
    "S3-N40-causal": Soft(40, 3, 1037, 129, True, False, "N=40, not a multiple of 16: m % Nb wraps inside a 16-row group; "
                                                         "129 frames; causal"),
    "SN2048": Soft(1024, 2, 1037, 129, False, False, "S*N=2048 = F16_MAX_ROWS: the mask contraction still on fp16 pieces"),
    "SN2560": Soft(512, 5, 1032, 128, False, False, "S*N=2560 > F16_MAX_ROWS: eff_math moves the mask contraction to tf32 pieces"),
    "SN2560-causal": Soft(512, 5, 1037, 129, True, False, "S*N=2560 > F16_MAX_ROWS, causal"),
    "logits110": Soft(40, 2, 1037, 129, False, True, "mask biases +-110 on alternate groups of 7 channels: logits beyond "
                                                     "+-100, where exp overflows fp32 without the max subtraction"),
    "logits110-causal": Soft(40, 2, 1037, 129, True, True, "logits beyond +-100, causal"),
}


def _soft_case(case):
    e = SOFTS[case]
    cfg = _cfg(n_basis=e.N, n_sources=e.S, sep_bottleneck_channels=32, sep_hidden_channels=64, sep_skip_channels=32,
               causal=e.causal, mask_nonlinear="softmax")
    sd = O.synth_state_dict(cfg, seed=621)
    if e.big:
        # The logits are made large through the bias: a bias of +-110 is exact, while an fp32 dot product of magnitude 100
        # carries an absolute error near 1e-4 in any implementation, which would move the peaked probabilities by about as
        # much as the bound.  Within the +110 group the softmax keeps its ordinary spread.
        m = torch.arange(e.S * e.N)
        sd["separator.mask_conv1d.bias"] = torch.where((m // 7) % 2 == 0, 110.0, -110.0) + sd["separator.mask_conv1d.bias"]
    mixture, _ = O.synth_batch(2, e.S, e.T, seed=622)
    w = 0.3 * torch.randn(2, e.N, e.frames, generator=torch.Generator().manual_seed(623)) + 0.05
    return cfg, sd, mixture, w


def _mask_logits(w, sd, cfg):
    """the mask_conv1d output of O.separator_fwd, before the softmax"""
    x = O._norm(w, sd, "separator.norm1d.", cfg.causal, cfg.eps)
    x = F_.conv1d(x, sd["separator.bottleneck_conv1d.weight"], sd["separator.bottleneck_conv1d.bias"])
    x = O.tdcn_fwd(x, sd, "separator.tdcn.", kernel_size=cfg.sep_kernel_size, num_blocks=cfg.sep_num_blocks,
                   num_layers=cfg.sep_num_layers, dilated=True, causal=cfg.causal, nonlinear=True, norm=True, eps=EPS)
    x = O.prelu(x, sd["separator.prelu.weight"])
    return F_.conv1d(x, sd["separator.mask_conv1d.weight"], sd["separator.mask_conv1d.bias"])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(SOFTS))
def test_softmax_mask_vs_fp64(case, mode):
    """Each SOFTS row: separator() (the mask itself) and the whole model (extract_latent and forward) against fp64."""
    e = SOFTS[case]
    cfg, sd, mixture, w = _soft_case(case)
    assert N.frames_of(e.T, cfg.kernel_size, cfg.stride)[0] == e.frames

    def fn():
        sd64 = {k: v.double() for k, v in sd.items()}
        logits = _mask_logits(w.double(), sd64, cfg)
        mask64 = O.separator_fwd(w.double(), sd64, cfg)
        m32 = _ratio(O.separator_fwd(w, sd, cfg), mask64, OUT_RTOL, OUT_ATOL * float(mask64.abs().max()))
        return mask64, m32, float(logits.min()), float(logits.max())
    mask64, m32, lo, hi = _cached(("softmax", case), fn)
    if e.big:
        assert lo < -100 and hi > 100, (lo, hi)
    rtol, atol = _tol(mode)
    with torch.no_grad():
        mask = _separator(cfg, sd, mode)(w.cuda()).cpu()
    # a softmax over S*N = 2560 channels puts most of the mask near 1 / 2560: atol is taken relative to the largest entry
    matol = atol * float(mask64.abs().max())
    torch.testing.assert_close(mask.double(), mask64, rtol=rtol, atol=matol,
                               msg=lambda m: "separator(): {} (fp32 oracle: {:.3f})".format(m, m32))
    out64, lat64, r32 = _model_reference(("softmax", case), cfg, sd, mixture)
    worst = _check_model(_build(cfg, sd, mode), mixture, out64, lat64, r32, mode, case)
    print("[softmax {} {}] mask {:.3f}, model {:.3f} of bound; fp32 oracle {:.3f} / {:.3f}; logits in [{:.1f}, {:.1f}] -- {}".format(
        case, mode, _ratio(mask, mask64, rtol, matol), worst, m32, r32, lo, hi, e.reaches))


# ---- C. multichannel filter banks --------------------------------------------------------------------------------------------
McMod = collections.namedtuple("McMod", "C L S T relu reaches")

MC_MODULES = {
    "C2-L2S1": McMod(2, 2, 1, 300, False, "k_encoder_mc (w_pitch = 299), k_decoder_mc_v<1,2>: L=2, stride 1: 299 frames"),
    "C3-L16S8-relu": McMod(3, 16, 8, 1037, True, "k_encoder_v4_mc<16,8>, k_decoder_mc_v<8,2>: ragged T: the module drops a 5-sample tail; ReLU encoder; 128 frames"),
    "C8-L20S10": McMod(8, 20, 10, 1290, False, "k_encoder_v4_mc<20,10>, k_decoder_mc_v<10,2>: L=20, stride 10; 128 frames"),
    "C64-L40S20": McMod(64, 40, 20, 2620, False, "k_encoder_mc, k_decoder_mc: C=64, the largest in_channels; L=40, stride 20; 130 frames"),
    "C3-L16S16": McMod(3, 16, 16, 2064, False, "k_encoder_mc, k_decoder_mc: stride = L: no overlap in the decoder; 129 frames"),
    "C8-L16S4-T=L": McMod(8, 16, 4, 16, False, "k_encoder_mc, k_decoder_mc: T = L: one frame; the decoder's f_lo / f_hi clamps at both ends"),
    "C2-L16S4": McMod(2, 16, 4, 532, False, "k_encoder_mc, k_decoder_mc: L / stride = 4 frames per output sample; 130 frames"),
}
MC_N = 40


@pytest.mark.parametrize("case", list(MC_MODULES))
def test_multichannel_filterbank_modules_vs_fp64(case):
    """Encoder(C, N) and Decoder(N, C) (ctn_encoder_mc_fwd / ctn_decoder_mc_fwd) within the fp32 dot-product bound of fp64
    conv1d / conv_transpose1d; the decoder is fed the fp64 encoder output rounded to fp32."""
    e = MC_MODULES[case]
    g = torch.Generator().manual_seed(631 + e.C * 100 + e.L)
    x = 0.5 * torch.randn(2, e.C, e.T, generator=g)
    We = (torch.rand(MC_N, e.C, e.L, generator=g) * 2 - 1) / (e.C * e.L) ** 0.5
    Wd = (torch.rand(MC_N, e.C, e.L, generator=g) * 2 - 1) / e.L ** 0.5
    enc = Encoder(e.C, MC_N, kernel_size=e.L, stride=e.S, nonlinear="relu" if e.relu else None)
    dec = Decoder(MC_N, e.C, kernel_size=e.L, stride=e.S)
    enc.load_state_dict({"conv1d.weight": We})
    dec.load_state_dict({"conv_transpose1d.weight": Wd})
    frames = (e.T - e.L) // e.S + 1
    Tu = (frames - 1) * e.S + e.L
    x64 = x[..., :Tu].double()
    w64 = F_.conv1d(x64, We.double(), stride=e.S)
    w_bound = e.C * e.L * U * F_.conv1d(x64.abs(), We.double().abs(), stride=e.S)
    if e.relu:
        w64 = torch.relu(w64)
    wq = w64.float()
    y64 = F_.conv_transpose1d(wq.double(), Wd.double(), stride=e.S)
    y_bound = MC_N * (e.L // e.S) * U * F_.conv_transpose1d(wq.double().abs(), Wd.double().abs(), stride=e.S)
    with torch.no_grad():
        w = enc.cuda()(x.cuda()).cpu()
        y = dec.cuda()(wq.cuda()).cpu()
    assert w.shape == (2, MC_N, frames) and y.shape == (2, e.C, Tu)
    worst = []
    for name, v, ref, bound in (("encoder", w, w64, w_bound), ("decoder", y, y64, y_bound)):
        err = (v.double() - ref).abs()
        share = float((err / bound.clamp_min(1e-300)).max())
        assert bool((err <= bound).all()), "{} {}: {:.2f}x the dot-product bound (max |err| {:.3e})".format(case, name, share, float(err.max()))
        worst.append(share)
    print("[filterbank {}] encoder {:.3f}, decoder {:.3f} of bound -- {}".format(case, worst[0], worst[1], e.reaches))


McModel = collections.namedtuple("McModel", "C L S T frames causal relu reaches")

MC_MODELS = {
    "C2-L2S1": McModel(2, 2, 1, 300, 299, False, False, "k_encoder_v4_mc<2,1>, k_decoder_mc_v<1,2>: L=2, stride 1: no padding"),
    "C3-L20S10-ragged": McModel(3, 20, 10, 1283, 128, False, False, "k_encoder_v4_mc<20,10>, k_decoder_mc_v<10,2>: pad 3 / 4: decoder crop_left = 3; 128 frames"),
    "C8-L16S4": McModel(8, 16, 4, 526, 129, False, False, "k_encoder_mc, k_decoder_mc: L / stride = 4, pad 1 / 1; 129 frames"),
    "C64-L40S20": McModel(64, 40, 20, 415, 20, False, False, "k_encoder_mc, k_decoder_mc: C=64, L=40, stride 20, pad 2 / 3"),
    "C3-L16S16-T=L": McModel(3, 16, 16, 16, 1, False, False, "k_encoder_mc, k_decoder_mc: stride = L and T = L: one frame, no padding"),
    "C8-L16S8-relu": McModel(8, 16, 8, 1037, 129, False, True, "k_encoder_v4_mc<16,8> past the 48 KB opt-in (64 KB), k_decoder_mc_v<8,2>: ReLU encoder and its gLN statistics; pad 1 / 2"),
    "C2-causal": McModel(2, 16, 8, 1037, 129, True, False, "k_encoder_v4_mc<16,8>, k_decoder_mc_v<8,2>: causal: the cLN pipeline between multichannel filter banks"),
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(MC_MODELS))
def test_multichannel_model_vs_fp64(case, mode):
    """ConvTasNet(in_channels=C) through the 4-D input (B, 1, C, T): output (B, S, C, T) and latent against fp64."""
    e = MC_MODELS[case]
    cfg = _cfg(kernel_size=e.L, stride=e.S, sep_skip_channels=16, in_channels=e.C, causal=e.causal,
               enc_nonlinear="relu" if e.relu else None)
    assert N.frames_of(e.T, e.L, e.S)[0] == e.frames
    sd = O.synth_state_dict(cfg, seed=641)
    x = 0.1 * torch.randn(2, 1, e.C, e.T, generator=torch.Generator().manual_seed(642 + e.C))
    out64, lat64, r32 = _model_reference(("mc", case), cfg, sd, x)
    worst = _check_model(_build(cfg, sd, mode), x, out64, lat64, r32, mode, case)
    print("[multichannel {} {}] {:.3f} of bound; fp32 oracle {:.3f} -- {}".format(case, mode, worst, r32, e.reaches))


def test_in_channels_65_raises_without_launching():
    """in_channels = 65 is outside the multichannel kernels: the modules refuse to build and the C entry points return
    CTN_EINVAL, and no kernel launches."""
    cfg = _cfg(in_channels=2)
    model = _build(cfg, O.synth_state_dict(cfg, seed=651), "fp32")
    dev = model.encoder.conv1d.weight.device
    n0 = N.ctn_total_launch_count()
    with pytest.raises(NotImplementedError):
        ConvTasNet(40, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, in_channels=65)
    with pytest.raises(NotImplementedError):
        Encoder(65, 40, kernel_size=16, stride=8)
    with pytest.raises(NotImplementedError):
        Decoder(40, 65, kernel_size=16, stride=8)
    ncfg = model.native_config()
    ncfg.in_channels = 65
    params, keep = model.native_params(dev)
    need = C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(ncfg), 2, 1037, C.byref(need)) == N.CTN_EINVAL
    x = torch.zeros(2, 65, 1037, device=dev)
    out = torch.zeros(2, 2, 65, 1037, device=dev)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=dev)
    base = (ws.data_ptr() + 255) & ~255
    assert N.ctn_convtasnet_fwd(C.byref(ncfg), C.byref(params), x.data_ptr(), 2, 1037, out.data_ptr(), None, base,
                                ws.numel() - 256, N.stream_ptr(dev)) == N.CTN_EINVAL
    assert N.ctn_total_launch_count() == n0


# ---- D. stand-alone gLN and DC offsets ---------------------------------------------------------------------------------------
Gln = collections.namedtuple("Gln", "B C T shape4 reaches")

GLNS = {
    "per608000": Gln(2, 64, 9500, None, "per-sample size 608000 > 296 x 2048: the chunk loop of k_gln_stats"),
    "T16385-C3": Gln(2, 3, 16385, None, "T=16385 > 64 x 256: the time loop of k_gln_apply"),
    "T100000-C1": Gln(1, 1, 100000, None, "one channel, T=100000: both loops"),
    "4D-C24": Gln(2, 24, 1230, (30, 41), "the 4-D input (B, C, S, K) of GlobalLayerNorm"),
}


@pytest.mark.parametrize("case", list(GLNS))
def test_gln_vs_fp64(case):
    """Each GLNS row through ctn_gln_fwd (NaN-filled output) or GlobalLayerNorm (4-D row) within the per-element norm bound"""
    e = GLNS[case]
    x, gamma, beta = _norm_inputs(e.B, e.C, e.T, seed=e.C * 100019 + e.T)
    y64, scale, r32 = _norm_reference(("gLN", case), "gLN", x, gamma, beta)
    if e.shape4 is None:
        y = _run_norm("gLN", x, gamma, beta)
    else:
        m = GlobalLayerNorm(e.C)
        m.load_state_dict({"norm.weight": gamma, "norm.bias": beta})
        with torch.no_grad():
            y4 = m.cuda()(x.reshape(e.B, e.C, *e.shape4).cuda())
        assert y4.shape == (e.B, e.C) + e.shape4
        y = y4.cpu().reshape(e.B, e.C, e.T)
    worst = _check_norm(y, y64, scale, r32, case)
    print("[gLN {}] {:.3f} of bound; fp32 oracle {:.3f} -- {}".format(case, worst, r32, e.reaches))


OFFSETS = (0.0, 1e1, 1e2, 1e3, 1e4)


@pytest.mark.parametrize("offset", OFFSETS)
@pytest.mark.parametrize("kind", ["gLN", "cLN"])
def test_norm_dc_offset_vs_fp64(kind, offset):
    """x = offset + N(0.3, 0.8^2), C=24, T=1301 (cLN: two frames per scan thread): within the per-element bound, which grows with
    |x| + |mean|, while the statistics have to resolve a variance offset^2 / 0.64 times smaller than E[x^2]."""
    x, gamma, beta = _norm_inputs(2, 24, 1301, seed=661, offset=offset)
    y64, scale, r32 = _norm_reference((kind, "offset", offset), kind, x, gamma, beta)
    y = _run_norm(kind, x, gamma, beta)
    worst = _check_norm(y, y64, scale, r32, "{} offset {:g}".format(kind, offset))
    print("[{} offset {:g}] {:.3f} of bound; fp32 oracle {:.3f}".format(kind, offset, worst, r32))


# Stand-alone non-causal separator() takes its gLN statistics from k_stats_pitch over the caller's w, and folds the gLN into the
# bottleneck 1x1: x0 = rstd (W gamma) w - rstd mean (W gamma) 1 + W beta + b.  That contraction sums the raw w, so even with exact
# statistics x0 carries fp32 rounding of order u (|w| + |mean|) rstd per term.  The bound adds to the model bound the change of
# the fp64 mask when x0 moves by that much in every element, with random signs:
#   e_x0 = 8 u max((|w| + |mean|) rstd) max_m sum_n |W[m, n] gamma_n|      (8 u (|x| + |mean|) rstd: the norm bound above)
# Statistics whose error exceeds the norm bound move the whole of x0 coherently and land outside it.  'tf32' is left out: one
# 10-bit-mantissa pass over an un-normalised w at offset / std ~ 1e4 has no meaningful error bound.
SepOff = collections.namedtuple("SepOff", "N frames reaches")

SEP_OFFSETS = {
    "N24": SepOff(24, 1301, "24 k_stats_pitch CTAs, one channel each, ~5 frames per thread"),
    "N512": SepOff(512, 2000, "64 k_stats_pitch CTAs, 8 channels each, ~8 frames per thread and channel"),
}
OFFSET_MODES = [m for m in MODES if m != "tf32"]


def _mask_from_head(x0, sd, cfg):
    """the rest of O.separator_fwd from the bottleneck output x0"""
    x = O.tdcn_fwd(x0, sd, "separator.tdcn.", kernel_size=cfg.sep_kernel_size, num_blocks=cfg.sep_num_blocks,
                   num_layers=cfg.sep_num_layers, dilated=True, causal=False, nonlinear=True, norm=True, eps=EPS)
    x = O.prelu(x, sd["separator.prelu.weight"])
    x = torch.sigmoid(F_.conv1d(x, sd["separator.mask_conv1d.weight"], sd["separator.mask_conv1d.bias"]))
    return x.view(x0.shape[0], cfg.n_sources, cfg.n_basis, x0.shape[-1])


@pytest.mark.parametrize("mode", OFFSET_MODES)
@pytest.mark.parametrize("offset", OFFSETS)
@pytest.mark.parametrize("case", list(SEP_OFFSETS))
def test_separator_dc_offset_vs_fp64(case, offset, mode):
    """Non-causal separator() on w = offset + N(0.3, 0.8^2): the mask within rtol 1e-4 / atol 2e-5 x max|mask| of fp64 plus the
    mask's response to the head's rounding budget e_x0 (see above)."""
    e = SEP_OFFSETS[case]
    cfg = _cfg(n_basis=e.N)
    sd = O.synth_state_dict(cfg, seed=671)
    w, _, _ = _norm_inputs(2, e.N, e.frames, seed=672 + e.N, offset=offset)

    def fn():
        sd64 = O.synth_state_dict(cfg, seed=671, dtype=torch.float64)
        w64 = w.double()
        g, b = sd64["separator.norm1d.norm.weight"], sd64["separator.norm1d.norm.bias"]
        Wb = sd64["separator.bottleneck_conv1d.weight"]
        x0 = F_.conv1d(O.gln(w64, g, b, EPS), Wb, sd64["separator.bottleneck_conv1d.bias"])
        mask64 = _mask_from_head(x0, sd64, cfg)
        flat = w64.reshape(2, -1)
        mean = flat.mean(1).view(2, 1, 1)
        rstd = 1.0 / torch.sqrt(flat.var(1, unbiased=False).view(2, 1, 1) + EPS)
        e_x0 = NORM_C * U * float(((w64.abs() + mean.abs()) * rstd).max()) * float((Wb[:, :, 0].abs() * g.abs()).sum(1).max())
        signs = torch.randint(0, 2, x0.shape, generator=torch.Generator().manual_seed(673), dtype=torch.int64).double() * 2 - 1
        slack = float((_mask_from_head(x0 + e_x0 * signs, sd64, cfg) - mask64).abs().max())
        m32 = O.separator_fwd(w, sd, cfg)
        tol = OUT_ATOL * float(mask64.abs().max()) + OUT_RTOL * mask64.abs() + slack
        return mask64, e_x0, slack, float(((m32.double() - mask64).abs() / tol).max())
    mask64, e_x0, slack, r32 = _cached(("sep-offset", case, offset), fn)
    with torch.no_grad():
        mask = _separator(cfg, sd, mode)(w.cuda()).cpu().double()
    tol = OUT_ATOL * float(mask64.abs().max()) + OUT_RTOL * mask64.abs() + slack
    share = (mask - mask64).abs() / tol
    worst = float(share.max())
    assert worst <= 1.0, "{} offset {:g} {}: max |mask - mask64| {:.3e} is {:.2f}x the bound (head budget e_x0 {:.2e} -> slack {:.2e}; " \
                         "fp32 oracle {:.2f}x)".format(case, offset, mode, float((mask - mask64).abs().max()), worst, e_x0, slack, r32)
    print("[separator offset {} {:g} {}] {:.3f} of bound (slack {:.2e}); fp32 oracle {:.3f} -- {}".format(
        case, offset, mode, worst, slack, r32, e.reaches))
