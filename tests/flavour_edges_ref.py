"""Rows, inputs and fp64 references of tests/test_train_flavour_edges_gpu.py (test infrastructure only): the softmax-mask and
multichannel training steps at the gLN step's edge geometries (test_train_edges_gpu.EDGES), batches of every non-causal flavour
with silent samples in them, and an fp64 restatement of the tail of the backward (mask backward -> encoder adjoint -> crop) that
tests/test_train_flavour_edges_cpu.py applies its mutants to.

Filter banks by geometry (ctn_encdec.cu): L = 16 / stride 8 runs k_decoder<8,2> (monaural) and k_encoder_v4_mc<16,8> /
k_decoder_mc_v<8,2> (C > 1); L = 20 / stride 10 k_decoder<10,2>; every other geometry of EDGES the generic decoders
(k_decoder_generic, k_decoder_mc) and, for C > 1 with L != 2 stride or L > 20, k_encoder_mc.  The mixture gradient d_x of the
softmax step is one ctn_decoder_fwd over the encoder weight, cropped by the encoder's left pad, so it runs through the same
decoder kernel as the estimate of its row.  fused_tcn (ctn_train.cu) is !causal && f16x3 && P == 3: every row with P != 3 runs
the un-fused f16x3 step.
"""
import collections

import torch
import torch.nn.functional as F

import causal_train_ref as CR
import convtasnet_oracle as O
import pit_variants_oracle as PV
from ctn_b200.criterion.distance import MeanSquaredError
from test_train_edges_gpu import EDGES

Row = collections.namedtuple("Row", "shape C batch T frames reaches")

SOFTMAX_REACHES = {
    "E1": "L=40 / stride 20: d_x and the estimate through k_decoder_generic, pads 0 / 0; P=4: un-fused f16x3 with the logits "
          "contraction, ctn_softmax_mask and k_softmax_mask_bwd",
    "E2": "L=64 / stride 32: d_x through k_decoder_generic with pads 4 / 4 (T=3000); P=8 = CTN_MAX_P, un-fused",
    "E4": "one frame: the softmax over the S*N=64 channels of a single frame; d_x over 16 samples through k_decoder<8,2>; P=3 fused",
    "E5": "encoder ReLU: d_x takes relu'(0) = 0 from k_dw_combine; 128 frames; P=2 un-fused",
    "E6": "B=5, 33 frames: L=8 / stride 4, d_x through k_decoder_generic; weight-gradient chunks cross samples; P=6 un-fused",
    "E7": "L=20 / stride 10: d_x through k_decoder<10,2> with pads 4 / 5 (T=1001); P=7 un-fused",
    "E8": "stride = L = 4: d_x through k_decoder_generic without overlap, pads 1 / 2 (T=301); P=1 un-fused",
    "E9": "S*N=2560 > F16_MAX_ROWS: the logits contraction on tf32 pieces in f16x3, no fused mask+decoder, SinkPIT over 5 outputs; "
          "P=3 fused",
}
SOFTMAX = {k: Row(EDGES[k].shape, 1, EDGES[k].batch, EDGES[k].T, EDGES[k].frames, r) for k, r in SOFTMAX_REACHES.items()}

MC_REACHES = {
    "E1": "C=2, L=40 / stride 20: k_encoder_mc, k_decoder_mc, k_encdec_wgrad_generic over 2 channels; P=4 un-fused",
    "E2": "C=2, L=64 / stride 32: k_encoder_mc, k_decoder_mc, pads 4 / 4; P=8 un-fused",
    "E5": "C=2, L=16 / stride 8: k_encoder_v4_mc<16,8> / k_decoder_mc_v<8,2>; encoder ReLU; 128 frames; P=2 un-fused",
    "E6": "C=2, B=5, 33 frames: k_encoder_v4_mc<8,4> and k_decoder_mc; P=6 un-fused",
    "E8": "C=2, stride = L = 4: k_encoder_mc and k_decoder_mc without overlap, pads 1 / 2; P=1 un-fused",
}
MULTICHANNEL = {k: Row(EDGES[k].shape, 2, EDGES[k].batch, EDGES[k].T, EDGES[k].frames, r) for k, r in MC_REACHES.items()}
MULTICHANNEL["M9"] = Row(dict(EDGES["E9"].shape, sep_kernel_size=4), 2, 2, 4000, 499,
                         "C=2, S*N=2560 > F16_MAX_ROWS: the mask contraction on tf32 pieces in f16x3, no fused mask+decoder; P=4 un-fused")

# PReLU is not differentiable at 0: an input within rounding of 0 takes a different slope in fp32 and fp64 and moves the
# gradients upstream by up to ~1e-2 of their role scale, which no fp32 implementation can match (test_train_edges_gpu.py's
# _assert_well_conditioned).  The softmax rows take the weights of seed 611 and the inputs of 612 (test_softmax_train_gpu.py's)
# except where that puts the fp32 oracle's criterion-driven gradients too far from fp64: E2 (a PReLU input of the output PReLU
# at 1.95e-4 of its role scale) and E9 (7.1e-5 for the encoder weight; 613 puts the output PReLU's slope at 3.8e-5) take
# the inputs of the seeds below.
SOFTMAX_INPUT_SEED = {"E2": 613, "E9": 614}


def softmax_setup(case):
    """(cfg, sd, mixture, sources, G) of a softmax row: 3-speaker targets for two outputs, else one target per output"""
    e = SOFTMAX[case]
    cfg = O.OracleConfig(causal=False, mask_nonlinear="softmax", **e.shape)
    sd = O.synth_state_dict(cfg, seed=611)
    g = torch.Generator().manual_seed(SOFTMAX_INPUT_SEED.get(case, 612))
    sources = 0.3 * torch.randn(e.batch, 3 if cfg.n_sources == 2 else cfg.n_sources, e.T, generator=g)
    mixture = sources.sum(dim=1, keepdim=True)
    G = torch.randn(e.batch, cfg.n_sources, e.T, generator=g)
    return cfg, sd, mixture, sources, G


# The multichannel rows take test_multichannel_train_gpu.py's seeds (weights 511, inputs 512) except M9, where inputs 512 put an
# input of the last block's PReLU1 at -9.5e-8, 4.7e-8 of that tensor's largest entry: fp32 and fp64 round it to the same side, so
# the fp32 oracle looks well conditioned, but the tensor-core modes' h_pre can land on the other side of the kink and move every
# gradient upstream of that block by up to 1.1e-2 of its role scale.  PRELU_MARGIN below keeps every row clear of that.
MC_INPUT_SEED = {"M9": 514}


def mc_setup(case):
    """(cfg, sd, mixture (B, 1, C, T), sources (B, S, C, T), G) of a multichannel row"""
    e = MULTICHANNEL[case]
    cfg = O.OracleConfig(causal=False, in_channels=e.C, **e.shape)
    sd = O.synth_state_dict(cfg, seed=511)
    g = torch.Generator().manual_seed(MC_INPUT_SEED.get(case, 512))
    mixture = 0.3 * torch.randn(e.batch, 1, cfg.in_channels, e.T, generator=g)
    sources = 0.1 * torch.randn(e.batch, cfg.n_sources, cfg.in_channels, e.T, generator=g)
    G = torch.randn(e.batch, cfg.n_sources, cfg.in_channels, e.T, generator=g)
    return cfg, sd, mixture, sources, G


# ---- silent batches ---------------------------------------------------------------------------------------------------------
SILENT_SHAPE = dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=48, sep_skip_channels=16,
                    sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=4, n_sources=2)
SILENT_T, SILENT_FRAMES = 16000, 1999
SILENT_ZERO, SILENT_FADE = 10000, 500
ORDINARY, ZERO, ONSET, NEAR = 0, 1, 2, 3  # the samples of a silent batch
NEAR_SCALE = 5e-5  # the near-silent sample's sources, relative to an ordinary one's: var(w) of gLN0 within 1 .. 100 x eps
SILENT_REACHES = ("sample 1 exact zeros: gLN0 variance 0, rstd = 1/sqrt(eps) = 1e6; sample 2 {} zeros and a {}-sample fade-in "
                  "(frames of w exactly 0); sample 3 near-silent, var(w) within 1 .. 100 x eps of gLN0").format(SILENT_ZERO, SILENT_FADE)
FLAVOURS = ("gln", "softmax", "mc")
MSE = MeanSquaredError(dim=-1, reduction="mean")


# inputs of seed 712, except where the fp32 oracle lands too far from fp64 at a PReLU kink (see SOFTMAX_INPUT_SEED): with the
# encoder ReLU and ORPIT, 712 puts the softmax batch's output PReLU slope at 5.8e-5 of its role scale
SILENT_INPUT_SEED = {("softmax", True): 713}


def silent_batch(flavour, relu):
    """(cfg, sd, mixture, sources, G) of the silent batch of a flavour: 'gln' (sigmoid mask), 'softmax' (3-speaker targets for
    ORPIT over two outputs) or 'mc' (C = 2, sigmoid)"""
    cfg = O.OracleConfig(causal=False, mask_nonlinear="softmax" if flavour == "softmax" else "sigmoid",
                         in_channels=2 if flavour == "mc" else 1, enc_nonlinear="relu" if relu else None, **SILENT_SHAPE)
    sd = O.synth_state_dict(cfg, seed=711)
    g = torch.Generator().manual_seed(SILENT_INPUT_SEED.get((flavour, relu), 712))
    n_tgt = 3 if flavour == "softmax" else cfg.n_sources
    sources = 0.1 * torch.randn(4, n_tgt, cfg.in_channels, SILENT_T, generator=g)
    sources[ZERO] = 0
    CR.silent_onset_(sources[ONSET], SILENT_ZERO, SILENT_FADE)
    sources[NEAR] *= NEAR_SCALE
    mixture = sources.sum(dim=1, keepdim=True)
    G = torch.randn(4, cfg.n_sources, cfg.in_channels, SILENT_T, generator=g)
    if cfg.in_channels == 1:
        return cfg, sd, mixture[:, :, 0], sources[:, :, 0], G[:, :, 0]
    return cfg, sd, mixture, sources, G


def encoder_pre(cfg, sd, mixture, dtype=torch.float64):
    """the encoder output before its ReLU, and the pads (pl, pr)"""
    x = mixture.to(dtype)
    x = x.reshape(x.shape[0], -1, x.shape[-1])
    K, S = cfg.kernel_size, cfg.stride
    pad = (S - (x.shape[-1] - K) % S) % S
    pl, pr = pad // 2, pad - pad // 2
    return F.conv1d(F.pad(x, (pl, pr)), sd["encoder.conv1d.weight"].to(dtype), stride=S), pl, pr


def gln0_var_over_eps(cfg, sd, mixture):
    """per sample: the variance gLN0 sees (biased, over all N x frames of relu?(w)) divided by its eps"""
    w, _, _ = encoder_pre(cfg, sd, mixture)
    if cfg.enc_nonlinear == "relu":
        w = torch.relu(w)
    return w.var(dim=(1, 2), unbiased=False) / cfg.eps


# ---- distance of the PReLU inputs from the kink -------------------------------------------------------------------------------
# A PReLU input within a kernel's rounding of 0 can take the other slope on the GPU.  _assert_well_conditioned only sees such an
# input when fp32 and fp64 round it to different sides; this margin sees it whatever the rounding.  Every PReLU input of an edge
# row (SOFTMAX, MULTICHANNEL) must sit at least PRELU_MARGIN of its tensor's largest |entry| away from 0 (a few fp32 ulps of it).
PRELU_MARGIN = 3e-7


def prelu_margins(cfg, sd, mixture):
    """[(min |x| / max |x|, call index)] over the PReLU calls of the fp64 oracle forward, in call order"""
    seen = []
    plain = O.prelu

    def record(x, a):
        v = x.detach().abs()
        seen.append((float(v.min() / v.max()), len(seen)))
        return plain(x, a)

    orig = O.prelu
    O.prelu = record
    try:
        with torch.no_grad():
            O.conv_tasnet_fwd(mixture.double(), {k: v.double() for k, v in sd.items()}, cfg)
    finally:
        O.prelu = orig
    return seen


# ---- the oracle with the criteria of every flavour ---------------------------------------------------------------------------
def crit_oracle(cfg, out, target):
    """the recipes' criteria on the oracle: (loss, permutation or None).  C > 1: MeanSquaredError; softmax: ORPIT over two
    outputs, Sinkhorn PIT otherwise (the permutation as argmax of its soft pattern); sigmoid: PIT(NegSISDR)"""
    if cfg.in_channels > 1:
        return MSE(out, target), None
    if cfg.mask_nonlinear == "softmax":
        if cfg.n_sources == 2:
            return PV.orpit(out, target)
        loss, P = PV.sinkpit(out, target)
        return loss, torch.argmax(P, dim=2)
    return O.pit_neg_sisdr(out, target, batch_mean=True)


def forward_kept(x, sdv, cfg, mask_grad_from=None):
    """O.conv_tasnet_fwd with the encoder output before and after its ReLU and the mask kept (retain_grad).  mask_grad_from: a
    sample index whose mask gradient is d_what instead of d_what * w (the forward is unchanged) -- a defect for the mutants"""
    B, T = x.shape[0], x.shape[-1]
    xr = x.reshape(B, -1, T)
    K, S = cfg.kernel_size, cfg.stride
    pad = (S - (T - K) % S) % S
    pl, pr = pad // 2, pad - pad // 2
    w_pre = F.conv1d(F.pad(xr, (pl, pr)), sdv["encoder.conv1d.weight"], stride=S)
    w = torch.relu(w_pre) if cfg.enc_nonlinear == "relu" else w_pre
    mask = O.separator_fwd(w, sdv, cfg)
    w_hat = w.unsqueeze(1) * mask
    if mask_grad_from is not None:
        k = torch.zeros_like(w_hat)
        k[mask_grad_from] = 1
        w_hat = w_hat + k * (mask - mask.detach())
    for t in (w_pre, w, mask, w_hat):
        if t.requires_grad:
            t.retain_grad()
    x_hat = O.decoder_fwd(w_hat.reshape(B * cfg.n_sources, cfg.n_basis, -1), sdv["decoder.conv_transpose1d.weight"], S)
    x_hat = x_hat.view(B, cfg.n_sources, -1) if x.dim() == 3 else x_hat.view(B, cfg.n_sources, xr.shape[1], -1)
    out = F.pad(x_hat, (-pl, -pr))
    return out, dict(w_pre=w_pre, w=w, mask=mask, w_hat=w_hat, pl=pl, pr=pr)


def oracle(cfg, sd, mixture, drive, dtype, x_grad=False, mask_grad_from=None):
    """oracle forward + backward in `dtype`: drive = a cotangent, or (targets,) for crit_oracle.  Returns
    (out, frames, {key: grad}, d_x or None, permutation or None, kept tensors of forward_kept with their .grad)"""
    sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    x = mixture.to(dtype).clone().requires_grad_(x_grad)
    out, kept = forward_kept(x, sdv, cfg, mask_grad_from)
    perm = None
    if isinstance(drive, tuple):
        loss, perm = crit_oracle(cfg, out, drive[0].to(dtype))
        loss.backward()
    else:
        out.backward(drive.to(dtype))
    return out.detach(), kept["w"].shape[-1], {k: v.grad for k, v in sdv.items()}, x.grad if x_grad else None, perm, kept


# ---- fp64 restatement of the tail of the backward ----------------------------------------------------------------------------
def mixture_grad(d_w, w_pre, enc_w, stride, pl, T, relu, mut=None):
    """d_x = crop(conv_transpose1d(relu'(w_pre) d_w, W_enc)), the encoder's adjoint as ctn_softmax_bwd forms it: k_dw_combine
    masks d_w where w_pre is not > 0, ctn_decoder_fwd crops pl samples on the left.  mut: 'relu_at_zero' (relu'(0) = 1) or
    'no_crop' (the crop left out)"""
    if relu:
        d_w = d_w * ((w_pre >= 0) if mut == "relu_at_zero" else (w_pre > 0)).to(d_w.dtype)
    full = F.conv_transpose1d(d_w, enc_w, stride=stride)
    left = 0 if mut == "no_crop" else pl
    return full[..., left:left + T]


def gln_eps_outside(x, gamma, beta, eps=O.EPS):
    """gLN with eps outside the sqrt, (x - mean) / (sqrt(var) + eps): the cLN's placement, a defect for gLN"""
    mean = x.mean(dim=(1, 2), keepdim=True)
    var = ((x - mean) ** 2).mean(dim=(1, 2), keepdim=True)
    return (x - mean) / (torch.sqrt(var) + eps) * gamma.view(1, -1, 1) + beta.view(1, -1, 1)
