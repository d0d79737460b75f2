"""Edge shapes of the TRAINING path (``-m gpu``): ctn_convtasnet_fwd_train / ctn_convtasnet_bwd against torch autograd over the
CPU oracle (oracle/convtasnet_oracle.py) run in FLOAT64, at shapes that reach the branches the toy shapes of test_train_gpu.py
leave alone: filter banks longer than ENCDEC_MAX_L, even and 1-/7-tap depthwise kernels, dilations past the padded sequence,
frame counts at the 32-frame weight-gradient chunks and the 128-frame activation tiles, contractions with several n-tiles,
the fp16-piece row limit (F16_MAX_ROWS), single-pass 'tf32' training, extreme operand magnitudes and cross-sample sums.

The backward is driven by a seeded random cotangent G through ``out.backward(G)``, which isolates the model backward from the
PIT loss; one PIT-driven case per shape keeps ctn_sisdr_pit_bwd in the loop.

Criterion (fp32, tf32x3, f16x3):
  * estimate within rtol 1e-4 / atol 2e-5 of the oracle, and the training forward equal to the inference forward;
  * every tensor: max|g - g64| <= 2e-4 * scale(role) + 1e-9, scale(role) = the largest |g64| entry among the tensors of the
    same role (all depthwise weights, all PReLU slopes, ...), so a tensor that is legitimately ~0 (e.g. depthwise taps that
    only ever see padding) is judged against its peers.  Failure messages carry the fp32 oracle's own distance to fp64.
"""
import collections

import pytest
import torch

import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import PIT1d
from ctn_b200.criterion.sdr import NegSISDR
from test_parity_gpu import build_model, _scaled_paperish
from test_train_gpu import _role

pytestmark = pytest.mark.gpu

MODES = ["fp32"] + (["tf32x3", "f16x3"] if N.ctn_has_tcgen05() else [])
OUT_RTOL, OUT_ATOL = 1e-4, 2e-5
GRAD_PER, GRAD_ATOL = 2e-4, 1e-9

Edge = collections.namedtuple("Edge", "shape batch T frames reaches")

EDGES = {
    "E1": Edge(dict(n_basis=24, kernel_size=40, stride=20, sep_bottleneck_channels=20, sep_hidden_channels=40, sep_skip_channels=12,
                    sep_kernel_size=4, sep_num_blocks=1, sep_num_layers=10, n_sources=2), 2, 2000, 99,
               "L=40 > ENCDEC_MAX_L: k_encdec_wgrad_generic; stride 20 / R=2 has no k_decoder specialisation: k_decoder_generic; "
               "P=4: asymmetric pad_left = (P-1)*d//2; dilation 512 > pitch: ld4_shift / dw_slab clamps"),
    "E2": Edge(dict(n_basis=64, kernel_size=64, stride=32, sep_bottleneck_channels=24, sep_hidden_channels=48, sep_skip_channels=16,
                    sep_kernel_size=8, sep_num_blocks=1, sep_num_layers=3, n_sources=2), 2, 3000, 93,
               "L=64 > ENCDEC_MAX_L (largest encoder case); P=8 = CTN_MAX_P, the register arrays of k_dw_bwd full"),
    "E3": Edge(dict(n_basis=100, kernel_size=16, sep_bottleneck_channels=96, sep_hidden_channels=136, sep_skip_channels=48,
                    sep_kernel_size=3, sep_num_blocks=2, sep_num_layers=3, n_sources=3), 3, 1040, 129,
               "Bc+Sc=144 > 128: two n-tiles of the fused TRAIN producer (f16x3, P=3), which stores dw_u_pre_out and the stage-2 "
               "statistics from n-tile 0 only; S*N=300: source boundaries inside a 128-row tile; split_row 96 inside a 128-row "
               "weight-gradient tile; 129 frames: one frame past a 128-frame tile"),
    "E4": Edge(dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16,
                    sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=4, n_sources=2), 2, 16, 1,
               "a single frame: every dilated tap reads padding, one partial WG_KT / WG_T chunk per sample"),
    "E5": Edge(dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=48, sep_skip_channels=16,
                    sep_kernel_size=2, sep_num_blocks=1, sep_num_layers=5, n_sources=2, enc_nonlinear="relu"), 1, 1032, 128,
               "128 frames: exactly one activation tile, four full 32-frame chunks; P=2; encoder ReLU backward"),
    "E6": Edge(dict(n_basis=24, kernel_size=8, sep_bottleneck_channels=20, sep_hidden_channels=40, sep_skip_channels=12,
                    sep_kernel_size=6, sep_num_blocks=2, sep_num_layers=2, n_sources=2), 5, 136, 33,
               "33 frames: one frame past a 32-frame chunk (WG_KT / WG_T), so split-K ranges cross sample boundaries; P=6"),
    "E7": Edge(dict(n_basis=40, kernel_size=20, stride=10, sep_bottleneck_channels=24, sep_hidden_channels=40, sep_skip_channels=24,
                    sep_kernel_size=7, sep_num_blocks=1, sep_num_layers=4, n_sources=2), 2, 1001, 100,
               "L=20, stride 10: k_encoder_v4<20,10> and k_decoder<10,2>; P=7"),
    "E8": Edge(dict(n_basis=16, kernel_size=4, stride=4, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16,
                    sep_kernel_size=1, sep_num_blocks=1, sep_num_layers=3, n_sources=2), 2, 301, 76,
               "stride = L (R=1): k_decoder_generic with no overlap; P=1: no dilated taps"),
    "E9": Edge(dict(n_basis=512, kernel_size=16, sep_bottleneck_channels=32, sep_hidden_channels=64, sep_skip_channels=32,
                    sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=2, n_sources=5), 2, 4000, 499,
               "S*N=2560 > F16_MAX_ROWS=2048: eff_math falls back to tf32 pieces for the mask contraction and maskdec_ok refuses "
               "the fused mask+decoder"),
}

_CACHE = {}


def _setup(case):
    e = EDGES[case]
    cfg = O.OracleConfig(causal=False, **e.shape)
    sd = O.synth_state_dict(cfg, seed=411)
    mixture, sources = O.synth_batch(e.batch, cfg.n_sources, e.T, seed=412)
    G = torch.randn(e.batch, cfg.n_sources, e.T, generator=torch.Generator().manual_seed(413))
    return cfg, sd, mixture, sources, G


def _oracle(cfg, sd, mixture, drive, dtype):
    """oracle forward + backward in `dtype`; drive = a cotangent tensor, or the sources for PIT(NegSISDR).
    Returns (out, latent frames, perm or None, {key: grad})."""
    sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    out, latent = O.conv_tasnet_fwd(mixture.to(dtype), sdv, cfg)
    perm = None
    if isinstance(drive, tuple):
        loss, perm = O.pit_neg_sisdr(out, drive[0].to(dtype), batch_mean=True)
        loss.backward()
    else:
        out.backward(drive.to(dtype))
    return out.detach(), latent.shape[-1], perm, {k: v.grad for k, v in sdv.items()}


def _reference(key, cfg, sd, mixture, drive):
    """fp64 answer and the fp32 oracle's distance to it, once per (case, driver) for all modes"""
    if key not in _CACHE:
        out64, frames, perm64, g64 = _oracle(cfg, sd, mixture, drive, torch.float64)
        _, _, perm32, g32 = _oracle(cfg, sd, mixture, drive, torch.float32)
        noise32 = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
        _CACHE[key] = (out64, frames, perm64, perm32, g64, noise32)
    return _CACHE[key]


def _role_scales(g64):
    group = {}
    for k, v in g64.items():
        group[_role(k)] = max(group.get(_role(k), 0.0), float(v.abs().max()))
    return group


def _assert_well_conditioned(g64, noise32):
    """The fp32 oracle itself must sit 10x inside the bound.  PReLU is not differentiable at 0: a pre-activation within
    rounding of 0 takes a different slope in fp32 and fp64 and moves a whole row of gradients by O(1e-2) of its scale (seed 211
    did that on E3), which no fp32 implementation can match -- such a seed says nothing about the kernels."""
    group = _role_scales(g64)
    worst = max((noise32[k] / (group[_role(k)] + 1e-30), k) for k in g64)
    assert worst[0] <= GRAD_PER / 10, "ill-conditioned case: the fp32 oracle is {:.2e} of its role scale from fp64 ({})".format(*worst)


def _check_grads(model, g64, noise32, per=GRAD_PER):
    """per-tensor role-scaled check; every failing tensor is listed in one message. Returns (worst ratio, key)."""
    group = _role_scales(g64)
    worst, bad = (0.0, None), []
    for k, p in model.named_parameters():
        assert p.grad is not None, k
        g, r = p.grad.detach().cpu().double(), g64[k]
        assert g.shape == r.shape, k
        scale = group[_role(k)]
        d = (g - r).abs()
        err = float(d.max())
        ratio = err / (scale + 1e-30)
        worst = max(worst, (ratio, k))
        if err > per * scale + GRAD_ATOL:
            at = tuple(int(i) for i in torch.nonzero(d == d.max())[0])
            bad.append("{}: |g-g64| {:.3e} at {} = {:.2e} of role scale {:.3e} (fp32 oracle: {:.2e})".format(
                k, err, at, ratio, scale, noise32[k] / (scale + 1e-30)))
    assert not bad, "{} tensor(s) over {:.0e} of their role scale:\n  ".format(len(bad), per) + "\n  ".join(bad)
    return worst


def _train_step(model, mixture, drive):
    model.zero_grad(set_to_none=True)
    out = model(mixture.cuda())
    assert out.requires_grad
    if isinstance(drive, tuple):
        loss, perm = PIT1d(NegSISDR(), model.n_sources)(out, drive[0].cuda())
        loss.backward()
        return out.detach(), perm.cpu()
    out.backward(drive.cuda())
    return out.detach(), None


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(EDGES))
def test_edge_shape_gradients_vs_fp64(case, mode):
    """Each EDGES row (its `reaches` field names the branch and the constant that selects it), backward driven by a random
    cotangent: estimate == oracle, training forward == inference forward, every gradient within 2e-4 of its role scale of fp64."""
    e = EDGES[case]
    cfg, sd, mixture, _, G = _setup(case)
    out64, frames, _, _, g64, noise32 = _reference((case, "G"), cfg, sd, mixture, G)
    assert frames == e.frames, (case, frames)
    _assert_well_conditioned(g64, noise32)
    model = build_model(cfg, sd, math=mode).train()
    out, _ = _train_step(model, mixture, G)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    worst = _check_grads(model, g64, noise32)
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL)
    print("[{} {}] worst gradient error / role scale {:.2e} ({}) -- {}".format(case, mode, worst[0], worst[1], e.reaches))


@pytest.mark.parametrize("case", list(EDGES))
def test_edge_shape_pit_gradients_vs_fp64(case):
    """Same shapes driven by PIT(NegSISDR) (ctn_sisdr_pit_bwd in the loop) in the default tensor-core mode: permutation equal to
    the fp64 oracle's, gradients within 2e-4 of their role scale."""
    mode = MODES[-1]
    cfg, sd, mixture, sources, _ = _setup(case)
    out64, _, perm64, perm32, g64, noise32 = _reference((case, "pit"), cfg, sd, mixture, (sources,))
    assert torch.equal(perm32, perm64)
    _assert_well_conditioned(g64, noise32)
    model = build_model(cfg, sd, math=mode).train()
    out, perm = _train_step(model, mixture, (sources,))
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    assert torch.equal(perm, perm64)
    worst = _check_grads(model, g64, noise32)
    print("[{} {} PIT] worst gradient error / role scale {:.2e} ({})".format(case, mode, worst[0], worst[1]))


def _rel_l2(model, g64):
    num = sum(float(((p.grad.detach().cpu().double() - g64[k]) ** 2).sum()) for k, p in model.named_parameters())
    den = sum(float((g64[k] ** 2).sum()) for k, _ in model.named_parameters())
    return (num / den) ** 0.5


MID = dict(n_basis=256, kernel_size=16, sep_bottleneck_channels=128, sep_hidden_channels=256, sep_skip_channels=128,
           sep_kernel_size=3, sep_num_blocks=2, sep_num_layers=4, n_sources=2)
TF32_L2 = 4e-2


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
@pytest.mark.parametrize("case", ["E3", "mid"])
def test_tf32_training_vs_fp64(case):
    """Single-pass 'tf32' training (launch_wg<1>, the NPASS = 1 raw contractions): one 10-bit-mantissa product per term, so the
    stated bound is on the whole gradient, ||g - g64||_2 / ||g64||_2 <= TF32_L2, plus the PIT permutation of the fp64 oracle
    and the forward's stated 'tf32' tolerance (rtol 2e-2, atol 5e-3).  'mid' is a paper-like N = H = 256, 2 x 4 blocks.
    Measured on an H100 80GB HBM3 at a 400 W power limit: 1.14e-2 (E3) and 2.23e-2 (mid); TF32_L2 = 4e-2."""
    if case == "mid":
        cfg = O.OracleConfig(causal=False, **MID)
        sd = O.synth_state_dict(cfg, seed=221)
        mixture, sources = O.synth_batch(2, cfg.n_sources, 8000, seed=222)
    else:
        cfg, sd, mixture, sources, _ = _setup(case)
    out64, _, perm64, _, g64, _ = _reference((case, "pit"), cfg, sd, mixture, (sources,))
    model = build_model(cfg, sd, math="tf32").train()
    out, perm = _train_step(model, mixture, (sources,))
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=2e-2, atol=5e-3)
    assert torch.equal(perm, perm64)
    l2 = _rel_l2(model, g64)
    print("[{} tf32] relative L2 of the whole gradient vs fp64 {:.2e}".format(case, l2))
    assert l2 <= TF32_L2, l2


def _magnitude_case(kind, value):
    """The perturbations of test_parity_gpu.py's test_split_modes_are_robust_*: (cfg, sd, mixture, forward atol)."""
    if kind == "weights":
        cfg = O.OracleConfig(n_basis=64, kernel_size=16, sep_hidden_channels=96, sep_bottleneck_channels=48, sep_skip_channels=32,
                             sep_num_blocks=2, sep_num_layers=3, causal=False, n_sources=2)
        sd = O.synth_state_dict(cfg, seed=77)
        g = torch.Generator().manual_seed(78)
        for k in list(sd):
            if k.endswith("separable_conv1d.norm1d.norm.weight"):      # gamma2 rows of 1e-5 .. 1e-3
                sd[k] = sd[k] * (10.0 ** (-5 + 2 * torch.rand(sd[k].shape, generator=g)))
            elif k.endswith("output_pointwise_conv1d.weight"):
                sd[k] = sd[k] * 3e3
            elif k.endswith("skip_pointwise_conv1d.weight"):
                sd[k] = sd[k] * 3e4
            elif k.endswith("bottleneck_conv1d.weight") and ".net." in k:
                sd[k] = sd[k] * 1e-3
        mixture, _ = O.synth_batch(2, 2, 3000, seed=79)
        return cfg, sd, mixture, 1.0
    if kind == "input":
        # PReLU has a kink at 0: an input within rounding of it takes a different slope on the GPU than in fp64, which moves the
        # gradients of its channel and of everything upstream by ~1e-3 of their role scale (see _assert_well_conditioned).  At
        # 3000 x 96 x 16 PReLU inputs the closest one sits ~1e-7 .. 1e-6 of its tensor's largest entry from 0, so the seed is
        # picked per scale: the forward test's 92 puts a PReLU2 input of block 1 layer 2 at 1.2e-8 when scaled by 1e3, and 99
        # puts one of block 1 layer 3 at 3.2e-7 when scaled by 1e-4, which the f16x3 forward rounds to the other side.
        cfg, sd = _scaled_paperish()
        mixture, _ = O.synth_batch(2, 2, 3000, seed=92 if value < 1 else 99)
        return cfg, sd, mixture * value, 1e-30
    cfg, sd = _scaled_paperish(seed=93)                              # "residual": residual stream and skip sum at `value`
    for k in list(sd):
        if k.startswith("separator.bottleneck_conv1d.") or k.endswith("output_pointwise_conv1d.weight") or k.endswith("output_pointwise_conv1d.bias") \
                or k.endswith("skip_pointwise_conv1d.weight") or k.endswith("skip_pointwise_conv1d.bias"):
            sd[k] = sd[k] * value
        if k == "separator.mask_conv1d.weight":
            sd[k] = sd[k] / value
    mixture, _ = O.synth_batch(2, 2, 3000, seed=94)
    return cfg, sd, mixture, 1.0


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
@pytest.mark.parametrize("mode", ["tf32x3", "f16x3"])
@pytest.mark.parametrize("kind,value", [("weights", None), ("input", 1e-4), ("input", 1e3), ("residual", 1e-3), ("residual", 1e4)])
def test_split_mode_training_is_robust_to_magnitudes(mode, kind, value):
    """The training forward uses its own instantiations of the split contractions and takes mask_scale from the fused stack:
    tiny gamma2 rows with huge output / skip weights, the mixture at 1e-4 / 1e3, and the residual stream and skip sum at
    1e-3 / 1e4, each through model.train().  Estimate at the forward tests' scaled tolerance, gradients within 2e-4 of their
    role scale of fp64 -- or twice the fp32 oracle's own worst distance where that is larger: the tiny-gamma2 weights make the
    problem ill-conditioned, and the fp32 oracle itself is 2.2e-4 of its role scale away from fp64 there."""
    cfg, sd, mixture, floor = _magnitude_case(kind, value)
    G = torch.randn(mixture.shape[0], cfg.n_sources, mixture.shape[-1], generator=torch.Generator().manual_seed(231))
    out64, _, _, _, g64, noise32 = _reference((kind, value, "G"), cfg, sd, mixture, G)
    group = _role_scales(g64)
    per = max(GRAD_PER, 2 * max(noise32[k] / (group[_role(k)] + 1e-30) for k in g64))
    model = build_model(cfg, sd, math=mode).train()
    out, _ = _train_step(model, mixture, G)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL * max(floor, float(out64.abs().max())))
    worst = _check_grads(model, g64, noise32, per=per)
    print("[{} {}={}] worst gradient error / role scale {:.2e} ({}), bound {:.1e}".format(mode, kind, value, worst[0], worst[1], per))


ADD_PER = 1e-5


@pytest.mark.parametrize("mode", MODES)
def test_gradients_are_additive_over_the_batch(mode):
    """Split-K ranges and the fp32 / fp64 atomics of the weight gradients span sample boundaries: with a fixed cotangent G, the
    gradients of a batch of 5 equal the sum of the gradients of each sample run alone with G[b], within fp32 summation-order
    slack (ADD_PER of the role scale).  E6's 33 frames put a 32-frame chunk edge inside every sample."""
    cfg, sd, mixture, _, G = _setup("E6")
    assert mixture.shape[0] == 5
    model = build_model(cfg, sd, math=mode).train()
    _train_step(model, mixture, G)
    batch = {k: p.grad.detach().double().cpu() for k, p in model.named_parameters()}
    alone = {k: torch.zeros_like(v) for k, v in batch.items()}
    for b in range(mixture.shape[0]):
        _train_step(model, mixture[b:b + 1], G[b:b + 1])
        for k, p in model.named_parameters():
            alone[k] += p.grad.detach().double().cpu()
    group = _role_scales(batch)
    worst, bad = (0.0, None), []
    for k in batch:
        err = float((batch[k] - alone[k]).abs().max())
        worst = max(worst, (err / (group[_role(k)] + 1e-30), k))
        if err > ADD_PER * group[_role(k)] + GRAD_ATOL:
            bad.append("{}: {:.3e} = {:.2e} of role scale".format(k, err, err / (group[_role(k)] + 1e-30)))
    assert not bad, "\n  ".join(bad)
    print("[additivity {}] worst difference / role scale {:.2e} ({})".format(mode, worst[0], worst[1]))
