"""Multichannel (in_channels = C > 1) TRAINING on the GPU (``-m gpu``): ConvTasNet(in_channels=C) with multichannel_training = True
through ctn_multichannel_fwd_train / ctn_multichannel_bwd, against torch autograd over the CPU oracle in FLOAT64, the reference
golden tiny_stereo_grad.pt, the MUSDB18 recipe architecture (N = 256, L = 20, H = 512, Bc = 256, Sc = 128, X = 10, R = 4, 4
sources) at a short segment and at its full 4 x 8 s shape, the multichannel filter-bank kernels at the recipe length, and the
node's contract.

Criterion (test_train_edges_gpu.py's): the backward is driven by a seeded cotangent G (B, S, C, T) or by the recipe's
MeanSquaredError; every gradient tensor within 2e-4 of its role scale of fp64, failure messages carry the fp32 oracle's own
distance."""
import collections
import os

import pytest
import torch
import torch.nn.functional as F_

import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.criterion.distance import MeanSquaredError
from ctn_b200.models.conv_tasnet import ConvTasNet
from ctn_b200.optim import FlatClipAdam
from test_train_edges_gpu import GRAD_PER, MODES, OUT_ATOL, OUT_RTOL, _assert_well_conditioned, _check_grads, _role_scales
from test_train_gpu import _role

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
MSE = MeanSquaredError(dim=-1, reduction="mean")  # the recipe's criterion (egs/musdb18/conv-tasnet, criterion='mse')

Edge = collections.namedtuple("Edge", "C shape batch T frames reaches")
SMALL = dict(n_basis=32, kernel_size=16, stride=8, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16,
             sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=3, n_sources=2)

EDGES = {
    "C2-L16-ragged-relu": Edge(2, dict(SMALL, enc_nonlinear="relu"), 2, 1037, 129,
                               "k_encoder_v4_mc<16,8> / k_decoder_mc_v<8,2>; T padded 1 / 2 on both sides; encoder ReLU backward"),
    "C2-L20-wide": Edge(2, dict(n_basis=40, kernel_size=20, stride=10, sep_bottleneck_channels=96, sep_hidden_channels=96,
                                sep_skip_channels=48, sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=2, n_sources=2), 2, 1995, 199,
                        "the recipe's 20 / 10: k_encoder_v4_mc<20,10>, k_decoder_mc_v<10,2>; Bc + Sc = 144 > 128"),
    "C3-L16S4": Edge(3, dict(SMALL, stride=4), 2, 803, 198,
                     "L / stride = 4: the fallback k_encoder_mc (also as the decoder adjoint) and k_decoder_mc"),
    "C8-L40": Edge(8, dict(SMALL, n_basis=24, kernel_size=40, stride=20), 2, 2000, 99,
                   "L = 40 > ENCDEC_MAX_L: k_encdec_wgrad_generic over 8 channels; fallback encoder and decoder"),
    "C64-L2": Edge(64, dict(SMALL, n_basis=16, kernel_size=2, stride=1), 2, 300, 299,
                   "C = 64, the largest in_channels, through k_encoder_v4_mc<2,1> (106 KB of shared memory) and k_decoder_mc_v<1,2>"),
    "C2-T=L": Edge(2, SMALL, 2, 16, 1, "T = L: one frame"),
    "C2-129f-B1-S1": Edge(2, dict(SMALL, n_sources=1), 1, 1040, 129, "129 frames: one past a 128-frame tile; B = 1; S = 1"),
    "C2-B3-S4": Edge(2, dict(SMALL, n_sources=4), 3, 600, 74, "B = 3, S = 4: decoder rows B*S = 12"),
}

_CACHE = {}


def _build(cfg, sd, math):
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, stride=cfg.stride, enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg.enc_nonlinear, sep_hidden_channels=cfg.sep_hidden_channels,
                   sep_bottleneck_channels=cfg.sep_bottleneck_channels, sep_skip_channels=cfg.sep_skip_channels,
                   sep_kernel_size=cfg.sep_kernel_size, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers,
                   mask_nonlinear=cfg.mask_nonlinear, causal=cfg.causal, n_sources=cfg.n_sources, eps=cfg.eps, in_channels=cfg.in_channels)
    m.load_state_dict(sd, strict=True)
    m.math = math
    m.multichannel_training = True
    return m.cuda().train()


def _inputs(cfg, batch, T, seed):
    g = torch.Generator().manual_seed(seed)
    mixture = 0.3 * torch.randn(batch, 1, cfg.in_channels, T, generator=g)
    sources = 0.1 * torch.randn(batch, cfg.n_sources, cfg.in_channels, T, generator=g)
    G = torch.randn(batch, cfg.n_sources, cfg.in_channels, T, generator=g)
    return mixture, sources, G


def _setup(case):
    e = EDGES[case]
    cfg = O.OracleConfig(causal=False, in_channels=e.C, **e.shape)
    sd = O.synth_state_dict(cfg, seed=511)
    return (cfg, sd) + _inputs(cfg, e.batch, e.T, 512)


def _oracle(cfg, sd, mixture, drive, dtype):
    """oracle forward + backward in `dtype`; drive = a cotangent tensor, or (sources,) for the recipe's MSE"""
    sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    out, latent = O.conv_tasnet_fwd(mixture.to(dtype), sdv, cfg)
    if isinstance(drive, tuple):
        MSE(out, drive[0].to(dtype)).backward()
    else:
        out.backward(drive.to(dtype))
    return out.detach(), latent.shape[-1], {k: v.grad for k, v in sdv.items()}


def _reference(key, cfg, sd, mixture, drive):
    if key not in _CACHE:
        out64, frames, g64 = _oracle(cfg, sd, mixture, drive, torch.float64)
        _, _, g32 = _oracle(cfg, sd, mixture, drive, torch.float32)
        _CACHE[key] = (out64, frames, g64, {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64})
    return _CACHE[key]


def _step(model, mixture, drive):
    model.zero_grad(set_to_none=True)
    out = model(mixture.cuda())
    assert out.requires_grad and out.shape == (mixture.shape[0], model.n_sources, model.in_channels, mixture.shape[-1])
    if isinstance(drive, tuple):
        loss = MSE(out, drive[0].cuda())
        loss.backward()
        return out.detach(), loss.detach()
    out.backward(drive.cuda())
    return out.detach(), None


def _run_case(cfg, sd, mixture, drive, key, mode, what, deep=False):
    """deep: a 40-block stack, where the fp32 oracle itself is farther than 2e-5 of a role scale from fp64; the bound is then
    twice the fp32 oracle's own worst distance where that exceeds 2e-4 (as test_split_mode_training_is_robust_to_magnitudes)"""
    out64, _, g64, noise32 = _reference(key, cfg, sd, mixture, drive)
    per = GRAD_PER
    if deep:
        group = _role_scales(g64)
        per = max(GRAD_PER, 2 * max(noise32[k] / (group[_role(k)] + 1e-30) for k in g64))
    else:
        _assert_well_conditioned(g64, noise32)
    model = _build(cfg, sd, mode)
    out, _ = _step(model, mixture, drive)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    worst = _check_grads(model, g64, noise32, per=per)
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL)
    print("[{} {}] worst gradient error / role scale {:.2e} ({}), bound {:.1e} -- {}".format(key[0], mode, worst[0], worst[1], per, what))
    return model


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(EDGES))
def test_gradients_vs_fp64(case, mode):
    """each EDGES row (`reaches` names the branch), driven by a seeded cotangent: estimate == oracle, training forward == inference
    forward, every gradient within 2e-4 of its role scale of fp64"""
    e = EDGES[case]
    cfg, sd, mixture, _, G = _setup(case)
    assert _reference((case, "G"), cfg, sd, mixture, G)[1] == e.frames
    _run_case(cfg, sd, mixture, G, (case, "G"), mode, e.reaches)


@pytest.mark.parametrize("case", list(EDGES))
def test_mse_gradients_vs_fp64(case):
    """the same rows driven by the recipe's MeanSquaredError in the default tensor-core mode"""
    cfg, sd, mixture, sources, _ = _setup(case)
    _run_case(cfg, sd, mixture, (sources,), (case, "mse"), MODES[-1], EDGES[case].reaches)


@pytest.mark.parametrize("mode", MODES)
def test_reference_golden(golden_dir, mode):
    """tiny_stereo_grad.pt, minted from the unmodified reference: output and loss, and every gradient within 2e-4 of its role scale
    of the reference's fp64 gradients"""
    r = torch.load(os.path.join(golden_dir, "tiny_stereo_grad.pt"), weights_only=False)
    cfg = O.OracleConfig(**r["cfg"])
    sd = O.synth_state_dict(cfg, seed=r["wseed"])
    model = _build(cfg, sd, mode)
    out, loss = _step(model, r["mixture"], (r["sources"],))
    torch.testing.assert_close(out.cpu(), r["out"], rtol=OUT_RTOL, atol=OUT_ATOL)
    assert abs(float(loss) - r["loss64"]) <= 1e-5 * r["loss64"]
    worst = _check_grads(model, r["grads64"], r["fp32_vs_fp64_maxabs"])
    print("[golden {}] worst gradient error / role scale {:.2e} ({})".format(mode, worst[0], worst[1]))


RECIPE = dict(n_basis=256, kernel_size=20, stride=10, sep_hidden_channels=512, sep_bottleneck_channels=256, sep_skip_channels=128,
              sep_kernel_size=3, sep_num_blocks=4, sep_num_layers=10, n_sources=4)
RECIPE_T = 352800  # 8 s at 44.1 kHz


def _recipe(seed=521):
    cfg = O.OracleConfig(causal=False, in_channels=2, **RECIPE)
    return cfg, O.synth_state_dict(cfg, seed=seed)


@pytest.mark.parametrize("mode", ["fp32"] + (["f16x3"] if N.ctn_has_tcgen05() else []))
def test_recipe_architecture_short_segment_vs_fp64(mode):
    """the recipe's separator (Bc = 256, H = 512, X = 10: dilation 512, 40 blocks) at B = 1 and 0.25 s of stereo at 44.1 kHz
    (1102 frames), cotangent-driven, against fp64"""
    cfg, sd = _recipe()
    mixture, _, G = _inputs(cfg, 1, 11025, 522)
    _run_case(cfg, sd, mixture, G, ("recipe-short", "G"), mode, "recipe architecture, 0.25 s", deep=True)


def _finite_grads(model):
    return all(bool(torch.isfinite(p.grad).all()) for p in model.parameters())


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
def test_recipe_shape_trains():
    """4 x 352 800 samples of stereo, f16x3: training forward == inference forward; a step with MSE, clip 5 and Adam; finite
    gradients that are additive over the batch; the loss falls over a few steps on one batch"""
    cfg, sd = _recipe()
    mixture, sources, G = _inputs(cfg, 4, RECIPE_T, 523)
    sources = sources * 3.0
    mixture = sources.sum(dim=1, keepdim=True)
    model = _build(cfg, sd, "f16x3")
    out, _ = _step(model, mixture, G)
    assert _finite_grads(model)
    batch = {k: p.grad.detach().double().cpu() for k, p in model.named_parameters()}
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL * max(1.0, float(out_inf.abs().max())))
    alone = {k: torch.zeros_like(v) for k, v in batch.items()}
    for b in range(4):
        _step(model, mixture[b:b + 1], G[b:b + 1])
        for k, p in model.named_parameters():
            alone[k] += p.grad.detach().double().cpu()
    group = _role_scales(batch)
    worst = max((float((batch[k] - alone[k]).abs().max()) / (group[_role(k)] + 1e-30), k) for k in batch)
    print("[recipe additivity] worst difference / role scale {:.2e} ({})".format(*worst))
    assert worst[0] <= 1e-4, worst
    # the B = 1 steps leave ~10 GB blocks in the caching allocator that a 4 x 8 s workspace (39 GB) cannot reuse
    del out, out_inf, batch, alone
    model.zero_grad(set_to_none=True)
    N.release_workspaces()
    torch.cuda.empty_cache()
    opt = FlatClipAdam(model, lr=3e-4, max_norm=5.0)  # the recipe's lr and max_norm
    losses = []
    for _ in range(4):
        model.zero_grad(set_to_none=True)
        loss = MSE(model(mixture.cuda()), sources.cuda())
        loss.backward()
        assert _finite_grads(model)
        opt.step()
        losses.append(float(loss))
    print("[recipe steps] MSE {}".format(", ".join("{:.5f}".format(v) for v in losses)))
    assert losses[-1] < losses[0], losses


# ---- kernels at the recipe length ------------------------------------------------------------------------------------------
probe_wgrad_mc = N._sig("ctn_probe_encdec_wgrad_mc", N._i, N._fp, N._fp, N._fp, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i,
                        N._fp)


def _dev(t):
    return t.contiguous().cuda()


@pytest.mark.parametrize("relu", [False, True])
def test_filterbank_kernels_at_recipe_length(relu):
    """ctn_encoder_mc_fwd (k_encoder_v4_mc<20,10>) and ctn_decoder_mc_fwd (k_decoder_mc_v<10,2>) over 2 x 352 800 stereo samples
    (35 279 frames, pad 5 / 5), within the order-independent fp32 dot-product bound of fp64; gLN statistics in the same pass"""
    Cc, L, S, N_, T = 2, 20, 10, 256, RECIPE_T
    frames, pl, pr = N.frames_of(T, L, S)
    pitch = N.ctn_pitch(frames)
    g = torch.Generator().manual_seed(531)
    x = 0.5 * torch.randn(2, Cc, T, generator=g)
    We = (torch.rand(N_, Cc, L, generator=g) * 2 - 1) / (Cc * L) ** 0.5
    Wd = (torch.rand(N_, Cc, L, generator=g) * 2 - 1) / L ** 0.5
    xp = F_.pad(x.double(), (pl, pr))
    w64 = F_.conv1d(xp, We.double(), stride=S)
    w_bound = Cc * L * U * F_.conv1d(xp.abs(), We.double().abs(), stride=S)
    if relu:
        w64 = torch.relu(w64)
    w = torch.full((2, N_, pitch), float("nan"), device="cuda")
    stats = torch.zeros(2, 2, dtype=torch.float64, device="cuda")
    N.check(N.ctn_encoder_mc_fwd(_dev(x).data_ptr(), _dev(We).data_ptr(), w.data_ptr(), 2, Cc, T, pl, pr, N_, L, S, int(relu), pitch,
                                 stats.data_ptr(), None), "ctn_encoder_mc_fwd")
    wq = w64.float()
    wpad = torch.zeros(2, N_, pitch)
    wpad[..., :frames] = wq
    y64 = F_.conv_transpose1d(wq.double(), Wd.double(), stride=S)[..., pl:pl + T]
    y_bound = N_ * (L // S) * U * F_.conv_transpose1d(wq.double().abs(), Wd.double().abs(), stride=S)[..., pl:pl + T]
    y = torch.full((2, Cc, T), float("nan"), device="cuda")
    N.check(N.ctn_decoder_mc_fwd(_dev(wpad).data_ptr(), _dev(Wd).data_ptr(), y.data_ptr(), 2, Cc, N_, frames, pitch, L, S, pl, T, None),
            "ctn_decoder_mc_fwd")
    torch.cuda.synchronize()
    w = w.cpu()
    assert bool((w[..., frames:] == 0).all())
    shares = []
    for name, v, ref, bound in (("encoder", w[..., :frames], w64, w_bound), ("decoder", y.cpu(), y64, y_bound)):
        err = (v.double() - ref).abs()
        assert bool((err <= bound).all()), "{}: {:.2f}x the dot-product bound".format(name, float((err / bound.clamp_min(1e-300)).max()))
        shares.append(float((err / bound.clamp_min(1e-300)).max()))
    ref_stats = torch.stack([w64.sum(dim=(1, 2)), (w64 ** 2).sum(dim=(1, 2))], dim=1)
    torch.testing.assert_close(stats.cpu(), ref_stats, rtol=1e-5, atol=1e-6 * float(ref_stats.abs().max()))
    print("[recipe filter banks relu={}] encoder {:.3f}, decoder {:.3f} of the bound".format(relu, *shares))


@pytest.mark.parametrize("R,L,S", [(4, 20, 10), (16, 20, 10), (2, 40, 20)])
def test_wgrad_mc_at_recipe_length(R, L, S):
    """ctn_probe_encdec_wgrad_mc over R rows x 2 channels x 352 800 samples: dW (N, 2, L) against fp64 within fp32 summation slack
    of the sum of |terms| (k_encdec_wgrad for L <= 32, k_encdec_wgrad_generic for L = 40); at C = 1 both probes meet channel 0's bound"""
    Cc, N_, T = 2, 256, RECIPE_T
    frames, pl, pr = N.frames_of(T, L, S)
    pitch = N.ctn_pitch(frames)
    g = torch.Generator().manual_seed(541 + R)
    act = torch.zeros(R, N_, pitch)
    act[..., :frames] = torch.randn(R, N_, frames, generator=g)
    sig = torch.randn(R * Cc, T, generator=g)
    sp = F_.pad(sig.double().view(R, Cc, T), (pl, pr))
    windows = sp.unfold(2, L, S)  # (R, C, frames, L)
    a64 = act[..., :frames].double()
    ref = torch.einsum("rnf,rcfk->nck", a64, windows)
    bound = 64 * U * torch.einsum("rnf,rcfk->nck", a64.abs(), windows.abs())
    dW = torch.zeros(N_, Cc, L, device="cuda")
    assert probe_wgrad_mc(_dev(act).data_ptr(), _dev(sig).data_ptr(), dW.data_ptr(), R, N_, Cc, frames, pitch, T, L, S, pl, None) == 0
    err = (dW.cpu().double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    # C = 1: the channel-0 rows alone through the monaural probe and the channel probe
    probe_wgrad = N._sig("ctn_probe_encdec_wgrad", N._i, N._fp, N._fp, N._fp, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._fp)
    sig0 = _dev(sig.view(R, Cc, T)[:, 0])
    d1, d2 = torch.zeros(N_, 1, L, device="cuda"), torch.zeros(N_, 1, L, device="cuda")
    assert probe_wgrad(_dev(act).data_ptr(), sig0.data_ptr(), d1.data_ptr(), R, N_, frames, pitch, T, L, S, pl, None) == 0
    assert probe_wgrad_mc(_dev(act).data_ptr(), sig0.data_ptr(), d2.data_ptr(), R, N_, 1, frames, pitch, T, L, S, pl, None) == 0
    for d in (d1, d2):  # fp32 atomics across the row-group CTAs land in any order: two runs agree to summation slack, not bits
        assert bool(((d.cpu().double() - ref[:, :1]).abs() <= bound[:, :1]).all())
    print("[wgrad_mc R={} L={}] {:.3f} of the bound".format(R, L, float((err / bound).max())))


# ---- contract ------------------------------------------------------------------------------------------------------------
def _mono_twin(cfg, sd):
    mcfg = O.OracleConfig(**dict(cfg.to_dict(), in_channels=1))
    msd = O.synth_state_dict(mcfg, seed=511)
    m = _build(mcfg, msd, None)
    m.multichannel_training = False
    return mcfg, m


@pytest.mark.parametrize("mode", MODES)
def test_launch_count_equals_the_monaural_step(mode):
    cfg, sd, mixture, _, G = _setup("C2-L20-wide")
    model = _build(cfg, sd, mode)
    _step(model, mixture, G)
    mcfg, mono = _mono_twin(cfg, sd)
    mono.math = mode
    mono.zero_grad(set_to_none=True)
    mono(mixture[:, :, 0].cuda()).backward(G[:, :, 0].cuda())
    assert (model.last_launches, model.last_bwd_launches) == (mono.last_launches, mono.last_bwd_launches)
    print("[launches {}] forward {}, backward {}".format(mode, model.last_launches, model.last_bwd_launches))


def test_refusals():
    cfg, sd, mixture, _, G = _setup("C2-L16-ragged-relu")
    model = _build(cfg, sd, None)
    x = mixture.cuda()
    model.multichannel_training = False
    with pytest.raises(NotImplementedError, match="multichannel_training"):
        model(x)
    model.multichannel_training = True
    with pytest.raises(NotImplementedError, match="mixture"):
        model(x.clone().requires_grad_(True))
    out = model(x)
    out.backward(G.cuda(), retain_graph=True)
    with pytest.raises(RuntimeError, match="already run"):
        out.backward(G.cuda())
    for kw in (dict(causal=True), dict(mask_nonlinear="softmax")):
        c2 = O.OracleConfig(**dict(cfg.to_dict(), **kw))
        m2 = _build(c2, O.synth_state_dict(c2, seed=511), None)
        m2.causal_training = True
        with pytest.raises(NotImplementedError):
            m2(x)


def test_flag_on_a_monaural_model_changes_nothing():
    cfg = O.OracleConfig(causal=False, **SMALL)
    sd = O.synth_state_dict(cfg, seed=551)
    mixture, _ = O.synth_batch(2, cfg.n_sources, 1037, seed=552)
    G = torch.randn(2, cfg.n_sources, 1037, generator=torch.Generator().manual_seed(553))
    res = []
    for flag in (False, True):
        m = _build(O.OracleConfig(**dict(cfg.to_dict(), in_channels=1)), sd, None)
        m.multichannel_training = flag
        out = m(mixture.cuda())
        out.backward(G.cuda())
        res.append((out.detach().cpu(), {k: p.grad.cpu() for k, p in m.named_parameters()}, m.last_launches, m.last_bwd_launches))
    # the same pipeline both times; only the order of fp32 / fp64 atomics may differ between two runs
    assert res[0][2:] == res[1][2:]
    torch.testing.assert_close(res[0][0], res[1][0], rtol=1e-6, atol=1e-7)
    for k in res[0][1]:
        torch.testing.assert_close(res[0][1][k], res[1][1][k], rtol=1e-5, atol=1e-6 * float(res[0][1][k].abs().max()) + 1e-12)
