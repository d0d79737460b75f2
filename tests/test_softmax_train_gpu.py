"""Softmax-mask TRAINING on the GPU (``-m gpu``): ConvTasNet(mask_nonlinear='softmax') with softmax_training = True through
ctn_softmax_fwd_train / ctn_softmax_bwd.  The softmax backward kernel k_softmax_mask_bwd is held to its fp64 bound through the
probe (tests/softmax_train_ref.py); whole models against torch autograd over the CPU oracle in FLOAT64, driven by a cotangent,
by ORPIT and by Sinkhorn PIT; the gradient w.r.t. the mixture; the ORPIT recipe's two-stage fine-tune step against the oracle and
the reference golden tiny_softmax_grad.pt; the ORPIT recipe shape (egs/wsj0-mix/orpit_conv-tasnet/train.sh); the node's contract.

Criterion (test_train_edges_gpu.py's): every gradient tensor within 2e-4 of its role scale of fp64; the mixture gradient within 2e-4
of its largest fp64 entry; failure messages carry the fp32 oracle's own distance."""
import collections
import os

import pytest
import torch

import convtasnet_oracle as O
import pit_variants_oracle as PV
import softmax_train_ref as R
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import ORPIT, SinkPIT
from ctn_b200.criterion.sdr import NegSISDR
from ctn_b200.models.conv_tasnet import ConvTasNet
from ctn_b200.optim import FlatClipAdam
from test_train_edges_gpu import GRAD_ATOL, GRAD_PER, MODES, OUT_ATOL, OUT_RTOL, _assert_well_conditioned, _check_grads

pytestmark = pytest.mark.gpu

probe = N._sig("ctn_probe_softmax_mask_bwd", N._i, N._fp, N._fp, N._fp, N._fp, N._i, N._i, N._i, N._i, N._i, N._fp)


# ---- the kernel ------------------------------------------------------------------------------------------------------------
def _pitched(x, pitch, fill):
    y = torch.full(x.shape[:-1] + (pitch,), fill, dtype=torch.float32)
    y[..., :x.shape[-1]] = x.float()
    return y.cuda()


@pytest.mark.parametrize("name", list(R.ROWS))
def test_softmax_mask_bwd_kernel(name):
    """k_softmax_mask_bwd against fp64: inputs carry NaN in their pad lanes and the outputs start as NaN, so a read past `frames`
    or an unwritten cell shows; pad lanes of d_z and d_wprod exactly 0; a repeat call gives the same bits; one launch"""
    B, S, Nn, F, _, reaches = R.ROWS[name]
    dwhat, w, m = R.inputs(name)
    pitch = N.ctn_pitch(F)
    outs = []
    for _ in range(2):
        dz = _pitched(dwhat.reshape(B, S * Nn, F), pitch, float("nan"))
        dp = torch.full((B, Nn, pitch), float("nan"), device="cuda")
        wd, md = _pitched(w, pitch, float("nan")), _pitched(m.reshape(B, S * Nn, F), pitch, float("nan"))
        assert probe(dz.data_ptr(), wd.data_ptr(), md.data_ptr(), dp.data_ptr(), B, S, Nn, F, pitch, None) == 0
        torch.cuda.synchronize()
        assert N.ctn_last_launch_count() == 1
        outs.append((dz.cpu(), dp.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))
    dz, dp = outs[0]
    assert bool((dz[..., F:] == 0).all()) and bool((dp[..., F:] == 0).all())
    ref = R.softmax_mask_bwd(dwhat, w, m)
    shares = []
    for key, got in (("dz", dz[..., :F].reshape(B, S, Nn, F)), ("dwprod", dp[..., :F])):
        val, bound = ref[key]
        err = (got.double() - val).abs()
        ok = torch.where(bound > 0, err <= bound, err == 0)
        r = float(torch.where(bound > 0, err / bound.clamp_min(1e-300), err).max())
        assert bool(ok.all()), "{} {}: {:.2f}x its bound".format(name, key, r)
        shares.append(r)
    print("[softmax_mask_bwd {}] d_z {:.3f}, d_wprod {:.3f} of the bound -- {}".format(name, shares[0], shares[1], reaches))


# ---- whole models ----------------------------------------------------------------------------------------------------------
Edge = collections.namedtuple("Edge", "shape batch T frames reaches")
SMALL = dict(n_basis=32, kernel_size=16, stride=8, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16,
             sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=3, n_sources=2)

EDGES = {
    "S1": Edge(dict(SMALL, n_sources=1), 2, 803, 100, "S = 1: the softmax runs over the N channels of one source"),
    "S2-ragged-relu": Edge(dict(SMALL, enc_nonlinear="relu"), 2, 1037, 129, "S = 2, T padded unevenly; encoder ReLU zeros in w"),
    "S5": Edge(dict(SMALL, n_sources=5), 2, 600, 74, "S = 5: the SinkPIT tutorial's outputs, S*N = 160"),
    "T=L": Edge(SMALL, 2, 16, 1, "T = L: one frame"),
    "129f-B1": Edge(SMALL, 1, 1040, 129, "129 frames: one past a 128-frame tile; B = 1"),
    "wide": Edge(dict(n_basis=40, kernel_size=16, stride=8, sep_bottleneck_channels=96, sep_hidden_channels=96, sep_skip_channels=48,
                      sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=2, n_sources=2), 2, 1595, 199, "Bc + Sc = 144 > 128"),
}
_CACHE = {}


def _build(cfg, sd, math, switch=True):
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, stride=cfg.stride, enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg.enc_nonlinear, sep_hidden_channels=cfg.sep_hidden_channels,
                   sep_bottleneck_channels=cfg.sep_bottleneck_channels, sep_skip_channels=cfg.sep_skip_channels,
                   sep_kernel_size=cfg.sep_kernel_size, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers,
                   mask_nonlinear=cfg.mask_nonlinear, causal=cfg.causal, n_sources=cfg.n_sources, eps=cfg.eps, in_channels=cfg.in_channels)
    m.load_state_dict(sd, strict=True)
    m.math = math
    m.softmax_training = switch
    return m.cuda().train()


def _setup(case):
    e = EDGES[case]
    cfg = O.OracleConfig(causal=False, mask_nonlinear="softmax", **e.shape)
    sd = O.synth_state_dict(cfg, seed=611)
    g = torch.Generator().manual_seed(612)
    sources = 0.3 * torch.randn(e.batch, 3 if cfg.n_sources == 2 else cfg.n_sources, e.T, generator=g)
    mixture = sources.sum(dim=1, keepdim=True)
    G = torch.randn(e.batch, cfg.n_sources, e.T, generator=g)
    return cfg, sd, mixture, sources, G


def _crit_oracle(cfg, out, sources):
    if cfg.n_sources == 2:
        return PV.orpit(out, sources)[0]
    return PV.sinkpit(out, sources)[0]


def _crit(cfg, out, sources):
    if cfg.n_sources == 2:
        return ORPIT(NegSISDR())(out, sources)[0]
    return SinkPIT(NegSISDR(), n_sources=cfg.n_sources)(out, sources)[0]


def _oracle(cfg, sd, mixture, drive, dtype):
    """oracle forward + backward in `dtype` with the mixture as a leaf that requires grad; drive = a cotangent, or (sources,) for
    ORPIT (two outputs) / SinkPIT.  Returns (out, frames, {key: grad}, d_x)"""
    sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    x = mixture.to(dtype).clone().requires_grad_(True)
    out, latent = O.conv_tasnet_fwd(x, sdv, cfg)
    if isinstance(drive, tuple):
        _crit_oracle(cfg, out, drive[0].to(dtype)).backward()
    else:
        out.backward(drive.to(dtype))
    return out.detach(), latent.shape[-1], {k: v.grad for k, v in sdv.items()}, x.grad


def _reference(key, cfg, sd, mixture, drive):
    if key not in _CACHE:
        out64, frames, g64, dx64 = _oracle(cfg, sd, mixture, drive, torch.float64)
        _, _, g32, dx32 = _oracle(cfg, sd, mixture, drive, torch.float32)
        noise = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
        _CACHE[key] = (out64, frames, g64, noise, dx64, float((dx32.double() - dx64).abs().max()))
    return _CACHE[key]


def _step(model, mixture, drive, cfg, x_grad=False):
    model.zero_grad(set_to_none=True)
    x = mixture.cuda().clone().requires_grad_(x_grad)
    out = model(x)
    assert out.requires_grad and out.shape == (mixture.shape[0], model.n_sources, mixture.shape[-1])
    if isinstance(drive, tuple):
        _crit(cfg, out, drive[0].cuda()).backward()
    else:
        out.backward(drive.cuda())
    return out.detach(), x.grad


def _run_case(case, drive_kind, mode, x_grad):
    e = EDGES[case]
    cfg, sd, mixture, sources, G = _setup(case)
    drive = (sources,) if drive_kind == "crit" else G
    out64, frames, g64, noise32, dx64, dxnoise = _reference((case, drive_kind), cfg, sd, mixture, drive)
    assert frames == e.frames, (case, frames)
    _assert_well_conditioned(g64, noise32)
    model = _build(cfg, sd, mode)
    out, dx = _step(model, mixture, drive, cfg, x_grad=x_grad)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    worst = _check_grads(model, g64, noise32)
    dx_share = None
    if x_grad:
        scale = float(dx64.abs().max())
        assert dxnoise <= GRAD_PER / 10 * scale, "ill-conditioned mixture gradient"
        err = float((dx.cpu().double() - dx64).abs().max())
        dx_share = err / (GRAD_PER * scale + GRAD_ATOL)
        assert err <= GRAD_PER * scale + GRAD_ATOL, "d_x: |err| {:.3e} = {:.2e} of its scale {:.3e}".format(err, err / scale, scale)
    else:
        assert dx is None
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL)
    print("[{} {} {}] worst gradient error {:.3f} of its bound ({}){} -- {}".format(
        case, drive_kind, mode, worst[0] / GRAD_PER, worst[1], "" if dx_share is None else ", d_x {:.3f} of its bound".format(dx_share),
        e.reaches))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(EDGES))
def test_gradients_vs_fp64(case, mode):
    """each EDGES row driven by a seeded cotangent with a mixture that requires grad: estimate == oracle, training forward ==
    inference forward, every gradient within 2e-4 of its role scale of fp64 and d_x within 2e-4 of its scale"""
    _run_case(case, "G", mode, x_grad=True)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", [k for k, e in EDGES.items() if e.shape["n_sources"] > 1])
def test_criterion_gradients_vs_fp64(case, mode):
    """the same rows driven by the recipes' criteria: ORPIT(NegSISDR()) over 3-speaker targets for two outputs, SinkPIT(NegSISDR())
    for five; the mixture does not require grad, so no d_x is formed"""
    _run_case(case, "crit", mode, x_grad=False)


# ---- the fine-tune step ----------------------------------------------------------------------------------------------------
def _finetune(model, mixture, sources):
    loss, ests = R.finetune_loss(model, mixture, sources, ORPIT(NegSISDR()))
    return loss, ests


@pytest.mark.parametrize("mode", MODES)
def test_finetune_two_stages_vs_oracle_and_golden(golden_dir, mode):
    """the ORPIT recipe's fine-tune step on 3-speaker targets (two stages, one backward; stage 2's gradient reaches stage 1 through
    d_x): loss and every gradient against the oracle running the same loop in fp64 and against the reference's fp64 golden; the
    two nodes share one flat bucket, so clip + Adam take the step"""
    r = torch.load(os.path.join(golden_dir, "tiny_softmax_grad.pt"), weights_only=False)["finetune"]
    cfg = O.OracleConfig(**r["cfg"])
    sd = O.synth_state_dict(cfg, seed=r["wseed"])
    model = _build(cfg, sd, mode)
    model.zero_grad(set_to_none=True)
    loss, ests = _finetune(model, r["mixture"].cuda(), r["sources"].cuda())
    loss.backward()
    assert len(ests) == 2
    torch.testing.assert_close(ests[0].detach().cpu(), r["out"], rtol=OUT_RTOL, atol=OUT_ATOL)
    assert abs(float(loss) - r["loss64"]) <= 1e-4 * abs(r["loss64"])
    worst = _check_grads(model, r["grads64"], r["fp32_vs_fp64_maxabs"])
    # the oracle running the same loop
    sdv = {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}
    loss64, _ = R.finetune_loss(lambda x: O.conv_tasnet_fwd(x, sdv, cfg)[0], r["mixture"].double(), r["sources"].double(),
                                lambda e, t: PV.orpit(e, t))
    loss64.backward()
    assert abs(float(loss) - float(loss64)) <= 1e-4 * abs(float(loss64))
    worst_o = _check_grads(model, {k: v.grad for k, v in sdv.items()}, r["fp32_vs_fp64_maxabs"])
    flat = model.last_flat_grad
    base, end = flat.data_ptr(), flat.data_ptr() + flat.numel() * 4
    assert all(base <= p.grad.data_ptr() < end for p in model.parameters())
    before = [p.detach().clone() for p in model.parameters()]
    FlatClipAdam(model, lr=1e-3, weight_decay=1e-5, max_norm=5.0).step()
    assert any(not torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))
    print("[finetune {}] worst gradient error {:.3f} of its bound vs the golden ({}), {:.3f} vs the oracle ({})".format(
        mode, worst[0] / GRAD_PER, worst[1], worst_o[0] / GRAD_PER, worst_o[1]))


@pytest.mark.parametrize("case", ["orpit", "sinkpit"])
def test_reference_golden(golden_dir, case):
    """tiny_softmax_grad.pt: ORPIT over a PackedSequence of 2- and 3-speaker targets, and SinkPIT at five outputs, in the default
    tensor-core mode: output, loss and every gradient against the reference's fp64 values"""
    from torch.nn.utils.rnn import pack_sequence
    r = torch.load(os.path.join(golden_dir, "tiny_softmax_grad.pt"), weights_only=False)[case]
    cfg = O.OracleConfig(**r["cfg"])
    model = _build(cfg, O.synth_state_dict(cfg, seed=r["wseed"]), MODES[-1])
    model.zero_grad(set_to_none=True)
    out = model(r["mixture"].cuda())
    if case == "orpit":
        loss, idx = ORPIT(NegSISDR())(out, pack_sequence([t.cuda() for t in r["targets"]], enforce_sorted=False))
        assert torch.equal(idx.cpu(), r["extra64"])
    else:
        loss, pattern = SinkPIT(NegSISDR(), n_sources=5)(out, r["sources"].cuda())
        assert torch.equal(pattern.cpu(), r["extra64"])
    loss.backward()
    torch.testing.assert_close(out.detach().cpu(), r["out"], rtol=OUT_RTOL, atol=OUT_ATOL)
    assert abs(float(loss) - r["loss64"]) <= 1e-4 * abs(r["loss64"])
    worst = _check_grads(model, r["grads64"], r["fp32_vs_fp64_maxabs"])
    print("[golden {}] worst gradient error {:.3f} of its bound ({})".format(case, worst[0] / GRAD_PER, worst[1]))


# ---- the ORPIT recipe shape ------------------------------------------------------------------------------------------------
RECIPE = dict(n_basis=512, kernel_size=16, stride=8, sep_hidden_channels=512, sep_bottleneck_channels=128, sep_skip_channels=128,
              sep_kernel_size=3, sep_num_blocks=3, sep_num_layers=8, n_sources=2)


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
def test_orpit_recipe_shape_trains():
    """egs/wsj0-mix/orpit_conv-tasnet/train.sh: 4 x 4 s at 8 kHz, f16x3, ORPIT over 3-speaker targets.  Finite gradients; the loss
    falls over 4 steps of FlatClipAdam(lr=1e-3, weight_decay=1e-5); launches equal the sigmoid step's of the same separator plus 1
    in the forward, the same in the backward, plus 1 more when the mixture requires grad"""
    cfg = O.OracleConfig(causal=False, mask_nonlinear="softmax", **RECIPE)
    sd = O.synth_state_dict(cfg, seed=621)
    g = torch.Generator().manual_seed(622)
    sources = (0.3 * torch.randn(4, 3, 32000, generator=g)).cuda()
    mixture = sources.sum(dim=1, keepdim=True)
    model = _build(cfg, sd, "f16x3")
    opt = FlatClipAdam(model, lr=1e-3, weight_decay=1e-5)
    losses = []
    for _ in range(4):
        opt.zero_grad()
        loss, _ = ORPIT(NegSISDR())(model(mixture), sources)
        loss.backward()
        assert all(bool(torch.isfinite(p.grad).all()) for p in model.parameters())
        opt.step()
        losses.append(float(loss))
    print("[orpit recipe steps] loss {}".format(", ".join("{:.4f}".format(v) for v in losses)))
    assert losses[-1] < losses[0], losses
    soft = (model.last_launches, model.last_bwd_launches)
    model.zero_grad(set_to_none=True)
    G = torch.randn(4, 2, 32000, device="cuda")
    model(mixture.clone().requires_grad_(True)).backward(G)
    soft_dx = model.last_bwd_launches
    scfg = O.OracleConfig(**dict(cfg.to_dict(), mask_nonlinear="sigmoid"))
    sig = _build(scfg, sd, "f16x3")
    sig.zero_grad(set_to_none=True)
    sig(mixture).backward(G)
    print("[orpit recipe launches] softmax {} / {} (+ d_x {}), sigmoid {} / {}".format(*soft, soft_dx, sig.last_launches,
                                                                                        sig.last_bwd_launches))
    assert soft == (sig.last_launches + 1, sig.last_bwd_launches)
    assert soft_dx == sig.last_bwd_launches + 1


# ---- contract --------------------------------------------------------------------------------------------------------------
def test_contract():
    cfg, sd, mixture, sources, G = _setup("S2-ragged-relu")
    x = mixture.cuda()
    model = _build(cfg, sd, None, switch=False)
    with pytest.raises(NotImplementedError, match="ctn_train_workspace_bytes"):  # switch off: refused as before
        model(x)
    with pytest.raises(NotImplementedError, match="mixture"):
        model(x.clone().requires_grad_(True))
    model.softmax_training = True
    out = model(x)
    out.backward(G.cuda(), retain_graph=True)
    with pytest.raises(RuntimeError, match="already run"):
        out.backward(G.cuda())
    out = model(x)
    with torch.no_grad():
        next(model.parameters()).add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.backward(G.cuda())
    for kw in (dict(causal=True), dict(in_channels=2)):
        c2 = O.OracleConfig(**dict(cfg.to_dict(), **kw))
        m2 = _build(c2, O.synth_state_dict(c2, seed=611), None)
        m2.causal_training = m2.multichannel_training = True
        with pytest.raises(NotImplementedError):
            m2(x if c2.in_channels == 1 else x.unsqueeze(2).expand(-1, -1, 2, -1).contiguous())


def test_switch_on_a_sigmoid_model_changes_nothing():
    cfg = O.OracleConfig(causal=False, **SMALL)
    sd = O.synth_state_dict(cfg, seed=631)
    mixture, _ = O.synth_batch(2, cfg.n_sources, 1037, seed=632)
    G = torch.randn(2, cfg.n_sources, 1037, generator=torch.Generator().manual_seed(633))
    res = []
    for flag in (False, True):
        m = _build(cfg, sd, None, switch=flag)
        out = m(mixture.cuda())
        out.backward(G.cuda())
        res.append((out.detach().cpu(), {k: p.grad.cpu() for k, p in m.named_parameters()}, m.last_launches, m.last_bwd_launches))
        with pytest.raises(NotImplementedError, match="mixture"):
            m(mixture.cuda().requires_grad_(True))
    assert res[0][2:] == res[1][2:]
    torch.testing.assert_close(res[0][0], res[1][0], rtol=1e-6, atol=1e-7)
    for k in res[0][1]:
        torch.testing.assert_close(res[0][1][k], res[1][1][k], rtol=1e-5, atol=1e-6 * float(res[0][1][k].abs().max()) + 1e-12)
