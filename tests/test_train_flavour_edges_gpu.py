"""Edge rows of the SOFTMAX-MASK and MULTICHANNEL training steps, and batches with SILENT samples for every non-causal flavour
(``-m gpu``): the shared fwd_train / bwd of ctn_train.cu against torch autograd over the CPU oracle in FLOAT64, at the gLN step's
edge geometries (test_train_edges_gpu.EDGES).  Rows and inputs live in tests/flavour_edges_ref.py; each row's `reaches` names
the branch it selects.

  A. softmax rows E1, E2, E4 .. E9: the un-fused f16x3 step (P != 3) with the logits contraction, ctn_softmax_mask and
     k_softmax_mask_bwd; the mixture gradient d_x through k_decoder_generic, k_decoder<10,2> and uneven pads; S*N > F16_MAX_ROWS.
     Driven by a cotangent with the mixture requiring grad, and by ORPIT (3-speaker targets) / SinkPIT (S = 5).
  B. multichannel rows (C = 2) at E1, E2, E5, E6, E8 and S*N = 2560, every one with P != 3; a cotangent and the recipe's MSE.
  C. silent batches: an ordinary sample, one of exact zeros, a silent onset and a near-silent one, per flavour, with and
     without the encoder ReLU.
  D. single-pass 'tf32'.  E. operand magnitudes.  F. additivity over the batch.

Criterion (test_train_edges_gpu.py's): estimate within rtol 1e-4 / atol 2e-5 of fp64 and the training forward equal to the
inference forward; every gradient within 2e-4 of its role scale of fp64; d_x within 2e-4 of its largest fp64 entry; the fp32
oracle 10x inside the bound.  Launch counts: the softmax step is the sigmoid step of the same separator + 1 forward launch, + 1
backward launch when d_x is formed; the multichannel step launches what its monaural twin does.
"""
import pytest
import torch

import convtasnet_oracle as O
import flavour_edges_ref as R
import test_multichannel_train_gpu as MC
import test_softmax_train_gpu as SM
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import ORPIT, PIT1d, SinkPIT
from ctn_b200.criterion.sdr import NegSISDR
from test_train_edges_gpu import ADD_PER, GRAD_ATOL, GRAD_PER, MODES, OUT_ATOL, OUT_RTOL, TF32_L2, _assert_well_conditioned, \
    _check_grads, _magnitude_case, _rel_l2, _role_scales
from test_train_gpu import _role

pytestmark = pytest.mark.gpu

_CACHE = {}
_LAUNCHES = {}


def _reference(key, cfg, sd, mixture, drive, x_grad):
    """fp64 answer and the fp32 oracle's distances to it, once per (row, driver) for all modes:
    (out64, frames, g64, noise32, dx64, dx noise32 per sample, perm64, perm32)"""
    if key not in _CACHE:
        out64, frames, g64, dx64, perm64, _ = R.oracle(cfg, sd, mixture, drive, torch.float64, x_grad=x_grad)
        _, _, g32, dx32, perm32, _ = R.oracle(cfg, sd, mixture, drive, torch.float32, x_grad=x_grad)
        noise = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
        dxn = None if dx64 is None else (dx32.double() - dx64).abs().flatten(1).max(dim=1).values
        _CACHE[key] = (out64, frames, g64, noise, dx64, dxn, perm64, perm32)
    return _CACHE[key]


def _build(cfg, sd, mode):
    return MC._build(cfg, sd, mode) if cfg.in_channels > 1 else SM._build(cfg, sd, mode)


def _crit(cfg, out, target):
    if cfg.in_channels > 1:
        return R.MSE(out, target), None
    if cfg.mask_nonlinear == "softmax":
        if cfg.n_sources == 2:
            return ORPIT(NegSISDR())(out, target)
        loss, pattern = SinkPIT(NegSISDR(), n_sources=cfg.n_sources)(out, target)
        return loss, pattern
    return PIT1d(NegSISDR(), cfg.n_sources)(out, target)


def _step(cfg, model, mixture, drive, x_grad=False):
    """one training step: (estimate, d_x or None, permutation or None)"""
    model.zero_grad(set_to_none=True)
    x = mixture.cuda().clone().requires_grad_(x_grad)
    out = model(x)
    assert out.requires_grad and out.shape[:2] == (mixture.shape[0], cfg.n_sources)
    perm = None
    if isinstance(drive, tuple):
        loss, perm = _crit(cfg, out, drive[0].cuda())
        loss.backward()
        perm = None if perm is None else perm.cpu()
    else:
        out.backward(drive.cuda())
    return out.detach(), x.grad, perm


def _grads(model):
    return {k: p.grad.detach().double().cpu() for k, p in model.named_parameters()}


def _dx_share(dx, dx64, dxnoise, per=GRAD_PER, per_sample=False):
    """max |d_x - dx64| over its bound, per * (largest |dx64| entry) + GRAD_ATOL, the scale taken over the batch or per sample;
    asserts the fp32 oracle's own d_x 10x inside the bound"""
    err = (dx.cpu().double() - dx64).abs().flatten(1).max(dim=1).values
    mag = dx64.abs().flatten(1).max(dim=1).values
    scale = mag if per_sample else mag.max().expand_as(mag)
    bound = per * scale + GRAD_ATOL
    assert bool((dxnoise <= bound / 10).all()), "ill-conditioned mixture gradient: fp32 oracle {} of bound {}".format(dxnoise.tolist(),
                                                                                                                  bound.tolist())
    share = err / bound
    assert bool((share <= 1).all()), "d_x: error / bound per sample {}".format([round(float(s), 3) for s in share])
    return float(share.max())


def _twin_launches(cfg, sd, mixture, mode):
    """(forward, backward) launches of the sigmoid step of the same separator (softmax) or of the monaural twin (C > 1)"""
    key = (cfg.to_dict().__repr__(), mixture.shape, mode)
    if key not in _LAUNCHES:
        if cfg.in_channels > 1:
            _, twin = MC._mono_twin(cfg, sd)
            x = mixture[:, :, 0]
        else:
            twin = SM._build(O.OracleConfig(**dict(cfg.to_dict(), mask_nonlinear="sigmoid")), sd, mode)
            x = mixture
        twin.math = mode
        twin.zero_grad(set_to_none=True)
        out = twin(x.cuda())
        out.backward(torch.ones_like(out))
        _LAUNCHES[key] = (twin.last_launches, twin.last_bwd_launches)
    return _LAUNCHES[key]


def _assert_launches(cfg, sd, mixture, mode, model, x_grad):
    f, b = _twin_launches(cfg, sd, mixture, mode)
    if cfg.in_channels > 1:
        want = (f, b)
    else:
        want = (f + 1, b + (1 if x_grad else 0))
    got = (model.last_launches, model.last_bwd_launches)
    assert got == want, "launches {} != {} (sigmoid / monaural twin {})".format(got, want, (f, b))


def _run_row(key, cfg, sd, mixture, drive, mode, reaches, frames=None, x_grad=False, perm=False):
    out64, fr, g64, noise32, dx64, dxnoise, perm64, perm32 = _reference(key, cfg, sd, mixture, drive, x_grad)
    if frames is not None:
        assert fr == frames, (key, fr)
    _assert_well_conditioned(g64, noise32)
    model = _build(cfg, sd, mode)
    out, dx, p = _step(cfg, model, mixture, drive, x_grad)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    worst = _check_grads(model, g64, noise32)
    share = None
    if x_grad:
        share = _dx_share(dx, dx64, dxnoise)
    else:
        assert dx is None
    if perm and perm64 is not None:
        assert torch.equal(perm32, perm64)
        assert torch.equal(p, perm64), (p, perm64)
    _assert_launches(cfg, sd, mixture, mode, model, x_grad)
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL)
    group = _role_scales(g64)
    noise = max(noise32[k] / (group[_role(k)] + 1e-30) for k in g64)
    print("[{} {} {}] worst gradient error {:.3f} of the bound ({}){}; fp32 oracle {:.3f} of the bound -- {}".format(
        key[0], key[1], mode, worst[0] / GRAD_PER, worst[1], "" if share is None else ", d_x {:.3f} of its bound".format(share),
        noise / GRAD_PER, reaches))


# ---- A. softmax rows --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(R.SOFTMAX))
def test_softmax_edge_gradients_vs_fp64(case, mode):
    """each softmax row driven by a seeded cotangent, the mixture requiring grad: estimate, every gradient and d_x against fp64;
    launches = the sigmoid step's + 1 forward, + 1 backward for d_x"""
    e = R.SOFTMAX[case]
    cfg, sd, mixture, _, G = R.softmax_setup(case)
    _run_row(("softmax-" + case, "G"), cfg, sd, mixture, G, mode, e.reaches, frames=e.frames, x_grad=True)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(R.SOFTMAX))
def test_softmax_edge_criterion_gradients_vs_fp64(case, mode):
    """the same rows driven by ORPIT(NegSISDR()) over 3-speaker targets (two outputs) or SinkPIT(NegSISDR()) (five): the
    permutation of fp64, every gradient against fp64; no d_x, so the backward launches what the sigmoid step's does"""
    e = R.SOFTMAX[case]
    cfg, sd, mixture, sources, _ = R.softmax_setup(case)
    _run_row(("softmax-" + case, "crit"), cfg, sd, mixture, (sources,), mode, e.reaches, frames=e.frames, perm=True)


# ---- B. multichannel rows ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(R.MULTICHANNEL))
@pytest.mark.parametrize("driver", ["G", "mse"])
def test_multichannel_edge_gradients_vs_fp64(case, driver, mode):
    """each multichannel row driven by a seeded cotangent (B, S, C, T) and by the recipe's MeanSquaredError: estimate and every
    gradient against fp64; launches equal those of the monaural twin"""
    e = R.MULTICHANNEL[case]
    cfg, sd, mixture, sources, G = R.mc_setup(case)
    drive = G if driver == "G" else (sources,)
    _run_row(("mc-" + case, driver), cfg, sd, mixture, drive, mode, e.reaches, frames=e.frames)


# ---- C. silent batches ------------------------------------------------------------------------------------------------------
# (flavour, driver): PIT(NegSISDR) for the sigmoid mask, a cotangent with d_x and ORPIT for softmax, MSE for C = 2
SILENT_CASES = [("gln", "crit"), ("softmax", "G"), ("softmax", "crit"), ("mc", "crit")]


def _per_sample_out(out, out64):
    """each sample within rtol 1e-4 of fp64 and atol 2e-5 of its own largest entry: the near-silent sample's estimate is ~1e-5"""
    for b in range(out.shape[0]):
        mag = float(out64[b].abs().max())
        if mag == 0.0:
            continue
        torch.testing.assert_close(out[b].cpu(), out64[b].float(), rtol=OUT_RTOL, atol=OUT_ATOL * mag, msg=lambda m: "sample {}: {}".format(b, m))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("relu", [False, True], ids=["linear", "relu"])
@pytest.mark.parametrize("flavour,driver", SILENT_CASES)
def test_silent_batch_vs_fp64(flavour, driver, relu, mode):
    """a batch of an ordinary sample, one of exact zeros, a silent onset and a near-silent one: the zero sample's estimate is
    bit-for-bit 0; every gradient finite and within 2e-4 of its role scale of fp64; each sample's estimate at its own scale;
    softmax with a cotangent: d_x per sample within 2e-4 of the sample's largest fp64 entry, the silent-onset frames included"""
    cfg, sd, mixture, sources, G = R.silent_batch(flavour, relu)
    drive = G if driver == "G" else (sources,)
    x_grad = driver == "G"
    out64, frames, g64, noise32, dx64, dxnoise, _, _ = _reference(("silent", flavour, driver, relu), cfg, sd, mixture, drive, x_grad)
    assert frames == R.SILENT_FRAMES
    assert torch.equal(out64[R.ZERO], torch.zeros_like(out64[R.ZERO]))
    _assert_well_conditioned(g64, noise32)
    model = _build(cfg, sd, mode)
    out, dx, _ = _step(cfg, model, mixture, drive, x_grad)
    assert torch.equal(out[R.ZERO], torch.zeros_like(out[R.ZERO])), "the silent sample's estimate is not exactly 0"
    grads = _grads(model)
    assert all(torch.isfinite(g).all() for g in grads.values()), [k for k, g in grads.items() if not torch.isfinite(g).all()]
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    _per_sample_out(out, out64)
    worst = _check_grads(model, g64, noise32)
    share = None
    if x_grad:
        assert bool(torch.isfinite(dx).all())
        share = _dx_share(dx, dx64, dxnoise, per_sample=True)
        if relu:  # windows of exact zeros: w_pre = 0, relu'(0) = 0 -- the zero sample's d_x is exactly 0
            assert torch.equal(dx[R.ZERO].cpu(), torch.zeros_like(dx[R.ZERO].cpu()))
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    assert torch.equal(out_inf[R.ZERO], torch.zeros_like(out_inf[R.ZERO]))
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL)
    group = _role_scales(g64)
    noise = max(noise32[k] / (group[_role(k)] + 1e-30) for k in g64)
    print("[silent {} {} relu={} {}] worst gradient error {:.3f} of the bound ({}){}; fp32 oracle {:.3f} of the bound -- {}".format(
        flavour, driver, relu, mode, worst[0] / GRAD_PER, worst[1], "" if share is None else ", d_x {:.3f} of its bound".format(share),
        noise / GRAD_PER, R.SILENT_REACHES))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("relu", [False, True], ids=["linear", "relu"])
@pytest.mark.parametrize("flavour", R.FLAVOURS)
def test_silent_sample_contributes_nothing(flavour, relu, mode):
    """with a fixed cotangent, the gradients of the silent batch equal those of the same batch without its zero sample within
    ADD_PER of the role scale (d_mask = d_what w = 0, the decoder's G x w_hat = 0 and the encoder's d_w x x = 0), and for
    softmax every other sample's d_x is unchanged"""
    cfg, sd, mixture, _, G = R.silent_batch(flavour, relu)
    keep = [b for b in range(mixture.shape[0]) if b != R.ZERO]
    x_grad = flavour == "softmax"
    model = _build(cfg, sd, mode)
    out, dx, _ = _step(cfg, model, mixture, G, x_grad)
    with_zero = _grads(model)
    out_k, dx_k, _ = _step(cfg, model, mixture[keep], G[keep], x_grad)
    without = _grads(model)
    group = _role_scales(with_zero)
    worst, bad = (0.0, None), []
    for k in with_zero:
        err = float((with_zero[k] - without[k]).abs().max())
        worst = max(worst, (err / (group[_role(k)] + 1e-30), k))
        if not err <= ADD_PER * group[_role(k)] + GRAD_ATOL:
            bad.append("{}: {:.3e} = {:.2e} of role scale".format(k, err, err / (group[_role(k)] + 1e-30)))
    assert not bad, "\n  ".join(bad)
    torch.testing.assert_close(out[keep], out_k, rtol=OUT_RTOL, atol=OUT_ATOL)
    if x_grad:
        for i, b in enumerate(keep):
            scale = float(dx[b].abs().max())
            assert float((dx[b] - dx_k[i]).abs().max()) <= ADD_PER * scale + GRAD_ATOL, b
    print("[silent additivity {} relu={} {}] worst difference / role scale {:.2e} ({})".format(flavour, relu, mode, *worst))


# ---- D. single-pass tf32 ----------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
@pytest.mark.parametrize("flavour", ["softmax", "mc"])
def test_tf32_training_vs_fp64(flavour):
    """single-pass 'tf32' at E7 (softmax, ORPIT: its permutation equals fp64's) and E2 (C = 2, MSE): the forward's 'tf32'
    tolerance (rtol 2e-2, atol 5e-3) and ||g - g64||_2 / ||g64||_2 <= TF32_L2"""
    if flavour == "softmax":
        cfg, sd, mixture, sources, _ = R.softmax_setup("E7")
        key = ("softmax-E7", "crit")
    else:
        cfg, sd, mixture, sources, _ = R.mc_setup("E2")
        key = ("mc-E2", "mse")
    out64, _, g64, _, _, _, perm64, _ = _reference(key, cfg, sd, mixture, (sources,), False)
    model = _build(cfg, sd, "tf32")
    out, _, perm = _step(cfg, model, mixture, (sources,))
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=2e-2, atol=5e-3)
    if perm64 is not None:
        assert torch.equal(perm, perm64)
    l2 = _rel_l2(model, g64)
    print("[{} tf32] relative L2 of the whole gradient vs fp64 {:.2e} (bound {:.0e})".format(key[0], l2, TF32_L2))
    assert l2 <= TF32_L2, l2


# ---- E. magnitudes ----------------------------------------------------------------------------------------------------------
MAGNITUDES = [("softmax", "input", 1e-4), ("softmax", "input", 1e3), ("softmax", "residual", 1e-3), ("softmax", "residual", 1e4),
              ("mc", "input", 1e-4), ("mc", "input", 1e3)]


def _magnitude_setup(flavour, kind, value):
    if flavour == "softmax":  # test_train_edges_gpu's perturbations with a softmax mask: the TCN and its PReLU inputs unchanged
        cfg, sd, mixture, floor = _magnitude_case(kind, value)
        cfg = O.OracleConfig(**dict(cfg.to_dict(), mask_nonlinear="softmax"))
    else:
        cfg, sd, mixture, _, _ = R.mc_setup("E5")
        mixture, floor = mixture * value, 1e-30
    # cotangent seed 231 as test_train_edges_gpu.py, except softmax: with the mixture at 1e3 it puts the output PReLU's slope
    # gradient on the kink (the fp32 oracle 1.4e-4 of its role scale from fp64); 233 leaves the fp32 oracle at 1.7e-6
    seed = 233 if flavour == "softmax" else 231
    G = torch.randn(mixture.shape[:1] + (cfg.n_sources,) + mixture.shape[2:], generator=torch.Generator().manual_seed(seed))
    return cfg, sd, mixture, floor, G


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
@pytest.mark.parametrize("mode", ["tf32x3", "f16x3"])
@pytest.mark.parametrize("flavour,kind,value", MAGNITUDES)
def test_split_modes_are_robust_to_magnitudes(flavour, kind, value, mode):
    """softmax: the mixture at 1e-4 / 1e3 and the residual stream and skip sum at 1e-3 / 1e4 (the mask weight divided by the same
    factor), with d_x; C = 2: the mixture at 1e-4 / 1e3.  Estimate at the scaled tolerance; gradients and d_x within 2e-4 of
    their scale of fp64, or twice the fp32 oracle's own worst distance where that is larger"""
    cfg, sd, mixture, floor, G = _magnitude_setup(flavour, kind, value)
    x_grad = flavour == "softmax"
    out64, _, g64, noise32, dx64, dxnoise, _, _ = _reference((flavour, kind, value, "G"), cfg, sd, mixture, G, x_grad)
    group = _role_scales(g64)
    per = max(GRAD_PER, 2 * max(noise32[k] / (group[_role(k)] + 1e-30) for k in g64))
    model = _build(cfg, sd, mode)
    out, dx, _ = _step(cfg, model, mixture, G, x_grad)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL * max(floor, float(out64.abs().max())))
    worst = _check_grads(model, g64, noise32, per=per)
    share = None
    if x_grad:
        scale = float(dx64.abs().max())
        dper = max(GRAD_PER, 2 * float(dxnoise.max()) / scale)
        share = _dx_share(dx, dx64, torch.zeros_like(dxnoise), per=dper)
    print("[{} {} {}={}] worst gradient error / role scale {:.2e} ({}), bound {:.1e}{}".format(
        flavour, mode, kind, value, worst[0], worst[1], per, "" if share is None else ", d_x {:.3f} of its bound".format(share)))


# ---- F. additivity over the batch ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("flavour", ["softmax", "mc"])
def test_gradients_are_additive_over_the_batch(flavour, mode):
    """E6 (B = 5, 33 frames: 32-frame chunks cross sample boundaries) with a fixed cotangent: the gradients of the batch equal
    the sum of those of each sample run alone within ADD_PER of the role scale; softmax: each sample's d_x equals its own run's"""
    if flavour == "softmax":
        cfg, sd, mixture, _, G = R.softmax_setup("E6")
    else:
        cfg, sd, mixture, _, G = R.mc_setup("E6")
    assert mixture.shape[0] == 5
    x_grad = flavour == "softmax"
    model = _build(cfg, sd, mode)
    _, dx, _ = _step(cfg, model, mixture, G, x_grad)
    batch = _grads(model)
    alone = {k: torch.zeros_like(v) for k, v in batch.items()}
    dx_alone = []
    for b in range(mixture.shape[0]):
        _, dxb, _ = _step(cfg, model, mixture[b:b + 1], G[b:b + 1], x_grad)
        dx_alone.append(dxb)
        for k, v in _grads(model).items():
            alone[k] += v
    group = _role_scales(batch)
    worst, bad = (0.0, None), []
    for k in batch:
        err = float((batch[k] - alone[k]).abs().max())
        worst = max(worst, (err / (group[_role(k)] + 1e-30), k))
        if not err <= ADD_PER * group[_role(k)] + GRAD_ATOL:
            bad.append("{}: {:.3e} = {:.2e} of role scale".format(k, err, err / (group[_role(k)] + 1e-30)))
    assert not bad, "\n  ".join(bad)
    dx_worst = 0.0
    if x_grad:
        scale = float(dx.abs().max())
        dx_worst = float((dx - torch.cat(dx_alone)).abs().max()) / scale
        assert dx_worst <= ADD_PER, dx_worst
    print("[{} additivity {}] worst difference / role scale {:.2e} ({}); d_x {:.2e} of its scale".format(flavour, mode, *worst, dx_worst))
