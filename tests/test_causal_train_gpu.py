"""Causal (cLN) training on the GPU (``-m gpu``): the cLN backward and causal depthwise kernels one at a time against fp64
(tests/causal_train_ref.py) with a bound from their fp32 arithmetic, the stand-alone CumulativeLayerNorm1d under autograd, and
the whole model (``model.causal_training = True``) against autograd over the oracle, the fp64 oracle at the paper size and the
reference's own backward (tests/golden/tiny_cln_grad.pt)."""
import ctypes as C
import os

import pytest
import torch

import causal_train_ref as R
import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import PIT1d
from ctn_b200.criterion.sdr import NegSISDR
from ctn_b200.modules.norm import CumulativeLayerNorm1d
from ctn_b200.optim import FlatClipAdam
from test_parity_gpu import build_model
from test_train_gpu import GRAD_RTOL, MODES, PAPER, SHAPES, _check_grads, _check_grads_vs_fp64, _oracle_grads, _oracle_grads64

pytestmark = pytest.mark.gpu

_fp, _i, _f = C.c_void_p, C.c_int, C.c_float


def _sig(name, *argtypes):
    fn = getattr(N.lib, name)
    fn.restype, fn.argtypes = C.c_int, list(argtypes)
    return fn


probe_cln_stats = _sig("ctn_probe_cln_stats", _fp, _fp, _i, _i, _i, _i, _f, _fp, _fp, _fp)
probe_cln_bwd = _sig("ctn_probe_cln_bwd", _fp, _fp, _fp, _fp, _fp, _fp, _f, _fp, _fp, _fp, _fp, _fp, _i, _i, _i, _i, _fp)
probe_cdw_train_fwd = _sig("ctn_probe_cdw_train_fwd", _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _i, _i, _i, _i, _i, _i, _fp)
probe_cdw_bwd = _sig("ctn_probe_cdw_bwd", _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _fp, _i, _i, _i, _i, _i, _i, _fp)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _pitched(x, pitch):
    """(B, C, T) -> device (B, C, pitch) with NaN in the padding"""
    B, Cc, T = x.shape
    p = torch.full((B, Cc, pitch), float("nan"), dtype=torch.float32, device="cuda")
    p[:, :, :T] = x.cuda()
    return p


def _ratio(got, want, mag, ulps, floor=1e-30):
    """worst |got - want| over the bound ulps * 2^-24 * mag"""
    return float(((got.double().cpu() - want).abs() / (ulps * R.U24 * mag + floor)).max())


FRAMES = [1, 127, 128, 129, 1003, 3999]


@pytest.mark.parametrize("slope", [None, 0.25])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Cc", [1, 20, 512])
@pytest.mark.parametrize("frames", FRAMES)
def test_cln_bwd_kernels_vs_fp64(frames, Cc, B, slope):
    if Cc == 512 and B == 3 and frames not in (129, 3999):
        pytest.skip("the large shape is covered at two frame counts")
    g = torch.Generator().manual_seed(frames * 7 + Cc + B)
    pre = torch.randn(B, Cc, frames, generator=g) + 0.3
    dy = torch.randn(B, Cc, frames, generator=g)
    gamma = 1.0 + 0.3 * torch.randn(Cc, generator=g)
    eps = 1e-8
    pitch = N.ctn_pitch(frames)
    want = R.cln_bwd(dy.double(), pre.double(), gamma.double(), eps, slope)
    d_pre, d_dy, d_g = _pitched(pre, pitch), _pitched(dy, pitch), gamma.cuda()
    d_a = None if slope is None else torch.tensor([slope], device="cuda")
    st = torch.empty(B, frames, 2, dtype=torch.float64, device="cuda")
    N.check(probe_cln_stats(d_pre.data_ptr(), N.ptr(d_a), B, Cc, frames, pitch, eps, st.data_ptr(), None, _st()), "stats")
    S, Q, _ = R.cln_stats(pre.double() if slope is None else R.prelu(pre.double(), slope))
    torch.testing.assert_close(st.cpu(), torch.stack([S, Q], -1), rtol=1e-12, atol=1e-9)
    scratch = torch.empty(18 * B * frames, dtype=torch.float64, device="cuda")
    acc = torch.zeros(4, max(Cc, 1), device="cuda")  # dgamma, dbeta, dslope, dbias
    # dx aliases dy, as the pipeline calls it
    N.check(probe_cln_bwd(d_dy.data_ptr(), d_pre.data_ptr(), d_dy.data_ptr(), N.ptr(d_a), d_g.data_ptr(), st.data_ptr(), eps,
                          scratch.data_ptr(), acc[0].data_ptr(), acc[1].data_ptr(), None if slope is None else acc[2].data_ptr(),
                          None if slope is None else acc[3].data_ptr(), B, Cc, frames, pitch, _st()), "cln_bwd")
    torch.cuda.synchronize()
    assert torch.equal(d_dy[:, :, frames:], torch.zeros_like(d_dy[:, :, frames:])), "padding of dx is not zero"
    mag = want["mag"]
    n_seq = 4 * ((frames + 1023) // 1024)  # terms a thread adds in fp32 before the block's double reduction
    # frames whose variance is exactly zero (one channel, frame 0) sit on the clamp: the kernel's float r = 1 / eps there
    worst = dict(dpre=_ratio(d_dy[:, :, :frames], want["dpre"], mag["dpre"], 24))
    worst["dgamma"] = _ratio(acc[0, :Cc], want["dgamma"], mag["dgamma"], 16 + n_seq)
    worst["dbeta"] = _ratio(acc[1, :Cc], want["dbeta"], mag["dbeta"], 8 + n_seq)
    if slope is not None:
        worst["dslope"] = _ratio(acc[2, :1], want["dslope"], mag["dslope"], 32 + n_seq)
        worst["dbias"] = _ratio(acc[3, :Cc], want["dbias"], mag["dbias"], 32 + n_seq)
    print("[cln_bwd frames={} C={} B={} slope={}] error / bound: {}".format(frames, Cc, B, slope, {k: round(v, 3) for k, v in worst.items()}))
    assert all(v <= 1.0 for v in worst.values()), worst


def test_cln_bwd_constant_input_is_finite():
    B, Cc, T = 2, 8, 64
    x = torch.full((B, Cc, T), 0.5, device="cuda")
    dy = torch.randn(B, Cc, T, device="cuda")
    dx, dg = torch.empty_like(x), torch.zeros(2, Cc, device="cuda")
    scratch = torch.empty(20 * B * T, dtype=torch.float64, device="cuda")
    N.check(N.ctn_cln_bwd(dy.data_ptr(), x.data_ptr(), torch.ones(Cc, device="cuda").data_ptr(), scratch.data_ptr(), dx.data_ptr(),
                          dg[0].data_ptr(), dg[1].data_ptr(), B, Cc, T, 1e-12, _st()), "ctn_cln_bwd")
    assert torch.isfinite(dx).all() and torch.isfinite(dg).all()


@pytest.mark.parametrize("shape", [(2, 5, 1), (3, 20, 129), (1, 512, 1003), (2, 24, 6, 25)])
def test_cln_module_autograd_vs_oracle(shape):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.randn(*shape, generator=g) + 0.2
    Cc = shape[1]
    gamma, beta = 1.0 + 0.3 * torch.randn(1, Cc, 1, generator=g), 0.2 * torch.randn(1, Cc, 1, generator=g)
    dy = torch.randn(*shape, generator=g)
    x64, g64, b64 = (t.double().requires_grad_(True) for t in (x, gamma, beta))
    flat = x64.reshape(shape[0], Cc, -1)
    (O.cln(flat, g64.view(-1), b64.view(-1), 1e-8).reshape(shape) * dy.double()).sum().backward()
    m = CumulativeLayerNorm1d(Cc, eps=1e-8)
    m.load_state_dict({"gamma": gamma, "beta": beta})
    m = m.cuda()
    xd = x.cuda().requires_grad_(True)
    y = m(xd)
    assert y.grad_fn is not None
    (y * dy.cuda()).sum().backward()
    for name, got, want in (("dx", xd.grad, x64.grad), ("dgamma", m.gamma.grad, g64.grad), ("dbeta", m.beta.grad, b64.grad)):
        torch.testing.assert_close(got.double().cpu(), want, rtol=1e-4, atol=1e-5 * float(want.abs().max()), msg=lambda s, n=name: n + ": " + s)
    with torch.no_grad():
        assert m(x.cuda()).grad_fn is None
    # parameters frozen, input needs grad: the gradient still flows
    m.gamma.requires_grad_(False), m.beta.requires_grad_(False)
    xd2 = x.cuda().requires_grad_(True)
    (m(xd2) * dy.cuda()).sum().backward()
    torch.testing.assert_close(xd2.grad, xd.grad)


@pytest.mark.parametrize("B,Cc", [(1, 1), (3, 20), (1, 512)])
@pytest.mark.parametrize("frames", FRAMES)
@pytest.mark.parametrize("P,dil", [(1, 1), (2, 8), (3, 128), (5, 1), (5, 8), (3, 1)])
def test_causal_depthwise_kernels_vs_fp64(P, dil, frames, B, Cc):
    g = torch.Generator().manual_seed(P * 100 + dil + frames + Cc)
    hpre = torch.randn(B, Cc, frames, generator=g) + 0.3
    du = torch.randn(B, Cc, frames, generator=g)
    g1, b1 = 1.0 + 0.3 * torch.randn(Cc, generator=g), 0.2 * torch.randn(Cc, generator=g)
    wd, bd = torch.randn(Cc, P, generator=g), torch.randn(Cc, generator=g)
    slope, eps = 0.25, 1e-8
    pitch = N.ctn_pitch(frames)
    h64 = R.prelu(hpre.double(), slope)
    hn = R.cln_fwd(h64, g1.double(), b1.double(), eps)
    u_ref = R.cdw_fwd(hn, wd.double(), bd.double(), dil)
    dhn_ref, dwd_ref, mhn, mwd = R.cdw_bwd(du.double(), hn, wd.double(), dil)
    d_h, d_du = _pitched(hpre, pitch), _pitched(du, pitch)
    d_a = torch.tensor([slope], device="cuda")
    st = torch.empty(B, frames, 2, dtype=torch.float64, device="cuda")
    mi = torch.empty(B, frames, 2, device="cuda")
    N.check(probe_cln_stats(d_h.data_ptr(), d_a.data_ptr(), B, Cc, frames, pitch, eps, st.data_ptr(), mi.data_ptr(), _st()), "stats")
    u = torch.full((B, Cc, pitch), float("nan"), device="cuda")
    dev = [t.cuda() for t in (g1, b1, wd, bd)]
    N.check(probe_cdw_train_fwd(d_h.data_ptr(), u.data_ptr(), mi.data_ptr(), dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(),
                                dev[3].data_ptr(), d_a.data_ptr(), B, Cc, frames, pitch, P, dil, _st()), "cdw_train_fwd")
    dhn = torch.full((B, Cc, pitch), float("nan"), device="cuda")
    dwd = torch.zeros(Cc, P, device="cuda")
    N.check(probe_cdw_bwd(d_du.data_ptr(), d_h.data_ptr(), dhn.data_ptr(), mi.data_ptr(), dev[0].data_ptr(), dev[1].data_ptr(),
                          d_a.data_ptr(), dev[2].data_ptr(), dwd.data_ptr(), B, Cc, frames, pitch, P, dil, _st()), "cdw_bwd")
    torch.cuda.synchronize()
    for t in (u, dhn):
        assert torch.equal(t[:, :, frames:], torch.zeros_like(t[:, :, frames:])), "padding is not zero"
    # hn carries the error of (x - m) r: 2^-24 (|x| + |m|) r |gamma| per element, folded into the bound through |hn| + that term
    S, Q, n = R.cln_stats(h64)
    m = S / n
    r = 1.0 / ((Q / n - m * m).clamp_min(0).sqrt() + eps)
    hn_mag = (h64.abs() + m.abs()[:, None]) * r[:, None] * g1.double().abs().view(1, -1, 1) + b1.double().abs().view(1, -1, 1)
    _, _, _, mwd_h = R.cdw_bwd(du.double(), hn_mag, wd.double().abs(), dil)
    u_mag = R.cdw_fwd(hn_mag, wd.double().abs(), bd.double().abs(), dil)
    n_seq = (frames + 255) // 256
    worst = dict(upre=_ratio(u[:, :, :frames], u_ref, u_mag, 8 + 2 * P), dhn=_ratio(dhn[:, :, :frames], dhn_ref, mhn, 2 + P, 1e-12),
                 dwd=_ratio(dwd, dwd_ref, mwd_h, 16 + n_seq, 1e-12))
    print("[cdw P={} dil={} frames={} C={} B={}] error / bound: {}".format(P, dil, frames, Cc, B, {k: round(v, 3) for k, v in worst.items()}))
    assert all(v <= 1.0 for v in worst.values()), worst


# ---- whole model -------------------------------------------------------------------------------------------------
def _causal_model(cfg, sd, mode=None):
    model = build_model(cfg, sd, math=mode).train()
    model.causal_training = True
    return model


def _affine(sd, seed=5):
    g = torch.Generator().manual_seed(seed)
    for k in sd:
        if k.endswith("gamma"):
            sd[k] = 1.0 + 0.3 * torch.randn(sd[k].shape, generator=g)
        elif k.endswith("beta"):
            sd[k] = 0.2 * torch.randn(sd[k].shape, generator=g)
    return sd


def expected_launches(cfg, mode):
    """DESIGN.md, "Causal training": g launches per 1x1 contraction, q for a block's two-part weight gradient"""
    g, q = (1, 2) if mode == "fp32" else (2, 1)
    RX = cfg.sep_num_blocks * cfg.sep_num_layers
    return 6 + 2 * g + RX * (9 + g), 19 + 2 * g + (RX - 1) * (14 + 2 * g + q) + (14 + 2 * g)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", SHAPES)
def test_model_gradients_vs_oracle_autograd(mode, shape):
    cfg = O.OracleConfig(causal=True, **shape)
    sd = _affine(O.synth_state_dict(cfg, seed=41))
    mixture, sources = O.synth_batch(3, cfg.n_sources, 1003, seed=42)
    ref_out, ref_loss, ref_perm, ref_grads = _oracle_grads(cfg, sd, mixture, sources)
    model = _causal_model(cfg, sd, mode)
    # a workspace full of NaN must change nothing: every buffer the step reads is written by the step
    need = C.c_size_t(0)
    N.check(N.ctn_causal_train_workspace_bytes(C.byref(model.native_config()), 3, 1003, C.byref(need)), "workspace")
    junk = torch.full((need.value // 4 + 256,), float("nan"), device="cuda")
    del junk  # the caching allocator hands the same block to the node's workspace
    out = model(mixture.cuda())
    assert out.requires_grad
    torch.testing.assert_close(out.detach().cpu(), ref_out, rtol=1e-4, atol=2e-5)
    fwd_launches = model.last_launches
    loss, perm = PIT1d(NegSISDR(), cfg.n_sources)(out, sources.cuda())
    assert torch.equal(perm.cpu(), ref_perm)
    torch.testing.assert_close(loss.detach().cpu(), ref_loss, rtol=0, atol=1e-4)
    loss.backward()
    worst = _check_grads(model, ref_grads, GRAD_RTOL)
    assert (fwd_launches, model.last_bwd_launches) == expected_launches(cfg, mode)
    assert model.last_flat_grad is not None
    print("[causal {} R={} X={}] worst relative gradient error {}; launches fwd {} bwd {}".format(
        mode, cfg.sep_num_blocks, cfg.sep_num_layers, worst, fwd_launches, model.last_bwd_launches))
    with torch.no_grad():  # the training forward and the inference forward are the same function
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out.detach(), out_inf, rtol=1e-4, atol=2e-5)


_PAPER_REF = {}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("S", [2, 3])
def test_paper_size_gradients_vs_fp64(mode, S):
    cfg = O.OracleConfig(causal=True, n_sources=S, **PAPER)
    sd = O.synth_state_dict(cfg, seed=113)
    mixture, sources = O.synth_batch(2, S, 8000, seed=113)
    if S not in _PAPER_REF:  # the CPU oracle's fp32 and fp64 backward, once for all modes
        _PAPER_REF[S] = _oracle_grads(cfg, sd, mixture, sources) + (_oracle_grads64(cfg, sd, mixture, sources),)
    ref_out, ref_loss, ref_perm, g32, g64 = _PAPER_REF[S]
    noise32 = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
    model = _causal_model(cfg, sd, mode)
    out = model(mixture.cuda())
    torch.testing.assert_close(out.detach().cpu(), ref_out, rtol=1e-4, atol=2e-5)
    loss, perm = PIT1d(NegSISDR(), S)(out, sources.cuda())
    assert torch.equal(perm.cpu(), ref_perm)
    torch.testing.assert_close(loss.detach().cpu(), ref_loss, rtol=0, atol=1e-4)
    loss.backward()
    assert len(g64) == 343
    g64max = {k: float(v.abs().max()) for k, v in g64.items()}
    worst, closer, l2 = _check_grads_vs_fp64([(k, p.grad.detach().cpu()) for k, p in model.named_parameters()], g64max, g64, noise32, mode)
    print("[causal paper size {} S={}] worst per-tensor error / role scale {:.2e} ({}); relative L2 of the whole gradient {:.2e}; "
          "at least as close to fp64 as the CPU fp32 oracle: {} / 343; launches fwd {} bwd {}".format(
              mode, S, worst[0], worst[1], l2, closer, model.last_launches, model.last_bwd_launches))
    assert (model.last_launches, model.last_bwd_launches) == expected_launches(cfg, mode)


def test_gradients_vs_reference_golden(golden_dir):
    rec = torch.load(os.path.join(golden_dir, "tiny_cln_grad.pt"), weights_only=False)
    cfg = O.OracleConfig(**rec["cfg"])
    assert cfg.causal
    sd = O.synth_state_dict(cfg, seed=rec["wseed"])
    mixture, sources = O.synth_batch(rec["batch"], cfg.n_sources, rec["T"], seed=rec["xseed"])
    model = _causal_model(cfg, sd)
    loss, perm = PIT1d(NegSISDR(), cfg.n_sources)(model(mixture.cuda()), sources.cuda())
    loss.backward()
    assert torch.equal(perm.cpu(), rec["perm"])
    torch.testing.assert_close(loss.detach().cpu(), rec["loss"], rtol=0, atol=1e-4)
    worst = (0.0, None)
    for k, p in model.named_parameters():
        r = rec["grads"][k]
        want, scale = r["sample64"].reshape(r["shape"]), r["absmax64"]
        err = float((p.grad.detach().cpu().double() - want).abs().max())
        # as close to the reference's fp64 backward as 2e-4 of the tensor's largest entry, or as the reference's own fp32 is
        assert err <= max(GRAD_RTOL * scale, 2 * r["fp32_vs_fp64_maxabs"]) + 1e-9, (k, err, scale, r["fp32_vs_fp64_maxabs"])
        worst = max(worst, (err / (scale + 1e-30), k))
    print("[causal golden] worst error vs the reference's fp64 backward / largest entry: {:.2e} ({})".format(*worst))


def test_autograd_node_contract():
    cfg = O.OracleConfig(n_basis=32, kernel_size=16, sep_hidden_channels=64, sep_bottleneck_channels=32, sep_skip_channels=32,
                         sep_num_blocks=1, sep_num_layers=2, causal=True, n_sources=2)
    sd = O.synth_state_dict(cfg, seed=3)
    mixture, sources = O.synth_batch(2, 2, 2000, seed=8)
    mixture, sources = mixture.cuda(), sources.cuda()
    crit = PIT1d(NegSISDR(), 2)
    off = build_model(cfg, sd).train()
    with pytest.raises(NotImplementedError, match="causal_training"):
        off(mixture)
    model = _causal_model(cfg, sd)
    loss, _ = crit(model(mixture), sources)
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError):
        loss.backward()
    loss, _ = crit(model(mixture), sources)
    with torch.no_grad():
        next(model.parameters()).add_(1.0)
    with pytest.raises(RuntimeError):
        loss.backward()
    with pytest.raises(NotImplementedError):
        model(mixture.clone().requires_grad_(True))


def test_native_steps_lower_the_loss_and_the_model_still_streams():
    """three clip + Adam steps on the flat gradient bucket; the stepped model's online stream equals its offline forward"""
    from test_online_gpu import ON_ATOL, ON_RTOL
    cfg = O.OracleConfig(n_basis=32, kernel_size=16, sep_hidden_channels=64, sep_bottleneck_channels=32, sep_skip_channels=32,
                         sep_num_blocks=2, sep_num_layers=3, causal=True, n_sources=2)
    model = _causal_model(cfg, O.synth_state_dict(cfg, seed=3))
    mixture, sources = O.synth_batch(4, 2, 4000, seed=8)
    mixture, sources = mixture.cuda(), sources.cuda()
    opt = FlatClipAdam(model, lr=1e-3, max_norm=5.0)
    crit = PIT1d(NegSISDR(), 2)
    losses = []
    for _ in range(4):
        opt.zero_grad()
        loss, _ = crit(model(mixture), sources)
        losses.append(loss.item())
        loss.backward()
        opt.step()
    assert losses[-1] < losses[0], losses
    model.eval()
    with torch.no_grad():
        off = model(mixture)
        sep = model.online(batch_size=4, max_chunk=50 * cfg.stride)
        ys = [sep.push(mixture[..., t:t + 50 * cfg.stride]) for t in range(0, 4000, 50 * cfg.stride)]
        z = sep.flush()
    D = cfg.kernel_size - cfg.stride
    s = torch.cat([torch.cat(ys, 2)[..., D:], z], 2)
    bound = ON_RTOL * off.double().abs() + ON_ATOL * float(off.abs().max())
    share = float(((s.double() - off.double()).abs() / bound).max())
    print("[causal train -> online] losses {}; stream vs offline {:.3g} of bound".format([round(v, 4) for v in losses], share))
    assert share <= 1.0
