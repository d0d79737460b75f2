"""Edge shapes of the CAUSAL (cLN) training path (``-m gpu``): ctn_causal_fwd_train / ctn_causal_bwd against torch autograd over
the CPU oracle (oracle/convtasnet_oracle.py, causal=True) run in FLOAT64, at the shapes of test_train_edges_gpu.py's EDGES with
causal=True and three causal-only rows: a long sequence (several frames per thread of the 1024-thread cLN scans), a mixture
that starts in digital silence (frames of exactly zero cumulative variance, where the backward takes e_t = 0) and cLNs with
fewer channels than CLN_BWD_SLICES.  Then the kernels of the path one at a time at their edge widths and frame counts.

Criterion (fp32, tf32x3, f16x3), as test_train_edges_gpu.py: estimate within rtol 1e-4 / atol 2e-5 of fp64, training forward
equal to the inference forward, every gradient within 2e-4 of its role scale of fp64; failure messages carry the fp32 oracle's
own distance, which is printed for the silent-onset row but not asserted: that row is held to the bound whatever the fp32
oracle's conditioning (a PReLU input within rounding of 0 puts any fp32 evaluation on the other side of the kink; see KINK_FREE).

The silent-onset row's fp64 reference swaps the oracle's cLN for causal_train_ref.cln_conv, whose backward takes the kernels'
documented e_t = 0 at v_t <= 0: the oracle's own autograd differentiates sqrt at 0 there and returns NaN for the encoder weight.
"""
import collections
import ctypes as C

import pytest
import torch

import causal_train_ref as R
import convtasnet_oracle as O
from ctn_b200 import _native as N
from test_causal_train_gpu import _affine, _causal_model, _pitched, _st, expected_launches, probe_cdw_bwd, probe_cdw_train_fwd, \
    probe_cln_bwd, probe_cln_stats
from test_train_edges_gpu import EDGES, GRAD_ATOL, GRAD_PER, MID, MODES, OUT_ATOL, OUT_RTOL, TF32_L2, _oracle, _rel_l2, _role_scales, \
    _train_step
from test_train_gpu import _role

pytestmark = pytest.mark.gpu

Edge = collections.namedtuple("Edge", "shape batch T frames reaches")

CAUSAL_REACHES = {
    "E1": "L=40: k_encdec_wgrad_generic and k_decoder_generic; P=4 with all 3*d of padding on the left; X=10: dilation 512 > 99 "
          "frames, so only tap P-1 lands inside in k_cdw_train_fwd / k_cdw_bwd",
    "E2": "P=8 = CTN_MAX_P: k_cdw_bwd's w / acc / part arrays full",
    "E3": "Bc+Sc=144: two m-tiles of [Wo; Ws] and of its transpose; H=136; S*N=300; split_row 96; 129 frames; B=3",
    "E4": "one frame: n_t = C, every tap but P-1 reads padding",
    "E5": "128 frames, P=2, encoder ReLU",
    "E6": "33 frames at B=5: weight-gradient chunks cross samples; P=6",
    "E7": "L=20 / stride 10, P=7",
    "E8": "stride = L, P=1: no dilated taps",
    "E9": "S*N=2560 > F16_MAX_ROWS in the causal EPI_MASK tail",
}
ROWS = {k: Edge(e.shape, e.batch, e.T, e.frames, CAUSAL_REACHES[k]) for k, e in EDGES.items()}
ROWS.update({
    "C10": Edge(dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=48, sep_skip_channels=16,
                     sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=4, n_sources=2), 2, 64000, 7999,
                "7999 frames: 8 frames per thread in k_cln_scan and k_cln_bwd_scan, k_cln_bwd_sums with grid.x = 63; every PReLU "
                "slope 1"),
    "C11": Edge(dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=48, sep_skip_channels=16,
                     sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=4, n_sources=2), 2, 16000, 1999,
                "silent onset: sample 0 is 10000 zeros and a 500-sample fade-in, so cLN0 has 1249 frames of exactly zero variance "
                "(e_t = 0) over many scan segments, then frames of tiny variance; sample 1 unchanged"),
    "C12": Edge(dict(n_basis=6, kernel_size=16, sep_bottleneck_channels=4, sep_hidden_channels=7, sep_skip_channels=4,
                     sep_kernel_size=3, sep_num_blocks=2, sep_num_layers=3, n_sources=2), 2, 2000, 249,
                "N=6, H=7, Bc=Sc=4: every cLN runs with fewer than CLN_BWD_SLICES = 8 slices"),
})
# PReLU is not differentiable at 0: a pre-activation within rounding of 0 takes a different slope in fp32 and fp64 and moves
# every gradient upstream of it by up to ~1e-2 of its role scale.  C10 has 6.4M PReLU inputs, so at fp32 rounding several sit
# that close to 0 whatever the seed (seed 411: the fp32 oracle itself lands 1.6e-3 of its role scale from fp64, and the kernels
# in fp32 mode at the same distance).  Its slopes are set to 1, which removes the kink and keeps every slope gradient: the row
# is about the long scans, and the other rows cover the PReLU branches.
KINK_FREE = ("C10",)
SILENT = "C11"
SILENT_ZERO, SILENT_FADE = 10000, 500
ENC = "encoder.conv1d.weight"

_CACHE = {}


def _setup(case):
    e = ROWS[case]
    cfg = O.OracleConfig(causal=True, **e.shape)
    sd = _affine(O.synth_state_dict(cfg, seed=411))
    if case in KINK_FREE:
        sd = {k: torch.ones_like(v) if k.endswith("nonlinear1d.weight") or k == "separator.prelu.weight" else v for k, v in sd.items()}
    mixture, sources = O.synth_batch(e.batch, cfg.n_sources, e.T, seed=412)
    if case == SILENT:
        R.silent_onset_(mixture[0], SILENT_ZERO, SILENT_FADE)
    G = torch.randn(e.batch, cfg.n_sources, e.T, generator=torch.Generator().manual_seed(413))
    return cfg, sd, mixture, sources, G


def _reference(key, cfg, sd, mixture, drive, conv=False):
    """fp64 answer and the fp32 oracle's distance to it, once per (case, driver) for all modes; conv: the oracle's cLN replaced by
    the convention-aware causal_train_ref.cln_conv"""
    key = key + (conv,)
    if key not in _CACHE:
        with pytest.MonkeyPatch.context() as mp:
            if conv:
                mp.setattr(O, "cln", R.cln_conv)
            out64, frames, perm64, g64 = _oracle(cfg, sd, mixture, drive, torch.float64)
            _, _, perm32, g32 = _oracle(cfg, sd, mixture, drive, torch.float32)
        noise32 = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
        _CACHE[key] = (out64, frames, perm64, perm32, g64, noise32)
    return _CACHE[key]


def _check_grads(grads, g64, noise32, per=GRAD_PER, atol=GRAD_ATOL, skip=()):
    """per-tensor role-scaled check of {key: grad}; every failing tensor is listed in one message. Returns (worst ratio, key)."""
    group = _role_scales({k: v for k, v in g64.items() if k not in skip})
    worst, bad = (0.0, None), []
    for k, g in grads.items():
        if k in skip:
            continue
        g, r = g.detach().cpu().double(), g64[k]
        assert g.shape == r.shape, k
        scale = group[_role(k)]
        d = (g - r).abs()
        err = float(d.max())
        ratio = err / (scale + 1e-30)
        worst = max(worst, (ratio, k))
        if not err <= per * scale + atol:
            at = tuple(int(i) for i in torch.nonzero(d == d.max())[0]) if torch.isfinite(d).all() else "non-finite"
            bad.append("{}: |g-g64| {:.3e} at {} = {:.2e} of role scale {:.3e} (fp32 oracle: {:.2e})".format(
                k, err, at, ratio, scale, noise32[k] / (scale + 1e-30)))
    assert not bad, "{} tensor(s) over {:.0e} of their role scale:\n  ".format(len(bad), per) + "\n  ".join(bad)
    return worst


def _grads(model):
    return {k: p.grad for k, p in model.named_parameters()}


def _noise(g64, noise32):
    group = _role_scales(g64)
    return max((noise32[k] / (group[_role(k)] + 1e-30), k) for k in g64)


def _nan_workspace(model, batch, T):
    """hand the node a workspace full of NaN: every buffer the step reads must be written by the step"""
    need = C.c_size_t(0)
    N.check(N.ctn_causal_train_workspace_bytes(C.byref(model.native_config()), batch, T, C.byref(need)), "workspace")
    junk = torch.full((need.value // 4 + 256,), float("nan"), device="cuda")
    del junk  # the caching allocator hands the same block to the node's workspace


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(ROWS))
def test_causal_edge_gradients_vs_fp64(case, mode):
    """Each row (its `reaches` field names the causal branch and the constant that selects it), backward driven by a random
    cotangent over a NaN-filled workspace: estimate == fp64, training forward == inference forward, every gradient within 2e-4
    of its role scale of fp64, and the launch counts of DESIGN.md "Causal training"."""
    e = ROWS[case]
    cfg, sd, mixture, _, G = _setup(case)
    silent = case == SILENT
    out64, frames, _, _, g64, noise32 = _reference((case, "G"), cfg, sd, mixture, G, conv=silent)
    assert frames == e.frames, (case, frames)
    model = _causal_model(cfg, sd, mode)
    _nan_workspace(model, e.batch, e.T)
    out, _ = _train_step(model, mixture, G)
    launches = (model.last_launches, model.last_bwd_launches)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    grads = _grads(model)
    assert all(torch.isfinite(g).all() for g in grads.values()), [k for k, g in grads.items() if not torch.isfinite(g).all()]
    worst = _check_grads(grads, g64, noise32)
    assert launches == expected_launches(cfg, mode), launches
    with torch.no_grad():
        out_inf = model(mixture.cuda())
    torch.testing.assert_close(out, out_inf, rtol=OUT_RTOL, atol=OUT_ATOL)
    extra = ""
    if silent:
        # the oracle's own cLN: NaN for the encoder weight only; every other tensor equals the convention-aware reference's
        _, _, _, _, gp, noisep = _reference((case, "G"), cfg, sd, mixture, G)
        assert torch.isnan(gp[ENC]).any()
        assert all(torch.isfinite(v).all() for k, v in gp.items() if k != ENC)
        worst_p = _check_grads(grads, gp, noisep, skip=(ENC,))
        extra = "; vs the oracle's own cLN (encoder weight excluded) {:.2e} ({}); fp32 oracle {:.2e} of its role scale ({})".format(
            *worst_p, *_noise(g64, noise32))
    print("[{} {}] worst gradient error / role scale {:.2e} = {:.3f} of the bound ({}){} -- {}".format(
        case, mode, worst[0], worst[0] / GRAD_PER, worst[1], extra, e.reaches))


@pytest.mark.parametrize("case", list(ROWS))
def test_causal_edge_pit_gradients_vs_fp64(case):
    """Same rows driven by PIT(NegSISDR) (ctn_sisdr_pit_bwd in the loop) in the default tensor-core mode: permutation equal to
    the fp64 oracle's, gradients within 2e-4 of their role scale."""
    mode = MODES[-1]
    e = ROWS[case]
    cfg, sd, mixture, sources, _ = _setup(case)
    out64, _, perm64, perm32, g64, noise32 = _reference((case, "pit"), cfg, sd, mixture, (sources,), conv=case == SILENT)
    assert torch.equal(perm32, perm64)
    model = _causal_model(cfg, sd, mode)
    out, perm = _train_step(model, mixture, (sources,))
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    assert torch.equal(perm, perm64)
    worst = _check_grads(_grads(model), g64, noise32)
    assert (model.last_launches, model.last_bwd_launches) == expected_launches(cfg, mode)
    print("[{} {} PIT] worst gradient error / role scale {:.2e} = {:.3f} of the bound ({})".format(
        case, mode, worst[0], worst[0] / GRAD_PER, worst[1]))


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
@pytest.mark.parametrize("case", ["E3", "mid"])
def test_causal_tf32_training_vs_fp64(case):
    """Single-pass 'tf32' causal training: the PIT permutation of the fp64 oracle, the forward's 'tf32' tolerance (rtol 2e-2,
    atol 5e-3) and ||g - g64||_2 / ||g64||_2 <= TF32_L2, the bound measured on the gLN path.  'mid' is MID with causal=True."""
    if case == "mid":
        cfg = O.OracleConfig(causal=True, **MID)
        sd = O.synth_state_dict(cfg, seed=221)
        mixture, sources = O.synth_batch(2, cfg.n_sources, 8000, seed=222)
    else:
        cfg, sd, mixture, sources, _ = _setup(case)
    out64, _, perm64, _, g64, _ = _reference((case, "pit"), cfg, sd, mixture, (sources,))
    model = _causal_model(cfg, sd, "tf32")
    out, perm = _train_step(model, mixture, (sources,))
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=2e-2, atol=5e-3)
    assert torch.equal(perm, perm64)
    l2 = _rel_l2(model, g64)
    print("[{} causal tf32] relative L2 of the whole gradient vs fp64 {:.2e} (bound {:.0e})".format(case, l2, TF32_L2))
    assert l2 <= TF32_L2, l2


MAG_SHAPE = dict(n_basis=64, kernel_size=16, sep_hidden_channels=96, sep_bottleneck_channels=48, sep_skip_channels=32,
                 sep_num_blocks=2, sep_num_layers=4, n_sources=2)


@pytest.mark.skipif(not N.ctn_has_tcgen05(), reason="tensor-core family not built")
@pytest.mark.parametrize("mode", ["tf32x3", "f16x3"])
@pytest.mark.parametrize("kind,value", [("input", 1e-4), ("input", 1e3), ("cotangent", 2.0 ** -30)])
def test_causal_split_modes_are_robust_to_magnitudes(mode, kind, value):
    """The mixture at 1e-4 / 1e3 and the cotangent at 2^-30 (gradients around 1e-9 and below, the absolute floor scaled with it):
    estimate and every gradient within their bounds of fp64.  The causal contractions run on tf32 pieces in f16x3 too (DESIGN.md
    "Causal training"); fp16 pieces would flush the smallest of these gradients to zero."""
    cfg = O.OracleConfig(causal=True, **MAG_SHAPE)
    sd = _affine(O.synth_state_dict(cfg, seed=91))
    mixture, _ = O.synth_batch(2, 2, 3000, seed=92)
    G = torch.randn(2, cfg.n_sources, 3000, generator=torch.Generator().manual_seed(231))
    if kind == "input":
        mixture = mixture * value
    else:
        G = G * value
    out64, _, _, _, g64, noise32 = _reference(("mag", kind, value), cfg, sd, mixture, G)
    model = _causal_model(cfg, sd, mode)
    out, _ = _train_step(model, mixture, G)
    torch.testing.assert_close(out.cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL * (float(out64.abs().max()) if kind == "input" else 1.0))
    atol = GRAD_ATOL * (value if kind == "cotangent" else 1.0)
    worst = _check_grads(_grads(model), g64, noise32, atol=atol)
    print("[causal {} {}={:.3g}] worst gradient error / role scale {:.2e} = {:.3f} of the bound ({}); largest |g64| {:.2e}".format(
        mode, kind, value, worst[0], worst[0] / GRAD_PER, worst[1], max(float(v.abs().max()) for v in g64.values())))


ADD_PER = 1e-5


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", ["E6", SILENT])
def test_causal_gradients_are_additive_over_the_batch(case, mode):
    """With a fixed cotangent G the gradients of a batch equal the sum of the gradients of each sample run alone with G[b],
    within ADD_PER of the role scale: cLN statistics and scans stay per sample, and the weight gradients' cross-sample chunks
    add up.  E6: 33 frames at B = 5; C11: a silent-onset sample next to an ordinary one."""
    cfg, sd, mixture, _, G = _setup(case)
    model = _causal_model(cfg, sd, mode)
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
        if not err <= ADD_PER * group[_role(k)] + GRAD_ATOL:
            bad.append("{}: {:.3e} = {:.2e} of role scale".format(k, err, err / (group[_role(k)] + 1e-30)))
    assert not bad, "\n  ".join(bad)
    print("[causal additivity {} {}] worst difference / role scale {:.2e} ({})".format(case, mode, worst[0], worst[1]))


# ---- kernels one at a time ---------------------------------------------------------------------------------------
def _share(got, want, bound):
    return float(((got.double().cpu() - want).abs() / bound).max())


@pytest.mark.parametrize("kind", R.CLN_INPUTS)
@pytest.mark.parametrize("slope", [None, 0.25])
@pytest.mark.parametrize("Cc", R.CLN_CHANNELS)
@pytest.mark.parametrize("frames", R.CLN_FRAMES)
def test_cln_bwd_edges_vs_fp64(frames, Cc, slope, kind):
    """k_cln_step / k_cln_scan / k_cln_bwd_sums / k_cln_bwd_scan / k_cln_bwd_apply through the probes, with 1, 2 and 16 frames per
    scan thread, fewer and more channels than the 8 slices, a silent onset and a large DC offset: NaN in the pad lanes, dx
    aliasing dy, pad columns exactly 0, every output within its bound of causal_train_ref.cln_bwd."""
    dy, pre, gamma = R.cln_row(frames, Cc, slope, kind)
    B, eps = R.CLN_B, R.EPS_PROBE
    want = R.cln_bwd(dy.double(), pre.double(), gamma.double(), eps, slope)
    bound = R.cln_bwd_bounds(want, frames, slope)
    pitch = N.ctn_pitch(frames)
    d_pre, d_dy, d_g = _pitched(pre, pitch), _pitched(dy, pitch), gamma.cuda()
    d_a = None if slope is None else torch.tensor([slope], device="cuda")
    st = torch.full((B, frames, 2), float("nan"), dtype=torch.float64, device="cuda")
    N.check(probe_cln_stats(d_pre.data_ptr(), N.ptr(d_a), B, Cc, frames, pitch, eps, st.data_ptr(), None, _st()), "stats")
    S, Q, _ = R.cln_stats(pre.double() if slope is None else R.prelu(pre.double(), slope))
    torch.testing.assert_close(st.cpu(), torch.stack([S, Q], -1), rtol=1e-12, atol=1e-9 * float(Q.abs().max()) / frames)
    scratch = torch.full((18 * B * frames,), float("nan"), dtype=torch.float64, device="cuda")
    acc = torch.zeros(4, Cc, device="cuda")  # dgamma, dbeta, dslope, dbias
    N.check(probe_cln_bwd(d_dy.data_ptr(), d_pre.data_ptr(), d_dy.data_ptr(), N.ptr(d_a), d_g.data_ptr(), st.data_ptr(), eps,
                          scratch.data_ptr(), acc[0].data_ptr(), acc[1].data_ptr(), None if slope is None else acc[2].data_ptr(),
                          None if slope is None else acc[3].data_ptr(), B, Cc, frames, pitch, _st()), "cln_bwd")
    torch.cuda.synchronize()
    assert torch.equal(d_dy[:, :, frames:], torch.zeros_like(d_dy[:, :, frames:])), "padding of dx is not zero"
    got = dict(dpre=d_dy[:, :, :frames], dgamma=acc[0], dbeta=acc[1])
    if slope is not None:
        got["dslope"], got["dbias"] = acc[2, :1], acc[3]
    assert all(torch.isfinite(v).all() for v in got.values())
    worst = {k: _share(got[k], want[k], bound[k]) for k in bound}
    print("[cln_bwd frames={} C={} slope={} {}] error / bound: {}".format(frames, Cc, slope, kind, {k: round(v, 3) for k, v in worst.items()}))
    assert all(v <= 1.0 for v in worst.values()), worst


@pytest.mark.parametrize("B,Cc", R.CDW_BC)
@pytest.mark.parametrize("frames", R.CDW_FRAMES)
@pytest.mark.parametrize("dil", R.CDW_DIL)
@pytest.mark.parametrize("P", R.CDW_P)
def test_causal_depthwise_edges_vs_fp64(P, dil, frames, B, Cc):
    """k_cdw_train_fwd / k_cdw_bwd at P = 4, 6, 7 and 8 = CTN_MAX_P, dilations up to past the frame count: outputs start as NaN,
    pad columns exactly 0, u_pre, d_hn and d_wd within their bounds of causal_train_ref."""
    hpre, du, g1, b1, wd, bd = R.cdw_row(P, dil, frames, B, Cc)
    want = R.cdw_expect(hpre, du, g1, b1, wd, bd, dil)
    pitch = N.ctn_pitch(frames)
    d_h, d_du = _pitched(hpre, pitch), _pitched(du, pitch)
    d_a = torch.tensor([R.SLOPE_PROBE], device="cuda")
    st = torch.empty(B, frames, 2, dtype=torch.float64, device="cuda")
    mi = torch.full((B, frames, 2), float("nan"), device="cuda")
    N.check(probe_cln_stats(d_h.data_ptr(), d_a.data_ptr(), B, Cc, frames, pitch, R.EPS_PROBE, st.data_ptr(), mi.data_ptr(), _st()),
            "stats")
    dev = [t.cuda() for t in (g1, b1, wd, bd)]
    u = torch.full((B, Cc, pitch), float("nan"), device="cuda")
    N.check(probe_cdw_train_fwd(d_h.data_ptr(), u.data_ptr(), mi.data_ptr(), dev[0].data_ptr(), dev[1].data_ptr(), dev[2].data_ptr(),
                                dev[3].data_ptr(), d_a.data_ptr(), B, Cc, frames, pitch, P, dil, _st()), "cdw_train_fwd")
    dhn = torch.full((B, Cc, pitch), float("nan"), device="cuda")
    dwd = torch.zeros(Cc, P, device="cuda")
    N.check(probe_cdw_bwd(d_du.data_ptr(), d_h.data_ptr(), dhn.data_ptr(), mi.data_ptr(), dev[0].data_ptr(), dev[1].data_ptr(),
                          d_a.data_ptr(), dev[2].data_ptr(), dwd.data_ptr(), B, Cc, frames, pitch, P, dil, _st()), "cdw_bwd")
    torch.cuda.synchronize()
    for t in (u, dhn):
        assert torch.equal(t[:, :, frames:], torch.zeros_like(t[:, :, frames:])), "padding is not zero"
    got = dict(upre=u[:, :, :frames], dhn=dhn[:, :, :frames], dwd=dwd)
    worst = {k: _share(got[k], *want[k]) for k in want}
    print("[cdw P={} dil={} frames={} C={} B={}] error / bound: {}".format(P, dil, frames, Cc, B, {k: round(v, 3) for k, v in worst.items()}))
    assert all(v <= 1.0 for v in worst.values()), worst


def _cln_bwd_direct(dy, x, gamma, dx, eps):
    B, Cc, T = x.shape
    scratch = torch.empty(20 * B * T, dtype=torch.float64, device="cuda")
    dg = torch.zeros(2, Cc, device="cuda")
    N.check(N.ctn_cln_bwd(dy.data_ptr(), x.data_ptr(), gamma.data_ptr(), scratch.data_ptr(), dx.data_ptr(), dg[0].data_ptr(),
                          dg[1].data_ptr(), B, Cc, T, eps, _st()), "ctn_cln_bwd")
    torch.cuda.synchronize()
    return dict(dpre=dx, dgamma=dg[0], dbeta=dg[1])


def _offset_copy(t, offset):
    """a contiguous device copy of t whose storage starts `offset` floats past a 256-byte boundary"""
    buf = torch.full((t.numel() + 64,), float("nan"), device="cuda")
    v = buf[offset:offset + t.numel()].view(t.shape)
    v.copy_(t)
    return v


@pytest.mark.parametrize("T,offset", [(4097, 0), (1024, 1)])
def test_public_cln_bwd_edges(T, offset):
    """ctn_cln_bwd (pitch = T) and CumulativeLayerNorm1d under autograd at T = 4097 (5 frames per scan thread, a row that is not a
    multiple of 4), and at T = 1024 on storage one float past a 16-byte boundary: pitch % 4 == 0 but the pointers are
    misaligned, so k_cln_bwd_apply must take its scalar branch."""
    from ctn_b200.modules.norm import CumulativeLayerNorm1d
    B, Cc, eps = 2, 24, 1e-8
    g = torch.Generator().manual_seed(T + offset)
    x = torch.randn(B, Cc, T, generator=g) + 0.2
    dy = torch.randn(B, Cc, T, generator=g)
    gamma, beta = 1.0 + 0.3 * torch.randn(Cc, generator=g), 0.2 * torch.randn(Cc, generator=g)
    want = R.cln_bwd(dy.double(), x.double(), gamma.double(), eps)
    bound = R.cln_bwd_bounds(want, T, None)
    d_x, d_dy, d_dx = _offset_copy(x.cuda(), offset), _offset_copy(dy.cuda(), offset), _offset_copy(torch.zeros(B, Cc, T, device="cuda"), offset)
    assert (d_x.data_ptr() % 16 != 0) == (offset != 0)
    got = _cln_bwd_direct(d_dy, d_x, gamma.cuda(), d_dx, eps)
    worst = {k: _share(got[k], want[k], bound[k]) for k in bound}
    assert all(v <= 1.0 for v in worst.values()), worst
    # the module under autograd, on the same (possibly misaligned) input
    m = CumulativeLayerNorm1d(Cc, eps=eps)
    m.load_state_dict({"gamma": gamma.view(1, Cc, 1), "beta": beta.view(1, Cc, 1)})
    m = m.cuda()
    xd = d_x.detach().requires_grad_(True)
    y = m(xd)
    ref_y = R.cln_fwd(x.double(), gamma.double(), beta.double(), eps)
    torch.testing.assert_close(y.detach().double().cpu(), ref_y, rtol=1e-5, atol=1e-5 * float(ref_y.abs().max()))
    y.backward(d_dy)
    mod = dict(dpre=xd.grad, dgamma=m.gamma.grad.view(-1), dbeta=m.beta.grad.view(-1))
    worst_m = {k: _share(mod[k], want[k], bound[k]) for k in bound}
    print("[ctn_cln_bwd T={} offset={}] error / bound: direct {}, module {}".format(
        T, offset, {k: round(v, 3) for k, v in worst.items()}, {k: round(v, 3) for k, v in worst_m.items()}))
    assert all(v <= 1.0 for v in worst_m.values()), worst_m
