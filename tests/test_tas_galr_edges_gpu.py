"""LSTM-TasNet's and GALRNet's kernels at their own edges against fp64 (tests/tas_galr_edges_ref.py), every bound taken per unit:
per (sequence, direction) for the recurrence, per sample and per (sample, frame) for the encoder and frame norm, per (sample,
chunk) for the globally attentive block, per sample for the GALR head, per (sample, source) for the models.

The recurrence's rows come from the geometry restated for this device's SM count and opt-in shared memory: H where U steps and
the last CTA owns one unit, the largest H, passes of `ctn_tas_lstm_group` sequences up to three of them, 1 to 49 steps around the
16-step prefetch tiles.  The GALR rows put Q and K around the down- and up-map's passes of 2048 / F rows and their 32-row staging
tiles.  Every entry row runs twice on outputs and workspaces pre-filled with NaN and must give the same bits with zero pad columns;
every refusal comes before any launch.  Each row prints its worst unit error over its bound."""
import pytest
import torch

import galrnet_ref as GR
import lstm_tasnet_ref as LR
import tas_galr_edges_ref as E
import tas_online_ref as O
from ctn_b200 import _native as N
from ctn_b200.models.galrnet import GALRNet
from ctn_b200.models.tasnet import TasNet
from test_tas_online_gpu import build as online_model, row as online_row, signal, sizes, stream, whole

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def device_limits():
    """(SMs, opt-in shared memory per block) of cuda:0; the H100 SXM's where there is no device (the rows are then skipped)"""
    if torch.cuda.is_available():
        p = torch.cuda.get_device_properties(0)
        return p.multi_processor_count, p.shared_memory_per_block_optin
    return E.H100_SMS, E.H100_SMEM_OPTIN


SMS, OPTIN = device_limits()


def nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device=DEV)


def nan_ws(nbytes):
    buf = torch.full(((int(nbytes) + 512) // 4 + 1,), float("nan"), dtype=torch.float32, device=DEV).view(torch.uint8)
    return N.aligned(buf), buf


def st():
    return N.stream_ptr(DEV)


def dev(t):
    return t.contiguous().to(DEV)


def twice(run, shapes, nbytes):
    """run(outs, base, nbytes) -> status, twice on fresh NaN outputs ((shape, dtype) each) and a fresh NaN workspace; the two
    results must agree bit for bit.  Returns the first call's outputs on the host and its launch count."""
    results, counts = [], []
    for _ in range(2):
        outs = [nan(*s) for s in shapes]
        (base, nb), keep = nan_ws(nbytes)
        N.check(run(outs, base, nb), "entry")
        counts.append(N.ctn_last_launch_count())
        torch.cuda.synchronize()
        results.append([o.cpu() for o in outs])
        del keep
    for a, b in zip(*results):
        assert torch.equal(a, b)
    assert counts[0] == counts[1]
    return results[0], counts[0]


def report(what, name, ratio, extra=""):
    print("[tas/galr edges] {:10s} {:44s} worst unit error / bound {:.3g} {}".format(what, name, ratio, extra))


def check(out, ref, lead, rel=E.D.BOUND_REL):
    E.check(out, ref, lead, rel)
    return E.excess(out, ref, lead, rel)


# ---- the recurrence (ctn_tas_lstm_fwd) ---------------------------------------------------------------------------------------------
LSTM_ROWS = E.lstm_rows(SMS, OPTIN)


def test_geometry_matches_the_device():
    for dirs in (1, 2):
        assert N.ctn_tas_lstm_max_hidden(dirs) == E.lstm_max_hidden(dirs, SMS, OPTIN)
        for label, H in E.hidden_rows(dirs, SMS, OPTIN) + [("500", 500)]:
            g = E.lstm_geo(H, dirs, SMS, OPTIN)
            assert N.ctn_tas_lstm_group(H, dirs) == g["group"], (dirs, H)
            print("[tas/galr edges] geometry SMs={} smem={} dirs={} H={}({}) U={} cpd={} nu={} group={}".format(
                SMS, OPTIN, dirs, label, H, g["U"], g["cpd"], g["nu"], g["group"]))


def run_lstm(x, ws, B, F, H, dirs, T, mode, skip=None):
    """(out, skip_out or None) on the host, (B, dirs H, pitch), with their pad columns checked; and the launch count"""
    pitch = N.ctn_pitch(T)
    xp = torch.zeros(B, F, pitch)
    xp[..., :T] = x
    xd = dev(xp)
    wd = [dev(t) for t in ws]
    wp = (N._fp * len(wd))(*[t.data_ptr() for t in wd])
    sk = None
    if skip is not None:
        sk = torch.zeros(B, dirs * H, pitch)
        sk[..., :T] = skip
        sk = dev(sk)
    shapes = [((B, dirs * H, pitch),)] * (2 if skip is not None else 1)

    def run(o, base, nb):
        return N.ctn_tas_lstm_fwd(xd.data_ptr(), wp, o[0].data_ptr(), N.ptr(sk), o[1].data_ptr() if skip is not None else None, B, F, H, dirs,
                                  T, pitch, N.MATH_NAMES[mode], base, nb, st())
    outs, n = twice(run, shapes, N.ctn_tas_lstm_workspace_bytes(B, F, H, dirs, pitch, N.MATH_NAMES[mode]))
    for o in outs:
        assert not o[..., T:].any()
    return outs[0], (outs[1] if skip is not None else None), n


@pytest.mark.parametrize("name", list(LSTM_ROWS))
def test_lstm_entry(name):
    r = LSTM_ROWS[name]
    B, F, H, dirs, T, mode = r["B"], r["F"], r["H"], r["dirs"], r["T"], r["mode"]
    geo = E.lstm_geo(H, dirs, SMS, OPTIN)
    ws = E.lstm_weights(F, H, dirs, F + H + T)
    x = E.lstm_input(r, B + T)
    skip = torch.randn(B, dirs * H, T, generator=torch.Generator().manual_seed(T)) if r["skip"] else None
    out, skip_out, n = run_lstm(x, ws, B, F, H, dirs, T, mode, skip)
    assert n == 3 + (mode != "fp32")
    ref = E.lstm_answer(x, ws, dirs, geo)
    u = lambda y: E.lstm_units(y, B, dirs, H)  # noqa: E731
    ratio = check(u(out[..., :T]), u(ref), 2, E.rel_of(mode))
    if skip is not None:
        ratio = max(ratio, check(u(skip_out[..., :T]), u(ref + skip.double()), 2, E.rel_of(mode)))
    if r["alone"]:
        for b in range(B):
            one, _, _ = run_lstm(x[b:b + 1], ws, 1, F, H, dirs, T, mode)
            assert torch.equal(one[0], out[b]), "sequence {} of {} differs from its run alone".format(b, B)
    report("lstm", name, ratio, "{} SMs U={} nu={} group={} passes={}".format(SMS, geo["U"], geo["nu"], geo["group"], -(-B // geo["group"])))


@pytest.mark.parametrize("dirs", [1, 2])
def test_lstm_entry_refuses_past_the_largest_hidden_before_launch(dirs):
    H, F, T, B = E.lstm_max_hidden(dirs, SMS, OPTIN) + 1, 8, 4, 1
    pitch = N.ctn_pitch(T)
    x, out = torch.zeros(B, F, pitch, device=DEV), torch.zeros(B, dirs * H, pitch, device=DEV)
    wd = [dev(t) for t in E.lstm_weights(F, H, dirs, 1)]
    wp = (N._fp * len(wd))(*[t.data_ptr() for t in wd])
    ws = torch.empty(N.ctn_tas_lstm_workspace_bytes(B, F, H, dirs, pitch, N.MATH_FP32) + 256, dtype=torch.uint8, device=DEV)
    base, nb = N.aligned(ws)
    torch.cuda.synchronize()
    assert N.ctn_tas_lstm_fwd(x.data_ptr(), wp, out.data_ptr(), None, None, B, F, H, dirs, T, pitch, N.MATH_FP32, base, nb,
                              st()) == N.CTN_EUNSUPPORTED
    assert N.ctn_last_launch_count() == 0


# ---- the gated encoder + frame norm (ctn_tas_enc_gated_fwd) ------------------------------------------------------------------------
ENC_ROWS = E.enc_rows()


def run_enc(x, p, N_, L, stride, pl, pr, eps=1e-12):
    """w, xn (B, N, pitch) and nrm (B,) on the host, pad columns checked, launches checked"""
    B, _, T = x.shape
    frames = (T + pl + pr - L) // stride + 1
    pitch = N.ctn_pitch(frames)
    xd = dev(x)
    d = {k: dev(v) for k, v in p.items()}

    def run(o, base, nb):
        return N.ctn_tas_enc_gated_fwd(xd.data_ptr(), d["encoder.conv1d_U.weight"].data_ptr(), d["encoder.conv1d_V.weight"].data_ptr(),
                                       d["separator.gamma"].data_ptr(), d["separator.beta"].data_ptr(), o[0].data_ptr(), o[1].data_ptr(),
                                       o[2].data_ptr(), B, T, pl, pr, N_, L, stride, pitch, 1e-12, eps, st())
    (w, xn, nrm), n = twice(run, [((B, N_, pitch),), ((B, N_, pitch),), ((B,), torch.float64)], 0)
    assert n == 2
    assert not w[..., frames:].any() and not xn[..., frames:].any()
    return w[..., :frames], xn[..., :frames], nrm


def enc_check(name, x, p, r, w, xn, nrm):
    rw, rxn = E.enc_answer(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12)
    ratio = max(check(w, rw, 1), check(xn.permute(0, 2, 1), rxn.permute(0, 2, 1), 2))
    rn = E.signal_norm(x, r["L"], r["stride"], r["pl"], r["pr"]).view(-1)
    assert float(((nrm - rn).abs() / (rn + 1e-300)).max()) < 1e-10
    report("encoder", name, ratio)


@pytest.mark.parametrize("name", list(ENC_ROWS))
def test_gated_encoder_entry(name):
    r = ENC_ROWS[name]
    p = E.enc_params(r["N"], r["L"], r["N"] + r["L"])
    x = E.enc_input(r, r["T"])
    w, xn, nrm = run_enc(x, p, r["N"], r["L"], r["stride"], r["pl"], r["pr"])
    enc_check(name, x, p, r, w, xn, nrm)


def test_gated_encoder_largest_channels_and_one_past():
    L, stride, pl, pr = 40, 20, 3, 5
    Nmax = E.enc_max_n(L, stride, OPTIN)
    r = dict(B=2, T=L + 30 * stride + 11, N=Nmax, L=L, stride=stride, pl=pl, pr=pr, amps=None, clicks=())
    p = E.enc_params(Nmax, L, 1)
    x = E.enc_input(r, 2)
    w, xn, nrm = run_enc(x, p, Nmax, L, stride, pl, pr)
    enc_check("40/20 N={} (largest)".format(Nmax), x, p, r, w, xn, nrm)
    p = {k: dev(v) for k, v in E.enc_params(Nmax + 1, L, 1).items()}
    frames = (r["T"] + pl + pr - L) // stride + 1
    pitch = N.ctn_pitch(frames)
    w_, xn_ = torch.zeros(2, Nmax + 1, pitch, device=DEV), torch.zeros(2, Nmax + 1, pitch, device=DEV)
    nrm_ = torch.zeros(2, dtype=torch.float64, device=DEV)
    xd = dev(x)
    torch.cuda.synchronize()
    assert N.ctn_tas_enc_gated_fwd(xd.data_ptr(), p["encoder.conv1d_U.weight"].data_ptr(), p["encoder.conv1d_V.weight"].data_ptr(),
                                   p["separator.gamma"].data_ptr(), p["separator.beta"].data_ptr(), w_.data_ptr(), xn_.data_ptr(),
                                   nrm_.data_ptr(), 2, r["T"], pl, pr, Nmax + 1, L, stride, pitch, 1e-12, 1e-12, st()) == N.CTN_EUNSUPPORTED
    assert N.ctn_last_launch_count() == 0


def test_gated_encoder_1000_seconds():
    """8,000,007 samples (1000 s at 8 kHz and a ragged tail of 7): the signal norm in double"""
    r = dict(B=1, T=8_000_007, N=33, L=40, stride=20, pl=0, pr=0, amps=None, clicks=())
    p = E.enc_params(33, 40, 3)
    x = E.enc_input(r, 4)
    w, xn, nrm = run_enc(x, p, 33, 40, 20, 0, 0)
    enc_check("1000 s", x, p, r, w, xn, nrm)


def test_gated_encoder_equal_channels_give_beta_exactly():
    """every channel's filters alike: each frame's N channels are equal, so the centred variance is 0 and xn is beta exactly (the
    reference's fp32 E[w^2] - mean^2 can be negative there and give NaN: DESIGN 16's documented deviation)"""
    Nc, L, stride = 33, 16, 8
    p = E.enc_params(Nc, L, 5)
    for k in ("encoder.conv1d_U.weight", "encoder.conv1d_V.weight"):
        p[k] = p[k][:1].expand(Nc, 1, L).contiguous()
    x = torch.randn(2, 1, 1001, generator=torch.Generator().manual_seed(6)) * torch.tensor([1.0, 1e3]).view(-1, 1, 1)
    w, xn, _ = run_enc(x, p, Nc, L, stride, 3, 2)
    assert (w[:, :1] > 0).any()
    assert torch.equal(xn, p["separator.beta"].expand(2, Nc, xn.shape[2]))


# ---- the frame norm alone (ctn_tas_frame_norm_fwd) ----------------------------------------------------------------------------------
FRAME_NORM = [(3, n, f) for n, f in zip(E.ENC_NS, (1, 8, 9, 100, 1000))]


def run_frame_norm(w, gamma, beta, frames, eps=1e-12):
    B, Nc, pitch = w.shape
    wd, gd, bd = dev(w), dev(gamma), dev(beta)
    (xn,), n = twice(lambda o, base, nb: N.ctn_tas_frame_norm_fwd(wd.data_ptr(), gd.data_ptr(), bd.data_ptr(), o[0].data_ptr(), B, Nc,
                                                                   frames, pitch, eps, st()), [((B, Nc, pitch),)], 0)
    assert n == 1
    assert not xn[..., frames:].any()
    return xn[..., :frames]


@pytest.mark.parametrize("B,Nc,frames", FRAME_NORM)
def test_frame_norm_entry(B, Nc, frames):
    """w of samples scaled 1e-3, 1 and 1e3 (the plain encoder's output scales with the input), random pad columns that must not
    be read; frame 0 of sample 0 has all channels equal and must give beta exactly"""
    p = E.enc_params(Nc, 4, Nc + frames)
    w = E.D.pitched(B, Nc, frames, N.ctn_pitch(frames), frames, pad="random") * torch.tensor([1e-3, 1.0, 1e3]).view(-1, 1, 1)
    w[0, :, 0] = 0.7
    xn = run_frame_norm(w, p["separator.gamma"], p["separator.beta"], frames)
    ref = E.frame_norm(w[..., :frames], p["separator.gamma"], p["separator.beta"], 1e-12)
    ratio = check(xn.permute(0, 2, 1), ref.permute(0, 2, 1), 2)
    if Nc > 1:
        assert torch.equal(xn[0, :, 0], p["separator.beta"].view(-1))
    report("framenorm", "B={} N={} frames={}".format(B, Nc, frames), ratio)


def test_frame_norm_largest_channels_and_one_past():
    Nmax, frames = E.frame_norm_max_n(OPTIN), 9
    p = E.enc_params(Nmax + 1, 4, 1)
    w = E.D.pitched(1, Nmax + 1, frames, N.ctn_pitch(frames), 2)
    g, b = p["separator.gamma"][:, :Nmax], p["separator.beta"][:, :Nmax]
    xn = run_frame_norm(w[:, :Nmax].contiguous(), g, b, frames)
    report("framenorm", "N={} (largest)".format(Nmax), check(xn.permute(0, 2, 1), E.frame_norm(w[:, :Nmax, :frames], g, b, 1e-12).permute(0, 2, 1), 2))
    wd, xd = dev(w), torch.zeros_like(w, device=DEV)
    gd, bd = dev(p["separator.gamma"]), dev(p["separator.beta"])
    torch.cuda.synchronize()
    assert N.ctn_tas_frame_norm_fwd(wd.data_ptr(), gd.data_ptr(), bd.data_ptr(), xd.data_ptr(), 1, Nmax + 1, frames, w.shape[2], 1e-12,
                                    st()) == N.CTN_EUNSUPPORTED
    assert N.ctn_last_launch_count() == 0


# ---- whole TasNet -----------------------------------------------------------------------------------------------------------------
TINY_GATED = dict(n_basis=32, kernel_size=16, stride=8, enc_basis="trainableGated", enc_nonlinear=None, sep_num_blocks=2, sep_num_layers=2,
                  sep_hidden_channels=24, causal=False, mask_nonlinear="sigmoid", n_sources=2, eps=1e-12)
TINY_PLAIN = dict(n_basis=24, kernel_size=8, stride=4, enc_basis="trainable", enc_nonlinear="relu", sep_num_blocks=2, sep_num_layers=1,
                  sep_hidden_channels=16, causal=False, mask_nonlinear="softmax", n_sources=3, eps=1e-12)
RECIPE = dict(n_basis=500, kernel_size=40, stride=20, enc_basis="trainableGated", enc_nonlinear=None, sep_num_blocks=2, sep_num_layers=2,
              sep_hidden_channels=500, causal=False, mask_nonlinear="sigmoid", n_sources=2, eps=1e-12)


def tasnet(cfg, mode=None, seed=7):
    c = dict(cfg)
    m = TasNet(c.pop("n_basis"), dec_basis="trainable", rnn_type="lstm", **c)
    sd = LR.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed)
    m.load_state_dict(sd)
    m.math = mode
    return m.to(DEV).eval(), sd


def forward(m, x):
    with torch.no_grad():
        out = m(x.to(DEV))
    torch.cuda.synchronize()
    return out.cpu()


def loud_batch(T, seed):
    return torch.randn(4, 1, T, generator=torch.Generator().manual_seed(seed)) * torch.tensor([1e-3, 1.0, 1e3, 0.0]).view(-1, 1, 1)


@pytest.mark.parametrize("mode", E.MODES)
@pytest.mark.parametrize("enc", ["gated", "plain"])
def test_tasnet_mixed_loudness(enc, mode):
    """samples x1e-3, x1, x1e3 and digital silence in one batch: each within the bound of its own (sample, source) and bit-identical
    to its run alone"""
    cfg = TINY_GATED if enc == "gated" else TINY_PLAIN
    m, sd = tasnet(cfg, mode)
    x = loud_batch(803, 1)
    out = forward(m, x)
    ratio = check(out, LR.tasnet_fwd(x, sd, cfg), 2, E.rel_of(mode))
    for b in range(x.shape[0]):
        assert torch.equal(forward(m, x[b:b + 1])[0], out[b]), "sample {} differs from its run alone".format(b)
    assert not out[3].any()
    report("tasnet", "{} {} loudness batch".format(enc, mode), ratio)


@pytest.mark.parametrize("mask", ["sigmoid", "softmax"])
@pytest.mark.parametrize("n_src", [1, 4])
def test_tasnet_sources(n_src, mask):
    cfg = dict(TINY_GATED, n_sources=n_src, mask_nonlinear=mask)
    m, sd = tasnet(cfg)
    x = torch.randn(2, 1, 603, generator=torch.Generator().manual_seed(n_src))
    report("tasnet", "{} sources {}".format(n_src, mask), check(forward(m, x), LR.tasnet_fwd(x, sd, cfg), 2))


@pytest.mark.parametrize("label", ["P+1", "max"])
def test_tasnet_hidden_edges(label):
    """a small bidirectional model at H = P + 1 (the last CTA owns one unit) and at the largest H of two directions"""
    H = dict(E.hidden_rows(2, SMS, OPTIN))[label]
    cfg = dict(TINY_GATED, n_basis=16, kernel_size=4, stride=2, sep_num_blocks=1, sep_num_layers=1, sep_hidden_channels=H)
    m, sd = tasnet(cfg)
    x = torch.randn(2, 1, 81, generator=torch.Generator().manual_seed(H))
    report("tasnet", "H={}({})".format(label, H), check(forward(m, x), LR.tasnet_fwd(x, sd, cfg), 2))


def test_tasnet_three_passes_at_the_recipe_hidden():
    B = 2 * N.ctn_tas_lstm_group(RECIPE["sep_hidden_channels"], 2) + 1
    m, sd = tasnet(RECIPE)
    x = torch.randn(B, 1, 800, generator=torch.Generator().manual_seed(B))
    report("tasnet", "recipe B={} (three passes)".format(B), check(forward(m, x), LR.tasnet_fwd(x, sd, RECIPE), 2))


def test_tasnet_20_seconds_at_the_recipe():
    """160,000 samples: 7,999 steps through 4 bi-LSTM layers"""
    m, sd = tasnet(RECIPE)
    x = torch.randn(1, 1, 160000, generator=torch.Generator().manual_seed(20))
    assert N.frames_of(160000, 40, 20)[0] == 7999
    report("tasnet", "recipe 20 s", check(forward(m, x), LR.tasnet_fwd(x, sd, RECIPE), 2))


# ---- online TasNet: test_tas_online_gpu's contract ------------------------------------------------------------------------------------
def online_rows():
    H = dict(E.hidden_rows(1, SMS, OPTIN))["P+1"]
    return {"H=P+1({})".format(H): online_row(H=H, T=8 * 60, pushes=(5,)),
            "B=2group+1": online_row(H=64, B=2 * E.lstm_geo(64, 1, SMS, OPTIN)["group"] + 1, T=8 * 40, pushes=(1, 17))}


@pytest.mark.parametrize("name", list(online_rows()))
def test_online_edges_match_offline_and_fp64(name):
    r = online_rows()[name]
    m, sd, cfg = online_model(r)
    x = signal(r)
    sep, Y, Z, launches = stream(m, x, sizes(r.T, r.S, r.pushes))
    got = whole(sep, Y, Z)
    with torch.no_grad():
        off = m(x.to(DEV))
    torch.cuda.synchronize()
    excess = float(((got - off).abs() - O.stream_bound(off)).max())
    share = float((got == off).double().mean())
    print("[tas/galr edges] online {:>14s} B={} H={} bit-identical {:.4%} worst excess {:.3g}".format(name, r.B, r.H, share, excess))
    assert excess <= 0 and share == 1.0, (name, excess, share)
    assert launches == {4 + 2 * r.X * r.R}
    report("online", name, check(got.cpu(), LR.tasnet_fwd(x, sd, cfg), 2))


# ---- the globally attentive block (ctn_galr_inter_fwd) ----------------------------------------------------------------------------------
GALR_ROWS = E.galr_rows()


def run_inter(x, sd, heads, Q, ln_eps, gn_eps, in_place=False):
    B, S, K, F = x.shape
    w = {k: dev(v) for k, v in sd.items()}
    div = dev(10000 ** (torch.arange(F // 2) / F))
    ptrs = [w[k].data_ptr() for k in E.INTER_KEYS]
    xd = dev(x)
    nbytes = N.ctn_galr_inter_workspace_bytes(B, S, K, Q, F)
    if in_place:
        (base, nb), keep = nan_ws(nbytes)
        N.check(N.ctn_galr_inter_fwd(xd.data_ptr(), *ptrs[:4], div.data_ptr(), heads, *ptrs[4:], xd.data_ptr(), B, S, K, Q, F, ln_eps,
                                     gn_eps, base, nb, st()), "ctn_galr_inter_fwd")
        torch.cuda.synchronize()
        return xd.cpu()
    (out,), n = twice(lambda o, base, nb: N.ctn_galr_inter_fwd(xd.data_ptr(), *ptrs[:4], div.data_ptr(), heads, *ptrs[4:], o[0].data_ptr(),
                                                               B, S, K, Q, F, ln_eps, gn_eps, base, nb, st()), [((B, S, K, F),)], nbytes)
    assert n == 6
    assert torch.equal(xd.cpu(), x)
    return out


@pytest.mark.parametrize("name", list(GALR_ROWS))
def test_galr_inter_entry(name):
    r = GALR_ROWS[name]
    sd = E.inter_weights(r["F"], r["K"], r["Q"], r["F"] + r["K"] + r["Q"])
    x = E.inter_input(r, r["S"] + r["Q"])
    out = run_inter(x, sd, r["heads"], r["Q"], r["ln_eps"], r["gn_eps"])
    ratio = check(out, E.inter_answer(x, sd, r["heads"], r["Q"], r["ln_eps"], r["gn_eps"]), 2)
    if r["amps"]:
        for b in range(r["B"]):
            assert torch.equal(run_inter(x[b:b + 1], sd, r["heads"], r["Q"], r["ln_eps"], r["gn_eps"])[0], out[b]), b
        assert torch.equal(run_inter(x, sd, r["heads"], r["Q"], r["ln_eps"], r["gn_eps"], in_place=True), out)
    report("galr", name, ratio, "heads={} passes down={} up={}".format(r["heads"], -(-r["Q"] // (GR.PASS_ELEMS // r["F"])),
                                                                       -(-r["K"] // (GR.PASS_ELEMS // r["F"]))))


def test_galr_inter_refusals_before_launch():
    F, K, Q = 128, 17, 17
    sd = E.inter_weights(F, K, Q, 1)
    w = {k: dev(v) for k, v in sd.items()}
    ptrs = [w[k].data_ptr() for k in E.INTER_KEYS]
    x = torch.zeros(1, 2, K, F, device=DEV)
    div = torch.ones(F // 2, device=DEV)
    ws = torch.empty(N.ctn_galr_inter_workspace_bytes(1, 2, K, K + 1, F) + 256, dtype=torch.uint8, device=DEV)
    base, nb = N.aligned(ws)
    torch.cuda.synchronize()
    for Q_, heads, F_ in ((K + 1, 8, F), (Q, 32, F), (Q, 8, 96)):          # Q > K, head dimension 4, F outside {32, 64, 128}
        assert N.ctn_galr_inter_fwd(x.data_ptr(), *ptrs[:4], div.data_ptr(), heads, *ptrs[4:], x.data_ptr(), 1, 2, K, Q_, F_, 1e-3, 1e-1,
                                    base, nb, st()) == N.CTN_EUNSUPPORTED
        assert N.ctn_last_launch_count() == 0


# ---- the separator head (ctn_dpt_head_fwd without a bottleneck) --------------------------------------------------------------------------
HEAD_ROWS = E.head_rows()


@pytest.mark.parametrize("name", list(HEAD_ROWS))
def test_galr_head_without_bottleneck_entry(name):
    r = HEAD_ROWS[name]
    B, F, frames, K, P = r["B"], r["F"], r["frames"], r["K"], r["P"]
    pitch = N.ctn_pitch(frames)
    w = E.D.pitched(B, F, frames, pitch, frames + K + P)
    if r["amps"]:
        w = w * torch.tensor(r["amps"]).view(-1, 1, 1)
    sd = E.head_params(F, F + K)
    pl, pr, S = GR.segment_geometry(frames, K, P)
    wd, g, b = dev(w), dev(sd["separator.norm2d.norm.weight"]), dev(sd["separator.norm2d.norm.bias"])
    (z,), n = twice(lambda o, base, nb: N.ctn_dpt_head_fwd(wd.data_ptr(), None, None, g.data_ptr(), b.data_ptr(), o[0].data_ptr(), B, F, F,
                                                           frames, pitch, K, P, pl, pr, 1e-12, N.MATH_NAMES["fp32"], base, nb, st()),
                    [((B, S, K, F),)], N.ctn_dpt_head_workspace_bytes(B, F, F, pitch, S, K))
    assert n == 3
    ref = GR.head(w[..., :frames].double(), sd, dict(sep_chunk_size=K, sep_hop_size=P, eps=1e-12))
    report("galr head", name, check(z, ref, 1))


def test_head_without_bottleneck_refuses_fewer_frames_before_launch():
    """with a hop of 1 the padding rule adds nothing, so 11 frames cannot fill a chunk of 16"""
    B, F, frames, K, P = 1, 32, 11, 16, 1
    assert GR.segment_geometry(frames, K, P)[:2] == (0, 0)
    pitch = N.ctn_pitch(frames)
    w, z = torch.zeros(B, F, pitch, device=DEV), torch.zeros(B, 1, K, F, device=DEV)
    g = torch.ones(F, device=DEV)
    ws = torch.empty(N.ctn_dpt_head_workspace_bytes(B, F, F, pitch, 1, K) + 256, dtype=torch.uint8, device=DEV)
    base, nb = N.aligned(ws)
    torch.cuda.synchronize()
    assert N.ctn_dpt_head_fwd(w.data_ptr(), None, None, g.data_ptr(), g.data_ptr(), z.data_ptr(), B, F, F, frames, pitch, K, P, 0, 0, 1e-12,
                              N.MATH_NAMES["fp32"], base, nb, st()) == N.CTN_EINVAL
    assert N.ctn_last_launch_count() == 0


# ---- whole GALRNet ---------------------------------------------------------------------------------------------------------------------
GALR_TINY = dict(n_basis=32, kernel_size=4, stride=2, enc_nonlinear="relu", sep_hidden_channels=32, sep_chunk_size=16, sep_hop_size=8,
                 sep_down_chunk_size=4, sep_num_blocks=2, sep_num_heads=4, sep_dropout=0.1, mask_nonlinear="sigmoid", eps=1e-12, n_sources=2)
GALR_RECIPE = dict(n_basis=64, kernel_size=16, stride=8, enc_nonlinear=None, sep_hidden_channels=128, sep_chunk_size=100, sep_hop_size=50,
                   sep_down_chunk_size=32, sep_num_blocks=6, sep_num_heads=8, sep_dropout=0.1, mask_nonlinear="relu", eps=1e-12, n_sources=2)


def galrnet(cfg, seed=3):
    c = cfg
    m = GALRNet(c["n_basis"], c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable", enc_nonlinear=c["enc_nonlinear"],
                sep_hidden_channels=c["sep_hidden_channels"], sep_chunk_size=c["sep_chunk_size"], sep_hop_size=c["sep_hop_size"],
                sep_down_chunk_size=c["sep_down_chunk_size"], sep_num_blocks=c["sep_num_blocks"], sep_num_heads=c["sep_num_heads"], sep_norm=True,
                sep_dropout=c["sep_dropout"], mask_nonlinear=c["mask_nonlinear"], low_dimension=True, causal=False, n_sources=c["n_sources"],
                eps=c["eps"])
    sd = GR.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], seed)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval(), sd


def test_galrnet_mixed_loudness():
    """each sample within 1e-6 of its own largest value of its run alone; not bit for bit, since the intra block's gLN statistics
    add double partials with atomics (DESIGN 17)"""
    m, sd = galrnet(GALR_TINY)
    x = loud_batch(1203, 2)
    out = forward(m, x)
    ratio = check(out, GR.galrnet_fwd(x, sd, GALR_TINY), 2)
    same = 0
    for b in range(x.shape[0]):
        one = forward(m, x[b:b + 1])[0]
        assert float((one - out[b]).abs().max()) <= 1e-6 * float(one.abs().max()), b
        same += int(torch.equal(one, out[b]))
    assert not out[3].any()
    report("galrnet", "loudness batch", ratio, "bit-identical to B=1: {} of {} samples".format(same, x.shape[0]))


GALR_VARIANTS = {"1 source": dict(n_sources=1), "4 sources": dict(n_sources=4),
                 "F=32 head dim 32": dict(sep_num_heads=1), "F=128 head dim 64": dict(n_basis=128, sep_num_heads=2, sep_hidden_channels=64),
                 "eps 1e-3": dict(eps=1e-3)}


@pytest.mark.parametrize("name", list(GALR_VARIANTS))
def test_galrnet_variants(name):
    cfg = dict(GALR_TINY, **GALR_VARIANTS[name])
    m, sd = galrnet(cfg)
    x = torch.randn(2, 1, 603, generator=torch.Generator().manual_seed(len(name)))
    report("galrnet", name, check(forward(m, x), GR.galrnet_fwd(x, sd, cfg), 2))


def test_galrnet_60_seconds_at_the_recipe():
    """480,000 samples: 59,999 frames in S = 1200 chunks, attention positions up to 38,400"""
    m, sd = galrnet(GALR_RECIPE)
    x = torch.randn(1, 1, 480000, generator=torch.Generator().manual_seed(60))
    report("galrnet", "recipe 60 s", check(forward(m, x), GR.galrnet_fwd(x, sd, GALR_RECIPE), 2))
