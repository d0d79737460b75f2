"""The stage entries called directly through the C ABI (``-m gpu``): ctn_sep_head_fwd, ctn_sep_tail_fwd, ctn_depthwise_conv1d_fwd,
ctn_pointwise_conv1d_fwd and ctn_stage_workspace_bytes, against the fp64 restatements and bounds of stage_entries_ref.py, in every
math mode; their refusals; and the stage timers (ctn_profile_enable / ctn_profile_read).

Every call writes into NaN-filled outputs, scratch and workspace, reads pitched inputs whose pad columns are NaN, and must:
  * stay within its bound (the worst share per row is printed);
  * give the same bits when repeated, and when the pads are zero instead (the pad contract of stage_entries_ref.py);
  * leave the pad columns of its pitched outputs exactly 0;
  * launch exactly the predicted number of kernels.
f16x3 must run the head, the mask contraction and the pointwise stage on the tf32 pieces: the bits and the kernels of tf32x3,
never k_maskdec.  Each refusal returns its code with zero launches.

Stage timers: StageTimer (csrc/ctn_common.cuh) brackets kernel groups of the Conv-TasNet pipelines only; nested timers fold into
the outermost one.  Launches outside every stage: the latent copy of ctn_convtasnet_fwd, the causal head's cLN0 (3 launches) and
bias rows (1), everything of the training path except the fused TCN forward's stages (ctn_tcn_train_fwd) and the loss (LOSS), and
every launch of the stage entries, the filter banks, the dual-path blocks and the DPRNN-TasNet path.  Measured (H100): the gLN
forward 23 of 23 launches inside stages, with a latent 24 of 25, causal 78 of 82, one training step 14 of 21.
"""
import ctypes as C

import pytest
import torch

import convtasnet_oracle as O
import gln_forward_edges_ref as G
import stage_entries_ref as R
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import PIT1d
from ctn_b200.criterion.sdr import NegSISDR
from ctn_b200.models import dprnn_tasnet
from ctn_b200.models.dprnn_tasnet import DPRNNTasNet
from ctn_b200.modules.conv import DepthwiseSeparableConv1d
from test_forward_edges_gpu import _build

pytestmark = pytest.mark.gpu

MODES = ["fp32"] + (["tf32x3", "f16x3", "tf32"] if N.ctn_has_tcgen05() else [])
MATH = N.MATH_NAMES
DEV = torch.device("cuda", 0)


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _nan_ws(nbytes):
    """all-ones bytes (NaN as float and double) -> (buffer, 256-aligned base, usable bytes)"""
    buf = torch.full((int(nbytes) + 512,), 255, dtype=torch.uint8, device=DEV)
    return (buf,) + N.aligned(buf)


def _exact_ws(nbytes):
    """a NaN workspace handed over with exactly nbytes -> (buffer, base, check): check() asserts nothing was written past them"""
    buf, base, _ = _nan_ws(nbytes)
    tail = buf[base - buf.data_ptr() + int(nbytes):]

    def check():
        assert bool((tail == 255).all()), "written past the {} workspace bytes the entry asked for".format(nbytes)
    return buf, base, check


def _pitched(x64, pad):
    """(B, C, F) float64 -> (B, C, pitch(F)) float32 on the GPU, pad columns = pad"""
    B, Cc, Fr = x64.shape
    out = torch.full((B, Cc, R.pitch(Fr)), pad, dtype=torch.float32, device=DEV)
    out[..., :Fr] = x64.float().to(DEV)
    return out


def _g(t):
    return None if t is None else t.float().to(DEV).contiguous()


def _st():
    return N.stream_ptr(DEV)


def _same(calls, what):
    """calls: outputs of the same entry (NaN pads, NaN pads again, zero pads) -> the first; every one must match it bit for bit"""
    first = calls[0]
    for k, other in enumerate(calls[1:]):
        for a, b in zip(first, other):
            if a is not None:
                assert torch.equal(a, b), "{}: call {} gives other bits".format(what, k + 2)
    return first


# ---- head ------------------------------------------------------------------------------------------------------------------
def _head_inputs(name, r):
    i = R.head_inputs(name, r)
    if r.enc:
        L, stride, T = r.enc
        frames, pl, pr = R.frames_of(T, L, stride)
        w = torch.empty(r.B, r.N, R.pitch(frames), device=DEV)
        stats = torch.zeros(r.B, 2, dtype=torch.float64, device=DEV)
        N.check(N.ctn_encoder_fwd(_g(i["x"]).data_ptr(), _g(i["enc_w"]).data_ptr(), w.data_ptr(), r.B, T, pl, pr, r.N, L, stride, 0,
                                  w.shape[2], stats.data_ptr(), _st()), "ctn_encoder_fwd")
        torch.cuda.synchronize()
        i["w"] = w[..., :frames].double().cpu()
        i["stats"] = stats.cpu()
    else:
        i["stats"] = R.stats_frames(i["w"])
    return i


def _head_call(i, r, mode, pad, math=None):
    B, Nn, Bc = r.B, r.N, r.Bc
    frames = i["w"].shape[2]
    w = _pitched(i["w"], pad)
    P = w.shape[2]
    x0 = _nan(B, Bc, P)
    nbytes = N.ctn_stage_workspace_bytes(Bc, Nn)
    ws, base, ws_check = _exact_ws(nbytes)
    st = i["stats"].to(DEV)
    args = [_g(i[k]) for k in ("gamma", "beta", "W", "bias")]
    s = N.ctn_sep_head_fwd(w.data_ptr(), st.data_ptr(), *[a.data_ptr() for a in args], x0.data_ptr(), B, Nn, Bc, frames, P, r.eps,
                           MATH[math or mode], base, nbytes, _st())
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert s == N.CTN_OK, "ctn_sep_head_fwd: status {}".format(s)
    ws_check()
    return (x0,), n


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(R.HEAD))
def test_head(name, mode):
    r = R.HEAD[name]
    i = _head_inputs(name, r)
    runs = [_head_call(i, r, mode, p) for p in (float("nan"), float("nan"), 0.0)]
    assert all(n == R.head_launches(mode) for _, n in runs), ([n for _, n in runs], R.head_launches(mode))
    (x0,) = _same([o for o, _ in runs], "head " + name)
    frames = i["w"].shape[2]
    assert torch.equal(x0[..., frames:], torch.zeros_like(x0[..., frames:])), "x0 pad columns not 0"
    ref, fold = R.head_reference(i["w"], i["stats"], i["gamma"], i["beta"], i["W"], i["bias"], r.eps)
    s = R.share(x0[..., :frames].cpu(), ref.out["D"][0], R.gate_allowance(ref, mode) + fold)
    print("head {} [{}] {}: {:.3f} of the bound".format(name, r.reaches, mode, s))
    assert s <= 1.0, "head {} {}: {:.2f}x the bound".format(name, mode, s)


# ---- tail ------------------------------------------------------------------------------------------------------------------
def _tail_call(i, r, mode, pad):
    B, Nn, Bc, S = r.B, r.N, r.Bc, r.S
    frames, pl, _ = R.frames_of(r.T, r.L, r.stride)
    y, w = _pitched(i["y"], pad), _pitched(i["w"], pad)
    P = y.shape[2]
    out = _nan(B, S, r.T)
    lat = _nan(B, S, Nn, frames) if r.latent else None
    what = _nan(B, S * Nn, P)
    nbytes = N.ctn_stage_workspace_bytes(S * Nn, Bc)
    ws, base, ws_check = _exact_ws(nbytes)
    a = torch.tensor([i["a"]], dtype=torch.float32, device=DEV)
    Wm, bm, Wd = _g(i["Wm"]), _g(i["bm"]), _g(i["Wd"])
    s = N.ctn_sep_tail_fwd(y.data_ptr(), w.data_ptr(), a.data_ptr(), Wm.data_ptr(), bm.data_ptr(), Wd.data_ptr(), out.data_ptr(),
                           N.ptr(lat), what.data_ptr(), B, Nn, Bc, S, frames, P, r.L, r.stride, pl, r.T, MATH[mode], base, nbytes,
                           _st())
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert s == N.CTN_OK, "ctn_sep_tail_fwd: status {}".format(s)
    ws_check()
    return (out, lat, what), n


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(R.TAIL))
def test_tail(name, mode):
    r = R.TAIL[name]
    i = R.tail_inputs(name, r)
    frames, pl, _ = R.frames_of(r.T, r.L, r.stride)
    want = R.tail_launches(mode, r.B, r.S, r.N, r.latent)
    runs = [_tail_call(i, r, mode, p) for p in (float("nan"), float("nan"), 0.0)]
    assert all(n == want for _, n in runs), ([n for _, n in runs], want)
    out, lat, what = _same([o for o, _ in runs], "tail " + name)
    assert torch.equal(what[..., frames:], torch.zeros_like(what[..., frames:])), "w_hat pad columns not 0"
    if lat is not None:
        assert torch.equal(lat, what[..., :frames].reshape(lat.shape)), "the latent is not w_hat's valid columns"
    out64, lat64 = R.tail64(i["y"], i["w"], i["a"], i["Wm"], i["bm"], i["Wd"], r.S, r.stride, pl, r.T)
    _, allowance = R.tail_reference(i["y"], i["w"], i["a"], i["Wm"], i["bm"], i["Wd"], r.S, r.stride, pl, r.T)
    alat, aout = allowance(mode)
    s_lat = R.share(what[..., :frames].reshape(lat64.shape).cpu(), lat64, alat)
    s_out = R.share(out.cpu(), out64, aout)
    print("tail {} [{}] {} {}: out {:.3f}, w_hat {:.3f} of the bound".format(name, r.reaches, R.decoder_kernel(r.L, r.stride), mode,
                                                                             s_out, s_lat))
    assert s_lat <= 1.0 and s_out <= 1.0, "tail {} {}: out {:.2f}x, w_hat {:.2f}x the bound".format(name, mode, s_out, s_lat)


def _kernels(fn):
    """names of the kernels fn launches (not the fills and copies of the harness's own tensors)"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "emcpy" not in e.name
             and "emset" not in e.name and "at::" not in e.name]
    return out, names


def test_f16x3_runs_the_stages_on_tf32_pieces():
    """f16x3 = tf32x3 bit for bit and kernel for kernel in the head, the tail (never k_maskdec, on the shape where the model path
    fuses it) and the pointwise stage: none of their operands carries an operand scale"""
    if "f16x3" not in MODES:
        pytest.skip("tensor-core modes not built")
    r = R.TAIL["s2_l16s8_n128"]
    i = R.tail_inputs("s2_l16s8_n128", r)
    (a, na), ka = _kernels(lambda: _tail_call(i, r, "f16x3", 0.0))
    (b, nb), kb = _kernels(lambda: _tail_call(i, r, "tf32x3", 0.0))
    assert na == nb == R.tail_launches("f16x3", r.B, r.S, r.N, False) == len(ka), (na, nb, ka)
    assert not any("maskdec" in k for k in ka) and sorted(ka) == sorted(kb), (ka, kb)
    assert any("k_pw_wgmma" in k for k in ka) and any("k_decoder" in k for k in ka), ka
    assert all(torch.equal(u, v) for u, v in zip(a, b) if u is not None)
    h = R.HEAD["bc129_n64_f127_b37"]
    hi = _head_inputs("bc129_n64_f127_b37", h)
    (a, _), ka = _kernels(lambda: _head_call(hi, h, "f16x3", 0.0))
    (b, _), kb = _kernels(lambda: _head_call(hi, h, "tf32x3", 0.0))
    assert torch.equal(a[0], b[0]) and sorted(ka) == sorted(kb), (ka, kb)
    p = R.PW["m129_k64_b37"]
    pi = R.pw_inputs("m129_k64_b37", p)
    (a, _), ka = _kernels(lambda: _pw_call(pi, p, "f16x3", 0.0))
    (b, _), kb = _kernels(lambda: _pw_call(pi, p, "tf32x3", 0.0))
    assert torch.equal(a[0], b[0]) and sorted(ka) == sorted(kb), (ka, kb)


# ---- depthwise / pointwise ---------------------------------------------------------------------------------------------------
def _dw_call(i, r):
    To = R.dw_out_len(r.T, r.K, r.stride, r.padding, r.dilation)
    yp = R.pitch(To) + r.extra
    x, w, b = _g(i["x"]), _g(i["w"]), _g(i["bias"])
    y = _nan(r.B, r.C, yp)
    s = N.ctn_depthwise_conv1d_fwd(x.data_ptr(), w.data_ptr(), N.ptr(b), y.data_ptr(), r.B, r.C, r.T, r.K, r.stride, r.padding,
                                   r.dilation, yp, _st())
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert s == N.CTN_OK, "ctn_depthwise_conv1d_fwd: status {}".format(s)
    return (y,), n


@pytest.mark.parametrize("name", list(R.DW))
def test_depthwise(name):
    r = R.DW[name]
    i = R.dw_inputs(name, r)
    To = R.dw_out_len(r.T, r.K, r.stride, r.padding, r.dilation)
    runs = [_dw_call(i, r) for _ in range(2)]
    assert all(n == R.DW_LAUNCHES for _, n in runs)
    (y,) = _same([o for o, _ in runs], "depthwise " + name)
    assert torch.equal(y[..., To:], torch.zeros_like(y[..., To:])), "columns [To, y_pitch) not 0"
    y64, m = R.depthwise64(i["x"], i["w"], i["bias"], r.stride, r.padding, r.dilation)
    s = R.share(y[..., :To].cpu(), y64, R.depthwise_bound(m, r.K))
    print("depthwise {} [{}] To {}: {:.3f} of the bound".format(name, r.reaches, To, s))
    assert s <= 1.0, "depthwise {}: {:.2f}x the bound".format(name, s)


def _pw_need(B, M, K, P):
    return 4 * B * M * P + N.ctn_stage_workspace_bytes(M, K) + 16 * B + 4096


def _pw_call(i, r, mode, pad):
    x = _pitched(i["x"], pad)
    P = x.shape[2]
    W, b = _g(i["W"]), _g(i["bias"])
    y = _nan(r.B, r.M, r.frames)
    ws, base, nbytes = _nan_ws(_pw_need(r.B, r.M, r.K, P))
    s = N.ctn_pointwise_conv1d_fwd(x.data_ptr(), W.data_ptr(), N.ptr(b), y.data_ptr(), r.B, r.M, r.K, r.frames, P, MATH[mode], base,
                                   nbytes, _st())
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert s == N.CTN_OK, "ctn_pointwise_conv1d_fwd: status {}".format(s)
    return (y,), n


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(R.PW))
def test_pointwise(name, mode):
    r = R.PW[name]
    i = R.pw_inputs(name, r)
    runs = [_pw_call(i, r, mode, p) for p in (float("nan"), float("nan"), 0.0)]
    assert all(n == R.pw_launches(mode, r.B, r.M) for _, n in runs), [n for _, n in runs]
    (y,) = _same([o for o, _ in runs], "pointwise " + name)
    ref = R.pointwise_reference(i["x"], i["W"], i["bias"])
    s = R.share(y.cpu(), ref.out["D"][0], R.gate_allowance(ref, mode))
    print("pointwise {} [{}] {}: {:.3f} of the bound".format(name, r.reaches, mode, s))
    assert s <= 1.0, "pointwise {} {}: {:.2f}x the bound".format(name, mode, s)


# ---- refusals ----------------------------------------------------------------------------------------------------------------
def _refusals(mode):
    """(what, expected status, thunk returning the entry's status)"""
    m = MATH[mode]
    st = _st()
    f = lambda *s: torch.zeros(*s, device=DEV)  # noqa: E731
    B, Nn, Bc, S, frames, P = 2, 64, 32, 2, 100, 128
    w, y, x0, what = f(B, Nn, P + 128), f(B, Bc, P + 128), f(B, Bc, P + 128), f(B, S * Nn, P + 128)
    stats = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
    g, bt, Wb, bb = f(Nn), f(Nn), f(Bc, Nn), f(Bc)
    a, Wm, bm, Wd, out = f(1), f(S * Nn, Bc), f(S * Nn), f(Nn, 16), f(B, S, 804)
    hbytes, tbytes = N.ctn_stage_workspace_bytes(Bc, Nn), N.ctn_stage_workspace_bytes(S * Nn, Bc)
    ws = torch.zeros(max(hbytes, tbytes) + 4096, dtype=torch.uint8, device=DEV)
    base = N.aligned(ws)[0]
    keep = [w, y, x0, what, stats, g, bt, Wb, bb, a, Wm, bm, Wd, out, ws]

    def head(wp=w.data_ptr(), pitch=P, wsb=base, nb=hbytes):
        return N.ctn_sep_head_fwd(wp, stats.data_ptr(), g.data_ptr(), bt.data_ptr(), Wb.data_ptr(), bb.data_ptr(), x0.data_ptr(), B, Nn,
                                  Bc, frames, pitch, 1e-8, m, wsb, nb, st)

    def tail(whatp=what.data_ptr(), pitch=P, wsb=base, nb=tbytes, L=16, stride=8, crop=4, T=804):
        return N.ctn_sep_tail_fwd(y.data_ptr(), w.data_ptr(), a.data_ptr(), Wm.data_ptr(), bm.data_ptr(), Wd.data_ptr(), out.data_ptr(),
                                  None, whatp, B, Nn, Bc, S, frames, pitch, L, stride, crop, T, m, wsb, nb, st)

    xd, wd, yd = f(65536), f(65536), f(65536 * 4)

    def dw(Bn=1, Cn=4, T=16, K=3, stride=1, pad=0, dil=1, yp=128):
        return N.ctn_depthwise_conv1d_fwd(xd.data_ptr(), wd.data_ptr(), None, yd.data_ptr(), Bn, Cn, T, K, stride, pad, dil, yp, st)

    xp, Wp, bp, yq = f(B, 40, 256), f(24, 40), f(24), f(B, 24, frames)
    pneed = _pw_need(B, 24, 40, 128)
    pws = torch.zeros(pneed + 512, dtype=torch.uint8, device=DEV)
    pbase = N.aligned(pws)[0]
    keep += [xd, wd, yd, xp, Wp, bp, yq, pws]

    def pw(xptr=xp.data_ptr(), pitch=128, wsb=pbase, nb=pneed):
        return N.ctn_pointwise_conv1d_fwd(xptr, Wp.data_ptr(), bp.data_ptr(), yq.data_ptr(), B, 24, 40, frames, pitch, m, wsb, nb, st)

    cases = [
        ("head: workspace one byte short", N.CTN_EWORKSPACE, lambda: head(nb=hbytes - 1)),
        ("head: workspace not 256-byte aligned", N.CTN_EALIGN, lambda: head(wsb=base + 16)),
        ("head: pitch 192", N.CTN_EALIGN, lambda: head(pitch=192)),
        ("head: pitch < frames", N.CTN_EALIGN, lambda: head(pitch=64)),
        ("head: w 4 bytes off", N.CTN_EALIGN, lambda: head(wp=w.data_ptr() + 4)),
        ("tail: workspace one byte short", N.CTN_EWORKSPACE, lambda: tail(nb=tbytes - 1)),
        ("tail: workspace not 256-byte aligned", N.CTN_EALIGN, lambda: tail(wsb=base + 64)),
        ("tail: pitch 200", N.CTN_EALIGN, lambda: tail(pitch=200)),
        ("tail: w_hat 4 bytes off", N.CTN_EALIGN, lambda: tail(whatp=what.data_ptr() + 4)),
        ("tail: crop_left + T one past the full length", N.CTN_EINVAL, lambda: tail(crop=5)),
        ("tail: L % stride != 0", N.CTN_EINVAL, lambda: tail(L=15)),
        ("depthwise: T + 2 padding < span", N.CTN_EINVAL, lambda: dw(T=4, K=3, dil=2)),
        ("depthwise: y_pitch < To", N.CTN_EINVAL, lambda: dw(yp=13)),
        ("depthwise: C = 65536", N.CTN_EUNSUPPORTED, lambda: dw(Cn=65536, T=1, K=1, yp=1)),
        ("depthwise: B = 65536", N.CTN_EUNSUPPORTED, lambda: dw(Bn=65536, Cn=1, T=1, K=1, yp=1)),
        ("pointwise: workspace short", N.CTN_EWORKSPACE, lambda: pw(nb=4096)),
        ("pointwise: pitch 129", N.CTN_EALIGN, lambda: pw(pitch=129)),
        ("pointwise: workspace not 256-byte aligned", N.CTN_EALIGN, lambda: pw(wsb=pbase + 128)),
        ("pointwise: x 4 bytes off", N.CTN_EALIGN, lambda: pw(xptr=xp.data_ptr() + 4)),
    ]
    return cases, (head, tail, dw, pw), keep


@pytest.mark.parametrize("mode", MODES)
def test_refusals_launch_nothing(mode):
    """a refused call returns its code before its first launch; the same arguments with the fault removed succeed"""
    cases, bases, keep = _refusals(mode)
    for fn in bases:
        assert fn() == N.CTN_OK and N.ctn_last_launch_count() > 0, "{} ({}): the call without a fault".format(fn.__name__, mode)
    for what, code, fn in cases:
        s = fn()
        n = N.ctn_last_launch_count()
        assert s == code, "{} ({}): status {}, expected {}".format(what, mode, s, code)
        assert n == 0, "{} ({}): {} launch(es) before the refusal".format(what, mode, n)
    torch.cuda.synchronize()
    del keep


def test_stage_workspace_bytes():
    """0 for an empty shape; grows with both dimensions; covers the weight image of every mode"""
    assert N.ctn_stage_workspace_bytes(0, 5) == 0 and N.ctn_stage_workspace_bytes(5, 0) == 0
    assert N.ctn_stage_workspace_bytes(129, 64) > N.ctn_stage_workspace_bytes(128, 64)
    assert N.ctn_stage_workspace_bytes(128, 65) > N.ctn_stage_workspace_bytes(128, 64)
    for M, K in ((1, 1), (129, 513), (516, 33)):  # Wf, v1, v2 and a two-piece image of 128-row n-tiles x 32-channel slabs
        assert N.ctn_stage_workspace_bytes(M, K) >= 4 * (M * K + 2 * M) + 2 * 4 * ((M + 127) // 128 * 128) * ((K + 31) // 32 * 32)


# ---- module wrappers -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bias", [True, False])
def test_depthwise_separable_module_is_the_c_rows(bias):
    """DepthwiseSeparableConv1d(x) gives the bits of the two C entries called as the rows above call them"""
    g = torch.Generator().manual_seed(7)
    mod = DepthwiseSeparableConv1d(5, 129, 3, padding=1, dilation=2, bias=bias).to(DEV).eval()
    mod.math = "f16x3" if "f16x3" in MODES else "fp32"
    x = torch.randn(37, 5, 301, generator=g).to(DEV)
    with torch.no_grad():
        got = mod(x)
    To = R.dw_out_len(301, 3, 3, 1, 2)
    dw = R.Dw(37, 5, 301, 3, 3, 1, 2, bias, 0, "module")
    (u,), _ = _dw_call(dict(x=x.double().cpu(), w=mod.depthwise_conv1d.weight.detach()[:, 0].double().cpu(),
                            bias=mod.depthwise_conv1d.bias.detach().double().cpu() if bias else None), dw)
    pw = R.Pw(37, 129, 5, To, bias, "module")
    (y,), _ = _pw_call(dict(x=u[..., :To].double().cpu(), W=mod.pointwise_conv1d.weight.detach()[:, :, 0].double().cpu(),
                            bias=mod.pointwise_conv1d.bias.detach().double().cpu() if bias else None), pw, mod.math, 0.0)
    assert torch.equal(got, y)


def test_dprnn_model_calls_the_stage_entries_as_the_rows_do(monkeypatch):
    """DPRNNTasNet passes the head and tail what the rows pass: frames / pitch / crop from the encoder geometry, workspaces of
    at least ctn_stage_workspace_bytes, 256-byte aligned, and a latent exactly for extract_latent"""
    calls = []

    def spy(name, fn):
        def f(*args):
            calls.append((name, args))
            return fn(*args)
        return f
    monkeypatch.setattr(dprnn_tasnet, "ctn_sep_head_fwd", spy("head", N.ctn_sep_head_fwd))
    monkeypatch.setattr(dprnn_tasnet, "ctn_sep_tail_fwd", spy("tail", N.ctn_sep_tail_fwd))
    m = DPRNNTasNet(64, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=32,
                    sep_bottleneck_channels=32, sep_chunk_size=10, sep_hop_size=5, sep_num_blocks=1, causal=False, n_sources=2)
    m = m.to(DEV).eval()
    T = 1001
    x = torch.randn(3, 1, T, generator=torch.Generator().manual_seed(9)).to(DEV)
    frames, pl, _ = R.frames_of(T, 16, 8)
    with torch.no_grad():
        out = m(x)
        out2, lat = m.extract_latent(x)
    assert torch.equal(out, out2) and lat.shape == (3, 2, 64, frames)
    assert [c[0] for c in calls] == ["head", "tail", "head", "tail"]
    for k, (name, a) in enumerate(calls):
        if name == "head":
            B, Nn, Bc, fr, P, ws, nb = a[7], a[8], a[9], a[10], a[11], a[14], a[15]
            assert (B, Nn, Bc, fr, P) == (3, 64, 32, frames, R.pitch(frames))
            assert nb >= N.ctn_stage_workspace_bytes(Bc, Nn) and ws % 256 == 0
        else:
            latp, B, Nn, Bc, S, fr, P, L, s, crop, Tt, ws, nb = a[7], *a[9:19], a[20], a[21]
            assert (B, Nn, Bc, S, fr, P, L, s, crop, Tt) == (3, 64, 32, 2, frames, R.pitch(frames), 16, 8, pl, T)
            assert nb >= N.ctn_stage_workspace_bytes(S * Nn, Bc) and ws % 256 == 0
            assert (latp is not None) == (k == 3)


# ---- stage timers ------------------------------------------------------------------------------------------------------------
def _read():
    return N.profile_read()


def _zero(rec):
    return all(ms == 0.0 and n == 0 for ms, n in rec.values())


def _conv_call(model, x, latent=False):
    cfg = model.native_config()
    params, keep = model.native_params(DEV)
    B, _, T = x.shape
    frames = N.frames_of(T, model.kernel_size, model.stride)[0]
    need = C.c_size_t(0)
    N.check(N.ctn_workspace_bytes(C.byref(cfg), B, T, C.byref(need)), "ctn_workspace_bytes")
    ws, base, nbytes = _nan_ws(need.value)
    out = _nan(B, model.n_sources, T)
    lat = _nan(B, model.n_sources, model.n_basis, frames) if latent else None
    N.check(N.ctn_convtasnet_fwd(C.byref(cfg), C.byref(params), x.data_ptr(), B, T, out.data_ptr(), N.ptr(lat), base, nbytes, _st()),
            "ctn_convtasnet_fwd")
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    return (out, lat), n


def _profiled(fn):
    N.ctn_profile_enable(1)
    try:
        res = fn()
        rec = _read()
    finally:
        N.ctn_profile_enable(0)
    assert _zero(_read()), "a second read with no call in between added something"
    return res, rec


@pytest.mark.parametrize("kind", ["gln", "gln_latent", "causal"])
def test_stage_timers_leave_the_forward_alone(kind):
    """the same bits with the timers on; the summed stage launches equal the call's launch count less the launches outside
    every stage (the latent copy; the causal head's cLN0 and bias rows)"""
    cfg = G.cfg_of(N=128, Bc=32, H=64, Sc=32, R=2, X=3)
    if kind == "causal":
        cfg.causal = True
    sd = O.synth_state_dict(cfg, seed=61)
    model = _build(cfg, sd, "f16x3" if "f16x3" in MODES else "fp32")
    x, _ = O.synth_batch(2, cfg.n_sources, 4003, seed=62)
    x = x.to(DEV)
    latent = kind == "gln_latent"
    (off, n_off) = _conv_call(model, x, latent)
    (on, n_on), rec = _profiled(lambda: _conv_call(model, x, latent))
    assert n_on == n_off
    assert all(torch.equal(a, b) for a, b in zip(off, on) if a is not None), "the timers changed the output bits"
    outside = {"gln": 0, "gln_latent": R.ceil_div(2 * cfg.n_sources * cfg.n_basis, R.COPY_ROWS), "causal": 3 + 1}[kind]
    staged = sum(n for _, n in rec.values())
    print("stage timers {}: {} launches, {} inside stages, {}".format(kind, n_on, staged, {k: v[1] for k, v in rec.items() if v[1]}))
    assert staged == n_on - outside, (staged, n_on, outside)
    assert all(ms > 0.0 for ms, n in rec.values() if n), rec


def test_stage_timers_leave_a_training_step_alone():
    """one gLN training forward + backward (through PIT1d(NegSISDR)): the same estimate bits with the timers on (gradients to the
    atomics' rounding); only the fused TCN forward's stages and the loss record, and they hold fewer launches than the step made"""
    cfg = G.cfg_of(N=64, Bc=32, H=64, Sc=32, R=1, X=3)
    sd = O.synth_state_dict(cfg, seed=63)
    x, tgt = O.synth_batch(2, cfg.n_sources, 2003, seed=64)
    x, tgt = x.to(DEV), tgt.to(DEV)
    crit = PIT1d(NegSISDR(), cfg.n_sources)

    def step():
        model = _build(cfg, sd, "f16x3" if "f16x3" in MODES else "fp32").train()
        t0 = N.ctn_total_launch_count()
        out = model(x)
        loss, _ = crit(out, tgt)
        loss.backward()
        torch.cuda.synchronize()
        return out.detach(), [p.grad.clone() for p in model.parameters()], N.ctn_total_launch_count() - t0
    out0, g0, n0 = step()
    (out1, g1, n1), rec = _profiled(step)
    assert n1 == n0 and torch.equal(out0, out1), "the timers changed the estimate"
    for a, b in zip(g0, g1):
        assert float((a - b).abs().max()) <= 1e-4 * float(a.abs().max()) + 1e-30
    staged = {k: v[1] for k, v in rec.items() if v[1]}
    print("stage timers training step: {} launches, {} inside stages {}".format(n1, sum(staged.values()), staged))
    assert set(staged) <= {"prep", "pw1", "dw", "pw2", "fin", "loss"} and {"pw1", "pw2", "loss"} <= set(staged), staged
    assert 0 < sum(staged.values()) < n1


def test_stage_timers_through_dprnn():
    """DPRNN-TasNet (encoder, head, segment, dual-path blocks, overlap-add, tail: several entry calls) records no stage, and the
    timer depth it leaves lets the next Conv-TasNet forward record all its launches"""
    m = DPRNNTasNet(64, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=32,
                    sep_bottleneck_channels=32, sep_chunk_size=10, sep_hop_size=5, sep_num_blocks=2, causal=False, n_sources=2)
    m = m.to(DEV).eval()
    x = torch.randn(2, 1, 2001, generator=torch.Generator().manual_seed(11)).to(DEV)
    with torch.no_grad():
        off = m(x)
    t0 = N.ctn_total_launch_count()
    N.ctn_profile_enable(1)
    try:
        with torch.no_grad():
            on = m(x)
        torch.cuda.synchronize()
        n = N.ctn_total_launch_count() - t0
        rec = _read()
        cfg = G.cfg_of(N=128, Bc=32, H=64, Sc=32, R=1, X=2)
        model = _build(cfg, O.synth_state_dict(cfg, seed=65), "fp32")
        xc, _ = O.synth_batch(2, cfg.n_sources, 1003, seed=66)
        _, nc = _conv_call(model, xc.to(DEV))
        rec2 = _read()
    finally:
        N.ctn_profile_enable(0)
    assert torch.equal(off, on)
    assert n > 0 and _zero(rec), rec
    assert sum(v[1] for v in rec2.values()) == nc, (rec2, nc)
