"""The fp16-piece operand scales the pipelines choose (``-m gpu``), read back from a real forward's workspace through the
verification hook (ctn_probe_tcn_envelope), against the fp64 envelope of tests/envelope_ref.py.

Per row (`reaches` names what it reaches):
  * every scale passes E.scale_score (power of two, s bound64 <= 2^15, the largest such one up to fp32 rounding), the row bounds
    vb pass E.vb_score, dwp matches its packing bit for bit (P = 3), x_0's bound matches (measured max |x| bit for bit, or the
    head's row bounds);
  * the fp64 operand of every fp16-piece contraction (x_i for pw1, u_i for pw2, PReLU(skip sum) for the mask) satisfies
    max |operand| s <= 2^15: saturation is impossible on these inputs, not merely absent; the headroom log2(2^15 / (max|op| s))
    of each contraction is printed;
  * the forward's output matches fp64 at the parity bound of smoke() (2e-5 + 1e-4 max |ref|), so that a scale wired to the wrong
    contraction shows up where it saturates.
The paper-config rows (PAPER) also hold blocks 0, 11 and 23 and the mask contraction, fed their fp64 operands at the scale the
pipeline chose, to the gate of tests/pw_criterion.py.
"""
import ctypes as C
import math

import pytest
import torch

import convtasnet_oracle as O
import envelope_ref as E
import pw_criterion as PC
import test_pw_contraction_gpu as PW
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-12
_p = C.c_void_p
probe_env = N._sig("ctn_probe_tcn_envelope", C.c_int, C.POINTER(N.Config), C.c_int, C.c_int, C.c_int, _p, _p, _p, _p, _p, _p)
probe_absmax = N._sig("ctn_probe_absmax_pitch", C.c_int, _p, C.c_int, C.c_int, C.c_int, _p, _p)
ENV_TCN, ENV_MODEL, ENV_TRAIN = 0, 1, 2


def _dev():
    return torch.device(DEV, torch.cuda.current_device())


def _parity(got, ref, what):
    err, top = float((got.double() - ref).abs().max()), float(ref.abs().max())
    assert err <= 2e-5 + 1e-4 * top, f"{what}: max error {err:.3e} vs max |ref| {top:.3e}"
    return err / (2e-5 + 1e-4 * top)


def _gen_blocks(seed, n, Bc, H, Sc, P, last_out=False, a2=0.25, g1=1.0, g2=1.0, taps="randn", bd=0.1, impulse=None):
    """fp32 values held as fp64, oracle-free synthetic blocks (the dict layout of E.blocks_of)"""
    g = torch.Generator().manual_seed(seed)

    def r(*shape, scale=1.0, shift=0.0):
        return (torch.randn(*shape, generator=g) * scale + shift).float().double()
    out = []
    for i in range(n):
        wd = r(H, P, scale=0.5)
        if taps == "same_sign":
            wd = wd.abs() + 0.2
        elif taps == "zero":
            wd = torch.zeros_like(wd)
        has_out = last_out or i < n - 1
        blk = dict(W1=r(H, Bc, scale=Bc ** -0.5), b1=r(H, scale=0.05), a1=0.25, g1=r(H, scale=0.1 * g1, shift=g1),
                   be1=r(H, scale=0.05), wd=wd, bd=torch.zeros(H, dtype=torch.float64) if taps == "zero" else r(H, scale=bd, shift=bd),
                   a2=a2, g2=r(H, scale=0.1 * g2, shift=g2), be2=r(H, scale=0.05),
                   Wo=r(Bc, H, scale=H ** -0.5) if has_out else None, bo=r(Bc, scale=0.05) if has_out else None,
                   Ws=r(Sc, H, scale=H ** -0.5), bs=r(Sc, scale=0.05))
        if impulse is not None and i == 0:
            # x is silent but for one element in channel `impulse`: with b1 = 0 and one non-zero weight in that column, h is 0 but
            # for one element, whose gLN1 value is sqrt(H frames - 1)
            blk["b1"] = torch.zeros(H, dtype=torch.float64)
            blk["W1"][:, impulse] = 0.0
            blk["W1"][3, impulse] = 1.5
        out.append(blk)
    return out


def _block_slots(blocks):
    f = lambda t: None if t is None else t.float().contiguous().to(DEV)  # noqa: E731
    s = lambda a: torch.tensor([float(a)], device=DEV)  # noqa: E731
    slots = []
    for i, b in enumerate(blocks):
        vals = (f(b["W1"]), f(b["b1"]), s(b["a1"]), f(b["g1"]), f(b["be1"]), f(b["wd"]), f(b["bd"]), s(b["a2"]), f(b["g2"]),
                f(b["be2"]), f(b["Wo"]), f(b["bo"]), f(b["Ws"]), f(b["bs"]))
        slots += [((i, name), t) for name, t in zip(N.BLOCK_FIELDS, vals)]
    return slots


def _readback(cfg, B, frames, path, ws_base):
    n = cfg.num_blocks * cfg.num_layers
    Hp = (cfg.hidden + 15) // 16 * 16
    scales = torch.full((2 * n + 1,), float("nan"), device=DEV)
    dwp = torch.full((n, Hp, 8), float("nan"), device=DEV)
    vbs = torch.full((n, cfg.bottleneck + cfg.skip), float("nan"), device=DEV)
    x0 = torch.full((cfg.bottleneck,), float("nan"), device=DEV)
    st = probe_env(C.byref(cfg), B, frames, path, ws_base, scales.data_ptr(), dwp.data_ptr(), vbs.data_ptr(), x0.data_ptr(),
                   N.stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    assert st == N.CTN_OK, st
    return scales.cpu().double(), dwp.cpu(), vbs.cpu().double(), x0.cpu()


def _check_envelope(name, cfg, blocks, frames, scales, dwp, vbs, x0_bound, mask_slope, K_x0):
    """scales / vb / dwp against fp64; returns (bounds64, report)"""
    n, Bc, Sc, H = len(blocks), cfg.bottleneck, cfg.skip, cfg.hidden
    bounds, vbs64 = E.envelope(blocks, H, frames, x0_bound, mask_slope)
    sl = E.slack(max(H, K_x0), n)
    worst, ratios, fails = 0.0, [], []
    for j, (s, b) in enumerate(zip(scales.tolist(), bounds)):
        sc, q = E.scale_score(s, b, sl)
        worst = max(worst, sc)
        ratios.append(q)
        if sc > 1.0:
            fails.append(f"scale[{j}] = 2^{math.log2(s) if s > 0 else s} for bound64 {b:.6g}: score {sc:.3g}")
    vworst = 0.0
    for i, ((vo, vs), blk) in enumerate(zip(vbs64, blocks)):
        if vo is not None:
            vworst = max(vworst, E.vb_score(vbs[i, :Bc], vo, H), E.vb_score(vbs[i, Bc:Bc + Sc], vs, H))
        else:
            vworst = max(vworst, E.vb_score(vbs[i, :Sc], vs, H))
        if cfg.sep_kernel == 3:
            assert torch.equal(dwp[i], E.dwp_pack(blk, H)), f"{name}: dwp of block {i} differs from its packing"
    assert not fails, f"{name}: " + "; ".join(fails)
    assert vworst <= 1.0, f"{name}: vb score {vworst:.3g}"
    q = sorted(set(ratios))
    return bounds, f"scale/fp64 in {{{', '.join(f'{v:g}' for v in q)}}} (score {worst:.3f}), vb score {vworst:.3f}"


def _headroom(name, scales, xmax, umax, mask_max):
    """asserts max|op| s <= 2^15 for every fp16-piece contraction; returns the headrooms (binades) [pw1_i, pw2_i, ..., mask]"""
    ops = [v for pair in zip(xmax, umax) for v in pair] + [mask_max]
    hr = []
    for j, (m, s) in enumerate(zip(ops, scales.tolist())):
        assert m * s <= E.TOP, f"{name}: operand {j} max {m:.6g} x scale {s:g} = {m * s:.6g} > 2^15: fp16 pieces can saturate"
        hr.append(math.log2(E.TOP / (m * s)) if m > 0 else math.inf)
    return hr


def _fmt_hr(hr):
    fin = [h for h in hr[:-1] if math.isfinite(h)]
    pw1, pw2 = [h for h in hr[0:-1:2] if math.isfinite(h)], [h for h in hr[1:-1:2] if math.isfinite(h)]
    rng = lambda v: f"{min(v):.1f}..{max(v):.1f}" if v else "-"  # noqa: E731
    return f"headroom pw1 {rng(pw1)} pw2 {rng(pw2)} mask {hr[-1]:.1f} binades" if fin or math.isfinite(hr[-1]) else "headroom -"


# ---- stand-alone TCN rows (ctn_tcn_blocks_fwd; |x_0| measured, no mask slope: the mask bound is S) --------------------------
def _trow(reaches, n=3, Bc=32, H=64, Sc=32, P=3, frames=1000, B=2, dil=None, **kw):
    r = dict(reaches=reaches, n=n, Bc=Bc, H=H, Sc=Sc, P=P, frames=frames, B=B, dil=dil or [2 ** (i % 8) for i in range(n)],
             x="randn")
    r.update(kw)
    return r


TCN_ROWS = {
    "h300_bc160_sc170": _trow("H = 300 > 256, not a multiple of 16 (padded channels, two passes of the partials loop); Bc + Sc = 330 > 256",
                              Bc=160, H=300, Sc=170),
    "p1": _trow("P = 1: k_dw + scaled PRO_NONE, no dwp", P=1, dil=[1, 1, 1]),
    "p2": _trow("P = 2", P=2, dil=[1, 2, 4]),
    "p4_d3": _trow("P = 4, dilation 3", P=4, dil=[1, 3, 2]),
    "p8": _trow("P = 8: the depthwise sum over 8 taps", P=8, dil=[2, 5, 1]),
    "p3_d3_unfused": _trow("P = 3 at dilation 3 and 6: outside the fused producer, dwp still packed", dil=[3, 6, 1]),
    "last_with_out": _trow("the last block has an out head (x chain over all blocks)", last_out=True),
    "n64_f1": _trow("R X = 4 x 16 = 64 = CTN_MAX_BLOCKS through ctn_tcn_fwd, frames = 1", n=64, Bc=16, H=48, Sc=16, frames=1, B=1,
                    tcn_fwd=(4, 16), dil=[2 ** (i % 16) for i in range(64)]),
    "slope2_m3_big_gamma": _trow("slope2 = -3 (|a2| > 1), gamma1 = gamma2 = 8", a2=-3.0, g1=8.0, g2=8.0),
    "same_sign_taps_big_bd": _trow("depthwise taps of one sign, bd = 5", taps="same_sign", bd=5.0),
    "zero_dw": _trow("all-zero depthwise weights and biases: U = 0, scale 1", taps="zero"),
    "impulse_after_silence": _trow("x = 0 but one element: one gLN1 value at sqrt(H frames - 1)", x="impulse", frames=4000, B=1,
                                   impulse=5),
    "dc_plus_spike": _trow("x = DC 3 + one spike of 200", x="dc_spike", frames=2000),
}


def _tcn_input(r, g):
    B, Bc, T = r["B"], r["Bc"], r["frames"]
    if r["x"] == "impulse":
        x = torch.zeros(B, Bc, T, dtype=torch.float64)
        x[:, r["impulse"], T // 2] = 1.0
        return x
    x = torch.randn(B, Bc, T, generator=g).float().double()
    if r["x"] == "dc_spike":
        x = 0.1 * x + 3.0
        x[:, 7, T // 3] = 200.0
    return x


@pytest.mark.parametrize("name", list(TCN_ROWS))
def test_tcn_scales_vs_fp64(name):
    r = TCN_ROWS[name]
    seed = sum(map(ord, name))
    g = torch.Generator().manual_seed(seed)
    blocks = _gen_blocks(seed, r["n"], r["Bc"], r["H"], r["Sc"], r["P"], r.get("last_out", False), r.get("a2", 0.25),
                         r.get("g1", 1.0), r.get("g2", 1.0), r.get("taps", "randn"), r.get("bd", 0.1), r.get("impulse"))
    x = _tcn_input(r, g)
    B, T, n = r["B"], r["frames"], r["n"]
    cfg = N.Config()
    cfg.bottleneck, cfg.hidden, cfg.skip, cfg.sep_kernel = r["Bc"], r["H"], r["Sc"], r["P"]
    cfg.num_blocks, cfg.num_layers, cfg.math, cfg.eps, cfg.eps_tcn = 1, n, N.MATH_F16X3, EPS, EPS
    if r.get("tcn_fwd"):  # ctn_tcn_fwd: num_blocks x num_layers with dilations 2^l
        cfg.num_blocks, cfg.num_layers = r["tcn_fwd"]
    slots = _block_slots(blocks)  # build_params does not keep the tensors alive
    params, keep = N.build_params(slots, _dev())
    dil = (C.c_int * n)(*r["dil"])
    need = C.c_size_t(0)
    assert N.ctn_tcn_workspace_bytes(C.byref(cfg), B, T, C.byref(need)) == N.CTN_OK
    wsbuf = torch.empty(need.value + 512, dtype=torch.uint8, device=DEV)
    base, nbytes = N.aligned(wsbuf)
    xd = x.float().to(DEV).contiguous()
    skip = torch.empty(B, r["Sc"], T, device=DEV)
    xo = torch.empty(B, r["Bc"], T, device=DEV) if r.get("last_out") else None
    if r.get("tcn_fwd"):
        st = N.ctn_tcn_fwd(C.byref(cfg), params.blocks, xd.data_ptr(), skip.data_ptr(), B, T, base, nbytes, N.stream_ptr(torch.device(DEV)))
    else:
        st = N.ctn_tcn_blocks_fwd(C.byref(cfg), params.blocks, n, dil, xd.data_ptr(), N.ptr(xo), skip.data_ptr(), B, T, base, nbytes,
                                  N.stream_ptr(torch.device(DEV)))
    assert st == N.CTN_OK, st
    scales, dwp, vbs, x0 = _readback(cfg, B, T, ENV_TCN, base)
    xmax32 = xd.abs().max().cpu()
    assert torch.equal(x0[:1], xmax32.view(1)), f"{name}: x0 bound {float(x0[0])} != max |x| {float(xmax32)}"
    _, rep = _check_envelope(name, cfg, blocks, T, scales, dwp, vbs, float(xmax32), None, r["H"])
    ref = E.tcn_forward(x.to(DEV), [{k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in b.items()} for b in blocks], r["dil"], EPS)
    hr = _headroom(name, scales, ref["xmax"], ref["umax"], float(ref["skip"].abs().max()))
    p = _parity(skip, ref["skip"], f"{name} skip")
    if xo is not None:
        p = max(p, _parity(xo, ref["x_out"], f"{name} x_out"))
    print(f"{name} [{r['reaches']}]: {rep}; {_fmt_hr(hr)}; output e/parity bound {p:.3f}")


# ---- ctn_absmax_pitch ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,frames,pre", [(1500, 129, 0.0), (3, 1, 0.0), (2100, 300, 1e4), (7, 128, 0.0)])
def test_absmax_pitch(rows, frames, pre):
    """more than 1024 rows (grid-stride loop), NaN past frames (ignored), -0, an output already holding a larger value"""
    g = torch.Generator().manual_seed(rows + frames)
    pitch = N.ctn_pitch(frames)
    x = torch.full((rows, pitch), float("nan"), device=DEV)
    v = torch.randn(rows, frames, generator=g) * 3.0
    v[rows // 2, frames // 2] = -50.0 - rows  # the largest magnitude is negative
    v[0, 0] = -0.0
    x[:, :frames] = v.to(DEV)
    out = torch.tensor([pre], device=DEV)
    assert probe_absmax(x.data_ptr(), rows, frames, pitch, out.data_ptr(), N.stream_ptr(torch.device(DEV))) == N.CTN_OK
    torch.cuda.synchronize()
    assert float(out) == max(pre, float(v.abs().max()))
    z = torch.full((1, 128), -0.0, device=DEV)
    out = torch.tensor([0.0], device=DEV)
    assert probe_absmax(z.data_ptr(), 1, 1, 128, out.data_ptr(), N.stream_ptr(torch.device(DEV))) == N.CTN_OK
    torch.cuda.synchronize()
    assert float(out) == 0.0 and not math.copysign(1.0, float(out)) < 0


# ---- model path (ctn_convtasnet_fwd / ctn_convtasnet_fwd_train; x_0 bound = the head's row bounds) ---------------------------
def _ocfg(N_, Bc, H, Sc, R, X, S=2):
    return O.OracleConfig(n_basis=N_, kernel_size=16, sep_bottleneck_channels=Bc, sep_hidden_channels=H, sep_skip_channels=Sc,
                          sep_kernel_size=3, sep_num_blocks=R, sep_num_layers=X, n_sources=S)


def _native_cfg(oc):
    cfg = N.Config()
    cfg.n_basis, cfg.kernel_size, cfg.stride = oc.n_basis, oc.kernel_size, oc.stride
    cfg.bottleneck, cfg.hidden, cfg.skip, cfg.sep_kernel = oc.sep_bottleneck_channels, oc.sep_hidden_channels, oc.sep_skip_channels, 3
    cfg.num_blocks, cfg.num_layers, cfg.n_sources = oc.sep_num_blocks, oc.sep_num_layers, oc.n_sources
    cfg.math, cfg.eps, cfg.eps_tcn, cfg.in_channels = N.MATH_F16X3, EPS, EPS, 1
    return cfg


def _model_slots(sd, oc):
    f = lambda k: sd[k].float().contiguous().to(DEV)  # noqa: E731
    top = dict(enc_w=f("encoder.conv1d.weight"), norm0_g=f("separator.norm1d.norm.weight"), norm0_b=f("separator.norm1d.norm.bias"),
               bn_w=f("separator.bottleneck_conv1d.weight"), bn_b=f("separator.bottleneck_conv1d.bias"),
               prelu_out=f("separator.prelu.weight"), mask_w=f("separator.mask_conv1d.weight"), mask_b=f("separator.mask_conv1d.bias"),
               dec_w=f("decoder.conv_transpose1d.weight"))
    blocks = E.blocks_of(sd, E.block_prefixes(oc.sep_num_blocks, oc.sep_num_layers))
    return [(k, top[k]) for k in N.TOP_FIELDS] + _block_slots(blocks), blocks


def _model_case(name, oc, sd, B, T, train=False, keep=()):
    """runs the native forward, reads the envelope back and checks it; returns what the gate rows need"""
    dev = _dev()
    cfg = _native_cfg(oc)
    slots, blocks = _model_slots(sd, oc)  # slots holds the parameter tensors for the whole call
    params, pkeep = N.build_params(slots, dev)
    frames, _, _ = N.frames_of(T, oc.kernel_size, oc.stride)
    need = C.c_size_t(0)
    sizer = N.ctn_train_workspace_bytes if train else N.ctn_workspace_bytes
    assert sizer(C.byref(cfg), B, T, C.byref(need)) == N.CTN_OK
    wsbuf = torch.empty(need.value + 512, dtype=torch.uint8, device=dev)
    base, nbytes = N.aligned(wsbuf)
    mix, _ = O.synth_batch(B, 2, T, seed=sum(map(ord, name)))
    xd = mix.to(dev).contiguous()
    out = torch.empty(B, oc.n_sources, T, device=dev)
    if train:
        st = N.ctn_convtasnet_fwd_train(C.byref(cfg), C.byref(params), xd.data_ptr(), B, T, out.data_ptr(), base, nbytes, N.stream_ptr(dev))
    else:
        st = N.ctn_convtasnet_fwd(C.byref(cfg), C.byref(params), xd.data_ptr(), B, T, out.data_ptr(), None, base, nbytes, N.stream_ptr(dev))
    assert st == N.CTN_OK, st
    scales, dwp, vbs, x0 = _readback(cfg, B, frames, ENV_TRAIN if train else ENV_MODEL, base)
    head64 = E.head_bound(sd["separator.bottleneck_conv1d.weight"], sd["separator.bottleneck_conv1d.bias"],
                          sd["separator.norm1d.norm.weight"], sd["separator.norm1d.norm.bias"], oc.n_basis, frames)
    hs = E.vb_score(x0.double(), head64, oc.n_basis)
    assert hs <= 1.0, f"{name}: head row bounds score {hs:.3g}"
    a_mask = float(sd["separator.prelu.weight"])
    bounds, rep = _check_envelope(name, cfg, blocks, frames, scales, dwp, vbs, float(head64.max()), a_mask, oc.n_basis)
    # fp64 operands on the GPU
    sd64 = {k: v.double().to(dev) for k, v in sd.items()}
    x64 = mix.double().to(dev)
    pad = (oc.stride - (T - oc.kernel_size) % oc.stride) % oc.stride
    w = O.encoder_fwd(torch.nn.functional.pad(x64, (pad // 2, pad - pad // 2)), sd64["encoder.conv1d.weight"], oc.stride)
    x0_64 = torch.nn.functional.conv1d(O.gln(w, sd64["separator.norm1d.norm.weight"], sd64["separator.norm1d.norm.bias"], EPS),
                                       sd64["separator.bottleneck_conv1d.weight"], sd64["separator.bottleneck_conv1d.bias"])
    b64 = [{k: (v.double().to(dev) if torch.is_tensor(v) else v) for k, v in b.items()} for b in blocks]
    ref = E.tcn_forward(x0_64, b64, [2 ** (i % oc.sep_num_layers) for i in range(len(blocks))], EPS, keep=keep)
    mop = E.prelu(ref["skip"], a_mask)
    hr = _headroom(name, scales, ref["xmax"], ref["umax"], float(mop.abs().max()))
    ref_out, _ = O.conv_tasnet_fwd(x64, sd64, oc)
    p = _parity(out, ref_out, f"{name} output")
    return dict(cfg=cfg, scales=scales, hr=hr, rep=rep, ref=ref, blocks=blocks, w=w, mop=mop, sd=sd, frames=frames, parity=p,
                bounds=bounds)


MODEL_ROWS = {
    "small_mask_slope_m4": dict(oc=(128, 32, 64, 32, 2, 3), B=2, T=4000, mask_slope=-4.0,
                                reaches="model path: x_0 from the head's row bounds (R = sqrt(N frames)); mask slope -4 (|a| > 1)"),
    "small_train": dict(oc=(128, 32, 64, 32, 2, 3), B=2, T=4000, mask_slope=0.25, train=True,
                        reaches="training forward (fused TCN): its own carve of the same envelope"),
}


@pytest.mark.parametrize("name", list(MODEL_ROWS))
def test_model_scales_vs_fp64(name):
    r = MODEL_ROWS[name]
    oc = _ocfg(*r["oc"])
    sd = {k: v.double() for k, v in O.synth_state_dict(oc, seed=sum(map(ord, name))).items()}
    sd["separator.prelu.weight"] = torch.tensor([r["mask_slope"]], dtype=torch.float64)
    c = _model_case(name, oc, sd, r["B"], r["T"], train=r.get("train", False))
    print(f"{name} [{r['reaches']}]: {c['rep']}; {_fmt_hr(c['hr'])}; output e/parity bound {c['parity']:.3f}")


# ---- the gate at the pipelines' own scales (paper config) --------------------------------------------------------------------
PAPER = {
    "cfg2_4s": dict(T=32000, B=2, reaches="paper config, 4 s at 8 kHz (3999 frames), B = 2"),
    "cfg5_16s": dict(T=128000, B=1, reaches="paper config, 15999 frames"),
    "long_60s": dict(T=480000, B=1, reaches="paper config, 60 s at 8 kHz (59999 frames)"),
}
GATE_BLOCKS = (0, 11, 23)


def _gate(W, P, mode_scale, pro, epi, B, M, K, frames, extra):
    """one contraction through ctn_probe_pw in the f16x3 mode at operand scale mode_scale; -> e / bound"""
    pitch = N.ctn_pitch(frames)
    dev = torch.device(DEV)
    keep = []
    a = PW.ProbeArgs()
    a.B, a.M, a.K, a.frames, a.pitch = B, M, K, frames, pitch
    A = PW._padded(P, pitch)
    Wf = W.float().contiguous()
    Pv = P.float().double()  # the operand as the kernel reads it
    a.A, a.W = A.data_ptr(), Wf.data_ptr()
    if pro == "prelu":
        Pm_val, _ = PC.pro_prelu(Pv, extra["pro_slope"])
        a.pro_slope = (t := torch.tensor([extra["pro_slope"]], device=dev)).data_ptr()
        keep.append(t)
    else:
        Pm_val = Pv
    if epi == "h":
        fe = PC.epi_h(extra["bias"], extra["slope"])
        bias, sl = extra["bias"].float().contiguous(), torch.tensor([extra["slope"]], device=dev)
        keep += [bias, sl]
        a.bias, a.slope = bias.data_ptr(), sl.data_ptr()
        stats = torch.zeros(B, 2, dtype=torch.float64, device=dev)
        a.stats_out = stats.data_ptr()
    elif epi == "mask":
        fe = PC.epi_mask(extra["bias"], extra["wenc"], extra["Nb"])
        bias = extra["bias"].float().contiguous()
        wenc = PW._padded(extra["wenc"], pitch)
        keep += [bias, wenc]
        a.bias, a.wenc, a.Nb = bias.data_ptr(), wenc.data_ptr(), extra["Nb"]
    else:
        fe = PC.epi_raw()
    ref = PC.Reference(Wf.double(), Pm_val, Pm_val.abs(), fe)
    D = torch.full((B, M, pitch), float("nan"), device=dev)
    a.D = D.data_ptr()
    s = torch.tensor([mode_scale], device=dev)
    a.act_scale = s.data_ptr()
    nbytes = PW.probe_wimg_bytes(M, K, N.MATH_F16X3)
    wimg = torch.empty(nbytes // 4 + 64, device=dev)
    st = PW.probe_pw(C.byref(a), PW.PRO[pro], PW.EPI[epi], N.MATH_F16X3, 0, wimg.data_ptr(), nbytes, N.stream_ptr(dev))
    torch.cuda.synchronize()
    assert st == N.CTN_OK, st
    e = PC.gate_e(D[..., :frames], ref.out["D"])
    return e / ref.bound("f16x3")


@pytest.mark.parametrize("name", list(PAPER))
def test_paper_config_scales_and_gate(name):
    r = PAPER[name]
    oc = _ocfg(512, 128, 512, 128, 3, 8)
    sd = {k: v.double() for k, v in O.synth_state_dict(oc, seed=111).items()}
    c = _model_case(name, oc, sd, r["B"], r["T"], keep=GATE_BLOCKS)
    ref, blocks, sc, frames, B = c["ref"], c["blocks"], c["scales"].tolist(), c["frames"], r["B"]
    gates = {}
    for i in GATE_BLOCKS:
        b = blocks[i]
        gates[f"pw1[{i}]"] = _gate(b["W1"].to(DEV), ref["x"][i], sc[2 * i], "none", "h", B, 512, 128, frames,
                                   dict(bias=b["b1"].to(DEV), slope=b["a1"]))
        Wcat = torch.cat([b["Wo"], b["Ws"]]) if b["Wo"] is not None else b["Ws"]
        Wf = (Wcat.float() * b["g2"].float().view(1, -1)).double().to(DEV)  # the gLN2 fold, as k_fold_batch rounds it
        gates[f"pw2[{i}]"] = _gate(Wf, ref["u"][i], sc[2 * i + 1], "none", "raw", B, Wf.shape[0], 512, frames, {})
    a_mask = float(c["sd"]["separator.prelu.weight"])
    gates["mask"] = _gate(c["sd"]["separator.mask_conv1d.weight"].squeeze(-1).to(DEV), ref["skip"], sc[-1], "prelu", "mask", B,
                          1024, 128, frames, dict(pro_slope=a_mask, bias=c["sd"]["separator.mask_conv1d.bias"].to(DEV),
                                                  wenc=c["w"].float().double(), Nb=512))
    worst = max(gates.values())
    print(f"{name} [{r['reaches']}]: {c['rep']}; {_fmt_hr(c['hr'])} (max {max(h for h in c['hr'] if math.isfinite(h)):.1f}); "
          f"output e/parity bound {c['parity']:.3f}; gate e/bound at the pipeline scales: "
          + ", ".join(f"{k} {v:.3f}" for k, v in gates.items()))
    assert worst <= 1.0, gates
