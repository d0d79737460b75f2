"""The inference forward's streaming kernels one at a time (``-m gpu``), through the verification hook
(include/ctn_b200_probe.h) and the public ctn_encoder_fwd / ctn_decoder_fwd, against the fp64 references and bounds of
tests/forward_kernel_ref.py (derivations there).

Conventions of test_train_kernels_gpu.py: every output buffer starts as NaN (or, for a "+=" output, as a random nonzero
base); every input's pad columns carry finite garbage (1e6 randn).  Element-wise outputs must be bit-identical to the same
call with zero pads and exactly 0 in [frames, pitch) wherever the kernel writes them; every output must lie within its
bound.  Each row prints its worst error / bound per output next to what it reaches.
"""
import ctypes as C

import pytest
import torch

import forward_kernel_ref as R
from ctn_b200 import _native as N
from test_train_kernels_gpu import DEV, Check, Pads, _call, _elem_checks, base, dev, dptr, fptr, nan, sptr

pytestmark = pytest.mark.gpu

_p, _i, _d, _f = C.c_void_p, C.c_int, C.c_double, C.c_float
_ok = C.c_int
DBL_ADDS = 2.0 ** -29  # Check.within's base allowance is adds * u |base|: one double atomic rounds at 2^-53 = 2^-29 u


class FoldProbe(C.Structure):
    _fields_ = [("W", _p), ("bias", _p), ("gamma", _p), ("beta", _p), ("M", C.c_int32), ("K", C.c_int32),
                ("row_offset", C.c_int32), ("R", C.c_float), ("Wf", _p), ("v1", _p), ("v2", _p), ("vb", _p)]


class SkipProbe(C.Structure):
    _fields_ = [("r", _p), ("v1", _p), ("v2", _p), ("stats2", _p), ("off", C.c_int32), ("Mt", C.c_int32)]


probe_fold = N._sig("ctn_probe_fold", _ok, C.POINTER(FoldProbe), _i, _p)
probe_dw = N._sig("ctn_probe_dw_fwd", _ok, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _f, _p)
probe_finish = N._sig("ctn_probe_finish", _ok, _p, _p, _p, _p, _d, _f, _p, _i, _i, _i, _i, _i, _p)
probe_skip = N._sig("ctn_probe_skip_reduce", _ok, C.POINTER(SkipProbe), _i, _d, _f, _p, _i, _i, _i, _i, _p)
probe_stats = N._sig("ctn_probe_stats_pitch", _ok, _p, _i, _i, _i, _i, _p, _p)
probe_plain = N._sig("ctn_probe_dw_plain", _ok, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p)
probe_res = N._sig("ctn_probe_res_skip", _ok, _p, _i, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p)
probe_bias = N._sig("ctn_probe_bias_rows", _ok, _p, _p, _i, _i, _i, _i, _p)
probe_cln = N._sig("ctn_probe_cln_pitch", _ok, _p, _p, _p, _p, _i, _i, _i, _i, _f, _p, _p)

A2 = R.A2


def _d64(*shape, g):
    return base(g, *shape, dtype=torch.float64)


# ---- gLN folds ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.FOLD))
def test_fold(name):
    r = R.FOLD[name]
    ck, jobs = Check("fold", name, r), r["jobs"]
    inputs, Rv = R.fold_inputs(name, r)
    inputs = R.shared_norm(inputs, r)
    rows, Ks = {}, {}
    for jb in jobs:
        rows[jb["grp"]] = max(rows.get(jb["grp"], 0), jb["off"] + jb["M"])
        Ks[jb["grp"]] = jb["K"]
    out = {gi: dict(Wf=nan(m, Ks[gi]), v1=nan(m), v2=nan(m), vb=nan(m)) for gi, m in rows.items()}
    arr = (FoldProbe * len(jobs))()
    for j, (jb, (W, bias, gamma, beta)) in enumerate(zip(jobs, inputs)):
        o = out[jb["grp"]]
        arr[j] = FoldProbe(fptr(W), None if bias is None else fptr(bias), fptr(gamma), fptr(beta), jb["M"], jb["K"], jb["off"], Rv,
                           o["Wf"].data_ptr(), o["v1"].data_ptr(), o["v2"].data_ptr(), None if r.get("novb") else o["vb"].data_ptr())
    _call(probe_fold, arr, len(jobs))
    for jb, (W, bias, gamma, beta) in zip(jobs, inputs):
        o, sl = out[jb["grp"]], slice(jb["off"], jb["off"] + jb["M"])
        ref = R.fold(dev(W), None if bias is None else dev(bias), dev(gamma), dev(beta), Rv)
        for k in ("Wf", "v1", "v2") + (() if r.get("novb") else ("vb",)):
            ck.within(k, o[k][sl], ref[k])
    for gi, o in out.items():
        for k in ("Wf", "v1", "v2"):
            if bool(torch.isnan(o[k]).any()):
                ck.fail.append(f"fold/{name}: group {gi} {k} has rows no job wrote")
        if r.get("novb") and not bool(torch.isnan(o["vb"]).all()):
            ck.fail.append(f"fold/{name}: vb written although null")
    ck.done()


# ---- depthwise stage (k_dw) ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.DW))
def test_dw_fwd(name):
    r = R.DW[name]
    ck, B, Cc, F, P, d = Check("dw", name, r), r["B"], r["C"], r["F"], r["P"], r["d"]
    pitch = R.pitch_of(F, r["extra"])

    def run(r, pads):
        h, g1, b1, wd, bd, stats1 = R.dw_inputs(name, r)
        u, s0 = nan(B, Cc, pitch), _d64(B, 2, g=R.gen("dwbase" + name))
        s = s0.clone()
        _call(probe_dw, pads(h, pitch).data_ptr(), u.data_ptr(), fptr(g1), fptr(b1), fptr(wd), fptr(bd), sptr(A2), dptr(stats1),
              s.data_ptr(), B, Cc, F, pitch, P, d, R.EPS)
        return dict(u=u, s=s, s0=s0, inp=(h, g1, b1, wd, bd, stats1))

    a, b = run(r, Pads(21, True)), run(r, Pads(21, False))
    _elem_checks(ck, a, b, ["u"], F)
    h, g1, b1, wd, bd, stats1 = (dev(t) for t in a["inp"])
    ck.within("u", a["u"][..., :F], R.dw_fwd(h, g1, b1, wd, bd, A2, stats1, Cc * F, R.EPS, P, d)["u"])
    nc = R.dw_cta(Cc, pitch)
    ck.within("stats2", a["s"], R.stats_fp32_quads(a["u"][..., :F].double(), nc), a["s0"], nc * DBL_ADDS)
    ck.done()


# ---- skip reduce -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.SKIP))
def test_skip_reduce(name):
    r = R.SKIP[name]
    ck, B, F, Sc = Check("skip_reduce", name, r), r["B"], r["F"], r["Sc"]
    pitch = R.pitch_of(F, r["extra"])

    def run(r, pads):
        jobs, n2 = R.skip_inputs(name, r)
        arr = (SkipProbe * len(jobs))()
        for i, jb in enumerate(jobs):
            arr[i] = SkipProbe(pads(jb["r"], pitch).data_ptr(), fptr(jb["v1"]), fptr(jb["v2"]), dptr(jb["stats"]), jb["off"], jb["Mt"])
        skip = nan(B, Sc, pitch)
        _call(probe_skip, arr, len(jobs), n2, R.EPS, skip.data_ptr(), B, Sc, F, pitch)
        return dict(skip=skip, inp=(jobs, n2))

    a, b = run(r, Pads(22, True)), run(r, Pads(22, False))
    _elem_checks(ck, a, b, ["skip"], F)
    jobs, n2 = a["inp"]
    jobs = [{k: dev(v) if torch.is_tensor(v) else v for k, v in jb.items()} for jb in jobs]
    ck.within("skip", a["skip"][..., :F], R.skip_reduce(jobs, Sc, n2, R.EPS)["skip"])
    ck.done()


# ---- finish (residual update) ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.FINISH))
def test_finish(name):
    r = R.FINISH[name]
    ck, B, F, Bc, Sc = Check("finish", name, r), r["B"], r["F"], r["Bc"], r["Sc"]
    pitch = R.pitch_of(F, r["extra"])

    def run(r, pads):
        x0, rr, v1, v2, stats, n2 = R.finish_inputs(name, r)
        x = pads(x0, pitch)
        _call(probe_finish, pads(rr, pitch).data_ptr(), fptr(v1), fptr(v2), dptr(stats), n2, R.EPS, x.data_ptr(), B, Bc, Sc, F, pitch)
        return dict(x=x, inp=(x0, rr, v1, v2, stats, n2))

    a, b = run(r, Pads(23, True)), run(r, Pads(23, False))
    _elem_checks(ck, a, b, ["x"], F)
    x0, rr, v1, v2, stats, n2 = a["inp"]
    ck.within("x", a["x"][..., :F], R.finish(dev(x0), dev(rr), dev(v1), dev(v2), dev(stats), n2, R.EPS, Bc)["x"])
    ck.done()


# ---- gLN0 statistics of stand-alone separator() (k_stats_pitch) --------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.STATS))
def test_stats_pitch(name):
    r = R.STATS[name]
    ck, B, Cc, F = Check("stats_pitch", name, r), r["B"], r["C"], r["F"]
    pitch = R.pitch_of(F, r["extra"])
    x = R.stats_inputs(name, r)
    s0 = _d64(B, 2, g=R.gen("stbase" + name))
    s = s0.clone()
    _call(probe_stats, Pads(24, True)(x, pitch).data_ptr(), B, Cc, F, pitch, s.data_ptr())
    ck.within("stats", s, R.stats_pitch(dev(x))["stats"], s0, min(Cc, 64) * DBL_ADDS)
    ck.done()


# ---- encoder ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ENC))
def test_encoder(name):
    r = R.ENC[name]
    ck, B, Nn, L, S = Check("encoder", name, r), r["B"], r["N"], r["L"], r["S"]
    relu = bool(r.get("relu"))
    x, W, pl, pr, F = R.enc_inputs(name, r)
    wp = R.pitch_of(F) + r.get("wpad", 0)
    off = r.get("woff", 0)
    buf = torch.full((B * Nn * wp + 4,), float("nan"), device=DEV)
    w = buf[off:off + B * Nn * wp].view(B, Nn, wp)
    s0 = _d64(B, 2, g=R.gen("encbase" + name))
    s = s0.clone()
    _call(N.ctn_encoder_fwd, fptr(x), fptr(W), w.data_ptr(), B, r["T"], pl, pr, Nn, L, S, int(relu), wp, s.data_ptr())
    ck.pads_zero("w", w, F)
    ck.within("w", w[..., :F], R.encoder(dev(x), dev(W), S, pl, pr, relu)["w"])
    v4 = L <= 20 and S * 2 == L and wp % 128 == 0 and off == 0
    nc = -(-wp // 128)
    ck.within("stats", s, R.encoder_stats(w[..., :F].double(), v4, nc)["stats"], s0, nc * DBL_ADDS)
    ck.done()


# ---- decoder ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.DEC))
def test_decoder(name):
    r = R.DEC[name]
    ck, BS, Nn, F, L, S = Check("decoder", name, r), r["B"], r["N"], r["F"], r["L"], r["S"]
    pitch = R.pitch_of(F)

    def run(r, pads):
        what, Wd, T_out = R.dec_inputs(name, r)
        y = nan(BS, T_out)
        _call(N.ctn_decoder_fwd, pads(what, pitch).data_ptr(), fptr(Wd), y.data_ptr(), BS, Nn, F, pitch, L, S, r["crop"], T_out)
        return dict(y=y, inp=(what, Wd, T_out))

    a, b = run(r, Pads(25, True)), run(r, Pads(25, False))
    ck.same("y", a["y"], b["y"])
    what, Wd, T_out = a["inp"]
    ck.within("y", a["y"], R.decoder(dev(what), dev(Wd), S, r["crop"], T_out)["y"])
    ck.done()


# ---- causal pipeline: k_dw_plain, k_res_skip, k_bias_rows, pitched cLN ----------------------------------------------------------
@pytest.mark.parametrize("name", list(R.PLAIN))
def test_dw_plain(name):
    r = R.PLAIN[name]
    ck, B, Cc, F, P, d = Check("dw_plain", name, r), r["B"], r["C"], r["F"], r["P"], r["d"]
    pitch = R.pitch_of(F, r["extra"])

    def run(r, pads):
        h, wd, bd = R.plain_inputs(name, r)
        u = nan(B, Cc, pitch)
        _call(probe_plain, pads(h, pitch).data_ptr(), u.data_ptr(), fptr(wd), fptr(bd), sptr(A2), B, Cc, F, pitch, P, d, (P - 1) * d)
        return dict(u=u, inp=(h, wd, bd))

    a, b = run(r, Pads(26, True)), run(r, Pads(26, False))
    _elem_checks(ck, a, b, ["u"], F)
    h, wd, bd = (dev(t) for t in a["inp"])
    ck.within("u", a["u"][..., :F], R.dw_plain(h, wd, bd, A2, P, d)["u"])
    ck.done()


@pytest.mark.parametrize("name", list(R.RES))
def test_res_skip(name):
    r = R.RES[name]
    ck, B, F, Bc, Sc = Check("res_skip", name, r), r["B"], r["F"], r["Bc"], r["Sc"]
    has_out, init, inplace = r["has_out"], r["init"], r["inplace"]
    pitch = R.pitch_of(F, r["extra"])
    Mt = Bc + Sc if has_out else Sc

    def run(r, pads):
        rr, xin, skip0, bo, bs = R.res_inputs(name, r)
        xi, sk = pads(xin, pitch), pads(skip0, pitch)
        xi0 = xi.clone()
        xo = xi if inplace else nan(B, Bc, pitch)
        _call(probe_res, pads(rr, pitch).data_ptr(), Mt, xi.data_ptr(), xo.data_ptr(), sk.data_ptr(),
              fptr(bo) if has_out else None, fptr(bs), Bc, Sc, has_out, init, B, F, pitch)
        return dict(x=xo, skip=sk, xin=xi, xin0=xi0, inp=(rr, xin, skip0, bo, bs))

    a, b = run(r, Pads(27, True)), run(r, Pads(27, False))
    _elem_checks(ck, a, b, ["skip"] + (["x"] if has_out else []), F)
    if not inplace or not has_out:
        assert torch.equal(a["xin"], a["xin0"]), f"{name}: xin changed"
    if not has_out and not inplace:
        assert bool(torch.isnan(a["x"]).all()), f"{name}: xout written without an output head"
    rr, xin, skip0, bo, bs = (dev(t) for t in a["inp"])
    ref = R.res_skip(rr, xin, skip0, bo, bs, Bc, has_out, init)
    if has_out:
        ck.within("x", a["x"][..., :F], ref["x"])
    ck.within("skip", a["skip"][..., :F], ref["skip"])
    ck.done()


@pytest.mark.parametrize("name", list(R.BIAS))
def test_bias_rows(name):
    r = R.BIAS[name]
    ck, B, Cc, F = Check("bias_rows", name, r), r["B"], r["C"], r["F"]
    pitch = R.pitch_of(F, r["extra"])

    def run(r, pads):
        g = R.gen("bias" + name)
        y0, bias = R.rnd(g, B, Cc, F), R.rnd(g, Cc, scale=0.3)
        y = pads(y0, pitch)
        _call(probe_bias, y.data_ptr(), fptr(bias), Cc, B, F, pitch)
        return dict(y=y, inp=(y0, bias))

    a, b = run(r, Pads(28, True)), run(r, Pads(28, False))
    _elem_checks(ck, a, b, ["y"], F)
    y0, bias = (dev(t) for t in a["inp"])
    ck.within("y", a["y"][..., :F], R.bias_rows(y0, bias)["y"])
    ck.done()


@pytest.mark.parametrize("name", list(R.CLN))
def test_cln_pitch_in_place(name):
    r = R.CLN[name]
    ck, B, Cc, F = Check("cln_pitch", name, r), r["B"], r["C"], r["F"]
    pitch = R.pitch_of(F, r["extra"])

    def run(r, pads):
        g = R.gen("cln" + name)
        x0 = R.f32(R.rnd(g, B, Cc, F, scale=0.8, shift_=0.3) * R.sample_scale(B))
        gm, bt = R.rnd(g, Cc, scale=0.1, shift_=1.0), R.rnd(g, Cc, scale=0.05)
        x = pads(x0, pitch)
        scratch = torch.full((B * F * 2,), float("nan"), dtype=torch.float64, device=DEV)
        _call(probe_cln, x.data_ptr(), fptr(gm), fptr(bt), x.data_ptr(), B, Cc, F, pitch, R.EPS, scratch.data_ptr())
        return dict(y=x, inp=(x0, gm, bt))

    a, b = run(r, Pads(29, True)), run(r, Pads(29, False))
    _elem_checks(ck, a, b, ["y"], F)
    x0, gm, bt = (dev(t) for t in a["inp"])
    ck.within("y", a["y"][..., :F], R.cln(x0, gm, bt, R.EPS)["y"])
    ck.done()
