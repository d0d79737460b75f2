"""The training path's streaming and filter-bank gradient kernels one at a time (``-m gpu``), through the verification hook
(include/ctn_b200_probe.h), against the fp64 references and bounds of tests/train_kernel_ref.py (derivations there).

Per row: every output buffer starts as NaN (or, for a "+=" output, as a random nonzero base); every input's pad columns
carry finite garbage (1e6 randn).  Element-wise outputs must be bit-identical to the same call with zero pads and exactly 0
in [frames, pitch); every output must lie within its bound.  Each row prints its worst error / bound per output next to
what it reaches.
"""
import ctypes as C

import pytest
import torch

import train_kernel_ref as R
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu

DEV = "cuda"
U = R.U
_p, _i, _d, _f, _sz = C.c_void_p, C.c_int, C.c_double, C.c_float, C.c_size_t
_ok = C.c_int
probe_bias = N._sig("ctn_probe_bias_prelu_stats", _ok, _p, _p, _p, _p, _i, _i, _i, _i, _p)
probe_dw_fwd = N._sig("ctn_probe_dw_train_fwd", _ok, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _d, _f,
                      _p)
probe_act_norm = N._sig("ctn_probe_act_norm", _ok, _p, _p, _p, _p, _p, _p, _d, _f, _i, _i, _i, _i, _p)
probe_gln = N._sig("ctn_probe_gln_prelu_bwd", _ok, _p, _p, _p, _p, _p, _p, _d, _f, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p)
probe_dw_bwd = N._sig("ctn_probe_dw_bwd", _ok, _p, _p, _p, _p, _p, _p, _p, _d, _f, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i,
                      _p)
probe_mask = N._sig("ctn_probe_mask_bwd", _ok, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p)
probe_prelu_apply = N._sig("ctn_probe_prelu_apply", _ok, _p, _p, _p, _i, _i, _i, _i, _p)
probe_prelu_bwd = N._sig("ctn_probe_prelu_bwd", _ok, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p)
probe_combine = N._sig("ctn_probe_dw_combine", _ok, _p, _p, _p, _i, _i, _i, _i, _i, _p)
probe_encdec = N._sig("ctn_probe_encdec_wgrad", _ok, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _i, _p)
probe_rowsum = N._sig("ctn_probe_rowsum", _ok, _p, _sz, _i, _i, _i, _i, _p, _p)
probe_rows = N._sig("ctn_probe_rows", _ok, _p, _sz, _p, _sz, _i, _i, _i, _i, _i, _p)
probe_transpose = N._sig("ctn_probe_transpose", _ok, _p, _p, _i, _i, _p)

A1, A2 = R.A1, R.A2


def _st():
    return N.stream_ptr(torch.device(DEV))


_KEEP = []  # device temporaries whose pointers are in flight: alive until the call has finished


def _call(fn, *args):
    st = fn(*args, _st())
    torch.cuda.synchronize()
    _KEEP.clear()
    assert st == N.CTN_OK, f"{fn.__name__}: status {st}"


def fptr(x, dtype=torch.float32):
    t = x.to(DEV, dtype).contiguous()
    _KEEP.append(t)
    return t.data_ptr()


def dptr(x):
    return fptr(x, torch.float64)


def sptr(v):
    return fptr(torch.tensor([v]))


class Pads:
    """pitched float32 buffers whose pad columns are finite garbage (1e6 randn, fixed per call site) or zero"""

    def __init__(self, seed, garbage):
        self.g = torch.Generator().manual_seed(seed)
        self.garbage = garbage

    def __call__(self, x, pitch):
        lead, F = x.shape[:-1], x.shape[-1]
        y = (torch.randn(*lead, pitch, generator=self.g, dtype=torch.float64) * 1e6).float()
        if not self.garbage:
            y.zero_()
        y[..., :F] = x.float()
        y = y.to(DEV)
        _KEEP.append(y)
        return y


def nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def base(g, *shape, dtype=torch.float32):
    return (torch.randn(*shape, generator=g, dtype=torch.float64) + 2.0).to(dtype).to(DEV)


def dev(x):
    return x.to(DEV)


def ratio(got, ref, bnd, b0=None, adds=1):
    """max |got - b0 - ref| / (bnd + adds u |b0|); b0: accumulator base, adds: float atomics onto one address (each rounds
    relative to the running total, which carries the base).  An element with a zero bound must match exactly."""
    got, ref, bnd = got.double(), dev(ref).double(), dev(bnd).double()
    if b0 is not None:
        got = got - b0.double()
        bnd = bnd + adds * U * b0.double().abs()
    err = (got - ref).abs()
    r = torch.where(bnd > 0, err / bnd.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, float("inf")), err))
    return float(r.max()) if r.numel() else 0.0


class Check:
    def __init__(self, fam, name, r):
        self.tag, self.r, self.res, self.fail = f"{fam}/{name}", r, {}, []

    def within(self, key, got, refb, b0=None, adds=1):
        q = ratio(got, refb[0], refb[1], b0, adds)
        self.res[key] = max(self.res.get(key, 0.0), q)
        if not q <= 1.0:
            self.fail.append(f"{self.tag}: {key} error / bound = {q:.3g}")

    def pads_zero(self, key, y, F):
        if not bool((y[..., F:] == 0).all()):
            self.fail.append(f"{self.tag}: {key} columns [frames, pitch) are not exactly 0")

    def same(self, key, a, b):
        if not torch.equal(a, b):
            self.fail.append(f"{self.tag}: {key} with garbage pads differs from the call with zero pads")

    def done(self):
        print(f"{self.tag} [{self.r['reaches']}] e/bound: " + " ".join(f"{k} {v:.3f}" for k, v in self.res.items()))
        assert not self.fail, "\n".join(self.fail)


def _twice(run, r, elem, seed):
    """run with garbage pads and with zero pads; element-wise outputs must match bit for bit"""
    a, b = run(r, Pads(seed, True)), run(r, Pads(seed, False))
    return a, b, elem


def _elem_checks(ck, a, b, elem, F):
    for k in elem:
        ck.pads_zero(k, a[k], F)
        ck.same(k, a[k], b[k])


# ---- bias + PReLU statistics ------------------------------------------------------------------------------------------------
def _run_bias(r, pads):
    g = R.gen("bias" + str(sorted(r.items())))
    B, Cc, F = r["B"], r["C"], r["F"]
    pitch = R.pitch_of(F, r["extra"])
    y, bias = R.activation(g, r), R.rnd(g, Cc, scale=0.3)
    yb, st0 = pads(y, pitch), base(g, B, 2, dtype=torch.float64)
    st = st0.clone()
    _call(probe_bias, yb.data_ptr(), fptr(bias), sptr(A1), st.data_ptr(), B, Cc, F, pitch)
    return dict(y=yb, stats=st, st0=st0, inp=(y, bias))


@pytest.mark.parametrize("name", list(R.ROWS["bias_prelu_stats"]))
def test_bias_prelu_stats(name):
    r = R.ROWS["bias_prelu_stats"][name]
    ck, F = Check("bias_prelu_stats", name, r), r["F"]
    a, b, elem = _twice(_run_bias, r, ["y"], 1)
    _elem_checks(ck, a, b, elem, F)
    y, bias = (dev(t) for t in a["inp"])
    ck.within("y", a["y"][..., :F], R.bias_prelu_stats(y, bias, A1)["y"])
    ck.within("stats", a["stats"], R.stats_from_output(a["y"][..., :F].double(), A1, F), a["st0"])
    ck.done()


# ---- act-norm -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["act_norm"]))
def test_act_norm(name):
    r = R.ROWS["act_norm"][name]
    ck, B, Cc, F = Check("act_norm", name, r), r["B"], r["C"], r["F"]
    sl = None if r.get("act") is False else A1

    def run(r, pads):
        g = R.gen("actnorm" + name)
        pitch = R.pitch_of(F, r["extra"])
        pre = R.activation(g, r)
        gm, bt = R.norm_params(g, Cc)
        stats = R.stats_of(R.act(pre, sl))
        y = nan(B, Cc, pitch)
        _call(probe_act_norm, pads(pre, pitch).data_ptr(), y.data_ptr(), None if sl is None else sptr(sl),
              fptr(gm), fptr(bt), dptr(stats), float(Cc * F), R.EPS, B, Cc, F, pitch)
        return dict(y=y, inp=(pre, gm, bt, stats))

    a, b, elem = _twice(run, r, ["y"], 2)
    _elem_checks(ck, a, b, elem, F)
    pre, gm, bt, stats = (dev(t) for t in a["inp"])
    ck.within("y", a["y"][..., :F], R.act_norm(pre, sl, gm, bt, stats, Cc * F, R.EPS)["y"])
    ck.done()


# ---- gLN / PReLU backward ---------------------------------------------------------------------------------------------------
GLN_ROWS = dict(R.ROWS["gln_bwd"])
GLN_ROWS["reduced"] = R._r("reduced = true: apply phase only, from given sums", reduced=True)
GLN_ROWS["reduced_C1025"] = R._r("reduced = true at C = 1025, aliasing", reduced=True, alias=True, C=1025, F=33)


@pytest.mark.parametrize("name", list(GLN_ROWS))
def test_gln_prelu_bwd(name):
    r = GLN_ROWS[name]
    ck, B, Cc, F = Check("gln_bwd", name, r), r["B"], r["C"], r["F"]
    n = Cc * F
    reduced, nulls = bool(r.get("reduced")), bool(r.get("nulls")) or r.get("act") is False

    def run(r, pads):
        g, sl, pre, dy, gm, stats = R.gln_inputs(name, r)
        pitch = R.pitch_of(F, r["extra"])
        dyb = pads(dy, pitch)
        dpre = dyb if r.get("alias") else nan(B, Cc, pitch)
        o = dict(dg0=base(g, Cc), db0=base(g, Cc), ds0=base(g, 1), dbias0=base(g, Cc))
        o.update(dg=o["dg0"].clone(), db=o["db0"].clone(), ds=o["ds0"].clone(), dbias=o["dbias0"].clone())
        if reduced:
            sums = dev(R.gln_reduce(dev(dy), dev(pre), sl, dev(gm), dev(stats), n, R.EPS)["sums"][0]).clone()
        else:
            sums = torch.full((B, 2), float("nan"), dtype=torch.float64, device=DEV)  # cleared by the launcher
        o["sums_in"] = sums.clone()
        _call(probe_gln, dyb.data_ptr(), pads(pre, pitch).data_ptr(), dpre.data_ptr(), None if sl is None else sptr(sl),
              fptr(gm), dptr(stats), float(n), R.EPS, sums.data_ptr(), o["dg"].data_ptr(),
              o["db"].data_ptr(), None if nulls else o["ds"].data_ptr(), None if nulls else o["dbias"].data_ptr(), B, Cc, F, pitch,
              int(reduced))
        o.update(dpre=dpre, sums=sums, inp=(sl, pre, dy, gm, stats))
        return o

    a, b, elem = _twice(run, r, ["dpre"], 3)
    _elem_checks(ck, a, b, elem, F)
    sl, pre, dy, gm, stats = a["inp"]
    pre, dy, gm, stats = dev(pre), dev(dy), dev(gm), dev(stats)
    if reduced:
        assert torch.equal(a["dg"], a["dg0"]) and torch.equal(a["db"], a["db0"]), f"{name}: reduced call touched dgamma / dbeta"
        assert torch.equal(a["sums"], a["sums_in"]), f"{name}: reduced call touched sums"
    else:
        red = R.gln_reduce(dy, pre, sl, gm, stats, n, R.EPS)
        ck.within("sums", a["sums"], red["sums"])
        ck.within("dgamma", a["dg"], red["dgamma"], a["dg0"], B)
        ck.within("dbeta", a["db"], red["dbeta"], a["db0"], B)
    ap = R.gln_apply(dy, pre, sl, gm, stats, n, R.EPS, a["sums"])
    ck.within("dpre", a["dpre"][..., :F], ap["dpre"])
    if nulls:
        assert torch.equal(a["ds"], a["ds0"]) and torch.equal(a["dbias"], a["dbias0"]), f"{name}: a null output was written"
    else:
        ck.within("dslope", a["ds"], (ap["dslope"][0].reshape(1), ap["dslope"][1].reshape(1)), a["ds0"], Cc * B)
        ck.within("dbias", a["dbias"], ap["dbias"], a["dbias0"], B)
    ck.done()


# ---- depthwise: training forward and backward -------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["dw"]))
def test_dw_train_fwd(name):
    r = R.ROWS["dw"][name]
    ck, B, Cc, F, P, d = Check("dw_train_fwd", name, r), r["B"], r["C"], r["F"], r["P"], r["d"]
    pl, n = R.pad_left_of(P, d), Cc * F

    def run(r, pads):
        g, h, g1, b1, wd, bd, dU, stats1 = R.dw_inputs(name, r)
        pitch = R.pitch_of(F, r["extra"])
        up, s20 = nan(B, Cc, pitch), base(g, B, 2, dtype=torch.float64)
        s2 = s20.clone()
        _call(probe_dw_fwd, pads(h, pitch).data_ptr(), up.data_ptr(), fptr(g1), fptr(b1),
              fptr(wd), fptr(bd), sptr(A1), sptr(A2),
              dptr(stats1), s2.data_ptr(), B, Cc, F, pitch, P, d, pl, float(n), R.EPS)
        return dict(upre=up, s2=s2, s20=s20, inp=(h, g1, b1, wd, bd, stats1))

    a, b, elem = _twice(run, r, ["upre"], 4)
    _elem_checks(ck, a, b, elem, F)
    h, g1, b1, wd, bd, stats1 = (dev(t) for t in a["inp"])
    ck.within("upre", a["upre"][..., :F], R.dw_train_fwd(h, g1, b1, wd, bd, A1, stats1, n, R.EPS, P, d, pl)["upre"])
    ck.within("stats2", a["s2"], R.stats_from_output(a["upre"][..., :F].double(), A2, F), a["s20"])
    ck.done()


@pytest.mark.parametrize("name", list(R.ROWS["dw"]))
def test_dw_bwd(name):
    r = R.ROWS["dw"][name]
    ck, B, Cc, F, P, d = Check("dw_bwd", name, r), r["B"], r["C"], r["F"], r["P"], r["d"]
    pl, n = R.pad_left_of(P, d), Cc * F

    def run(r, pads):
        g, h, g1, b1, wd, bd, dU, stats1 = R.dw_inputs(name, r)
        pitch = R.pitch_of(F, r["extra"])
        o = dict(dwd0=base(g, Cc, P), sums0=base(g, B, 2, dtype=torch.float64), dg0=base(g, Cc), db0=base(g, Cc))
        o.update({k[:-1]: v.clone() for k, v in list(o.items())})
        dhn = nan(B, Cc, pitch)
        _call(probe_dw_bwd, pads(dU, pitch).data_ptr(), pads(h, pitch).data_ptr(), dhn.data_ptr(), sptr(A1),
              fptr(g1), fptr(b1), dptr(stats1), float(n), R.EPS,
              fptr(wd), o["dwd"].data_ptr(), o["sums"].data_ptr(), o["dg"].data_ptr(),
              o["db"].data_ptr(), B, Cc, F, pitch, P, d, pl)
        o.update(dhn=dhn, inp=(h, g1, b1, wd, dU, stats1))
        return o

    a, b, elem = _twice(run, r, ["dhn"], 5)
    _elem_checks(ck, a, b, elem, F)
    h, g1, b1, wd, dU, stats1 = (dev(t) for t in a["inp"])
    ref = R.dw_bwd(dU, h, A1, g1, b1, stats1, n, R.EPS, wd, P, d, pl)
    ck.within("dhn", a["dhn"][..., :F], ref["dhn"])
    ck.within("dwd", a["dwd"], ref["dwd"], a["dwd0"], B)
    ck.within("sums", a["sums"], ref["sums"], a["sums0"])
    ck.within("dgamma", a["dg"], ref["dgamma"], a["dg0"], B)
    ck.within("dbeta", a["db"], ref["dbeta"], a["db0"], B)
    ck.done()


# ---- mask backward --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["mask_bwd"]))
def test_mask_bwd(name):
    r = R.ROWS["mask_bwd"][name]
    ck, B, S, Nn, F = Check("mask_bwd", name, r), r["B"], r["S"], r["N"], r["F"]

    def run(r, pads):
        g = R.gen("mask" + name)
        pitch = R.pitch_of(F, r["extra"])
        dwhat = R.f32(R.rnd(g, B, S, Nn, F) * R.sample_scale(B)[:, :, :, None])
        w = R.rnd(g, B, Nn, F).abs()
        m = R.f32(torch.sigmoid(R.rnd(g, B, S, Nn, F, scale=3.0)))
        if r.get("edges"):
            sel = torch.randint(0, 4, m.shape, generator=g)
            m = torch.where(sel == 0, torch.zeros_like(m), m)
            m = torch.where(sel == 1, torch.ones_like(m), m)
            m = torch.where(sel == 2, torch.full_like(m, 1.0 - 2.0 ** -24), m)
        dw = pads(dwhat, pitch)
        dp = nan(B, Nn, pitch)
        _call(probe_mask, dw.data_ptr(), pads(w, pitch).data_ptr(), pads(m, pitch).data_ptr(), dp.data_ptr(), B, S, Nn, F, pitch)
        return dict(dmpre=dw, dwprod=dp, inp=(dwhat, w, m))

    a, b, elem = _twice(run, r, ["dmpre", "dwprod"], 6)
    _elem_checks(ck, a, b, elem, F)
    ref = R.mask_bwd(*(dev(t) for t in a["inp"]))
    ck.within("dmpre", a["dmpre"][..., :F], ref["dmpre"])
    ck.within("dwprod", a["dwprod"][..., :F], ref["dwprod"])
    ck.done()


# ---- PReLU apply / backward -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["prelu"]))
def test_prelu_apply_bwd(name):
    r = R.ROWS["prelu"][name]
    ck, B, Cc, F = Check("prelu", name, r), r["B"], r["C"], r["F"]

    def run(r, pads):
        g = R.gen("prelu" + name)
        pitch = R.pitch_of(F, r["extra"])
        x = R.activation(g, r)
        dy = R.rnd(g, B, Cc, F)
        xb = pads(x, pitch)
        y, dpre, ds0 = nan(B, Cc, pitch), nan(B, Cc, pitch), base(g, 1)
        ds = ds0.clone()
        _call(probe_prelu_apply, xb.data_ptr(), y.data_ptr(), sptr(A1), B, Cc, F, pitch)
        _call(probe_prelu_bwd, pads(dy, pitch).data_ptr(), xb.data_ptr(), dpre.data_ptr(), sptr(A1), ds.data_ptr(), B, Cc,
              F, pitch)
        return dict(y=y, dpre=dpre, ds=ds, ds0=ds0, inp=(x, dy))

    a, b, elem = _twice(run, r, ["y", "dpre"], 7)
    _elem_checks(ck, a, b, elem, F)
    x, dy = (dev(t) for t in a["inp"])
    ck.within("y", a["y"][..., :F], R.prelu_apply(x, A1)["y"])
    ref = R.prelu_bwd(dy, x, A1)
    ck.within("dpre", a["dpre"][..., :F], ref["dpre"])
    ck.within("dslope", a["ds"], (ref["dslope"][0].reshape(1), ref["dslope"][1].reshape(1)), a["ds0"], Cc * B)
    ck.done()


# ---- dw-combine -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["dw_combine"]))
def test_dw_combine(name):
    r = R.ROWS["dw_combine"][name]
    ck, B, Cc, F = Check("dw_combine", name, r), r["B"], r["C"], r["F"]
    relu = bool(r.get("relu"))

    def run(r, pads):
        g = R.gen("comb" + name)
        pitch = R.pitch_of(F, r["extra"])
        dw, dwp = R.rnd(g, B, Cc, F), R.rnd(g, B, Cc, F, scale=3.0)
        w = R.activation(g, r)
        dwb = pads(dw, pitch)
        _call(probe_combine, dwb.data_ptr(), pads(dwp, pitch).data_ptr(), pads(w, pitch).data_ptr(), int(relu), B, Cc, F, pitch)
        return dict(dw=dwb, inp=(dw, dwp, w))

    a, b, elem = _twice(run, r, ["dw"], 8)
    _elem_checks(ck, a, b, elem, F)
    dw, dwp, w = (dev(t) for t in a["inp"])
    ck.within("dw", a["dw"][..., :F], R.dw_combine(dw, dwp, w, relu)["dw"])
    ck.done()


# ---- rowsum / rows / transpose ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["rowsum"]))
def test_rowsum(name):
    r = R.ROWS["rowsum"][name]
    ck, B, Cc, F = Check("rowsum", name, r), r["B"], r["C"], r["F"]
    g = R.gen("rowsum" + name)
    pitch = R.pitch_of(F, r["extra"])
    dy = R.f32(R.rnd(g, B, Cc, F, shift_=0.3) * R.sample_scale(B))
    bs = Cc * pitch + (3 * pitch + 64 if r.get("stride") else 0)
    buf = (torch.randn(B * bs, generator=g, dtype=torch.float64) * 1e6).float().to(DEV)  # finite garbage around the rows
    for bb in range(B):
        buf[bb * bs:bb * bs + Cc * pitch].view(Cc, pitch)[:, :F] = dev(dy[bb]).float()
    out0 = base(g, Cc)
    out = out0.clone()
    _call(probe_rowsum, buf.data_ptr(), bs, Cc, B, F, pitch, out.data_ptr())
    ck.within("out", out, R.rowsum(dev(dy))["out"], out0, B)
    ck.done()


@pytest.mark.parametrize("name", list(R.ROWS["rows"]))
def test_rows(name):
    r = R.ROWS["rows"][name]
    ck, B, Cc, F = Check("rows", name, r), r["B"], r["C"], r["F"]
    g = R.gen("rows" + name)
    pitch = R.pitch_of(F, r["extra"])
    wide = r.get("strides")
    dbs, sbs = Cc * pitch + (pitch * 2 + 128 if wide else 0), Cc * pitch + (pitch + 256 if wide else 0)
    src = (torch.randn(B * sbs, generator=g) * 1e6).to(DEV)  # finite garbage everywhere, data in the first C rows of each sample
    dst = (torch.randn(B * dbs, generator=g)).to(DEV)
    dst0 = dst.clone()
    acc = int(bool(r.get("acc")))
    _call(probe_rows, dst.data_ptr(), dbs, src.data_ptr(), sbs, Cc, B, acc, F, pitch)
    for bb in range(B):
        s = src[bb * sbs:bb * sbs + Cc * pitch].view(Cc, pitch)
        d, d0 = dst[bb * dbs:(bb + 1) * dbs], dst0[bb * dbs:(bb + 1) * dbs]
        want = s[:, :F] + d0[:Cc * pitch].view(Cc, pitch)[:, :F] if acc else s[:, :F]
        dv = d[:Cc * pitch].view(Cc, pitch)
        assert torch.equal(dv[:, :F], want), f"{name}: sample {bb} rows differ"
        assert bool((dv[:, F:] == 0).all()), f"{name}: columns past frames are not 0"
        assert torch.equal(d[Cc * pitch:], d0[Cc * pitch:]), f"{name}: written past C rows of sample {bb}"
    ck.res["bit-exact"] = 0.0
    ck.done()


@pytest.mark.parametrize("name", list(R.ROWS["transpose"]))
def test_transpose(name):
    r = R.ROWS["transpose"][name]
    ck, M, K = Check("transpose", name, r), r["M"], r["K"]
    g = R.gen("tr" + name)
    W = torch.randn(M, K, generator=g).to(DEV)
    Wt = nan(K * M + 64)
    _call(probe_transpose, W.data_ptr(), Wt.data_ptr(), M, K)
    assert torch.equal(Wt[:K * M].view(K, M), W.t()), name
    assert bool(torch.isnan(Wt[K * M:]).all()), f"{name}: written past K M"
    ck.res["bit-exact"] = 0.0
    ck.done()


# ---- filter-bank weight gradient --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ROWS["encdec"]))
def test_encdec_wgrad(name):
    r = R.ROWS["encdec"][name]
    ck, Rr, Nn, L, S, T = Check("encdec", name, r), r["R"], r["N"], r["L"], r["stride"], r["T"]
    F, pl = R.encdec_geometry(r)
    g = R.gen("encdec" + name)
    pitch = R.pitch_of(F)
    act_ = R.rnd(g, Rr, Nn, F)
    sig = R.f32(R.rnd(g, Rr, T) * R.sample_scale(Rr)[:, :, 0])
    off = r.get("off", 0)
    sbuf = (torch.randn(Rr * T + 8, generator=g) * 1e6).float().to(DEV)
    sbuf[off:off + Rr * T] = dev(sig).float().reshape(-1)
    dW0 = base(g, Nn, L)
    dW = dW0.clone()
    _call(probe_encdec, Pads(10, True)(act_, pitch).data_ptr(), sbuf[off:].data_ptr(), dW.data_ptr(), Rr, Nn, F, pitch, T, L, S, pl)
    ck.within("dW", dW, R.encdec_wgrad(dev(act_), dev(sig), L, S, pl)["dW"], dW0, R.encdec_gy(Rr, Nn) if L <= 32 else 1)
    ck.done()


# ---- composed: gLN2/PReLU2 backward -> k_dw_bwd -> gLN1/PReLU1 backward (reduced), as ctn_convtasnet_bwd chains them ---------
COMPOSED_TOL = 2.0 ** -14


def _gln(x, gamma, beta, eps):
    mean = x.mean((1, 2), keepdim=True)
    var = ((x - mean) ** 2).mean((1, 2), keepdim=True)
    return gamma[None, :, None] * (x - mean) / torch.sqrt(var + eps) + beta[None, :, None]


@pytest.mark.parametrize("name", list(R.COMPOSED))
def test_composed_block_backward_vs_autograd(name):
    """u = dwconv(gLN1(PReLU1(h))) + bd, y = gLN2(PReLU2(u)): every gradient of sum(y dy) within 2^-14 of its largest entry
    (per sample for d_h).  A wiring defect between the fused phase-1 sums of k_dw_bwd and the apply phase moves a gradient by
    1/frames or more, >= 2.4e-4 at the longest row here."""
    r = R.COMPOSED[name]
    B, Cc, F, P, d = r["B"], r["C"], r["F"], r["P"], r["d"]
    pl, n, pitch = R.pad_left_of(P, d), Cc * F, R.pitch_of(F, r["extra"])
    g, h, g1, b1, wd, bd, _, _ = R.dw_inputs(name, r)
    g2, b2 = R.norm_params(g, Cc)
    dy = R.rnd(g, B, Cc, F)
    eps = float(torch.tensor(R.EPS, dtype=torch.float32))
    leaves = {k: dev(v).clone().requires_grad_(True) for k, v in dict(h=h, g1=g1, b1=b1, wd=wd, bd=bd, g2=g2, b2=b2,
                                                                        a1=torch.tensor(A1, dtype=torch.float64),
                                                                        a2=torch.tensor(A2, dtype=torch.float64)).items()}
    L_ = leaves
    hn = _gln(torch.where(L_["h"] >= 0, L_["h"], L_["a1"] * L_["h"]), L_["g1"], L_["b1"], eps)
    u = L_["bd"][None, :, None] + sum(L_["wd"][None, :, k, None] * R.shift(hn, k * d - pl) for k in range(P))
    y = _gln(torch.where(u >= 0, u, L_["a2"] * u), L_["g2"], L_["b2"], eps)
    (y * dev(dy)).sum().backward()
    upre = R.f32(u.detach())
    stats1, stats2 = R.stats_of(R.prelu(dev(h), A1)), R.stats_of(R.prelu(upre, A2))
    pads = Pads(11, True)
    G = pads(dy, pitch)
    z = lambda *s: torch.zeros(*s, device=DEV)
    out = dict(dg2=z(Cc), db2=z(Cc), da2=z(1), dbd=z(Cc), dwd=z(Cc, P), dg1=z(Cc), db1=z(Cc), da1=z(1), dbias=z(Cc))
    sums = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
    upb, hb = pads(upre, pitch), pads(h, pitch)
    f = fptr
    _call(probe_gln, G.data_ptr(), upb.data_ptr(), G.data_ptr(), sptr(A2), f(g2), stats2.data_ptr(), float(n), R.EPS,
          sums.data_ptr(), out["dg2"].data_ptr(), out["db2"].data_ptr(), out["da2"].data_ptr(), out["dbd"].data_ptr(), B, Cc, F,
          pitch, 0)
    sums.zero_()
    G2 = nan(B, Cc, pitch)
    _call(probe_dw_bwd, G.data_ptr(), hb.data_ptr(), G2.data_ptr(), sptr(A1), f(g1), f(b1), dptr(stats1),
          float(n), R.EPS, f(wd), out["dwd"].data_ptr(), sums.data_ptr(), out["dg1"].data_ptr(), out["db1"].data_ptr(), B, Cc, F,
          pitch, P, d, pl)
    _call(probe_gln, G2.data_ptr(), hb.data_ptr(), G2.data_ptr(), sptr(A1), f(g1), dptr(stats1), float(n),
          R.EPS, sums.data_ptr(), out["dg1"].data_ptr(), out["db1"].data_ptr(), out["da1"].data_ptr(), out["dbias"].data_ptr(), B, Cc,
          F, pitch, 1)
    hg = L_["h"].grad
    want = dict(dg2=L_["g2"].grad, db2=L_["b2"].grad, da2=L_["a2"].grad.reshape(1), dbd=L_["bd"].grad, dwd=L_["wd"].grad,
                dg1=L_["g1"].grad, db1=L_["b1"].grad, da1=L_["a1"].grad.reshape(1), dbias=hg.sum((0, 2)))
    res, fails = {}, []
    for k, w in want.items():
        q = float((out[k].double() - w).abs().max() / w.abs().max().clamp_min(1e-300)) / COMPOSED_TOL
        res[k] = q
        if not q <= 1.0:
            fails.append(f"{name}: {k} {q:.3g} of the tolerance")
    dh = G2[..., :F].double()
    q = float(((dh - hg).abs().amax((1, 2)) / hg.abs().amax((1, 2)).clamp_min(1e-300)).max()) / COMPOSED_TOL
    res["dh"] = q
    if not q <= 1.0:
        fails.append(f"{name}: d_h {q:.3g} of the tolerance")
    if not bool((G2[..., F:] == 0).all()):
        fails.append(f"{name}: d_h columns past frames are not 0")
    print(f"composed/{name} [{r['reaches']}] e/tol: " + " ".join(f"{k} {v:.3f}" for k, v in res.items()))
    assert not fails, "\n".join(fails)


# ---- the launchers' move left the training pipeline's launches alone ----------------------------------------------------------
@pytest.mark.parametrize("mode,fwd,bwd", [("fp32", 41, 108), ("f16x3", 24, 117)])
def test_training_launch_counts(mode, fwd, bwd):
    """per-step launches of ctn_convtasnet_fwd_train / ctn_convtasnet_bwd at a 2 x 3-block config (the counts from before the
    streaming kernels got their own launchers)"""
    import convtasnet_oracle as O
    from test_parity_gpu import build_model
    cfg = O.OracleConfig(causal=False, n_basis=24, kernel_size=8, sep_hidden_channels=40, sep_bottleneck_channels=20,
                         sep_skip_channels=12, sep_num_blocks=2, sep_num_layers=3, n_sources=2)
    m = build_model(cfg, O.synth_state_dict(cfg, seed=3), math=mode).train()
    mix, _ = O.synth_batch(3, 2, 1003, seed=4)
    m(mix.cuda()).square().sum().backward()
    torch.cuda.synchronize()
    assert (m.last_launches, m.last_bwd_launches) == (fwd, bwd)
