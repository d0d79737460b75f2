"""DPRNN-TasNet's kernels at their edges against fp64 (tests/dprnn_unit_edges_ref.py), every bound taken per unit: per (sequence,
direction) for the shared bi-LSTM, per sample for the gLN + residual, bit for bit for segmentation and overlap-add, per (sample,
source) for the model.

Every entry call runs twice, on NaN-filled outputs and an exactly sized NaN workspace followed by a guard region that must stay
untouched, and the two calls must give the same bits.  The gLN + residual entries are the exception: their statistics add one
double partial per CTA with atomics, so the order of those adds changes between calls.  Under a DC offset of 1e4 the variance is
the small difference of two sums near 1e8 n, and the last bits of the double sums then reach the float rstd (measured on an H100:
the two calls of the 1e4 row differ).  Both calls are held to the bound instead, and the row reports whether the bits matched.
The bi-LSTM, segmentation and overlap-add use no atomics and must repeat bit for bit.  Every
refusal returns its code before any launch and leaves the outputs untouched.  Each row prints its worst unit error over its bound
and the branch it exists for."""
import math

import pytest
import torch

import dprnn_oracle as DO
import dprnn_unit_edges_ref as E
from ctn_b200 import _native as N
from ctn_b200.models.dprnn_tasnet import DPRNNTasNet
from test_dprnn_gpu import MODES

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
GUARD = 4096
_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def st():
    return N.stream_ptr(DEV)


def dev(t):
    return t.contiguous().to(DEV)


def nan(shape, dtype=torch.float32):
    """NaN-filled, or all ones bits for an integer word"""
    return torch.full(shape, float("nan") if dtype.is_floating_point else -1, dtype=dtype, device=DEV)


class Workspace:
    """nbytes exactly, 256-byte aligned, NaN-filled (0xff bytes), followed by GUARD bytes that must stay 0xff"""

    def __init__(self, nbytes):
        self.buf = torch.full((int(nbytes) + 256 + GUARD,), 0xFF, dtype=torch.uint8, device=DEV)
        self.off = (-self.buf.data_ptr()) % 256
        self.base, self.nbytes = self.buf.data_ptr() + self.off, int(nbytes)

    def guard_intact(self):
        g = self.buf[self.off + self.nbytes:self.off + self.nbytes + GUARD]
        return bool((g == 0xFF).all())


def twice(run, shapes, nbytes, exact=True):
    """run(outs, base, nbytes) -> status, twice on fresh NaN outputs ((shape, dtype) each) and a fresh exactly sized NaN workspace
    with an untouched guard after it; the two calls must agree bit for bit (exact).  Returns the first call's outputs on the host
    and its launch count; with exact=False the second call's outputs too, for the caller to hold to the same bound."""
    results, counts = [], []
    for _ in range(2):
        outs = [nan(*s) if s is not None else None for s in shapes]
        ws = Workspace(nbytes)
        N.check(run(outs, ws.base, ws.nbytes), "entry")
        counts.append(N.ctn_last_launch_count())
        torch.cuda.synchronize()
        assert ws.guard_intact(), "the call wrote past its workspace"
        results.append([o.cpu() if o is not None else None for o in outs])
    assert counts[0] == counts[1]
    if not exact:
        return results, counts[0]
    for a, b in zip(*results):
        if a is not None:
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b), \
                "a repeated call gave other bits"
    return results[0], counts[0]


def refused(call, code, outs):
    """call() returns `code` with no launch and leaves every output's bits as they were"""
    torch.cuda.synchronize()
    before = [o.clone() for o in outs]
    assert call() == code
    assert N.ctn_last_launch_count() == 0
    torch.cuda.synchronize()
    for o, b in zip(outs, before):
        assert torch.equal(o.view(torch.uint8), b.view(torch.uint8)), "a refused call wrote its output"


def report(what, name, ratio, reaches=""):
    print("[dprnn edges] {:6s} {:24s} worst unit error / bound {:.3g} -- {}".format(what, name, ratio, reaches))


# ---- A. the bi-LSTM: ctn_bilstm_proj_fwd and ctn_bilstm_relu_proj_fwd --------------------------------------------------------------
LSTM_ROWS = E.lstm_rows()


def lstm_weights_on_device(sd):
    w = [dev(sd["rnn." + n]) for n in E.NAMES]
    return w, (N._fp * 8)(*[t.data_ptr() for t in w]), dev(sd["fc.weight"])


def run_lstm(r, sd, z):
    """(hout or None, P or None, launches) of a row, run twice"""
    NSEQ, T, F, H, Fo = r["NSEQ"], r["T"], r["F"], r["H"], r["Fo"]
    want_h, want_p = r["outs"] in ("both", "h"), r["outs"] in ("both", "P")
    zd = dev(z)
    w, ptrs, fc = lstm_weights_on_device(sd)
    nbytes = N.ctn_bilstm_workspace_bytes(F, H, Fo if want_p else 0)
    assert nbytes > 0
    shapes = [((2, NSEQ, T, Fo),) if want_p else None, ((NSEQ, T, 2 * H),) if want_h else None]

    def run(o, base, nb):
        P, h = N.ptr(o[0]), N.ptr(o[1])
        fcp = fc.data_ptr() if want_p else None
        if r["entry"] == "relu":
            return N.ctn_bilstm_relu_proj_fwd(zd.data_ptr(), NSEQ, T, F, H, ptrs, fcp, Fo, P, h, base, nb, st())
        return N.ctn_bilstm_proj_fwd(zd.data_ptr(), NSEQ, T, F, H, ptrs, fcp, Fo, P, h, None, base, nb, st())
    (P, h), n = twice(run, shapes, nbytes)
    return h, P, n


def lstm_reference(name, r, sd, z, idx):
    return _cached(("lstm", name), lambda: E.lstm_answer(z[idx], sd, r["entry"] == "relu"))


@pytest.mark.parametrize("name", list(LSTM_ROWS))
def test_bilstm_entry(name):
    """h per (sequence, direction) within H_FLOOR and P per (direction, sequence) within 1e-4 max|fp64| + 1e-6, except the row's
    fp32 groups (the x1e3 sequences of the loudness row), held to H_C x the fp32 CPU recurrence's worst error on them; hout is the
    raw h also next to a ReLU projection; 2 launches"""
    r = LSTM_ROWS[name]
    assert N.ctn_bilstm_supported(r["F"], r["H"], r["Fo"])
    sd, z = E.lstm_case(r)
    h, P, n = run_lstm(r, sd, z)
    assert n == 2
    idx = torch.tensor(r["idx"] if r["idx"] else list(range(r["NSEQ"])))
    h64, P64 = lstm_reference(name, r, sd, z, idx)
    hs = h[idx] if h is not None else None
    Ps = P[:, idx] if P is not None else None
    m = E.fp32_mask(r, idx)
    extra = ""
    if m is None:
        ratio = E.lstm_excess(hs, Ps, h64 if h is not None else None, P64)
    else:
        h32, P32 = E.lstm_answer(z[idx], sd, r["entry"] == "relu", dtype=torch.float32)
        ratio = E.lstm_excess(hs, Ps, h64, P64, (m, h32, P32))
        quiet = E.lstm_excess(hs[~m], Ps[:, ~m], h64[~m], P64[:, ~m])
        assert quiet <= 1.0, "{}: the quiet sequences miss the floors by {:.3g}".format(name, quiet)
        extra = "; quiet sequences {:.3g} of the floors; x1e3 under H_C x the fp32 CPU error {:.2e}".format(
            quiet, float(E.h_unit_errors(h32, h64).view(-1, 2)[m].max()))
    assert ratio <= 1.0, "{}: worst unit error / bound {:.3g}{}".format(name, ratio, extra)
    report("lstm", name, ratio, r["reaches"] + extra)


def test_bilstm_refusals_before_launch():
    F, H, Fo, NSEQ, T = 64, 128, 64, 65, 3
    sd = E.lstm_weights(F, H, Fo, 1)
    w, ptrs, fc = lstm_weights_on_device(sd)
    # sized for the largest Fo and H the refused calls name, so a refusal that regressed fails the assert and writes nothing past them
    zbuf = torch.zeros(NSEQ * T * 128 + 64, device=DEV)
    Pbuf, hbuf = nan((2 * NSEQ * T * 160 + 64,)), nan((NSEQ * T * 2 * 128 + 64,))
    nbytes = N.ctn_bilstm_workspace_bytes(F, H, Fo)
    ws = Workspace(nbytes)
    z, P, h = zbuf.data_ptr(), Pbuf.data_ptr(), hbuf.data_ptr()
    outs = [Pbuf, hbuf, ws.buf]

    def proj(z=z, NSEQ=NSEQ, T=T, F=F, H=H, fc=fc.data_ptr(), Fo=Fo, P=P, h=h, base=ws.base, nb=nbytes):
        return lambda: N.ctn_bilstm_proj_fwd(z, NSEQ, T, F, H, ptrs, fc, Fo, P, h, None, base, nb, st())

    def relu(fc=fc.data_ptr(), P=P, h=h):
        return lambda: N.ctn_bilstm_relu_proj_fwd(z, NSEQ, T, F, H, ptrs, fc, Fo, P, h, ws.base, nbytes, st())
    cases = [
        (proj(F=48), N.CTN_EUNSUPPORTED, "F=48"), (proj(H=96), N.CTN_EUNSUPPORTED, "H=96"), (proj(Fo=160), N.CTN_EUNSUPPORTED, "Fo=160"),
        (proj(Fo=48), N.CTN_EUNSUPPORTED, "Fo % 32 != 0"), (proj(Fo=0), N.CTN_EUNSUPPORTED, "Fo=0 with w_fc"),
        (proj(z=z + 4), N.CTN_EALIGN, "z 4 bytes off"), (proj(P=P + 4), N.CTN_EALIGN, "P 4 bytes off"),
        (proj(h=h + 4), N.CTN_EALIGN, "hout 4 bytes off"), (proj(base=ws.base + 4, nb=nbytes), N.CTN_EALIGN, "workspace 4 bytes off"),
        (proj(nb=nbytes - 1), N.CTN_EWORKSPACE, "workspace 1 byte short"),
        (relu(fc=None, P=None), N.CTN_EINVAL, "ReLU without w_fc"), (proj(P=None), N.CTN_EINVAL, "w_fc without P"),
        (proj(fc=None, P=None, h=None), N.CTN_EINVAL, "no output"), (proj(NSEQ=0), N.CTN_EINVAL, "NSEQ=0"),
        (proj(NSEQ=-1), N.CTN_EINVAL, "NSEQ<0"), (proj(T=0), N.CTN_EINVAL, "T=0"), (proj(T=-3), N.CTN_EINVAL, "T<0"),
    ]
    for call, code, what in cases:
        try:
            refused(call, code, outs)
        except AssertionError as e:
            raise AssertionError("{}: {}".format(what, e))
    assert ws.guard_intact()


# ---- B. gLN + residual: ctn_dprnn_norm_res2_fwd and the fallback ctn_dprnn_norm_res_fwd ---------------------------------------------
NORM_ROWS = E.norm_rows()
NORM_CASES = [pytest.param(name, entry, id="{}-{}".format(entry, name)) for name, r in NORM_ROWS.items() for entry in r["entries"]]


def run_norm(entry, r, P, bias, R, gamma, beta):
    """(out, out_absmax or None) of a row, run twice; the scratch double[2B] is the workspace"""
    B, D1, D2, F, swap, eps = r["B"], r["D1"], r["D2"], r["F"], r["swap"], r["eps"]
    oshape = (B, D2, D1, F) if swap else (B, D1, D2, F)
    Rd, gd, bd = dev(R), dev(gamma), dev(beta)
    if entry == "res2":
        Pd, fb = dev(P), dev(bias)

        def run(o, base, nb):
            return N.ctn_dprnn_norm_res2_fwd(Pd.data_ptr(), fb.data_ptr(), Rd.data_ptr(), gd.data_ptr(), bd.data_ptr(), o[0].data_ptr(), B, D1, D2,
                                             F, eps, swap, base, o[1].data_ptr(), st())
        return twice(run, [(oshape,), ((1,), torch.int32)], 16 * B, exact=False)
    Yd = dev(E.fallback_y(P, bias))
    return twice(lambda o, base, nb: N.ctn_dprnn_norm_res_fwd(Yd.data_ptr(), Rd.data_ptr(), gd.data_ptr(), bd.data_ptr(), o[0].data_ptr(), B,
                                                              D1, D2, F, eps, swap, base, st()), [(oshape,), None], 16 * B, exact=False)


@pytest.mark.parametrize("name,entry", NORM_CASES)
def test_norm_residual_entry(name, entry):
    """every element within NORM_C u scale, per sample; out_absmax bit-equal to max|out|; 2 launches"""
    r = NORM_ROWS[name]
    P, bias, R, gamma, beta = E.norm_case(r)
    runs, n = run_norm(entry, r, P, bias, R, gamma, beta)
    assert n == 2
    parts = [P[0], P[1], bias] if entry == "res2" else [E.fallback_y(P, bias)]
    ref, scale = E.norm_answer(parts, R, gamma, beta, r["eps"], r["swap"])
    for out, amax in runs:
        ratio = E.norm_excess(out, ref, scale)
        per_sample = [E.norm_excess(out[b], ref[b], scale[b]) for b in range(r["B"])]
        assert ratio <= 1.0, "{} {}: worst element error / bound {:.3g}, per sample {}".format(entry, name, ratio, per_sample)
        if amax is not None:
            want = int(out.abs().max().view(torch.int32))
            assert int(amax.item()) == want, "out_absmax {:#x} != bits of max|out| {:#x}".format(int(amax.item()), want)
    same = torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    report(entry, name, ratio, r["reaches"] + "; per sample " + " ".join("{:.2g}".format(x) for x in per_sample)
           + "; repeat bit-identical: {}".format(same))


def test_norm_residual_refusals_before_launch():
    B, D1, D2, F = 2, 3, 4, 8
    # sized for the B = 65536 and F = 1028 calls (the scratch memset, the reads of P and the stores of out), so a refusal that
    # regressed fails the assert without touching memory past these buffers
    Bmax = E.GRID_LIMIT + 1
    t = torch.zeros(2 * Bmax * D1 * D2 * F + 64, device=DEV)
    out = nan((Bmax * D1 * D2 * F + 64,))
    scratch = nan((2 * Bmax,), torch.float64)
    amax = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    p, o, s = t.data_ptr(), out.data_ptr(), scratch.data_ptr()

    def res2(B=B, F=F, swap=0, out=o):
        return lambda: N.ctn_dprnn_norm_res2_fwd(p, p, p, p, p, out, B, D1, D2, F, E.DO.EPS, swap, s, amax.data_ptr(), st())

    def res(B=B, F=F, swap=0, out=o):
        return lambda: N.ctn_dprnn_norm_res_fwd(p, p, p, p, out, B, D1, D2, F, E.DO.EPS, swap, s, st())
    for call, code, what in ((res2(F=6), N.CTN_EINVAL, "F % 4"), (res2(F=1028), N.CTN_EUNSUPPORTED, "F > 1024"),
                             (res2(swap=1, out=p), N.CTN_EINVAL, "swap in place"), (res2(B=65536), N.CTN_EUNSUPPORTED, "B = 65536"),
                             (res2(B=0), N.CTN_EINVAL, "B = 0"), (res(swap=1, out=p), N.CTN_EINVAL, "swap in place"),
                             (res(B=65536), N.CTN_EUNSUPPORTED, "B = 65536"), (res(B=0), N.CTN_EINVAL, "B = 0")):
        try:
            refused(call, code, [out, scratch, amax])
        except AssertionError as e:
            raise AssertionError("{}: {}".format(what, e))


# ---- C. segmentation and overlap-add --------------------------------------------------------------------------------------------------
SEG_ROWS = E.seg_rows()
SEG_GROUPS = {"K12P5": [n for n in SEG_ROWS if n.startswith("K12P5")], "K250P125": [n for n in SEG_ROWS if n.startswith("K250P125")]}
SEG_GROUPS.update({n: [n] for n in SEG_ROWS if not n.startswith("K")})


def seg_one(name, channels_last):
    B, F, frames, K, P, reaches = SEG_ROWS[name]
    pl, pr, S = E.segment_geometry(frames, K, P)
    pitch = N.ctn_pitch(frames)
    x = torch.randn(B, F, pitch, generator=torch.Generator().manual_seed(frames))
    x[..., frames:] = float("nan")
    xd = dev(x)
    zshape = (B, S, K, F) if channels_last else (B, F, S, K)
    (Z,), n = twice(lambda o, base, nb: N.ctn_segment_fwd(xd.data_ptr(), o[0].data_ptr(), B, F, frames, pitch, K, P, pl, pr, channels_last, st()),
                    [(zshape,)], 0)
    assert n == 1
    ref = E.segment(x[..., :frames], K, P, pl, pr, channels_last)
    assert torch.equal(Z, ref), "{} channels_last={}: segmentation differs ({})".format(name, channels_last, reaches)
    out_pitch = N.ctn_pitch(frames)
    Zd = dev(ref)
    (y,), n = twice(lambda o, base, nb: N.ctn_overlap_add_fwd(Zd.data_ptr(), o[0].data_ptr(), B, F, S, K, P, pl, frames, out_pitch, channels_last,
                                                              st()), [((B, F, out_pitch),)], 0)
    assert n == 1
    assert torch.equal(y, E.overlap_add(ref, K, P, pl, frames, out_pitch, channels_last)), \
        "{} channels_last={}: overlap-add differs ({})".format(name, channels_last, reaches)


@pytest.mark.parametrize("channels_last", [1, 0])
@pytest.mark.parametrize("group", list(SEG_GROUPS))
def test_segment_and_overlap_add_exact(group, channels_last):
    """pitched input with NaN pad columns; segmentation bit-equal to the padded copy, overlap-add bit-equal to the fp32 sum in chunk
    order with the pitch tail 0"""
    for name in SEG_GROUPS[group]:
        seg_one(name, channels_last)
    report("seg", "{} cl={}".format(group, channels_last), 0.0, "{} row(s), bit for bit".format(len(SEG_GROUPS[group])))


def test_segment_overlap_add_refuse_past_the_grid_before_launch():
    """B = 65536 would put a batch index past the grid's y / z limit: refused with no launch, the memset of hop > chunk included"""
    B, F, frames, K, P = E.GRID_LIMIT + 1, 4, 30, 10, 15
    # sized for what the calls would touch (x: B F frames; Z: the hop > chunk memset of B S K F = B 2 10 F floats, and the
    # overlap-add's B F 20 stores), so a refusal that regressed fails the assert without writing past them
    x = torch.zeros(B * F * frames, device=DEV)
    Z = nan((B * F * 20,))
    for cl in (1, 0):
        refused(lambda: N.ctn_segment_fwd(x.data_ptr(), Z.data_ptr(), B, F, frames, frames, K, P, 0, 5, cl, st()), N.CTN_EUNSUPPORTED, [Z])
        refused(lambda: N.ctn_overlap_add_fwd(x.data_ptr(), Z.data_ptr(), B, F, 2, K, P, 0, 20, 20, cl, st()), N.CTN_EUNSUPPORTED, [Z])


# ---- D. the model ------------------------------------------------------------------------------------------------------------------------
MODEL_ROWS = E.model_rows()


def build(cfg, seed, mode):
    c = DO.DPRNNConfig(**cfg)
    sd = DO.synth_state_dict(c, seed=seed)
    m = DPRNNTasNet(c.n_basis, c.kernel_size, stride=c.stride, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None,
                    sep_hidden_channels=c.sep_hidden_channels, sep_bottleneck_channels=c.sep_bottleneck_channels, sep_chunk_size=c.sep_chunk_size,
                    sep_hop_size=c.sep_hop_size, sep_num_blocks=c.sep_num_blocks, sep_norm=True, mask_nonlinear="sigmoid", causal=False,
                    rnn_type="lstm", n_sources=c.n_sources, eps=c.eps)
    m.load_state_dict(sd, strict=True)
    m.math = mode
    return m.to(DEV).eval(), sd


def forward(m, x):
    with torch.no_grad():
        out = m(x.to(DEV))
    torch.cuda.synchronize()
    return out.cpu()


def model_reference(name, x, sd, cfg):
    """(fp64 answer, the fp32 oracle's worst unit error over the bound)"""
    def fn():
        out64 = E.model_answer(x, sd, cfg)
        return out64, E.D.excess(E.model_answer(x, sd, cfg, torch.float32), out64, 2)
    return _cached(("model", name), fn)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(MODEL_ROWS))
def test_model(name, mode):
    """each (sample, source) within 1e-4 max|fp64| + 1e-6, the fp32 oracle within 0.1 of that bound; the launch count of the native
    rows pinned; in the loudness batch each sample within 1e-6 of its run alone and digital silence exactly 0"""
    cfg, batch, samples, amps, reaches = MODEL_ROWS[name]
    m, sd = build(cfg, 7, mode)
    x = E.model_input(batch, samples, amps, samples)
    native = bool(N.ctn_bilstm_supported(cfg["sep_bottleneck_channels"], cfg["sep_hidden_channels"], cfg["sep_bottleneck_channels"]))
    assert native == (name != "fallback")
    torch.cuda.synchronize()
    n0 = N.ctn_total_launch_count()
    out = forward(m, x)
    launches = N.ctn_total_launch_count() - n0
    if native:
        assert launches == E.model_launches(cfg, mode), (launches, E.model_launches(cfg, mode))
    out64, r32 = model_reference(name, x, sd, cfg)
    assert r32 <= 0.1, "the fp32 oracle is {:.2f} of the bound from fp64: the row says nothing".format(r32)
    ratio = E.D.excess(out, out64, 2)
    assert ratio <= 1.0, "{} {}: worst (sample, source) error / bound {:.3g}".format(name, mode, ratio)
    extra = ""
    if amps:
        same = 0
        for b in range(batch):
            one = forward(m, x[b:b + 1])[0]
            assert float((one - out[b]).abs().max()) <= 1e-6 * float(one.abs().max()), b
            same += int(torch.equal(one, out[b]))
        assert not out[0].any(), "digital silence gave a nonzero estimate"
        extra = "; bit-identical to its run alone: {} of {} samples".format(same, batch)
    report("model", "{} {}".format(name, mode), ratio, "{}; fp32 oracle {:.3f} of the bound; {} launches{}".format(reaches, r32, launches, extra))


def test_model_graph_replay_gives_the_same_bits():
    cfg = E.SMALL
    m, sd = build(cfg, 7, None)
    x = E.model_input(2, 403, None, 1).to(DEV)
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.no_grad(), torch.cuda.stream(s):
        eager = m(x).clone()  # warm-up on the capture stream: the workspaces and kernel attributes exist before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = m(x)
    torch.cuda.current_stream(DEV).wait_stream(s)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)
    x2 = E.model_input(2, 403, None, 2)
    x.copy_(x2.to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = m(x)
    torch.cuda.synchronize()
    assert torch.equal(out, ref) and not torch.equal(out, eager)
    report("model", "graph replay", E.D.excess(out.cpu(), E.model_answer(x2, sd, cfg), 2), "captured once, replayed on new input")


def test_model_refuses_a_batch_past_the_grid_before_the_encoder():
    m, _ = build(E.SMALL, 7, None)
    x = torch.zeros(E.GRID_LIMIT + 1, 1, 40, device=DEV)
    torch.cuda.synchronize()
    n0 = N.ctn_total_launch_count()
    with torch.no_grad(), pytest.raises(NotImplementedError):
        m(x)
    assert N.ctn_total_launch_count() == n0
    assert math.isfinite(float(forward(m, x[:1].cpu()).abs().max()))
