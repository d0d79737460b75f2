"""Edge shapes of the DPRNN-TasNet path (BASELINE cfg4; ``-m gpu``) against plain float64 references.

test_lstm_gpu.py and test_dprnn_gpu.py check these kernels at toy lengths, in the reference layout, or through the whole model
against the fp32 oracle.  Here each kernel runs at the shapes that select its branches, and every row's `reaches` field names
the branch and the constant that selects it:
  A. ctn_bilstm_proj_fwd at the cfg4 recurrence lengths (T = 250 intra, ~255 inter, NSEQ up to 4080), every (F, H) instantiation
     and so every weight-ring depth, the Fo < 128 store guard, saturated gates, and each output alone.  Oracle: DO._bilstm.
  B. ctn_dprnn_norm_res2_fwd (k_sample_stats2 + k_norm_res2) at every block shape, including the ones whose last warp is
     partial, and its out_absmax word.
  C. ctn_dprnn_norm_res_fwd (the cuDNN-fallback gLN + residual) on its scalar and float4 branches, with samples that do not
     start on a 16-byte boundary.
  D. Channels-last ctn_segment_fwd / ctn_overlap_add_fwd on a pitched input with fused pads and crop.
  E. The whole DPRNNTasNet against DO.dprnn_tasnet_fwd in float64, in every math mode.

Every output buffer starts as NaN, so a cell a kernel never writes shows up.  The float64 answer and the fp32 oracle's own
distance to it are computed once per case (_CACHE).

Bounds:
  A. max|h - h64| <= max(2e-5, H_C x max|h32 - h64|), h32 = the CPU fp32 recurrence; projection rtol 1e-4 / atol 2e-5 x max|y64|.
  B, C. rtol / atol NORM_TOL (x max|ref|); out_absmax bit-equal to max|out|.
  D. segment bit-exact; overlap-add rtol / atol 1e-6 (x max|ref|), the pitch tail exactly 0.
  E. estimate and latent rtol 1e-4 / atol 2e-5 x max|ref|, the PIT permutation of the fp64 oracle; the fp32 oracle must sit
     10x inside that bound, or the case says nothing about the kernels.
"""
import collections

import pytest
import torch
import torch.nn.functional as F_

import convtasnet_oracle as O
import dprnn_oracle as DO
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import PIT1d
from ctn_b200.criterion.sdr import NegSISDR
from test_dprnn_gpu import MODES, build
from test_lstm_gpu import _ref, _run, _weights

pytestmark = pytest.mark.gpu

_CACHE = {}


def _cached(key, fn):
    if key not in _CACHE:
        _CACHE[key] = fn()
    return _CACHE[key]


def _ratio(x, ref, rtol, atol):
    """max over elements of |x - ref| / (atol + rtol |ref|): <= 1 passes torch.testing.assert_close(rtol, atol)"""
    return float(((x.double() - ref.double()).abs() / (atol + rtol * ref.double().abs())).max())


# ---- A. bi-LSTM + projection ------------------------------------------------------------------------------------------------
# Measured on an H100 80GB HBM3 at a 700 W power limit: over 250-257 steps the kernel's h sits 1e-6 .. 3e-6 from fp64, 2.6x ..
# 9.3x the fp32 CPU recurrence's own distance, all well inside the 2e-5 floor; only with weights x 8 (saturated gates, 8x larger
# pre-activations) does the scaled term bind: 2.5e-5 = 3.9x the fp32 recurrence's 6.4e-6.  H_C = 8 leaves 2x on that row.
H_FLOOR, H_C = 2e-5, 8.0
P_RTOL, P_ATOL = 1e-4, 2e-5


def _ring(F, H):
    """(ring depth nst, weight slabs per step) of k_bilstm: lstm_fixed_smem, SMEM_LIMIT, MAX_NST and lstm_per_step of ctn_lstm.cu"""
    fixed = 2048 + (F // 32 + H // 32) * 16384 + 64 * H * 4
    return min(4, (232448 - fixed) // 32768), (H // 32) * (F // 32 + H // 32) + H // 32


def _ring_text(F, H, T):
    nst, per_step = _ring(F, H)
    return "nst={}, per_step={}: {} slabs per CTA through the ring, each of its mbarriers completes {} phases".format(
        nst, per_step, T * per_step, T * per_step // nst)


Lstm = collections.namedtuple("Lstm", "F H Fo NSEQ T wscale every reaches")

LSTMS = {
    "intra": Lstm(64, 128, 64, 130, 250, 1.0, 1, "cfg4 intra length T=250; NSEQ=130 = 2 full CTAs + a 2-row CTA (LSEQ=64); "
                  + _ring_text(64, 128, 250)),
    "inter": Lstm(64, 128, 64, 129, 257, 1.0, 1, "cfg4 inter length T=257; NSEQ=129 = 2 full CTAs + a 1-row CTA"),
    "fo96": Lstm(64, 128, 96, 65, 250, 1.0, 1, "Fo=96 < 128 projection columns: the o < Fo guard of the P store"),
    "grid4080": Lstm(64, 128, 64, 4080, 250, 1.0, 67, "cfg4 intra grid NSEQ=4080 (64 x 2 CTAs, the last with 48 rows), every 67th "
                                                        "sequence and the last"),
    "wx8": Lstm(64, 128, 64, 65, 250, 8.0, 1, "weights x 8: saturated gates held over 250 steps"),
}
for _F in (32, 64, 128):
    for _H in (32, 64, 128):
        LSTMS["F{}H{}".format(_F, _H)] = Lstm(_F, _H, _F, 65, 250, 1.0, 1, "k_bilstm<NCH={}, KSX={}>, ".format(_H // 32, _F // 32)
                                              + _ring_text(_F, _H, 250))


def _lstm_case(case):
    e = LSTMS[case]
    sd = _weights(e.F, e.H, e.Fo, seed=e.NSEQ + e.T + e.F + e.H, wscale=e.wscale)
    z = torch.randn(e.NSEQ, e.T, e.F, generator=torch.Generator().manual_seed(e.T + e.F)) * 1.5
    idx = torch.tensor(sorted(set(range(0, e.NSEQ, e.every)) | {e.NSEQ - 1}))
    return sd, z, idx


def _lstm_reference(case, sd, z, idx):
    """(h64, y64, max|h32 - h64|) on the checked sequences; sequences are independent, so a subset needs only its own inputs"""
    def fn():
        zs = z[idx]
        h64, y64 = _ref(zs, sd, torch.float64)
        h32, _ = _ref(zs, sd, torch.float32)
        return h64, y64, float((h32.double() - h64).abs().max())
    return _cached(("lstm", case), fn)


@pytest.mark.parametrize("case", list(LSTMS))
def test_bilstm_long_sequences_vs_fp64(case):
    """Each LSTMS row: h within max(H_FLOOR, H_C x the fp32 CPU recurrence's own error) of fp64, the projection P0 + P1 + bias
    within rtol 1e-4 / atol 2e-5 x max|y64|, no cell left unwritten."""
    e = LSTMS[case]
    if not N.ctn_bilstm_supported(e.F, e.H, e.Fo):
        pytest.fail("({}, {}, {}) is inside the native envelope".format(e.F, e.H, e.Fo))
    sd, z, idx = _lstm_case(case)
    h, P = _run(z, sd, e.H, e.Fo)
    assert torch.isfinite(h).all() and torch.isfinite(P).all(), "cells left unwritten"
    h64, y64, err32 = _lstm_reference(case, sd, z, idx)
    err = float((h[idx].double() - h64).abs().max())
    bound = max(H_FLOOR, H_C * err32)
    assert err <= bound, "max|h - h64| {:.3e} > bound {:.3e} (fp32 CPU recurrence: {:.3e}, ratio {:.2f})".format(err, bound, err32,
                                                                                                             err / err32)
    y = (P[0] + P[1] + sd["fc.bias"])[idx]
    atol = P_ATOL * float(y64.abs().max())
    torch.testing.assert_close(y.double(), y64, rtol=P_RTOL, atol=atol)
    print("[lstm {}] h: {:.2e} = {:.3f} of bound (fp32 CPU {:.2e}, kernel / fp32 {:.2f}); projection {:.3f} of bound -- {}".format(
        case, err, err / bound, err32, err / err32, _ratio(y, y64, P_RTOL, atol), e.reaches))


def test_bilstm_outputs_alone_match_both():
    """hout only (P null) and P only at T=250: bit-equal to the run that writes both"""
    e = LSTMS["intra"]
    sd, z, _ = _lstm_case("intra")
    h, P = _run(z, sd, e.H, e.Fo)
    h_only, _ = _run(z, sd, e.H, e.Fo, want_p=False)
    _, p_only = _run(z, sd, e.H, e.Fo, want_h=False)
    assert torch.equal(h_only, h)
    assert torch.equal(p_only, P)


# ---- B, C. gLN + residual (+ path swap) -------------------------------------------------------------------------------------
# fp64 statistics, fp32 normalisation: measured within 8e-8 (x max|ref|) of fp64 on an H100; 2e-6 is about 17 float ulps
NORM_TOL = 2e-6
EPS = DO.EPS


def _gln_res64(Y, R, gamma, beta, swap):
    """fp64 GroupNorm(1, F) per sample over (D1, D2, F) channels-last, * gamma + beta, + R; swap stores (B, D2, D1, F)"""
    Y, R = Y.double(), R.double()
    B = Y.shape[0]
    flat = Y.reshape(B, -1)
    mean = flat.mean(1).view(B, 1, 1, 1)
    var = flat.var(1, unbiased=False).view(B, 1, 1, 1)
    out = (Y - mean) / torch.sqrt(var + EPS) * gamma.double() + beta.double() + R
    return out.transpose(1, 2).contiguous() if swap else out


def _norm_inputs(shape, F, seed):
    g = torch.Generator().manual_seed(seed)
    R = torch.randn(shape, generator=g)
    gamma = 1.0 + 0.2 * (torch.rand(F, generator=g) - 0.5)
    beta = 0.1 * (torch.rand(F, generator=g) - 0.5)
    return g, R, gamma, beta


def _block_text(F):
    q = F // 4
    ty = max(1, 256 // q)
    return ty, "block ({}, {}) = {} threads{}".format(q, ty, q * ty, ", partial last warp" if (q * ty) % 32 else "")


def _norm2_cases():
    cases = []
    for F in (4, 12, 32, 48, 64, 96, 128, 1024):
        ty, text = _block_text(F)
        for D2, what in ((1, "D2=1: no TY step"), (ty - 1, "D2=TY-1: a partial TY step"), (4 * ty + 1, "D2=4TY+1: one cell past a full 4-cell step")):
            if D2 >= 1:
                cases.append(pytest.param(F, D2, "F={}: {}; {}".format(F, text, what), id="F{}-D2={}".format(F, D2)))
    return cases


@pytest.mark.parametrize("F,D2,reaches", _norm2_cases())
def test_norm_res2_vs_fp64(F, D2, reaches):
    """ctn_dprnn_norm_res2_fwd (gLN(P0 + P1 + bias) + R, swap 0 / 1) for D1 in {1, 7}, B in {1, 3}; out_absmax ==
    float_as_uint(max|out|) bit for bit"""
    dev = torch.device("cuda")
    worst = 0.0
    for B in (1, 3):
        for D1 in (1, 7):
            g, R, gamma, beta = _norm_inputs((B, D1, D2, F), F, seed=F * 1000 + D2 * 10 + B + D1)
            P = torch.randn(2, B, D1, D2, F, generator=g) * 0.7 + 0.3
            bias = 0.2 * torch.randn(F, generator=g)
            for swap in (0, 1):
                ref = _gln_res64(P[0].double() + P[1].double() + bias.double(), R, gamma, beta, swap)
                Pd, Rd, bd, gd, betad = (t.to(dev).contiguous() for t in (P, R, bias, gamma, beta))
                out = torch.full(ref.shape, float("nan"), device=dev)
                scratch = torch.empty(2 * B, dtype=torch.float64, device=dev)
                amax = torch.full((1,), -1, dtype=torch.int32, device=dev)
                N.check(N.ctn_dprnn_norm_res2_fwd(Pd.data_ptr(), bd.data_ptr(), Rd.data_ptr(), gd.data_ptr(), betad.data_ptr(),
                                                  out.data_ptr(), B, D1, D2, F, EPS, swap, scratch.data_ptr(), amax.data_ptr(),
                                                  N.stream_ptr(dev)), "ctn_dprnn_norm_res2_fwd")
                what = "B={} D1={} swap={}".format(B, D1, swap)
                torch.testing.assert_close(out.cpu().double(), ref, rtol=NORM_TOL, atol=NORM_TOL * float(ref.abs().max()),
                                           msg=lambda m: "{}: {}".format(what, m))
                want = int(out.abs().max().view(torch.int32))
                assert int(amax.item()) == want, "{}: out_absmax {:#x} != bits of max|out| {:#x}".format(what, int(amax.item()), want)
                worst = max(worst, _ratio(out.cpu(), ref, NORM_TOL, NORM_TOL * float(ref.abs().max())))
    print("[norm_res2 F={} D2={}] worst {:.3f} of bound -- {}".format(F, D2, worst, reaches))


def test_norm_res2_envelope():
    dev = torch.device("cuda")
    t = torch.zeros(2 * 4 * 1028, device=dev)
    scratch = torch.empty(2, dtype=torch.float64, device=dev)
    st = N.stream_ptr(dev)

    def call(F, out, swap):
        p = t.data_ptr()
        return N.ctn_dprnn_norm_res2_fwd(p, p, p, p, p, out, 1, 1, 1, F, EPS, swap, scratch.data_ptr(), None, st)
    other = torch.zeros(1028, device=dev).data_ptr()
    assert call(6, other, 0) == N.CTN_EINVAL                # F % 4 != 0
    assert call(1028, other, 0) == N.CTN_EUNSUPPORTED       # F > 1024: more than 256 threads per row
    assert call(64, t.data_ptr(), 1) == N.CTN_EINVAL        # the swap cannot run in place (out == R)


Norm = collections.namedtuple("Norm", "F D1 D2 reaches")

NORMS = {
    "F5-odd": Norm(5, 3, 7, "F=5: scalar k_norm_res; n=105 odd: scalar k_sample_stats"),
    "F33-odd-3blocks": Norm(33, 13, 25, "F=33 scalar; n=10725 odd over 3 stats blocks: the grid-strided scalar loop"),
    "F33-model-intra": Norm(33, 21, 10, "F=33 scalar; n=6930 = 2 mod 4: DPRNNTasNet F=33, K=10, S=21 (sample 1 starts 8 bytes "
                                        "off a 16-byte boundary)"),
    "F33-n4": Norm(33, 4, 10, "F=33 scalar k_norm_res; n=1320 = 0 mod 4: float4 k_sample_stats"),
    "F8": Norm(8, 5, 9, "F=8: float4 k_norm_res and k_sample_stats"),
    "F12-2blocks": Norm(12, 7, 61, "F=12: float4, 3 float4 per lane; n=5124 over 2 stats blocks"),
}


@pytest.mark.parametrize("case", list(NORMS))
def test_norm_res_fallback_vs_fp64(case):
    """ctn_dprnn_norm_res_fwd (the gLN + residual of the cuDNN-fallback LSTM), B=3, swap 0 / 1"""
    e = NORMS[case]
    B, dev = 3, torch.device("cuda")
    g, R, gamma, beta = _norm_inputs((B, e.D1, e.D2, e.F), e.F, seed=e.F * 100 + e.D1 * 10 + e.D2)
    Y = torch.randn(B, e.D1, e.D2, e.F, generator=g) * 0.8 - 0.4
    Yd, Rd, gd, bd = (t.to(dev).contiguous() for t in (Y, R, gamma, beta))
    scratch = torch.empty(2 * B, dtype=torch.float64, device=dev)
    worst = 0.0
    for swap in (0, 1):
        ref = _gln_res64(Y, R, gamma, beta, swap)
        out = torch.full(ref.shape, float("nan"), device=dev)
        N.check(N.ctn_dprnn_norm_res_fwd(Yd.data_ptr(), Rd.data_ptr(), gd.data_ptr(), bd.data_ptr(), out.data_ptr(), B, e.D1, e.D2,
                                         e.F, EPS, swap, scratch.data_ptr(), N.stream_ptr(dev)), "ctn_dprnn_norm_res_fwd")
        atol = NORM_TOL * float(ref.abs().max())
        torch.testing.assert_close(out.cpu().double(), ref, rtol=NORM_TOL, atol=atol, msg=lambda m: "swap={}: {}".format(swap, m))
        worst = max(worst, _ratio(out.cpu(), ref, NORM_TOL, atol))
    for alias in (Yd, Rd):  # the path swap cannot run in place
        assert N.ctn_dprnn_norm_res_fwd(Yd.data_ptr(), Rd.data_ptr(), gd.data_ptr(), bd.data_ptr(), alias.data_ptr(), B, e.D1, e.D2,
                                        e.F, EPS, 1, scratch.data_ptr(), N.stream_ptr(dev)) == N.CTN_EINVAL
    print("[norm_res {}] worst {:.3f} of bound -- {}".format(case, worst, e.reaches))


# ---- D. channels-last segmentation and overlap-add --------------------------------------------------------------------------
OLA_TOL = 1e-6

Seg = collections.namedtuple("Seg", "B F frames K P pl pr reaches")

SEGS = {
    "overlap-F33": Seg(2, 33, 300, 40, 15, 3, 9, "hop < chunk (up to 3 chunks per frame); F=33: a second 32-channel tile with 1 "
                                                 "channel; ragged padded tail dropped"),
    "hop=chunk-F5": Seg(2, 5, 200, 25, 25, 1, 4, "hop = chunk: one chunk per frame; F=5 inside one tile"),
    "hop>chunk-F64": Seg(3, 64, 250, 20, 30, 2, 7, "hop > chunk: frames in the gaps land in no chunk, the cudaMemsetAsync branch"),
    "S1-F33": Seg(1, 33, 90, 100, 50, 4, 6, "S=1: the whole padded sequence is one chunk"),
    "cfg4-F64": Seg(2, 64, 997, 250, 125, 1, 2, "cfg4 K=250 P=125, S=7, pad_left != pad_right"),
}


def _seg_geometry(e):
    Tp = e.frames + e.pl + e.pr
    S = (Tp - e.K) // e.P + 1
    T_out = min(e.frames, (S - 1) * e.P + e.K - e.pl)
    return S, T_out


@pytest.mark.parametrize("case", list(SEGS))
def test_segment_channels_last_pitched(case):
    """ctn_segment_fwd(channels_last=1) on a pitched input (NaN in the pad columns [frames, pitch)): bit-equal to
    DO.segment1d of the padded input, permuted to (B, S, K, F); every cell of Z written"""
    e = SEGS[case]
    dev = torch.device("cuda")
    pitch = N.ctn_pitch(e.frames)
    assert pitch > e.frames
    S, _ = _seg_geometry(e)
    x = torch.randn(e.B, e.F, pitch, generator=torch.Generator().manual_seed(e.frames + e.F))
    x[..., e.frames:] = float("nan")
    ref = DO.segment1d(F_.pad(x[..., :e.frames], (e.pl, e.pr)), e.K, e.P).permute(0, 2, 3, 1).contiguous()
    assert ref.shape == (e.B, S, e.K, e.F)
    xd = x.to(dev)
    Z = torch.full((e.B, S, e.K, e.F), float("nan"), device=dev)
    N.check(N.ctn_segment_fwd(xd.data_ptr(), Z.data_ptr(), e.B, e.F, e.frames, pitch, e.K, e.P, e.pl, e.pr, 1, N.stream_ptr(dev)),
            "ctn_segment_fwd")
    assert torch.equal(Z.cpu(), ref), e.reaches


@pytest.mark.parametrize("case", list(SEGS))
def test_overlap_add_channels_last_crop_pitch(case):
    """ctn_overlap_add_fwd(channels_last=1) with crop_left = pad_left > 0 into a pitched output (out_pitch > T_out): fp64
    DO.overlap_add1d + crop within 1e-6 relative, columns [T_out, out_pitch) exactly 0"""
    e = SEGS[case]
    dev = torch.device("cuda")
    S, T_out = _seg_geometry(e)
    out_pitch = N.ctn_pitch(T_out)
    assert out_pitch > T_out and e.pl > 0
    Z = torch.randn(e.B, S, e.K, e.F, generator=torch.Generator().manual_seed(S + e.K))
    ref = DO.overlap_add1d(Z.double().permute(0, 3, 1, 2), e.K, e.P)[..., e.pl:e.pl + T_out]
    Zd = Z.to(dev)
    y = torch.full((e.B, e.F, out_pitch), float("nan"), device=dev)
    N.check(N.ctn_overlap_add_fwd(Zd.data_ptr(), y.data_ptr(), e.B, e.F, S, e.K, e.P, e.pl, T_out, out_pitch, 1, N.stream_ptr(dev)),
            "ctn_overlap_add_fwd")
    y = y.cpu()
    atol = OLA_TOL * float(ref.abs().max())
    torch.testing.assert_close(y[..., :T_out].double(), ref, rtol=OLA_TOL, atol=atol)
    assert torch.equal(y[..., T_out:], torch.zeros_like(y[..., T_out:])), "pitch tail not zeroed"
    print("[overlap_add {}] worst {:.3f} of bound -- {}".format(case, _ratio(y[..., :T_out], ref, OLA_TOL, atol), e.reaches))


# ---- E. the whole model -----------------------------------------------------------------------------------------------------
OUT_RTOL, OUT_ATOL = 1e-4, 2e-5

Model = collections.namedtuple("Model", "cfg batch T S reaches")

MODELS = {
    "cfg4": Model(dict(n_basis=64, kernel_size=2, sep_bottleneck_channels=64, sep_hidden_channels=128, sep_chunk_size=250,
                       sep_hop_size=125, sep_num_blocks=2), 2, 4000, 31,
                  "cfg4 dimensions: native LSTM at T=250 (intra) and T=31 over NSEQ=500 (inter); segment pads 0 / 1"),
    "S1": Model(dict(n_basis=32, kernel_size=4, sep_bottleneck_channels=32, sep_hidden_channels=64, sep_chunk_size=99,
                     sep_hop_size=33, sep_num_blocks=2), 2, 200, 1,
                "frames == chunk: S=1, the inter-chunk LSTM runs T=1, no padding"),
    "hop>chunk": Model(dict(n_basis=16, kernel_size=4, sep_bottleneck_channels=32, sep_hidden_channels=32, sep_chunk_size=20,
                            sep_hop_size=30, sep_num_blocks=2), 2, 420, 8,
                       "K=20 < P=30: frames in the gaps between chunks, overlap-add leaves them 0; pads 10 / 11"),
    "fallback-F33": Model(dict(n_basis=16, kernel_size=2, sep_bottleneck_channels=33, sep_hidden_channels=24, sep_chunk_size=10,
                               sep_hop_size=5, sep_num_blocks=2), 2, 108, 21,
                          "F=33, H=24 outside the native LSTM: cuDNN + ctn_dprnn_norm_res_fwd; n = 10 x 21 x 33 = 2 mod 4 with "
                          "batch 2: sample 1 of the statistics is not 16-byte aligned"),
    "F32-3src": Model(dict(n_basis=24, kernel_size=8, sep_bottleneck_channels=32, sep_hidden_channels=32, sep_chunk_size=15,
                           sep_hop_size=7, sep_num_blocks=2, n_sources=3), 3, 1000, 35,
                      "F=H=32 (k_bilstm<1,1>), K=15 P=7, 3 sources, batch 3"),
    "F128-H64": Model(dict(n_basis=32, kernel_size=2, sep_bottleneck_channels=128, sep_hidden_channels=64, sep_chunk_size=20,
                           sep_hop_size=10, sep_num_blocks=2), 3, 229, 22,
                      "F=128 H=64 (k_bilstm<2,4>); intra NSEQ = 3 x 22 = 66: a 64-row CTA and a 2-row CTA"),
}


def _model_case(case):
    e = MODELS[case]
    cfg = DO.DPRNNConfig(**e.cfg)
    sd = DO.synth_state_dict(cfg, seed=501)
    mixture, sources = O.synth_batch(e.batch, cfg.n_sources, e.T, seed=502)
    return cfg, sd, mixture, sources


def _model_reference(case, cfg, sd, mixture, sources):
    """fp64 (out, latent, perm) and the fp32 oracle's distance to it, as a share of the bound, and its permutation"""
    def fn():
        sd64 = {k: v.double() for k, v in sd.items()}
        out64, lat64 = DO.dprnn_tasnet_fwd(mixture.double(), sd64, cfg)
        _, perm64 = O.pit_neg_sisdr(out64, sources.double(), batch_mean=False)
        out32, lat32 = DO.dprnn_tasnet_fwd(mixture, sd, cfg)
        _, perm32 = O.pit_neg_sisdr(out32, sources, batch_mean=False)
        r32 = max(_ratio(out32, out64, OUT_RTOL, OUT_ATOL * float(out64.abs().max())),
                  _ratio(lat32, lat64, OUT_RTOL, OUT_ATOL * float(lat64.abs().max())))
        return out64, lat64, perm64, perm32, r32
    return _cached(("model", case), fn)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", list(MODELS))
def test_dprnn_tasnet_edges_vs_fp64(case, mode):
    """Each MODELS row through DPRNNTasNet.extract_latent: estimate and latent within rtol 1e-4 / atol 2e-5 x max|ref| of the
    fp64 oracle, PIT permutation equal to the fp64 oracle's"""
    e = MODELS[case]
    cfg, sd, mixture, sources = _model_case(case)
    native = case != "fallback-F33"
    F, H = cfg.sep_bottleneck_channels, cfg.sep_hidden_channels
    assert bool(N.ctn_bilstm_supported(F, H, F)) == native, case
    out64, lat64, perm64, perm32, r32 = _model_reference(case, cfg, sd, mixture, sources)
    assert torch.equal(perm32, perm64)
    assert r32 <= 0.1, "ill-conditioned case: the fp32 oracle is {:.2f} of the bound from fp64".format(r32)
    model = build(cfg, sd, math=mode)
    frames = N.frames_of(e.T, cfg.kernel_size, cfg.stride)[0]
    assert model.separator.segment_geometry(frames)[2] == e.S
    with torch.no_grad():
        out, latent = model.extract_latent(mixture.cuda())
        _, perm = PIT1d(NegSISDR(), cfg.n_sources)(out, sources.cuda(), batch_mean=False)
    out, latent = out.cpu(), latent.cpu()
    atol_o, atol_l = OUT_ATOL * float(out64.abs().max()), OUT_ATOL * float(lat64.abs().max())
    torch.testing.assert_close(out.double(), out64, rtol=OUT_RTOL, atol=atol_o)
    torch.testing.assert_close(latent.double(), lat64, rtol=OUT_RTOL, atol=atol_l)
    assert torch.equal(perm.cpu(), perm64)
    print("[model {} {}] estimate {:.3f}, latent {:.3f} of bound; fp32 oracle {:.3f} of bound -- {}".format(
        case, mode, _ratio(out, out64, OUT_RTOL, atol_o), _ratio(latent, lat64, OUT_RTOL, atol_l), r32, e.reaches))
