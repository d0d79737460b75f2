"""Every 1x1 contraction kernel on its own (``-m gpu``), through the verification hook (include/ctn_b200_probe.h), against fp64.

The models' tests see k_pw_wgmma / k_pw_simt / k_wgrad_wgmma only behind gLN renormalisation, sigmoids and the decoder, which
dilute a contraction's error: a pointwise contraction that lost one of its three split passes still passes them.  Here each
output is held to the gate of tests/pw_criterion.py (e <= E_drop / 8 for the 3-pass modes, see there), which such a loss
fails, at the shapes and branches where the kernels can go wrong.  Every row of ROWS names in `reaches` what it reaches.

Per row and mode:
  * D (prefilled with NaN, or zero for EPI_MASKDEC whose seams are added) passes the gate; columns [frames, pitch) are exactly 0;
  * the side outputs: gLN statistics (stats_out, dw_stats_out) within 64 u sum|.| of the fp64 sums of the kernel's own output,
    mask_out through the gate, dw_u_pre_out / res_x_out within 8 u of their magnitude and exactly 0 past frames;
  * modes: fp32 (FFMA), tf32x3, tf32, f16x3 with the operand scale at the top of its legal range (fp16 pieces), f16x3 without
    an operand scale (tf32 pieces); some rows add f16x3 with the scale 2^-15 lower (the headroom the pipelines leave unused);
  * combinations a mode does not implement must return CTN_EUNSUPPORTED.
"""
import ctypes as C
import math

import pytest
import torch

import pw_criterion as PC
import train_kernel_ref as TKR
from ctn_b200 import _native as N

pytestmark = pytest.mark.gpu

U = PC.U
PRO = {"none": 0, "prelu": 1, "dw": 2, "res": 3}
EPI = {"raw": 0, "head": 1, "h": 2, "mask": 3, "maskdec": 4}
MATH = {"fp32": N.MATH_FP32, "tf32x3": N.MATH_TF32X3, "tf32": N.MATH_TF32, "f16x3": N.MATH_F16X3, "f16x3-tf32": N.MATH_F16X3,
        "f16x3-low": N.MATH_F16X3}
MODES = ["fp32", "tf32x3", "tf32", "f16x3", "f16x3-tf32"]
SIMT = {("none", "raw"), ("none", "head"), ("none", "h"), ("prelu", "mask")}  # k_pw_simt's combinations
EPS = 1e-8
DEV = "cuda"

_p, _i, _d, _f = C.c_void_p, C.c_int32, C.c_double, C.c_float


class ProbeArgs(C.Structure):
    _fields_ = [("A", _p), ("W", _p), ("D", _p), ("B", _i), ("M", _i), ("K", _i), ("frames", _i), ("pitch", _i),
                ("pro_slope", _p), ("dw_norm_g", _p), ("dw_norm_b", _p), ("dw_w", _p), ("dw_b", _p), ("dw_stats_in", _p),
                ("dw_stats_out", _p), ("dw_dilation", _i), ("dw_pad_left", _i), ("dw_eps", _f), ("bias", _p), ("slope", _p),
                ("v1", _p), ("v2", _p), ("stats_in", _p), ("n_in", _d), ("eps", _f), ("stats_out", _p), ("store_pre", _i),
                ("wenc", _p), ("Nb", _i), ("mask_out", _p), ("mask_logits", _i), ("dec_w", _p), ("dec_crop_left", _i),
                ("dec_T_out", _i), ("res_r", _p), ("res_Mt", _i), ("res_v1", _p), ("res_v2", _p), ("res_stats", _p),
                ("res_n", _d), ("res_eps", _f), ("res_x_out", _p), ("act_scale", _p), ("dw_in_slope", _p), ("dw_u_pre_out", _p)]


probe_pw = N._sig("ctn_probe_pw", C.c_int, C.POINTER(ProbeArgs), C.c_int, C.c_int, C.c_int, C.c_int, _p, C.c_size_t, _p)
probe_wimg_bytes = N._sig("ctn_probe_pw_wimg_bytes", C.c_size_t, C.c_int, C.c_int, C.c_int)
probe_wgrad = N._sig("ctn_probe_wgrad", C.c_int, _p, C.c_size_t, _p, C.c_size_t, _p, _p, C.c_int, C.c_int, C.c_int, C.c_int,
                     C.c_int, C.c_int, C.c_int, _p)


def _row(pro, epi, M, K, frames, reaches, B=1, **kw):
    r = dict(pro=pro, epi=epi, M=M, K=K, frames=frames, B=B, reaches=reaches, extra_pitch=0, modes=MODES, routes=False)
    r.update(kw)
    return r


ROWS = {
    # ---- shapes (PRO_NONE / EPI_RAW unless named) ----
    "k1_m1_f1": _row("none", "raw", 1, 1, 1, "K = 1 (one partial k-slab), M = 1, one frame"),
    "k31_m17_f4_b3": _row("none", "raw", 17, 31, 4, "K = 31 < one slab, M = 17, B = 3", B=3),
    "k32_m128_f127": _row("none", "raw", 128, 32, 127, "one full k-slab, one full n-tile, frames one short of a tile"),
    "k33_m129_f128": _row("none", "raw", 129, 33, 128, "K = 33: a 1-channel last slab; M = 129: a 1-row last n-tile"),
    "k100_m300_f129_b3": _row("none", "raw", 300, 100, 129, "three n-tiles, K % 32 = 4, one frame into the second tile; routes",
                              B=3, routes=True, modes=MODES + ["f16x3-low"]),
    "k512_m128_f1000": _row("none", "raw", 128, 512, 1000, "16 k-slabs through the 2-stage ring, 8 time tiles"),
    "k1056_m128_f1000": _row("none", "raw", 128, 1056, 1000, "K = 1056 (33 slabs, the largest dense contraction); fp16 headroom",
                             modes=MODES + ["f16x3-low"]),
    "k64_m2048_f129": _row("none", "raw", 2048, 64, 129, "M = 2048 = F16_MAX_ROWS: fp16 pieces, batched builder past 8 n-tiles; routes",
                           routes=True),
    "k64_m2049_f129": _row("none", "raw", 2049, 64, 129, "M = 2049 > F16_MAX_ROWS: f16x3 falls back to tf32 pieces; routes",
                           routes=True),
    "k96_m128_f4_wide": _row("none", "raw", 128, 96, 4, "pitch = ctn_pitch(frames) + 256: two tiles wholly past frames",
                             extra_pitch=256),
    "head_k100_m129_b3": _row("none", "head", 129, 100, 1000, "EPI_HEAD: folded gLN (rstd, v1, v2) in the epilogue", B=3),
    "h_k96_m300": _row("none", "h", 300, 96, 1000, "EPI_H: bias + PReLU, gLN statistics of the output", B=3),
    "h_pre_k33_m129": _row("none", "h", 129, 33, 129, "EPI_H store_pre: pre-activation stored, statistics of PReLU(.)",
                           store_pre=True, modes=[m for m in MODES if m != "fp32"]),
    # ---- PRO_DW ----
    "dw_d1_k96": _row("dw", "raw", 128, 96, 1000, "PRO_DW d = 1 (DCLS 1), K = 96: interior and boundary tiles", d=1, B=3),
    "dw_d2_k100": _row("dw", "raw", 128, 100, 1000, "PRO_DW d = 2 (DCLS 2), K = 100: never interior", d=2),
    "dw_d4_k96": _row("dw", "raw", 300, 96, 1000, "PRO_DW d = 4 (DCLS 4), interior + boundary, three n-tiles", d=4,
                      modes=MODES + ["f16x3-low"]),
    "dw_d12_k100": _row("dw", "raw", 128, 100, 129, "PRO_DW d = 12, K = 100", d=12, B=3),
    "dw_d128_k96": _row("dw", "raw", 128, 96, 1000, "PRO_DW d = 128 = two 64-frame tiles", d=128),
    "dw_d520_k96": _row("dw", "raw", 128, 96, 500, "PRO_DW d = 520 > pitch = 512: every outer tap is padding", d=520),
    "dw_train_d2_k96": _row("dw", "raw", 300, 96, 1000, "PRO_DW TRAIN: PReLU on load, dw_u_pre_out, d = 2", d=2, train=True, B=3),
    "dw_train_d12_k100": _row("dw", "raw", 128, 100, 129, "PRO_DW TRAIN, boundary tiles only, d = 12", d=12, train=True),
    # ---- PRO_RES ----
    "res_k100_m300": _row("res", "h", 300, 100, 1000, "PRO_RES: x_new from n-tile 0 of three, K % 32 != 0", B=3),
    "res_k96_m300_wide": _row("res", "h", 300, 96, 129, "PRO_RES with pitch + 256", extra_pitch=256),
    # ---- EPI_MASK ----
    "mask_nb40": _row("prelu", "mask", 80, 96, 1000, "EPI_MASK Nb = 40 (S = 2), mask_out on", Nb=40, mask_out=True, B=3),
    "mask_nb40_nomask": _row("prelu", "mask", 80, 33, 129, "EPI_MASK Nb = 40, mask_out off", Nb=40),
    "mask_nb512": _row("prelu", "mask", 1024, 128, 129, "EPI_MASK Nb = 512 (S = 2), mask_out on", Nb=512, mask_out=True),
    "mask_logits": _row("prelu", "mask", 1024, 128, 1000, "EPI_MASK mask_logits (softmax first pass), mask_out on", Nb=512,
                        logits=True, mask_out=True),
    # ---- EPI_MASKDEC (fp16 pieces only: every other mode must refuse) ----
    "maskdec_nb128_s1_f1": _row("prelu", "maskdec", 128, 96, 1, "EPI_MASKDEC one frame", Nb=128, crop=0),
    "maskdec_nb128_s2_f129": _row("prelu", "maskdec", 256, 96, 129, "EPI_MASKDEC frames = 129: a seam, crop 4", Nb=128, crop=4,
                                  B=3),
    "maskdec_nb128_s4_f128": _row("prelu", "maskdec", 512, 33, 128, "EPI_MASKDEC one full tile, S = 4", Nb=128, crop=0),
    "maskdec_nb512_s4_f1000": _row("prelu", "maskdec", 2048, 96, 1000, "EPI_MASKDEC nt_per_cta = 4, 8 tiles, crop 4", Nb=512,
                                   crop=4),
    "maskdec_nb512_s1_f129": _row("prelu", "maskdec", 512, 128, 129, "EPI_MASKDEC Nb = 512, S = 1", Nb=512, crop=0),
    "maskdec_nb40": _row("prelu", "maskdec", 80, 96, 129, "EPI_MASKDEC refused: Nb = 40 is no multiple of 128", Nb=40, crop=0,
                         refuse=True),
    # ---- the pipelines' own shapes on the fp16 channel-split tile (64 frames x 2 n-tiles; side outputs from n-tile 0 only) ----
    "res_k128_m512_b3": _row("res", "h", 512, 128, 1000, "pw1 shape: four n-tiles = two full groups, every warpgroup live", B=3),
    "res_k128_m128": _row("res", "h", 128, 128, 1000, "one n-tile: warpgroup 1 idle in every CTA"),
    "h_k128_m512": _row("none", "h", 512, 128, 1000, "block 0's pw1 shape (PRO_NONE)"),
    **{f"dw_k512_m256_d{d}": _row("dw", "raw", 256, 512, 1000, f"pw2 shape, d = {d}" + (" = one 64-frame tile" if d == 64 else ""),
                                  d=d) for d in (1, 2, 4, 64, 128)},
    "dw_train_k512_m256_d2": _row("dw", "raw", 256, 512, 1000, "pw2 shape, TRAIN variant, d = 2", d=2, train=True),
    "dw_k512_m128": _row("dw", "raw", 128, 512, 1000, "the last block's pw2 (skip head only): one n-tile", d=1),
    **{f"res_k128_m512_f{T}": _row("res", "h", 512, 128, T, f"pw1 shape, frames = {T} at a 64-frame tile edge") for T in (63, 64, 65, 4001)},
    **{f"dw_k512_m256_f{T}": _row("dw", "raw", 256, 512, T, f"pw2 shape, frames = {T} at a 64-frame tile edge", d=4)
       for T in (63, 64, 65, 4001)},
}

# Headroom sweep: the f16x3 mode with the operand scale 2^k below the top of its range, on the pipelines' (pro, epi) pairs and
# shapes.  The lo piece x s - hi is stored as a plain fp16, so far below the top it turns subnormal and the gate eventually
# breaks; it must hold SWEEP_REQUIRED binades below the top, at least two more than the largest headroom test_act_envelope_gpu.py
# measured on the paper config (17.3 binades at 60 s, DESIGN section 2).
SWEEP_SHIFTS = (0, 9, 15, 18, 21)
SWEEP_REQUIRED = 21
SWEEP_ROWS = {
    "pw1_res": _row("res", "h", 512, 128, 1000, "PRO_RES / EPI_H", B=2),
    "pw1_none": _row("none", "h", 512, 128, 1000, "PRO_NONE / EPI_H (block 0)"),
    "pw2_dw": _row("dw", "raw", 256, 512, 1000, "PRO_DW / EPI_RAW", d=4),
    "pw2_dw_m128": _row("dw", "raw", 128, 512, 1000, "PRO_DW / EPI_RAW, M = 128 (last block)", d=4),
    "mask": _row("prelu", "mask", 1024, 128, 1000, "PRO_PRELU / EPI_MASK", Nb=512),
    "maskdec": _row("prelu", "maskdec", 1024, 128, 1000, "PRO_PRELU / EPI_MASKDEC", Nb=512, crop=4),
}


def _pitch(frames, extra=0):
    return N.ctn_pitch(frames) + extra


def _padded(x, pitch, fill=float("nan")):
    """(B, C, T) -> float32 (B, C, pitch) on cuda, columns [T, pitch) = fill"""
    B, Cc, T = x.shape
    y = torch.full((B, Cc, pitch), fill, dtype=torch.float32, device=DEV)
    y[..., :T] = x.float()
    return y


def _rnd(g, *shape, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=g) * scale + shift).float().double()


def _case(name, r):
    """inputs (fp32 values held as fp64 on cuda), the fp64 reference and the probe arguments of row r"""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    B, M, K, T = r["B"], r["M"], r["K"], r["frames"]
    pitch = _pitch(T, r["extra_pitch"])
    dev = torch.device(DEV)
    c = dict(pitch=pitch, keep=[])
    W = _rnd(g, M, K, scale=1.0 / math.sqrt(K)).to(dev)
    A = _rnd(g, B, K, T, scale=0.8, shift=0.1).to(dev)
    a = ProbeArgs()
    a.B, a.M, a.K, a.frames, a.pitch = B, M, K, T, pitch

    def dptr(x, dtype=torch.float32):
        x = x.to(device=dev, dtype=dtype).contiguous()
        c["keep"].append(x)
        return x.data_ptr()

    pro = r["pro"]
    if pro == "none":
        P, Pm = PC.pro_none(A)
    elif pro == "prelu":
        P, Pm = PC.pro_prelu(A, 0.25)
        a.pro_slope = dptr(torch.tensor([0.25]))
    elif pro == "dw":
        d = r["d"]
        g1, b1 = _rnd(g, K, scale=0.3, shift=1.0).to(dev), _rnd(g, K, scale=0.1).to(dev)
        wd, bd = _rnd(g, K, 3, scale=0.5).to(dev), _rnd(g, K, scale=0.1).to(dev)
        slope, in_slope = -0.2, (0.3 if r.get("train") else None)
        hin = PC.prelu(A, in_slope) if in_slope is not None else A
        stats = PC.gln_stats(hin)
        P, Pm, pre = PC.pro_dw(A, g1, b1, wd, bd, slope, d, stats, EPS, in_slope)
        c.update(u=P, umag=Pm, pre=pre)
        a.pro_slope = dptr(torch.tensor([slope]))
        a.dw_norm_g, a.dw_norm_b, a.dw_w, a.dw_b = dptr(g1), dptr(b1), dptr(wd), dptr(bd)
        a.dw_stats_in = dptr(stats, torch.float64)
        a.dw_dilation, a.dw_pad_left, a.dw_eps = d, d, EPS
        if in_slope is not None:
            a.dw_in_slope = dptr(torch.tensor([in_slope]))
    elif pro == "res":
        r_ = _rnd(g, B, K, T, scale=2.0).to(dev)
        v1, v2 = _rnd(g, K, scale=0.2).to(dev), _rnd(g, K, scale=0.5).to(dev)
        stats, n = PC.gln_stats(_rnd(g, B, K + 7, T, scale=1.5, shift=0.2).to(dev)), (K + 7) * T
        P, Pm = PC.pro_res(A, r_, v1, v2, stats, n, EPS)
        c.update(xnew=P, xmag=Pm)
        Mt = K + 5
        rr = torch.cat([r_, torch.full((B, Mt - K, T), float("nan"), device=dev, dtype=torch.float64)], 1)
        c["keep"].append(rr_p := _padded(rr, pitch))
        a.res_r, a.res_Mt = rr_p.data_ptr(), Mt
        a.res_v1, a.res_v2, a.res_stats, a.res_n, a.res_eps = dptr(v1), dptr(v2), dptr(stats, torch.float64), float(n), EPS

    epi = r["epi"]
    if epi == "raw":
        fe = PC.epi_raw()
    elif epi == "head":
        v1, v2 = _rnd(g, M, scale=0.2).to(dev), _rnd(g, M, scale=0.5).to(dev)
        stats, n = PC.gln_stats(_rnd(g, B, 64, T, scale=1.2, shift=-0.3).to(dev)), 64 * T
        fe = PC.epi_head(v1, v2, stats, n, EPS)
        a.v1, a.v2, a.stats_in, a.n_in, a.eps = dptr(v1), dptr(v2), dptr(stats, torch.float64), float(n), EPS
    elif epi == "h":
        bias = _rnd(g, M, scale=0.2).to(dev)
        fe = PC.epi_h(bias, 0.25, r.get("store_pre", False))
        a.bias, a.slope, a.store_pre = dptr(bias), dptr(torch.tensor([0.25])), int(r.get("store_pre", False))
    else:
        Nb = r["Nb"]
        bias = _rnd(g, M, scale=0.2).to(dev)
        wenc = _rnd(g, B, Nb, T, scale=1.0).to(dev).abs()
        c["keep"].append(wenc_p := _padded(wenc, pitch))
        a.bias, a.wenc, a.Nb = dptr(bias), wenc_p.data_ptr(), Nb
        if epi == "mask":
            fe = PC.epi_mask(bias, wenc, Nb, r.get("logits", False))
            a.mask_logits = int(r.get("logits", False))
        else:
            dec = _rnd(g, Nb, 16, scale=0.3).to(dev)
            c["T_out"] = 8 * T + 8 - 2 * r["crop"]
            fe = PC.epi_maskdec(bias, wenc, Nb, dec, r["crop"], c["T_out"])
            a.dec_w, a.dec_crop_left, a.dec_T_out = dptr(dec), r["crop"], c["T_out"]
    c["ref"] = PC.Reference(W, P, Pm, fe)
    c["pmax"] = float(P.abs().max())
    c["A"], c["W"] = _padded(A, pitch), W.float().contiguous()
    a.A, a.W = c["A"].data_ptr(), c["W"].data_ptr()
    c["args"] = a
    return c


def _supported(r, mode):
    if r.get("refuse"):
        return False
    if r["epi"] == "maskdec":
        return mode in ("f16x3", "f16x3-low") and r["M"] <= 2048
    if mode == "fp32":
        return (r["pro"], r["epi"]) in SIMT and not r.get("store_pre")
    return True


def _run(c, r, mode, route=0, shift=None):
    """one probe call -> (status, outputs on cuda); shift: f16x3 with the operand scale 2^shift below the top of its range"""
    B, M, K, T, pitch = r["B"], r["M"], r["K"], r["frames"], c["pitch"]
    a = ProbeArgs.from_buffer_copy(c["args"])
    out = {}
    if r["epi"] == "maskdec":
        out["D"] = torch.zeros(B, M // r["Nb"], c["T_out"], device=DEV)
    else:
        out["D"] = torch.full((B, M, pitch), float("nan"), device=DEV)
    a.D = out["D"].data_ptr()
    if r.get("mask_out"):
        out["mask"] = torch.full((B, M, pitch), float("nan"), device=DEV)
        a.mask_out = out["mask"].data_ptr()
    if r["epi"] == "h":
        out["stats"] = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
        a.stats_out = out["stats"].data_ptr()
    if r["pro"] == "dw":
        out["dw_stats"] = torch.zeros(B, 2, dtype=torch.float64, device=DEV)
        a.dw_stats_out = out["dw_stats"].data_ptr()
        if r.get("train"):
            out["upre"] = torch.full((B, K, pitch), float("nan"), device=DEV)
            a.dw_u_pre_out = out["upre"].data_ptr()
    if r["pro"] == "res":
        out["xnew"] = torch.full((B * K + 1, pitch), float("nan"), device=DEV)  # one guard row past the last sample
        a.res_x_out = out["xnew"].data_ptr()
    scale = None
    if mode in ("f16x3", "f16x3-low"):
        # |operand| * s in [2^14, 2^15): the top of the legal range; f16x3-low: 2^-15 of that
        if shift is None:
            shift = 15 if mode == "f16x3-low" else 0
        e = 14 - math.floor(math.log2(c["pmax"])) - shift
        scale = torch.tensor([2.0 ** e], device=DEV)
        a.act_scale = scale.data_ptr()
    nbytes = probe_wimg_bytes(M, K, MATH[mode])
    wimg = torch.full((nbytes // 4 + 64,), float("nan"), device=DEV)
    st = probe_pw(C.byref(a), PRO[r["pro"]], EPI[r["epi"]], MATH[mode], route, wimg.data_ptr(), nbytes,
                  N.stream_ptr(torch.device(DEV)))
    torch.cuda.synchronize()
    return st, out


def _check(name, c, r, mode, out):
    """gate and exactness checks of one run; returns {output: e / bound}"""
    T, ref, res = r["frames"], c["ref"], {}
    for key in ("D", "mask"):
        if key not in out:
            continue
        y = out[key]
        if r["epi"] != "maskdec":
            pad = y[..., T:]
            assert bool((pad == 0).all()), f"{name} {mode}: {key} columns past frames are not 0"
            y = y[..., :T]
        e, b = PC.gate_e(y, ref.out[key]), ref.bound(mode, key)
        res[key] = e / b
        assert e <= b, f"{name} {mode}: {key} e = {e:.3e} > bound {b:.3e} (E_drop {ref.e_drop[key]:.3e}, E_onepass {ref.e_one[key]:.3e})"
    if "stats" in out:
        v = out["D"][..., :T].double()
        if r.get("store_pre"):
            v = PC.prelu(v, 0.25)
        se = PC.stats_error(out["stats"], v, ref.out["act"][2])
        res["stats"] = se
        assert se <= 1.0, f"{name} {mode}: stats_out {se:.2f} of the bound"
    if "dw_stats" in out:
        if "upre" in out:
            up = out["upre"]
            assert bool((up[..., T:] == 0).all()), f"{name} {mode}: dw_u_pre_out past frames is not 0"
            up = up[..., :T].double()
            pre_e = float(((up - c["pre"]).abs() / (c["umag"] + 1e-30)).max())
            res["upre"] = pre_e / (8 * U)
            assert pre_e <= 8 * U, f"{name} {mode}: dw_u_pre_out {pre_e / U:.1f} u"
            u = PC.prelu(up, -0.2)
        else:
            u = c["u"]
        se = PC.stats_error(out["dw_stats"], u, c["umag"])
        res["dw_stats"] = se
        assert se <= 1.0, f"{name} {mode}: dw_stats_out {se:.2f} of the bound"
    if "xnew" in out:
        B, K = r["B"], r["K"]
        xo = out["xnew"]
        assert bool(torch.isnan(xo[B * K]).all()), f"{name} {mode}: res_x_out written past the last channel"
        xo = xo[:B * K].view(B, K, -1)
        assert bool((xo[..., T:] == 0).all()), f"{name} {mode}: res_x_out past frames is not 0"
        xe = float(((xo[..., :T].double() - c["xnew"]).abs() / c["xmag"]).max())
        res["xnew"] = xe / (8 * U)
        assert xe <= 8 * U, f"{name} {mode}: res_x_out {xe / U:.1f} u"
    return res


@pytest.mark.parametrize("name", list(ROWS))
def test_pw_contraction_vs_fp64(name):
    r = ROWS[name]
    c = _case(name, r)
    report, failures = [], []
    for mode in r["modes"]:
        try:
            report.append(f"{mode}: " + _run_mode(name, c, r, mode))
        except AssertionError as ex:  # every mode is run and reported, the row fails at the end
            report.append(f"{mode}: FAILED")
            failures.append(str(ex))
    print(f"{name} [{r['reaches']}] e/bound: " + "; ".join(report) +
          f"  (E_drop {c['ref'].e_drop['D']:.2e}, K = {r['K']})")
    assert not failures, "\n".join(failures)


def _run_mode(name, c, r, mode):
    st, out = _run(c, r, mode)
    if not _supported(r, mode):
        assert st == N.CTN_EUNSUPPORTED, f"{name} {mode}: status {st}, expected CTN_EUNSUPPORTED"
        return "refused"
    assert st == N.CTN_OK, f"{name} {mode}: status {st}"
    res = _check(name, c, r, mode, out)
    if r["epi"] == "maskdec":
        st2, out2 = _run(c, r, mode)
        assert st2 == N.CTN_OK and torch.equal(out2["D"], out["D"]), f"{name} {mode}: second call differs"
    if r["routes"] and mode in ("tf32x3", "f16x3"):
        st1, out1 = _run(c, r, mode, route=1)
        assert st1 == N.CTN_OK and torch.equal(out1["D"], out["D"]), f"{name} {mode}: batched weight image differs"
    return " ".join(f"{k} {v:.3f}" for k, v in res.items())


@pytest.mark.parametrize("name", list(SWEEP_ROWS))
def test_pw_headroom_sweep(name):
    r = SWEEP_ROWS[name]
    c = _case("sweep_" + name, r)
    ratios = {}
    for k in SWEEP_SHIFTS:
        st, out = _run(c, r, "f16x3", shift=k)
        assert st == N.CTN_OK, (name, k, st)
        y = out["D"] if r["epi"] == "maskdec" else out["D"][..., :r["frames"]]
        ratios[k] = PC.gate_e(y, c["ref"].out["D"]) / c["ref"].bound("f16x3")
    broken = [k for k in SWEEP_SHIFTS if ratios[k] > 1.0]
    print(f"sweep {name} [{r['reaches']}]: e/bound " + ", ".join(f"2^-{k}: {v:.3f}" for k, v in ratios.items()) +
          f"; gate breaks at {('2^-%d' % broken[0]) if broken else 'none of these'}")
    assert all(ratios[k] <= 1.0 for k in SWEEP_SHIFTS if k <= SWEEP_REQUIRED), ratios


def test_pw_host_refusals():
    r = ROWS["k33_m129_f128"]
    c = _case("refusals", r)
    bad = ProbeArgs.from_buffer_copy(c["args"])
    bad.pitch = c["pitch"] - 64  # rows 256-byte aligned but pitch % 128 != 0
    wimg = torch.zeros(probe_wimg_bytes(r["M"], r["K"], N.MATH_TF32X3) // 4 + 64, device=DEV)
    D = torch.zeros(r["B"], r["M"], c["pitch"], device=DEV)
    bad.D = D.data_ptr()
    st = probe_pw(C.byref(bad), 0, 0, N.MATH_TF32X3, 0, wimg.data_ptr(), wimg.numel() * 4, N.stream_ptr(torch.device(DEV)))
    assert st == N.CTN_EALIGN
    bad = ProbeArgs.from_buffer_copy(c["args"])
    bad.D = D.data_ptr()
    bad.A = c["A"].data_ptr() + 4  # misaligned activations
    st = probe_pw(C.byref(bad), 0, 0, N.MATH_TF32X3, 0, wimg.data_ptr(), wimg.numel() * 4, N.stream_ptr(torch.device(DEV)))
    assert st == N.CTN_EALIGN
    torch.cuda.synchronize()
    assert bool((D == 0).all()), "a refused call wrote its output"


# ---- weight gradient ---------------------------------------------------------------------------------------------------------
WGRAD_ROWS = {
    "m1_k1_f1": dict(M=1, K=1, B=1, frames=1, split=None, reaches="one element, one partial time chunk"),
    "m33_k144_f31_b5": dict(M=33, K=144, B=5, frames=31, split=None, reaches="K = 144: two k-tiles, frames < one chunk"),
    "m144_k33_f32_split": dict(M=144, K=33, B=1, frames=32, split=96, reaches="split_row 96 of 144, one full chunk"),
    "m144_k144_f33_b5_stride": dict(M=144, K=144, B=5, frames=33, split=96, extra_bs=384,
                                    reaches="batch strides past M pitch, frames one past a chunk"),
    "m33_k1_f1000": dict(M=33, K=1, B=1, frames=1000, split=None, reaches="long reduction split across CTAs"),
    "m144_k144_f800_b5": dict(M=144, K=144, B=5, frames=800, split=96, reaches="B frames = 4000"),
    "m144_k144_f4000_b32": dict(M=144, K=144, B=32, frames=4000, split=None, summation_only=True,
                                reaches="32 x 4000: fp32 summation bound only"),
}


@pytest.mark.parametrize("name", list(WGRAD_ROWS))
def test_wgrad_vs_fp64(name):
    r = WGRAD_ROWS[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    M, K, B, T = r["M"], r["K"], r["B"], r["frames"]
    pitch = _pitch(T)
    dy, x = _rnd(g, B, M, T).to(DEV), _rnd(g, B, K, T, shift=0.2).to(DEV)
    dy_bs, x_bs = M * pitch + r.get("extra_bs", 0), K * pitch + r.get("extra_bs", 0) + 128
    dyb = torch.full((B * dy_bs,), float("nan"), device=DEV)
    xb = torch.full((B * x_bs,), float("nan"), device=DEV)
    for b in range(B):
        dyb[b * dy_bs:b * dy_bs + M * pitch].view(M, pitch)[:, :T] = dy[b].float()
        xb[b * x_bs:b * x_bs + K * pitch].view(K, pitch)[:, :T] = x[b].float()
    ref = torch.einsum("bmt,bkt->mk", dy, x)
    den = torch.einsum("bmt,bkt->mk", dy.abs(), x.abs())
    smag = ref.abs()
    e_drop = PC.gate_e(torch.einsum("bmt,bkt->mk", PC.round_sig(dy), x), (ref, den, smag))
    e_one = PC.gate_e(torch.einsum("bmt,bkt->mk", PC.round_sig(dy), PC.round_sig(x)), (ref, den, smag))
    split = r["split"]
    report = []
    for mode in ("fp32", "tf32x3", "tf32", "f16x3"):
        dWa = torch.zeros(split if split else M, K, device=DEV)
        dWb = torch.zeros(M - split, K, device=DEV) if split else None
        st = probe_wgrad(dyb.data_ptr(), dy_bs, xb.data_ptr(), x_bs, dWa.data_ptr(), N.ptr(dWb), split if split else M, M, K, B, T,
                         pitch, MATH[mode], N.stream_ptr(torch.device(DEV)))
        torch.cuda.synchronize()
        assert st == N.CTN_OK, (name, mode, st)
        dW = torch.cat([dWa, dWb]) if split else dWa
        e = PC.gate_e(dW, (ref, den, smag))
        if mode == "fp32":  # FFMA split-K: one thread's chain of 32 units_per_cta terms, then one fp32 atomic per split
            b = TKR.wgrad_fp32_chain(M, K, B, T, split) * U
        elif r.get("summation_only"):
            b = (B * T + 8) * U
        else:
            b = PC.bound(mode, B * T, e_drop, e_one)
        rho = float((dW.double() - ref).norm() / den.norm())
        report.append(f"{mode}: e/bound {e / b:.3f} rho {rho:.2e}")
        assert e <= b, f"{name} {mode}: e = {e:.3e} > {b:.3e} (E_drop {e_drop:.3e})"
    print(f"wgrad {name} [{r['reaches']}]: " + "; ".join(report) + f"  (E_drop {e_drop:.2e})")
