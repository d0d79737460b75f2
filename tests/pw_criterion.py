"""fp64 references and the accuracy gate of the 1x1 contraction kernels (ctn_pw: k_pw_wgmma / k_pw_simt; ctn_wgrad_wgmma).

Plain torch on the CPU, no import of the native library: test_pw_contraction_cpu.py checks here that the gate accepts the
kernel's arithmetic and rejects its likely regressions, test_pw_contraction_gpu.py applies it to the kernels.

Every prologue / epilogue below returns, next to its fp64 value, a magnitude: the same expression evaluated on absolute values
with every subtraction turned into an addition.  For an output element,

    den = |W| . |pro(A)|  pushed through the epilogue the same way (plus |bias| and the folded shifts' magnitudes),

so |D - D64| / den is the error of that element relative to the size of the terms that produced it, whatever the cancellation.
The sigmoid epilogues are linearised: their den carries sigmoid'(logit), the factor by which they scale a logit's error.
Each element may also deviate by SLACK_ULPS ulps of the epilogue's own magnitude (its fp32 rounding, which no accuracy of the
contraction can remove), and

    e = max over elements of  max(|D - D64| - SLACK_ULPS u smag, 0) / den.

What e must satisfy depends on the mode (bound()):
  tf32x3 / f16x3: e <= E_drop / GATE_DIV, where E_drop is e of an fp64 evaluation on the same data with W rounded to 11
    significant bits, i.e. with the hi.lo product of the 3-pass split dropped.  A row scaling by a power of two leaves
    significands alone, so the same emulation stands for the tf32 and the fp16 pieces.  Normwise, a correct 3-pass
    contraction sits 19x or more below the dropped-piece one even with a truncating fp32 accumulator (DESIGN section 2).
  tf32 (one pass): e <= ONEPASS_MUL * E_onepass, E_onepass = e with both W and pro(A) rounded to 11 significant bits.
  fp32 (FFMA): e <= (K + 8) u, the forward error bound of a K-term fp32 dot product plus the epilogue.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -24
GATE_DIV = 8.0
ONEPASS_MUL = 2.0
SLACK_ULPS = 8.0
STATS_ULPS = 64.0
PIECE_BITS = 11


def round_sig(x, bits=PIECE_BITS):
    """x rounded to nearest at `bits` significant bits (fp64)"""
    m, e = torch.frexp(x)
    s = float(2 ** bits)
    return torch.ldexp(torch.round(m * s) / s, e)


def prelu(x, a):
    return torch.where(x >= 0, x, a * x)


def gln_stats(x):
    """(B, 2) float64 (sum, sum of squares) of each sample of x (B, C, T)"""
    x = x.double()
    return torch.stack([x.sum(dim=(1, 2)), (x * x).sum(dim=(1, 2))], dim=1)


def mean_rstd(stats, n, eps):
    """gln_mean_rstd (ctn_common.cuh) in fp64 -> (mean, rstd), each (B, 1, 1)"""
    mean = stats[:, 0] / n
    var = (stats[:, 1] / n - mean * mean).clamp_min(0.0)
    return mean.view(-1, 1, 1), (1.0 / torch.sqrt(var + eps)).view(-1, 1, 1)


# ---- prologues: (B, K, T) -> (P, |P| bound) -------------------------------------------------------------------------------
def pro_none(A):
    return A, A.abs()


def pro_prelu(A, a):
    P = prelu(A, a)
    return P, P.abs()


def pro_dw(h, g1, b1, w, bd, slope, d, stats, eps, in_slope=None):
    """PReLU(dwconv3_d(gLN1(h)) + bd), pad_left = d, zero outside [0, T).  in_slope: h is a pre-activation, PReLU on load.
    Returns (u, |u| bound, pre-activation)."""
    if in_slope is not None:
        h = prelu(h, in_slope)
    K = h.shape[1]
    mean, rstd = mean_rstd(stats, K * h.shape[2], eps)
    hn = (h - mean) * rstd * g1.view(1, -1, 1) + b1.view(1, -1, 1)
    hm = (h.abs() + mean.abs()) * rstd * g1.abs().view(1, -1, 1) + b1.abs().view(1, -1, 1)
    pre = F.conv1d(F.pad(hn, (d, d)), w.view(K, 1, 3), bd, dilation=d, groups=K)
    mag = F.conv1d(F.pad(hm, (d, d)), w.abs().view(K, 1, 3), bd.abs(), dilation=d, groups=K)
    return prelu(pre, slope), mag * max(1.0, abs(slope)), pre


def pro_res(x, r, v1, v2, stats, n, eps):
    """x_new = x + rstd r + (v1 - mean rstd v2): the previous block's deferred residual update"""
    mean, rstd = mean_rstd(stats, n, eps)
    xn = x + rstd * r + (v1.view(1, -1, 1) - mean * rstd * v2.view(1, -1, 1))
    mag = x.abs() + rstd * r.abs() + v1.abs().view(1, -1, 1) + mean.abs() * rstd * v2.abs().view(1, -1, 1)
    return xn, mag


# ---- epilogues: (Z = W P, Zm = |W| |P|) -> {output: (value, den, smag)} ------------------------------------------------------
def epi_raw():
    return lambda Z, Zm: {"D": (Z, Zm, Z.abs())}


def epi_head(v1, v2, stats, n, eps):
    def f(Z, Zm):
        mean, rstd = mean_rstd(stats, n, eps)
        D = rstd * Z + (v1.view(1, -1, 1) - mean * rstd * v2.view(1, -1, 1))
        den = rstd * Zm + v1.abs().view(1, -1, 1) + mean.abs() * rstd * v2.abs().view(1, -1, 1)
        return {"D": (D, den, D.abs())}
    return f


def epi_h(bias, slope, store_pre=False):
    """PReLU(Z + bias), or Z + bias itself (store_pre); "act" is what the gLN statistics sum"""
    def f(Z, Zm):
        pre = Z + bias.view(1, -1, 1)
        lm = Zm + bias.abs().view(1, -1, 1)
        act = prelu(pre, slope)
        if store_pre:
            return {"D": (pre, lm, pre.abs()), "act": (act, lm, act.abs())}
        lm = lm * max(1.0, abs(slope))
        return {"D": (act, lm, act.abs()), "act": (act, lm, act.abs())}
    return f


def _per_basis(wenc, M, Nb):
    return wenc[:, torch.arange(M, device=wenc.device) % Nb, :]


def epi_mask(bias, wenc, Nb, logits=False):
    """sigmoid(Z + bias) * wenc[n % Nb] (and the mask itself), or the logits"""
    def f(Z, Zm):
        logit = Z + bias.view(1, -1, 1)
        lm = Zm + bias.abs().view(1, -1, 1)
        if logits:
            return {"D": (logit, lm, logit.abs()), "mask": (logit, lm, logit.abs())}
        s = torch.sigmoid(logit)
        sp = s * (1.0 - s)
        wn = _per_basis(wenc, Z.shape[1], Nb)
        return {"D": (s * wn, wn.abs() * sp * lm, (s * wn).abs()), "mask": (s, sp * lm, s)}
    return f


def epi_maskdec(bias, wenc, Nb, dec_w, crop_left, T_out):
    """ConvTranspose1d(Nb, 1, 16, stride 8) of sigmoid(Z + bias) * wenc per source, then the crop [crop_left, crop_left + T_out)"""
    def f(Z, Zm):
        B, M, T = Z.shape
        S = M // Nb
        logit = Z + bias.view(1, -1, 1)
        lm = Zm + bias.abs().view(1, -1, 1)
        s = torch.sigmoid(logit)
        wn = _per_basis(wenc, M, Nb)

        def dec(x, wd):
            y = F.conv_transpose1d(x.reshape(B * S, Nb, T), wd.view(Nb, 1, 16), stride=8).view(B, S, -1)
            y = F.pad(y, (0, max(0, crop_left + T_out - y.shape[-1])))
            return y[..., crop_left:crop_left + T_out]
        o = s * wn
        return {"D": (dec(o, dec_w), dec(wn.abs() * s * (1.0 - s) * lm, dec_w.abs()), dec(o.abs(), dec_w.abs()))}
    return f


# ---- evaluation -------------------------------------------------------------------------------------------------------------
def contract(W, P, Pm, epi):
    return epi(torch.einsum("nk,bkt->bnt", W, P), torch.einsum("nk,bkt->bnt", W.abs(), Pm))


def gate_e(D, ref):
    """e of D against ref = (D64, den, smag); inf when D has a non-finite element or misses where den == 0"""
    D64, den, smag = ref
    D = D.double()
    if not bool(torch.isfinite(D).all()):
        return math.inf
    err = ((D - D64).abs() - SLACK_ULPS * U * smag).clamp_min(0.0)
    r = torch.where(den > 0, err / den.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


class Reference:
    """fp64 outputs of one contraction and the gate's yardsticks E_drop / E_onepass per output"""

    def __init__(self, W, P, Pm, epi):
        self.K = W.shape[1]
        self.out = contract(W, P, Pm, epi)
        W11 = round_sig(W)
        drop = contract(W11, P, Pm, epi)
        one = contract(W11, round_sig(P), Pm, epi)
        self.e_drop = {k: gate_e(drop[k][0], v) for k, v in self.out.items()}
        self.e_one = {k: gate_e(one[k][0], v) for k, v in self.out.items()}

    def bound(self, mode, key="D"):
        return bound(mode, self.K, self.e_drop[key], self.e_one[key])


def bound(mode, K, e_drop, e_one):
    if mode == "fp32":
        return (K + 8) * U
    if mode == "tf32":
        return ONEPASS_MUL * e_one
    return e_drop / GATE_DIV


def stats_error(got, vals, mags):
    """worst |stats - fp64 sums| / (STATS_ULPS u sum|.|) over the (sum, sum of squares) of each sample; <= 1 passes.
    vals: (B, ...) the values the kernel summed (its own output, fp64); mags: their magnitude bounds."""
    got = got.double().cpu()
    v = vals.double().cpu().flatten(1)
    m = torch.maximum(mags.double().cpu().flatten(1), v.abs())
    ref = torch.stack([v.sum(1), (v * v).sum(1)], 1)
    tol = STATS_ULPS * U * torch.stack([m.sum(1), (m * m).sum(1)], 1) + 1e-300
    return float(((got - ref).abs() / tol).max())


# ---- emulation of the tensor-core arithmetic (numpy, bit level) ------------------------------------------------------------
def _bits(x):
    return np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)


def tf32_rna(x):
    """cvt.rna.tf32.f32: nearest, ties away, at 10 explicit mantissa bits (weight pieces)"""
    return ((_bits(x) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_trunc(x):
    """the tensor core's reading of an fp32 operand as tf32: low 13 mantissa bits dropped"""
    return (_bits(x) & np.uint32(0xFFFFE000)).view(np.float32)


def f32_rz(x64):
    """fp64 -> fp32 rounded toward zero (a truncating accumulator, the pessimistic reading)"""
    f = x64.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x64)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def emulate_3xtf32(W, A, drop_w_lo=False, drop_a_lo=False, single_pass_from=None):
    """D = W A as k_pw_wgmma computes it in the tf32x3 mode: per k8 step, hi.hi, lo.hi (A_lo), hi.lo (W_lo) in that order, each
    an exact 8-term product sum added to the fp32 accumulator with truncation.  W (M, K), A (K, T) float32.
    single_pass_from: k from which only hi.hi is computed (a slab that lost its split passes)."""
    M, K = W.shape
    Kp = -(-K // 32) * 32
    Wp = np.zeros((M, Kp), np.float32)
    Wp[:, :K] = W
    Ap = np.zeros((Kp, A.shape[1]), np.float32)
    Ap[:K] = A
    Wh = tf32_rna(Wp)
    Wl = tf32_rna(Wp - Wh)
    Ah = tf32_rna(Ap)  # hi_tf32: the same rounding as cvt.rna
    Al = tf32_trunc(Ap - Ah)
    Wh, Wl, Ah, Al = (x.astype(np.float64) for x in (Wh, Wl, Ah, Al))
    acc = np.zeros((M, A.shape[1]), np.float32)
    for k0 in range(0, Kp, 8):
        sl = slice(k0, k0 + 8)
        passes = [(Wh, Ah)]
        full = single_pass_from is None or k0 < single_pass_from
        if full and not drop_a_lo:
            passes.append((Wh, Al))
        if full and not drop_w_lo:
            passes.append((Wl, Ah))
        for w, a in passes:
            acc = f32_rz(acc.astype(np.float64) + w[:, sl] @ a[sl])
    return acc
