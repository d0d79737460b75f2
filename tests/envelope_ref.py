"""fp64 reference of the fp16-piece activation envelope (ctn_act_scales, ctn_internal.h) and the checks its results must pass.

Plain torch, no import of the native library: test_act_envelope_cpu.py checks here that the checks accept an fp32 emulation of
k_scale_partials / k_scale_chain and reject its likely regressions, test_act_envelope_gpu.py applies them to what a forward
left in its workspace (ctn_probe_tcn_envelope).

In the f16x3 mode every contraction of the TCN stack meets the tensor core as fp16 pieces hi = fp16(x s), lo = fp16(x s - hi),
with a power-of-two operand scale s chosen per forward from a bound on |x| derived from the weights alone, so that |x s| <= 2^15
and cvt.rn.satfinite never clips.  Per residual block i (R = sqrt(H frames) >= max |gLN-normalised value|):

    |gLN(.)|  <= |gamma| R + |beta|
    vb[n]      = sum_k |W[n][k]| (|gamma_k| R + |beta_k|) + |b_n|                          (row bound of a gLN-folded 1x1 conv)
    U_i        = max(1, |a2|) max_c ((|g1_c| R + |b1_c|) sum_k |wd_ck| + |bd_c|)          (u_i, operand of pw2)
    X_{i+1}    = X_i + max_n vb_out_i[n]                                                   (x_i, operand of pw1)
    S          = sum_i max_n vb_skip_i[n]
    mask bound = max(1, |a_mask|) S                                                        (PReLU(skip sum), mask operand)

X_0 is the head's row bound max_n vb_head[n] with R = sqrt(N frames) (model path), or the measured max |x| (stand-alone TCN).
scales[2i] maps X_i, scales[2i + 1] maps U_i and scales[2n] the mask bound.

Checks (each returns a score, <= 1 passes):
  * scale_score: s is a power of two, s bound64 <= 2^15 (the hard safety property: no fp16 piece can saturate) and s is the
    largest such power of two.  The library computes the bounds in fp32 with R inflated by 1.0001, so a scale one binade
    lower is accepted only where bound64 lies within SLACK(K, n) = 1e-4 + (K + n + 16) u (u = 2^-24) of a power of two:
    1e-4 for the margin on R, K u for the K-term fp32 row sums, n u for the chain of n fp32 additions, 16 u for the rest.
    A zero or non-finite bound must give s = 1.
  * vb_score: vb within [vb64 (1 - t), vb64 (1 + 1e-4 + t)], t = (K + 8) u: the error of its K-term fp32 sum plus the R margin.
  * dwp (the packed depthwise parameters {g1, b1, w0, w1, w2, bd, 0, 0} per channel, zeros for channels [H, ceil16(H))) and
    the measured max |x| are compared bit for bit.
"""
import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24
TOP = 2.0 ** 15
R_MARGIN = 1e-4


def slack(K, n):
    return R_MARGIN + (K + n + 16) * U


def vb(W, b, g, beta, R):
    """row bounds of W gLN(.) + b, fp64"""
    W = W.reshape(W.shape[0], -1).double()
    r = W.abs() @ (g.double().abs() * R + beta.double().abs())
    return r + b.double().abs() if b is not None else r


def u_bound(blk, R):
    a2 = max(1.0, abs(float(blk["a2"])))
    wsum = blk["wd"].double().abs().sum(1)
    return a2 * float(((blk["g1"].double().abs() * R + blk["be1"].double().abs()) * wsum + blk["bd"].double().abs()).max())


def envelope(blocks, H, frames, x0, mask_slope):
    """fp64 bounds [X_0, U_0, X_1, U_1, ..., mask] and the row bounds (vb_out | None, vb_skip) of each block.
    x0: the bound of |x_0|; mask_slope: float or None."""
    R = math.sqrt(H * frames)
    X, S, bounds, vbs = float(x0), 0.0, [], []
    for b in blocks:
        vo = vb(b["Wo"], b["bo"], b["g2"], b["be2"], R) if b["Wo"] is not None else None
        vs = vb(b["Ws"], b["bs"], b["g2"], b["be2"], R)
        bounds += [X, u_bound(b, R)]
        vbs.append((vo, vs))
        if vo is not None:
            X += float(vo.max())
        S += float(vs.max())
    am = max(1.0, abs(float(mask_slope))) if mask_slope is not None else 1.0
    bounds.append(am * S)
    return bounds, vbs


def head_bound(bn_w, bn_b, g0, b0, N, frames):
    """X_0 of the model path: the head's row bounds with R = sqrt(N frames)"""
    return vb(bn_w, bn_b, g0, b0, math.sqrt(N * frames))


def best_scale(bound):
    """the largest power of two s with s bound <= 2^15; 1 for a zero or non-finite bound"""
    if not (bound > 0.0) or not math.isfinite(bound):
        return 1.0
    m, e = math.frexp(bound)  # bound = m 2^e, m in [0.5, 1)
    return 2.0 ** (16 - e) if m == 0.5 else 2.0 ** (15 - e)


def scale_score(s, bound, sl):
    """<= 1 passes (see the module docstring); also returns s / best_scale(bound), the scale's ratio to fp64"""
    s = float(s)
    ratio = s / best_scale(bound)
    m, _ = math.frexp(s) if s > 0 else (0.0, 0)
    if not (s > 0.0) or m != 0.5:
        return math.inf, ratio
    if not (bound > 0.0) or not math.isfinite(bound):
        return (0.0 if s == 1.0 else math.inf), ratio
    over = s * bound / TOP - 1.0
    under = (TOP / 2) / (s * bound) - 1.0
    if over > 0.0:
        return 1.0 + over / sl, ratio
    return max(under / sl, 0.0), ratio


def vb_score(got, ref, K):
    """<= 1 passes: worst deviation of the row bounds from [ref (1 - t), ref (1 + 1e-4 + t)], in units of t ref"""
    got, ref = got.double().cpu(), ref.double().cpu()
    t = (K + 8) * U
    zero = ref == 0
    if bool((got[zero] != 0).any()):
        return math.inf
    rel = got[~zero] / ref[~zero] - 1.0
    if rel.numel() == 0:
        return 0.0
    return float(torch.maximum(rel - R_MARGIN, -rel).max()) / t


def dwp_pack(blk, H):
    """{g1, b1, w0, w1, w2, bd, 0, 0} per channel for P = 3, zero rows for [H, ceil16(H)): float32 (ceil16(H), 8)"""
    Hp = (H + 15) // 16 * 16
    d = torch.zeros(Hp, 8, dtype=torch.float32)
    wd = blk["wd"].float().cpu()
    d[:H, 0], d[:H, 1], d[:H, 5] = blk["g1"].float().cpu(), blk["be1"].float().cpu(), blk["bd"].float().cpu()
    d[:H, 2:5] = wd
    return d


# ---- fp64 forward of the stack: the operands of the fp16-piece contractions ----------------------------------------------------
def gln(x, g, b, eps):
    return F.group_norm(x, 1, g.double(), b.double(), eps)


def prelu(x, a):
    return torch.where(x >= 0, x, float(a) * x)


def tcn_forward(x, blocks, dilations, eps, keep=()):
    """fp64 forward of a run of residual blocks (ResidualBlock1d, non-causal gLN).  Returns dict: xmax[i] = max |x_i| and
    umax[i] = max |u_i| (the operands of pw1 / pw2 of block i), skip (sum of the skip heads), x_out (after the last block with an
    out head), and x[i] / u[i] for i in keep."""
    x = x.double()
    res = dict(xmax=[], umax=[], x={}, u={})
    skip = 0.0
    for i, (b, d) in enumerate(zip(blocks, dilations)):
        P = b["wd"].shape[1]
        res["xmax"].append(float(x.abs().max()))
        if i in keep:
            res["x"][i] = x
        h = prelu(torch.einsum("hc,bct->bht", b["W1"].double(), x) + b["b1"].double().view(1, -1, 1), b["a1"])
        hn = gln(h, b["g1"], b["be1"], eps)
        pl = ((P - 1) * d) // 2
        u = F.conv1d(F.pad(hn, (pl, (P - 1) * d - pl)), b["wd"].double().unsqueeze(1), b["bd"].double(), dilation=d,
                     groups=hn.shape[1])
        u = prelu(u, b["a2"])
        res["umax"].append(float(u.abs().max()))
        if i in keep:
            res["u"][i] = u
        un = gln(u, b["g2"], b["be2"], eps)
        skip = skip + torch.einsum("sh,bht->bst", b["Ws"].double(), un) + b["bs"].double().view(1, -1, 1)
        if b["Wo"] is not None:
            x = x + torch.einsum("ch,bht->bct", b["Wo"].double(), un) + b["bo"].double().view(1, -1, 1)
        del h, hn, u, un
    res["skip"], res["x_out"] = skip, x
    return res


def block_prefixes(num_blocks, num_layers, prefix="separator.tdcn."):
    return [f"{prefix}net.{r}.net.{l}." for r in range(num_blocks) for l in range(num_layers)]


def blocks_of(sd, prefixes):
    """the residual blocks of an oracle-style state dict (convtasnet_oracle.state_dict_spec names), one per prefix -> [dict]"""
    out = []
    for p in prefixes:
        q = p + "separable_conv1d."
        o = sd.get(q + "output_pointwise_conv1d.weight")
        out.append(dict(
            W1=sd[p + "bottleneck_conv1d.weight"].squeeze(-1), b1=sd[p + "bottleneck_conv1d.bias"], a1=float(sd[p + "nonlinear1d.weight"]),
            g1=sd[p + "norm1d.norm.weight"], be1=sd[p + "norm1d.norm.bias"],
            wd=sd[q + "depthwise_conv1d.weight"].squeeze(1), bd=sd[q + "depthwise_conv1d.bias"], a2=float(sd[q + "nonlinear1d.weight"]),
            g2=sd[q + "norm1d.norm.weight"], be2=sd[q + "norm1d.norm.bias"],
            Wo=None if o is None else o.squeeze(-1), bo=sd.get(q + "output_pointwise_conv1d.bias"),
            Ws=sd[q + "skip_pointwise_conv1d.weight"].squeeze(-1), bs=sd[q + "skip_pointwise_conv1d.bias"]))
    return out
