"""fp64 restatement of DPTNet (reference src/models/dptnet.py, src/models/gtu.py) stage by stage, with seeded weights.

Every stage is written out from its definition, not imported from the reference: encoder, bottleneck 1x1, padding +
Segment1d, gLN over the segmented tensor, per block an intra- and an inter-chunk ImprovedTransformer (x <- gLN_seq(x + MHA(x)),
x <- gLN_seq(x + fc(ReLU(biLSTM(x)))), statistics per sequence), OverlapAdd1d + crop, PReLU, map, GTU1d, the mask
nonlinearity, w * mask and the transposed-conv decoder.  ``defect`` plants one known mistake, so a test can show that the bound
the GPU tests use tells it apart from the right answer.
"""
import math

import torch
import torch.nn.functional as F_

DEFECTS = ("scale_full_width", "residual_after_norm", "per_sample_stats", "relu_in_recurrence", "gtu_swapped", "drop_last_key_tile")


def bound(ref):
    """the bound every GPU comparison of this path uses: |out - fp64| <= 1e-4 max|fp64| + 1e-6"""
    return 1e-4 * float(ref.abs().max()) + 1e-6


def synth_state_dict(keys_shapes, seed):
    """seeded fp32 weights for a list of (key, shape): fan-in scaled normals, norm gains near 1, PReLU slopes near 0.25"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in keys_shapes:
        r = torch.randn(shape, generator=g, dtype=torch.float64)
        if k.endswith("prelu.weight"):
            v = 0.25 + 0.05 * r
        elif ".norm.weight" in k:
            v = 1.0 + 0.1 * r
        elif len(shape) == 1:
            v = 0.1 * r
        else:
            fan_in = 1
            for s in shape[1:]:
                fan_in *= s
            v = r / math.sqrt(fan_in)
        sd[k] = v.float()
    return sd


def gln_seq(x, g, b, eps, defect=None):
    """x (n, T, F): GroupNorm(1, F) per sequence (statistics over T and F)"""
    m = x.mean(dim=(1, 2), keepdim=True)
    v = ((x - m) ** 2).mean(dim=(1, 2), keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * g + b


def mha(x, sd, p, heads, defect=None):
    """nn.MultiheadAttention(F, heads)(x, x, x) on x (n, T, F), batch-first here"""
    n, T, F = x.shape
    d = F // heads
    qkv = x @ sd[p + "in_proj_weight"].double().t() + sd[p + "in_proj_bias"].double()
    q, k, v = qkv.split(F, dim=-1)
    q, k, v = (t.reshape(n, T, heads, d).transpose(1, 2) for t in (q, k, v))
    scale = 1.0 / math.sqrt(F if defect == "scale_full_width" else d)
    s = (q * scale) @ k.transpose(-1, -2)
    if defect == "drop_last_key_tile" and T > 64:
        s[..., 64 * ((T - 1) // 64):] = -math.inf
    o = torch.softmax(s, dim=-1) @ v
    o = o.transpose(1, 2).reshape(n, T, F)
    return o @ sd[p + "out_proj.weight"].double().t() + sd[p + "out_proj.bias"].double()


def lstm_dir(x, wih, whh, bih, bhh, reverse, relu_state=False):
    n, T, _ = x.shape
    H = whh.shape[1]
    h = x.new_zeros(n, H)
    c = x.new_zeros(n, H)
    out = x.new_zeros(n, T, H)
    steps = range(T - 1, -1, -1) if reverse else range(T)
    for t in steps:
        gates = x[:, t] @ wih.t() + bih + h @ whh.t() + bhh
        i, f, gg, o = gates.chunk(4, dim=-1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        if relu_state:
            h = torch.relu(h)
        out[:, t] = h
    return out


def bilstm(x, sd, p, relu_state=False):
    d = lambda k: sd[p + k].double()  # noqa: E731
    hf = lstm_dir(x, d("weight_ih_l0"), d("weight_hh_l0"), d("bias_ih_l0"), d("bias_hh_l0"), False, relu_state)
    hb = lstm_dir(x, d("weight_ih_l0_reverse"), d("weight_hh_l0_reverse"), d("bias_ih_l0_reverse"), d("bias_hh_l0_reverse"), True,
                  relu_state)
    return torch.cat([hf, hb], dim=-1)


def norm_res(y, x, sd, p, eps, defect, n_batch):
    """gLN(y + x) per sequence; the planted defects: the residual after the norm, statistics per sample"""
    g, b = sd[p + "norm.weight"].double(), sd[p + "norm.bias"].double()
    if defect == "residual_after_norm":
        return gln_seq(y, g, b, eps) + x
    if defect == "per_sample_stats":
        z = y + x
        n, T, F = z.shape
        zz = z.reshape(n_batch, -1, T, F)
        m = zz.mean(dim=(1, 2, 3), keepdim=True)
        v = ((zz - m) ** 2).mean(dim=(1, 2, 3), keepdim=True)
        return ((zz - m) / torch.sqrt(v + eps) * g + b).reshape(n, T, F)
    return gln_seq(y + x, g, b, eps)


def mha_block(x, sd, p, heads, eps, defect=None, n_batch=1):
    return norm_res(mha(x, sd, p + "multihead_attn.", heads, defect), x, sd, p + "norm1d.", eps, defect, n_batch)


def ff_block(x, sd, p, eps, defect=None, n_batch=1):
    h = bilstm(x, sd, p + "rnn.", relu_state=defect == "relu_in_recurrence")
    y = torch.relu(h) @ sd[p + "fc.weight"].double().t() + sd[p + "fc.bias"].double()
    return norm_res(y, x, sd, p + "norm1d.", eps, defect, n_batch)


def improved_transformer(x, sd, p, heads, eps, defect=None, n_batch=1):
    """x (n, T, F) batch-first sequences"""
    x = mha_block(x, sd, p + "multihead_attn_block.", heads, eps, defect, n_batch)
    return ff_block(x, sd, p + "subnet.", eps, defect, n_batch)


def dual_path(z, sd, cfg, defect=None):
    """z (B, S, K, F) channels-last through every DualPathTransformerBlock"""
    B, S, K, F = z.shape
    for i in range(cfg["sep_num_blocks"]):
        p = "separator.dptransformer.net.{}.".format(i)
        z = improved_transformer(z.reshape(B * S, K, F), sd, p + "intra_chunk_block.transformer.", cfg["sep_num_heads"], cfg["eps"],
                                 defect, B).reshape(B, S, K, F)
        zt = z.transpose(1, 2).reshape(B * K, S, F)
        zt = improved_transformer(zt, sd, p + "inter_chunk_block.transformer.", cfg["sep_num_heads"], cfg["eps"], defect, B)
        z = zt.reshape(B, K, S, F).transpose(1, 2)
    return z


def segment_geometry(frames, K, P):
    padding = (P - (frames - K) % P) % P
    pl = padding // 2
    return pl, padding - pl, (frames + padding - K) // P + 1


def dptnet_fwd(x, sd, cfg, defect=None):
    """x (B, 1, T) -> (B, n_sources, T), all in fp64"""
    d = lambda k: sd[k].double()  # noqa: E731
    x = x.double()
    B, _, T = x.shape
    L, st = cfg["kernel_size"], cfg["stride"]
    padding = (st - (T - L) % st) % st
    pl0, pr0 = padding // 2, padding - padding // 2
    w = F_.conv1d(F_.pad(x, (pl0, pr0)), d("encoder.conv1d.weight"), stride=st)
    if cfg.get("enc_nonlinear") == "relu":
        w = torch.relu(w)
    frames = w.shape[-1]
    K, P = cfg["sep_chunk_size"], cfg["sep_hop_size"]
    pl, pr, S = segment_geometry(frames, K, P)
    h = F_.conv1d(w, d("separator.bottleneck_conv1d.weight"), d("separator.bottleneck_conv1d.bias"))
    h = F_.pad(h, (pl, pr))
    seg = h.unfold(2, K, P)                                   # (B, F, S, K)
    m = seg.mean(dim=(1, 2, 3), keepdim=True)
    v = ((seg - m) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    seg = (seg - m) / torch.sqrt(v + cfg["eps"]) * d("separator.norm2d.norm.weight").view(1, -1, 1, 1) + \
        d("separator.norm2d.norm.bias").view(1, -1, 1, 1)
    z = dual_path(seg.permute(0, 2, 3, 1), sd, cfg, defect)   # (B, S, K, F)
    Fc = z.shape[-1]
    y = h.new_zeros(B, Fc, (S - 1) * P + K)
    for s in range(S):
        y[:, :, s * P:s * P + K] += z[:, s].transpose(1, 2)
    y = y[:, :, pl:pl + frames]
    a = d("separator.prelu.weight")
    y = torch.where(y >= 0, y, a * y)
    mk = F_.conv1d(y, d("separator.map.weight"), d("separator.map.bias"))
    Nb, ns = cfg["n_basis"], cfg["n_sources"]
    mk = mk.reshape(B * ns, Nb, frames)
    gm, gg = ("map_gate", "map") if defect == "gtu_swapped" else ("map", "map_gate")
    u = torch.tanh(F_.conv1d(mk, d("separator.gtu.{}.weight".format(gm)), d("separator.gtu.{}.bias".format(gm)))) * \
        torch.sigmoid(F_.conv1d(mk, d("separator.gtu.{}.weight".format(gg)), d("separator.gtu.{}.bias".format(gg))))
    mask = torch.relu(u) if cfg["mask_nonlinear"] == "relu" else torch.sigmoid(u)
    what = (w.unsqueeze(1) * mask.reshape(B, ns, Nb, frames)).reshape(B * ns, Nb, frames)
    out = F_.conv_transpose1d(what, d("decoder.conv_transpose1d.weight"), stride=st).reshape(B, ns, -1)
    return out[..., pl0:out.shape[-1] - pr0]
