"""fp64 restatement of SepFormer (reference src/models/sepformer.py, src/models/transformer.py, src/models/gtu.py) stage by stage,
with seeded weights.

Every stage is written out from its definition, not imported from the reference: encoder, gLN + bottleneck_conv1d_in, padding +
Segment1d, per block an IntraTransformer (sequences = the C frames of a chunk) and an InterTransformer (sequences = the S chunks
of a frame), each being x <- x + (x + pe), post-norm encoder layers (x <- LN(x + MHA(x)), x <- LN(x + W2 ReLU(W1 x))), the final
gLN per sequence and the outer residual (the block input, without the encoding); OverlapAdd1d + crop, PReLU, map, GTU1d,
bottleneck_conv1d_out, the mask nonlinearity, w * mask and the transposed-conv decoder.  ``defect`` plants one known mistake,
so a test can show that the bound the GPU tests use tells it apart from the right answer.
"""
import math

import torch
import torch.nn.functional as F_

DEFECTS = ("pe_not_interleaved", "pe_in_residual", "pre_norm", "final_gln_per_sample", "inter_within_chunk", "skip_bottleneck_out",
           "scale_full_width", "ln_over_tokens")
PE_KEY = "positional_encoding.positional_encoding"


def bound(ref):
    """the bound every GPU comparison of this path uses: |out - fp64| <= 1e-4 max|fp64| + 1e-6"""
    return 1e-4 * float(ref.abs().max()) + 1e-6


def positional_encoding(num_features, max_len=5000, base=10000):
    """the reference's buffer (transformer.py:13-22) with the same fp32 torch operations, so the bits agree: (max_len, 1, F),
    [sin_0, cos_0, sin_1, cos_1, ...] along the features"""
    position = torch.arange(max_len)
    index = torch.arange(0, num_features, 2) / num_features
    indices = position.unsqueeze(dim=1) / (base ** index.unsqueeze(dim=0))
    return torch.stack([torch.sin(indices), torch.cos(indices)], dim=-1).view(max_len, 1, num_features)


def synth_state_dict(keys_shapes, seed):
    """seeded fp32 weights for a list of (key, shape): fan-in scaled normals, norm gains near 1, PReLU slopes near 0.25; the
    positional-encoding buffers are the reference's own, not random"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in keys_shapes:
        if k.endswith(PE_KEY):
            sd[k] = positional_encoding(shape[-1], max_len=shape[0])
            continue
        r = torch.randn(shape, generator=g, dtype=torch.float64)
        if k.endswith("prelu.weight"):
            v = 0.25 + 0.05 * r
        elif k.endswith(("norm.weight", "norm1.weight", "norm2.weight")):
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


def gln_seq(x, g, b, eps):
    """x (n, T, F): GroupNorm(1, F) per sequence (statistics over T and F)"""
    m = x.mean(dim=(1, 2), keepdim=True)
    v = ((x - m) ** 2).mean(dim=(1, 2), keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * g + b


def layer_norm(x, g, b, eps, defect=None):
    """nn.LayerNorm(F) on x (n, T, F); the planted defect normalises over the tokens instead"""
    dim = 1 if defect == "ln_over_tokens" else -1
    m = x.mean(dim=dim, keepdim=True)
    v = ((x - m) ** 2).mean(dim=dim, keepdim=True)
    return (x - m) / torch.sqrt(v + eps) * g + b


def mha(x, sd, p, heads, defect=None):
    """nn.MultiheadAttention(F, heads)(x, x, x) on x (n, T, F), batch-first here"""
    n, T, F = x.shape
    d = F // heads
    qkv = x @ sd[p + "in_proj_weight"].double().t() + sd[p + "in_proj_bias"].double()
    q, k, v = qkv.split(F, dim=-1)
    q, k, v = (t.reshape(n, T, heads, d).transpose(1, 2) for t in (q, k, v))
    scale = 1.0 / math.sqrt(F if defect == "scale_full_width" else d)
    o = torch.softmax((q * scale) @ k.transpose(-1, -2), dim=-1) @ v
    o = o.transpose(1, 2).reshape(n, T, F)
    return o @ sd[p + "out_proj.weight"].double().t() + sd[p + "out_proj.bias"].double()


def encoder_layer(x, sd, p, heads, eps, defect=None):
    """nn.TransformerEncoderLayer(F, heads, d_ff, activation='relu', norm_first=False) in eval mode on x (n, T, F)"""
    d = lambda k: sd[p + k].double()  # noqa: E731
    ln1 = lambda t: layer_norm(t, d("norm1.weight"), d("norm1.bias"), eps, defect)  # noqa: E731
    ln2 = lambda t: layer_norm(t, d("norm2.weight"), d("norm2.bias"), eps, defect)  # noqa: E731
    ff = lambda t: torch.relu(t @ d("linear1.weight").t() + d("linear1.bias")) @ d("linear2.weight").t() + d("linear2.bias")  # noqa: E731
    if defect == "pre_norm":
        x = x + mha(ln1(x), sd, p + "self_attn.", heads, defect)
        return x + ff(ln2(x))
    x = ln1(x + mha(x, sd, p + "self_attn.", heads, defect))
    return ln2(x + ff(x))


def path_transformer(z, sd, p, layers, heads, eps, intra, defect=None):
    """IntraTransformer (intra) / InterTransformer on z (B, F, S, C)"""
    B, F, S, C = z.shape
    within = intra or defect == "inter_within_chunk"
    x = z.permute(0, 2, 3, 1).reshape(B * S, C, F) if within else z.permute(0, 3, 2, 1).reshape(B * C, S, F)
    T = x.shape[1]
    pe = sd[p + PE_KEY].double()[:T, 0, :]
    if defect == "pe_not_interleaved":
        pe = torch.cat([pe[:, 0::2], pe[:, 1::2]], dim=-1)
    residual = x + pe if defect == "pe_in_residual" else x
    x = x + (x + pe)
    for i in range(layers):
        x = encoder_layer(x, sd, p + "transformer.layers.{}.".format(i), heads, eps, defect)
    g, b = sd[p + "transformer.norm.norm1d.norm.weight"].double(), sd[p + "transformer.norm.norm1d.norm.bias"].double()
    if defect == "final_gln_per_sample":
        xx = x.reshape(B, -1, F)
        m = xx.mean(dim=(1, 2), keepdim=True)
        v = ((xx - m) ** 2).mean(dim=(1, 2), keepdim=True)
        x = ((xx - m) / torch.sqrt(v + eps) * g + b).reshape(x.shape)
    else:
        x = gln_seq(x, g, b, eps)
    x = x + residual
    if within:
        return x.reshape(B, S, C, F).permute(0, 3, 1, 2)
    return x.reshape(B, C, S, F).permute(0, 3, 2, 1)


def backbone(z, sd, cfg, defect=None):
    for i in range(cfg["sep_num_blocks"]):
        p = "separator.dptransformer.net.{}.".format(i)
        z = path_transformer(z, sd, p + "intra_transformer.", cfg["sep_num_layers_intra"], cfg["sep_num_heads_intra"], cfg["eps"], True,
                             defect)
        z = path_transformer(z, sd, p + "inter_transformer.", cfg["sep_num_layers_inter"], cfg["sep_num_heads_inter"], cfg["eps"], False,
                             defect)
    return z


def segment_geometry(frames, K, P):
    padding = (P - (frames - K) % P) % P
    pl = padding // 2
    return pl, padding - pl, (frames + padding - K) // P + 1


def sepformer_fwd(x, sd, cfg, defect=None):
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
    m = w.mean(dim=(1, 2), keepdim=True)
    v = ((w - m) ** 2).mean(dim=(1, 2), keepdim=True)
    wn = (w - m) / torch.sqrt(v + cfg["eps"]) * d("separator.norm1d.norm.weight").view(1, -1, 1) + \
        d("separator.norm1d.norm.bias").view(1, -1, 1)
    h = F_.conv1d(wn, d("separator.bottleneck_conv1d_in.weight"), d("separator.bottleneck_conv1d_in.bias"))
    K, P = cfg["sep_chunk_size"], cfg["sep_hop_size"]
    pl, pr, S = segment_geometry(frames, K, P)
    seg = F_.pad(h, (pl, pr)).unfold(2, K, P)                # (B, F, S, K)
    z = backbone(seg, sd, cfg, defect)
    Fc = z.shape[1]
    y = h.new_zeros(B, Fc, (S - 1) * P + K)
    for s in range(S):
        y[:, :, s * P:s * P + K] += z[:, :, s]
    y = y[:, :, pl:pl + frames]
    a = d("separator.prelu.weight")
    y = torch.where(y >= 0, y, a * y)
    mk = F_.conv1d(y, d("separator.map.weight"), d("separator.map.bias"))
    Nb, ns = cfg["n_basis"], cfg["n_sources"]
    mk = mk.reshape(B * ns, Nb, frames)
    u = torch.tanh(F_.conv1d(mk, d("separator.gtu.map.weight"), d("separator.gtu.map.bias"))) * \
        torch.sigmoid(F_.conv1d(mk, d("separator.gtu.map_gate.weight"), d("separator.gtu.map_gate.bias")))
    if defect != "skip_bottleneck_out":
        u = F_.conv1d(u, d("separator.bottleneck_conv1d_out.weight"), d("separator.bottleneck_conv1d_out.bias"))
    mask = torch.relu(u) if cfg["mask_nonlinear"] == "relu" else torch.sigmoid(u)
    what = (w.unsqueeze(1) * mask.reshape(B, ns, Nb, frames)).reshape(B * ns, Nb, frames)
    out = F_.conv_transpose1d(what, d("decoder.conv_transpose1d.weight"), stride=st).reshape(B, ns, -1)
    return out[..., pl0:out.shape[-1] - pr0]
