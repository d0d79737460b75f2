"""fp64 (and, where the kernel is a copy or a plain sum, exact fp32) restatements of the stage entries of DPTNet, SepFormer and
LSTM-TasNet that the edge tests call one at a time: DPTNet's head (bottleneck 1x1, pad, Segment1d, gLN per sample over the
segmented tensor) and tail (PReLU, map, GTU1d, mask, w * mask, decoder); SepFormer's segmentation, overlap-add and positional
encoding on the pitched channel-first layout, and one Intra/InterTransformer through ``sepformer_ref.path_transformer``;
LSTM-TasNet's tail (fc, the mask over the sources, w * mask, decoder).  The model-level and attention references stay in
``dptnet_ref``, ``sepformer_ref`` and ``lstm_tasnet_ref``.

Every comparison is held to the paths' bound, 1e-4 max|fp64| + 1e-6, taken per unit (a sample, a (sample, source) pair or a
sequence), so a loud unit in the batch cannot hide an error in a quiet one.  ``defect`` plants one known mistake per stage, so a
CPU test can show the bound tells it apart from the right answer at the shapes the GPU tests use.
"""
import math

import torch
import torch.nn.functional as F_

import sepformer_ref

BOUND_REL, BOUND_ABS = 1e-4, 1e-6
TF32_REL = 1e-2  # the single tf32 pass (mode 'tf32'): the looser bound of the LSTM-TasNet model test
DEFECTS = ("pad_split_swapped", "ola_drop_last_chunk", "pe_row_shifted", "head_gln_without_padding", "layers_past_64_from_layer_0",
           "softmax_without_max", "mask_on_pad_columns")
PE_ROWS = 5000


def unit_errors(out, ref, lead):
    """per unit (the first `lead` dims flattened): the largest |out - ref| (infinite where out is not finite) and the bound"""
    o, r = out.double().cpu(), ref.double().cpu()
    assert o.shape == r.shape, (o.shape, r.shape)
    n = math.prod(r.shape[:lead])
    err = (o - r).abs().reshape(n, -1)
    err[~torch.isfinite(err)] = math.inf
    return err.max(dim=1).values, r.abs().reshape(n, -1).max(dim=1).values


def excess(out, ref, lead, rel=BOUND_REL):
    """the worst unit's error over its bound: <= 1 passes"""
    err, mx = unit_errors(out, ref, lead)
    return float((err / (rel * mx + BOUND_ABS)).max())


def check(out, ref, lead, rel=BOUND_REL):
    err, mx = unit_errors(out, ref, lead)
    ratio = err / (rel * mx + BOUND_ABS)
    worst = int(ratio.argmax())
    assert float(ratio[worst]) <= 1.0, ("unit", worst, float(err[worst]), rel * float(mx[worst]) + BOUND_ABS)


def rel_of(math_name):
    return TF32_REL if math_name == "tf32" else BOUND_REL


def segment_geometry(frames, K, P):
    """the padding rule of dptnet.py / sepformer.py -> (pad_left, pad_right, S)"""
    padding = (P - (frames - K) % P) % P
    pl = padding // 2
    return pl, padding - pl, (frames + padding - K) // P + 1


# ---- DPTNet head / tail ------------------------------------------------------------------------------------------------------------
def dpt_head(w, bn_w, bn_b, g, b, K, P, pl, pr, eps, defect=None):
    """w (B, N, frames) -> z (B, S, K, Bc): gLN per sample over Segment1d(pad(Wb w + bb)), overlap duplicates and padding zeros
    in the statistics (dptnet.py:334-337)"""
    if defect == "pad_split_swapped":
        pl, pr = pr, pl
    h = F_.conv1d(w.double(), bn_w.double().unsqueeze(-1), bn_b.double())
    frames = h.shape[-1]
    seg = F_.pad(h, (pl, pr)).unfold(2, K, P)                  # (B, Bc, S, K)
    if defect == "head_gln_without_padding":
        real = F_.pad(torch.ones(frames, dtype=torch.float64), (pl, pr)).unfold(0, K, P).bool()   # (S, K)
        vals = seg[:, :, real]                                                                      # (B, Bc, n real)
        m = vals.mean(dim=(1, 2)).view(-1, 1, 1, 1)
        v = ((vals - m.view(-1, 1, 1)) ** 2).mean(dim=(1, 2)).view(-1, 1, 1, 1)
    else:
        m = seg.mean(dim=(1, 2, 3), keepdim=True)
        v = ((seg - m) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    z = (seg - m) / torch.sqrt(v + eps) * g.double().view(1, -1, 1, 1) + b.double().view(1, -1, 1, 1)
    return z.permute(0, 2, 3, 1)


def _finish_tail(w, mask, n_src, dec_w, stride, crop_left, T, frames, defect):
    """w (B, N, pitch), mask (B, n_src, N, pitch) -> out (B, n_src, T), what (B, n_src, N, pitch) with its pad columns zero"""
    B, Nb, pitch = w.shape
    what = w.double().unsqueeze(1) * mask
    if defect != "mask_on_pad_columns":
        what[..., frames:] = 0
    full = F_.conv_transpose1d(what[..., :frames].reshape(B * n_src, Nb, frames), dec_w.double(), stride=stride).reshape(B, n_src, -1)
    return full[..., crop_left:crop_left + T], what


def dpt_tail(y, w, p, n_src, mask_relu, stride, crop_left, T, frames, defect=None):
    """y (B, Bc, pitch) with zero pad columns, w (B, N, pitch) (its pad columns may hold anything), p = the tail's weights by name
    (prelu, map_w, map_b, gtu_w, gtu_b, gate_w, gate_b, dec_w) -> out (B, n_src, T), what (B, n_src, N, pitch)"""
    d = {k: v.double() for k, v in p.items()}
    B, Nb, pitch = w.shape
    yy = y.double()
    yy = torch.where(yy >= 0, yy, d["prelu"] * yy)
    m = F_.conv1d(yy, d["map_w"].unsqueeze(-1), d["map_b"]).reshape(B * n_src, Nb, pitch)
    u = torch.tanh(F_.conv1d(m, d["gtu_w"].unsqueeze(-1), d["gtu_b"])) * torch.sigmoid(F_.conv1d(m, d["gate_w"].unsqueeze(-1), d["gate_b"]))
    mask = (torch.relu(u) if mask_relu else torch.sigmoid(u)).reshape(B, n_src, Nb, pitch)
    return _finish_tail(w, mask, n_src, d["dec_w"], stride, crop_left, T, frames, defect)


# ---- LSTM-TasNet tail ----------------------------------------------------------------------------------------------------------------
def tas_tail(skip, w, fc_w, fc_b, dec_w, n_src, softmax, stride, crop_left, T, frames, defect=None):
    """skip (B, Hd, pitch) with zero pad columns, w (B, N, pitch) -> out (B, n_src, T), what (B, n_src, N, pitch): fc (row s N + n),
    then softmax over the sources or sigmoid (tasnet.py:365-381).  The planted defect takes the softmax without subtracting the
    max, in fp32 as a kernel would: logits near 90 overflow expf."""
    B, Nb, pitch = w.shape
    y = (fc_w.double() @ skip.double() + fc_b.double().view(-1, 1)).reshape(B, n_src, Nb, pitch)
    if not softmax:
        mask = torch.sigmoid(y)
    elif defect == "softmax_without_max":
        e = torch.exp(y.float())
        mask = (e / e.sum(dim=1, keepdim=True)).double()
    else:
        mask = torch.softmax(y, dim=1)
    return _finish_tail(w, mask, n_src, dec_w, stride, crop_left, T, frames, defect)


# ---- SepFormer stages on the pitched channel-first layout ---------------------------------------------------------------------------
def sfm_segment(x, K, P, pl, pr, z_pitch, defect=None):
    """x (B, F, frames) -> Z (B, F, z_pitch), Z[b][f][s K + k] = the zero-padded x at frame s P + k - pad_left; a copy, so exact"""
    if defect == "pad_split_swapped":
        pl, pr = pr, pl
    seg = F_.pad(x, (pl, pr)).unfold(2, K, P)                  # (B, F, S, K)
    B, Fc, S, _ = seg.shape
    Z = torch.zeros(B, Fc, z_pitch, dtype=x.dtype)
    Z[..., :S * K] = seg.reshape(B, Fc, S * K)
    return Z


def sfm_overlap_add(Z, S, K, P, crop_left, T_out, out_pitch, defect=None):
    """Z (B, F, z_pitch) fp32 -> y (B, F, out_pitch): each output frame the fp32 sum of its chunks' values, s ascending, from 0"""
    B, Fc, _ = Z.shape
    y = torch.zeros(B, Fc, (S - 1) * P + K, dtype=torch.float32)
    for s in range(S - 1 if defect == "ola_drop_last_chunk" else S):
        y[..., s * P:s * P + K] += Z[..., s * K:(s + 1) * K].float()
    out = torch.zeros(B, Fc, out_pitch, dtype=torch.float32)
    out[..., :T_out] = y[..., crop_left:crop_left + T_out]
    return out


def sfm_pos_enc(X, pe, S, C, intra, defect=None):
    """X (B, F, pitch) fp32, pe (5000, 1, F) -> X + (X + pe[pos]) in fp32 at token s C + k, pos = k (intra) or s (inter); pad 0"""
    B, Fc, pitch = X.shape
    tok = torch.arange(S * C)
    pos = tok % C if intra else tok // C
    if defect == "pe_row_shifted":
        pos = pos + 1
    e = pe.float()[:, 0, :][pos.clamp(max=pe.shape[0] - 1)].t()    # (F, S C)
    x = X[..., :S * C].float()
    out = torch.zeros(B, Fc, pitch, dtype=torch.float32)
    out[..., :S * C] = x + (x + e)
    return out


def transformer_keys(F, d_ff, layers):
    """the keys of one Intra/InterTransformer in the order of the entry's pointer array: 12 per layer, the encoding, the final gLN"""
    ks = []
    for i in range(layers):
        q = "transformer.layers.{}.".format(i)
        ks += [(q + "self_attn.in_proj_weight", (3 * F, F)), (q + "self_attn.in_proj_bias", (3 * F,)),
               (q + "self_attn.out_proj.weight", (F, F)), (q + "self_attn.out_proj.bias", (F,)), (q + "linear1.weight", (d_ff, F)),
               (q + "linear1.bias", (d_ff,)), (q + "linear2.weight", (F, d_ff)), (q + "linear2.bias", (F,)),
               (q + "norm1.weight", (F,)), (q + "norm1.bias", (F,)), (q + "norm2.weight", (F,)), (q + "norm2.bias", (F,))]
    return ks + [(sepformer_ref.PE_KEY, (PE_ROWS, 1, F)), ("transformer.norm.norm1d.norm.weight", (F,)),
                 ("transformer.norm.norm1d.norm.bias", (F,))]


IMAGED = ("self_attn.in_proj_weight", "self_attn.out_proj.weight", "linear1.weight", "linear2.weight")


def sfm_transformer(X, sd, S, C, layers, heads, eps, intra, defect=None):
    """X (B, F, pitch) -> out (B, F, pitch) of one Intra/InterTransformer (sepformer_ref.path_transformer), pad columns zero.
    The planted defect runs the layers from 64 on with layer 0's four contraction weights (the batched weight images)."""
    if defect == "layers_past_64_from_layer_0":
        sd = dict(sd)
        for i in range(64, layers):
            for k in IMAGED:
                sd["transformer.layers.{}.{}".format(i, k)] = sd["transformer.layers.0." + k]
    B, Fc, pitch = X.shape
    z = X[..., :S * C].double().reshape(B, Fc, S, C)
    y = sepformer_ref.path_transformer(z, sd, "", layers, heads, eps, bool(intra))
    out = torch.zeros(B, Fc, pitch, dtype=torch.float64)
    out[..., :S * C] = y.reshape(B, Fc, S * C)
    return out


def sequences(X, S, C, intra):
    """(B, F, pitch) -> (B, nseq, len, F): the sequences of the path, for per-sequence bounds"""
    B, Fc, _ = X.shape
    z = X[..., :S * C].reshape(B, Fc, S, C)
    return z.permute(0, 2, 3, 1) if intra else z.permute(0, 3, 2, 1)


# ---- seeded inputs the CPU and the GPU tests share -----------------------------------------------------------------------------
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def pitched(B, C, frames, pitch, seed, pad=0.0):
    """(B, C, pitch) normals in the first `frames` columns, `pad` (a number, or 'random') in the rest"""
    g = _gen(seed)
    x = torch.randn(B, C, pitch, generator=g)
    if pad != "random":
        x[..., frames:] = pad
    return x


def dpt_head_params(N, Bc, seed):
    g = _gen(seed)
    return {"bn_w": torch.randn(Bc, N, generator=g) / math.sqrt(N), "bn_b": 0.1 * torch.randn(Bc, generator=g),
            "g": 1 + 0.1 * torch.randn(Bc, generator=g), "b": 0.1 * torch.randn(Bc, generator=g)}


def dpt_tail_params(N, Bc, n_src, L, seed):
    g = _gen(seed)
    r = lambda *s: torch.randn(*s, generator=g)  # noqa: E731
    return {"prelu": 0.25 + 0.05 * r(1), "map_w": r(n_src * N, Bc) / math.sqrt(Bc), "map_b": 0.1 * r(n_src * N),
            "gtu_w": r(N, N) / math.sqrt(N), "gtu_b": 0.1 * r(N), "gate_w": r(N, N) / math.sqrt(N), "gate_b": 0.1 * r(N),
            "dec_w": r(N, 1, L) / math.sqrt(N)}


DPT_TAIL_ORDER = ("prelu", "map_w", "map_b", "gtu_w", "gtu_b", "gate_w", "gate_b", "dec_w")


def tas_tail_params(N, Hd, n_src, L, seed, logit_scale=1.0):
    """fc scaled so the logits reach about logit_scale * 3 in magnitude (skip of unit variance)"""
    g = _gen(seed)
    return {"fc_w": logit_scale * torch.randn(n_src * N, Hd, generator=g) / math.sqrt(Hd),
            "fc_b": 0.1 * torch.randn(n_src * N, generator=g), "dec_w": torch.randn(N, 1, L, generator=g) / math.sqrt(N)}


def transformer_sd(F, d_ff, layers, seed):
    return sepformer_ref.synth_state_dict(transformer_keys(F, d_ff, layers), seed)
