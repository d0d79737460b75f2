"""fp64 restatement of GALRNet (reference src/models/galrnet.py, src/models/galr.py) stage by stage, with seeded weights.

Every stage is written out from its definition, not imported from the reference: encoder, padding + Segment1d, gLN over the
segmented tensor, per block the intra-chunk DPRNN block (x <- gLN_sample(fc(biLSTM(x))) + x) and the low-dimension globally
attentive block (fc_map along the chunk axis, LayerNorm over channels, positional encoding, attention over the S chunks of each
down-sampled frame + residual, gLN per sample, fc_inv, + the block input), OverlapAdd1d + crop, PReLU, map, GTU1d, the mask
nonlinearity, w * mask and the transposed-conv decoder.  The positional encoding is the reference's fp32 table (formed by its
own expression), taken as an input here.  ``defect`` plants one known mistake, so a test can show that the bound the GPU tests
use tells it apart from the right answer.
"""
import torch
import torch.nn.functional as F_

from dptnet_ref import bilstm, bound, mha, segment_geometry, synth_state_dict  # noqa: F401  (shared with DPTNet)

DEFECTS = ("interleaved_encoding", "exponent_2f", "encoding_before_ln", "ln_over_tokens", "attention_within_chunk", "gln_per_sequence",
           "residual_after_gln", "fc_inv_bias_dropped", "outer_residual_omitted")
# mistakes at the kernels' own edges, planted by tests/tas_galr_edges_ref.py: the gLN eps outside its sqrt, and the down- or
# up-map skipping its last pass of PASS_ELEMS / F rows (the rows keep 0, or the block input where the block runs in place)
EDGE_DEFECTS = ("galr_gln_eps_placement", "galr_down_last_pass_dropped", "galr_up_last_pass_dropped")
PASS_ELEMS = 2048  # k_galr_down / k_galr_up: (256 / F) threads per row x 8 rows, so 2048 / F rows per pass
MHA_ELEMS = 1 << 24  # scores per attention slice: long sequences go through mha in slices of sequences, to bound the memory


def last_pass_start(rows, F):
    return (rows - 1) // (PASS_ELEMS // F) * (PASS_ELEMS // F)


def mha_sliced(z, sd, p, heads):
    """mha over z (n, T, F) in slices of sequences (each sequence is independent)"""
    n, T, _ = z.shape
    step = max(1, MHA_ELEMS // (heads * T * T))
    return torch.cat([mha(z[i:i + step], sd, p, heads) for i in range(0, n, step)])


def pe_table(length, F, defect=None):
    """(length, F) positional encoding of galr.py:61-78 in fp32 as the reference forms it: position / 10000^(j / F), then
    [sin | cos]; returned in fp64"""
    position = torch.arange(length).unsqueeze(1)
    index = torch.arange(F // 2) / F
    if defect == "exponent_2f":
        index = 2 * index
    ind = position / 10000 ** index.unsqueeze(0)
    if defect == "interleaved_encoding":
        return torch.stack([torch.sin(ind), torch.cos(ind)], dim=2).reshape(length, F).double()
    return torch.cat([torch.sin(ind), torch.cos(ind)], dim=1).double()


def intra_block(z, sd, p, eps):
    """IntraChunkRNN (dprnn.py:70-94) on z (B, S, K, F): gLN per sample of fc(biLSTM over K) + z"""
    B, S, K, F = z.shape
    h = bilstm(z.reshape(B * S, K, F), sd, p + "rnn.")
    y = (h @ sd[p + "fc.weight"].double().t() + sd[p + "fc.bias"].double()).reshape(B, S, K, F)
    m = y.mean(dim=(1, 2, 3), keepdim=True)
    v = ((y - m) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    return (y - m) / torch.sqrt(v + eps) * sd[p + "norm1d.norm.weight"].double() + sd[p + "norm1d.norm.bias"].double() + z


def inter_block(x, sd, p, heads, Q, eps, pe=None, defect=None, gn_eps=None):
    """LowDimensionGloballyAttentiveBlock (galr.py:161-197) on x (B, S, K, F) channels-last.  pe: (S*Q, F) encoding (fp64 of
    the fp32 table), formed here when None.  eps is the LayerNorm's; gn_eps the gLN's (eps when None)."""
    d = lambda k: sd[p + k].double()  # noqa: E731
    B, S, K, F = x.shape
    gn_eps = eps if gn_eps is None else gn_eps
    if pe is None:
        pe = pe_table(S * Q, F, defect)
    pe = pe.reshape(S, Q, F)
    z = torch.einsum("bskf,qk->bsqf", x, d("fc_map.weight")) + d("fc_map.bias").view(1, 1, Q, 1)
    if defect == "encoding_before_ln":
        z = z + pe
    dim = 2 if defect == "ln_over_tokens" else 3
    m = z.mean(dim=dim, keepdim=True)
    v = ((z - m) ** 2).mean(dim=dim, keepdim=True)
    z = (z - m) / torch.sqrt(v + eps) * d("norm2d_in.norm.weight") + d("norm2d_in.norm.bias")
    if defect != "encoding_before_ln":
        z = z + pe
    if defect == "galr_down_last_pass_dropped":
        z[:, :, last_pass_start(Q, F):] = 0
    if defect == "attention_within_chunk":
        y = mha_sliced(z.reshape(B * S, Q, F), sd, p + "multihead_attn.", heads).reshape(B, S, Q, F)
    else:
        y = mha_sliced(z.permute(0, 2, 1, 3).reshape(B * Q, S, F), sd, p + "multihead_attn.", heads).reshape(B, Q, S, F).permute(0, 2, 1, 3)
    u = y if defect == "residual_after_gln" else y + z
    dims = (1, 3) if defect == "gln_per_sequence" else (1, 2, 3)
    m = u.mean(dim=dims, keepdim=True)
    v = ((u - m) ** 2).mean(dim=dims, keepdim=True)
    sd_ = torch.sqrt(v) + gn_eps if defect == "galr_gln_eps_placement" else torch.sqrt(v + gn_eps)
    g = (u - m) / sd_ * d("norm2d_out.norm.weight") + d("norm2d_out.norm.bias")
    if defect == "residual_after_gln":
        g = g + z
    out = torch.einsum("bsqf,kq->bskf", g, d("fc_inv.weight"))
    if defect != "fc_inv_bias_dropped":
        out = out + d("fc_inv.bias").view(1, 1, K, 1)
    if defect == "galr_up_last_pass_dropped":
        out[:, :, last_pass_start(K, F):] = 0
    if defect != "outer_residual_omitted":
        out = out + x
    return out


def galr(z, sd, cfg, defect=None):
    """z (B, S, K, F) through every GALRBlock"""
    for i in range(cfg["sep_num_blocks"]):
        p = "separator.galr.net.{}.".format(i)
        z = intra_block(z, sd, p + "intra_chunk_block.", cfg["eps"])
        z = inter_block(z, sd, p + "inter_chunk_block.", cfg["sep_num_heads"], cfg["sep_down_chunk_size"], cfg["eps"], defect=defect)
    return z


def head(w, sd, cfg):
    """pad + Segment1d + gLN over the segmented tensor (galrnet.py:233-239): w (B, F, frames) -> (B, S, K, F)"""
    frames = w.shape[-1]
    K, P = cfg["sep_chunk_size"], cfg["sep_hop_size"]
    pl, pr, S = segment_geometry(frames, K, P)
    seg = F_.pad(w, (pl, pr)).unfold(2, K, P)                      # (B, F, S, K)
    m = seg.mean(dim=(1, 2, 3), keepdim=True)
    v = ((seg - m) ** 2).mean(dim=(1, 2, 3), keepdim=True)
    seg = (seg - m) / torch.sqrt(v + cfg["eps"]) * sd["separator.norm2d.norm.weight"].double().view(1, -1, 1, 1) + \
        sd["separator.norm2d.norm.bias"].double().view(1, -1, 1, 1)
    return seg.permute(0, 2, 3, 1)


def galrnet_fwd(x, sd, cfg, defect=None):
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
    z = galr(head(w, sd, cfg), sd, cfg, defect)               # (B, S, K, F)
    Fc = z.shape[-1]
    y = w.new_zeros(B, Fc, (S - 1) * P + K)
    for s in range(S):
        y[:, :, s * P:s * P + K] += z[:, s].transpose(1, 2)
    y = y[:, :, pl:pl + frames]
    a = d("separator.prelu.weight")
    y = torch.where(y >= 0, y, a * y)
    mk = F_.conv1d(y, d("separator.map.weight"), d("separator.map.bias"))
    Nb, ns = cfg["n_basis"], cfg["n_sources"]
    mk = mk.reshape(B * ns, Nb, frames)
    u = torch.tanh(F_.conv1d(mk, d("separator.gtu.map.weight"), d("separator.gtu.map.bias"))) * \
        torch.sigmoid(F_.conv1d(mk, d("separator.gtu.map_gate.weight"), d("separator.gtu.map_gate.bias")))
    mask = torch.relu(u) if cfg["mask_nonlinear"] == "relu" else torch.sigmoid(u)
    what = (w.unsqueeze(1) * mask.reshape(B, ns, Nb, frames)).reshape(B * ns, Nb, frames)
    out = F_.conv_transpose1d(what, d("decoder.conv_transpose1d.weight"), stride=st).reshape(B, ns, -1)
    return out[..., pl0:out.shape[-1] - pr0]
