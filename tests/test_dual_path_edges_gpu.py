"""The stage entries of DPTNet, SepFormer and LSTM-TasNet one at a time, and the DPTNet and SepFormer models, at their edges
against fp64 (tests/dual_path_edges_ref.py, dptnet_ref, sepformer_ref): every padding remainder of the hop, hops that equal,
divide or do not divide the chunk, a hop past the chunk, 1 to 4 sources, odd crops, every numeric mode, 1, 3 and 65 encoder
layers, sequences of exactly 5000 chunks, softmax logits that overflow expf without the max subtraction, digital silence, a
CUDA-graph replay, a reference checkpoint, and the attention past 65535 sequences (DPTNet at B = 4097, a GALR block at
B Q > 65535).  Every entry call runs twice on outputs and workspaces pre-filled with NaN and must give the same bits; every
bound is taken per sample, per source or per sequence."""
import os

import pytest
import torch

import dptnet_ref
import dual_path_edges_ref as R
import galrnet_ref
import sepformer_ref
from ctn_b200 import _native as N
from ctn_b200.models.dptnet import DPTNet
from ctn_b200.models.sepformer import SepFormer

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
EPS = 1e-12
MODES = ("fp32", "tf32", "tf32x3", "f16x3")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DPT_GOLD = torch.load(os.path.join(GOLDEN, "dptnet.pt"), weights_only=False)
SFM_GOLD = torch.load(os.path.join(GOLDEN, "sepformer.pt"), weights_only=False)


def nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def nan_ws(nbytes):
    buf = torch.full(((int(nbytes) + 512) // 4 + 1,), float("nan"), dtype=torch.float32, device=DEV).view(torch.uint8)
    return N.aligned(buf), buf


def st():
    return N.stream_ptr(DEV)


def twice(run, shapes, nbytes):
    """run(outs, base, nbytes) -> status, twice on fresh NaN outputs and a fresh NaN workspace; the two results must agree bit for
    bit.  Returns the first call's outputs (on the host) and its launch count."""
    results, counts = [], []
    for _ in range(2):
        outs = [nan(*s) for s in shapes]
        (base, nb), keep = nan_ws(nbytes)
        N.check(run(outs, base, nb), "entry")
        counts.append(N.ctn_last_launch_count())
        torch.cuda.synchronize()
        results.append([o.cpu() for o in outs])
        del keep
    for a, b in zip(*results):
        assert torch.equal(a, b)
    assert counts[0] == counts[1]
    return results[0], counts[0]


def dev(t):
    return t.contiguous().to(DEV)


# ---- ctn_dpt_head_fwd ---------------------------------------------------------------------------------------------------------------
def _head_cases():
    cases = []
    for K, P in ((16, 8), (16, 16), (16, 24)):               # every padding remainder at the small geometries, hop past the chunk
        cases += [(3, 32, K, P, K + j) for j in range(P)]
    cases += [(1, 64, 16, 8, 40), (3, 128, 16, 16, 47)]
    cases += [(1, 64, 100, 30, f) for f in (100, 101, 115, 129, 250)] + [(3, 128, 100, 30, 131)]
    cases += [(1, 64, 250, 125, f) for f in (250, 251, 300, 374)] + [(3, 32, 250, 125, 600), (3, 128, 250, 125, 375)]
    return cases


@pytest.mark.parametrize("B,Bc,K,P,frames", _head_cases())
def test_dpt_head_against_fp64(B, Bc, K, P, frames):
    Nb = 64
    pitch = N.ctn_pitch(frames)
    pl, pr, S = R.segment_geometry(frames, K, P)
    w = R.pitched(B, Nb, frames, pitch, frames + K)
    p = R.dpt_head_params(Nb, Bc, Bc + P)
    d = {k: dev(v) for k, v in p.items()}
    wd = dev(w)
    ref = R.dpt_head(w[..., :frames], p["bn_w"], p["bn_b"], p["g"], p["b"], K, P, pl, pr, EPS)
    for mode in MODES:
        run = lambda o, base, nb: N.ctn_dpt_head_fwd(wd.data_ptr(), d["bn_w"].data_ptr(), d["bn_b"].data_ptr(), d["g"].data_ptr(),  # noqa: E731
                                                     d["b"].data_ptr(), o[0].data_ptr(), B, Nb, Bc, frames, pitch, K, P, pl, pr, EPS,
                                                     N.MATH_NAMES[mode], base, nb, st())
        (z,), _ = twice(run, [(B, S, K, Bc)], N.ctn_dpt_head_workspace_bytes(B, Nb, Bc, pitch, S, K))
        R.check(z, ref, 2, R.rel_of(mode))


# ---- ctn_dpt_tail_fwd ---------------------------------------------------------------------------------------------------------------
TAIL = [(n_src, MODES[i], (n_src + i) % 2, i % 2) for n_src in (1, 2, 3, 4) for i in range(4)]


@pytest.mark.parametrize("n_src,mode,mask_relu,latent", TAIL)
def test_dpt_tail_against_fp64(n_src, mode, mask_relu, latent):
    B, Nb, Bc, frames, L, stride, crop = 2, 64, 32, 37, 4, 2, 1
    pitch = N.ctn_pitch(frames)
    T = (frames - 1) * stride + L - 3                          # odd, and cropped on both sides
    y = R.pitched(B, Bc, frames, pitch, 20 + n_src)
    w = R.pitched(B, Nb, frames, pitch, 30 + n_src, pad="random")   # the pad columns of w must not reach what
    p = R.dpt_tail_params(Nb, Bc, n_src, L, 40 + n_src)
    d = {k: dev(v) for k, v in p.items()}
    yd, wd = dev(y), dev(w)
    shapes = [(B, n_src, T), (B, n_src * Nb, pitch)] + ([(B, n_src, Nb, frames)] if latent else [])

    def run(o, base, nb):
        return N.ctn_dpt_tail_fwd(yd.data_ptr(), wd.data_ptr(), *[d[k].data_ptr() for k in R.DPT_TAIL_ORDER], o[0].data_ptr(),
                                  o[2].data_ptr() if latent else None, o[1].data_ptr(), B, Nb, Bc, n_src, frames, pitch, L, stride, crop,
                                  T, mask_relu, N.MATH_NAMES[mode], base, nb, st())
    outs, _ = twice(run, shapes, N.ctn_dpt_tail_workspace_bytes(B, Nb, Bc, n_src, pitch))
    ref_out, ref_what = R.dpt_tail(y, w, p, n_src, mask_relu, stride, crop, T, frames)
    what = outs[1].reshape(B, n_src, Nb, pitch)
    assert not what[..., frames:].any()
    rel = R.rel_of(mode)
    R.check(what, ref_what, 2, rel)
    R.check(outs[0], ref_out, 2, rel)
    if latent:
        assert torch.equal(outs[2], what[..., :frames])


def test_dpt_tail_refuses_too_many_rows_before_launch():
    B, n_src, Nb, Bc, frames, L, stride = 16384, 4, 8, 8, 8, 2, 1  # B * n_src = 65536
    pitch = N.ctn_pitch(frames)
    T = (frames - 1) * stride + L
    y, w = torch.zeros(B, Bc, pitch, device=DEV), torch.zeros(B, Nb, pitch, device=DEV)
    out, what = torch.zeros(B, n_src, T, device=DEV), torch.zeros(B, n_src * Nb, pitch, device=DEV)
    p = {k: dev(v) for k, v in R.dpt_tail_params(Nb, Bc, n_src, L, 1).items()}
    ws = torch.empty(N.ctn_dpt_tail_workspace_bytes(B, Nb, Bc, n_src, pitch) + 256, dtype=torch.uint8, device=DEV)
    base, nb = N.aligned(ws)
    torch.cuda.synchronize()
    n0 = N.ctn_total_launch_count()
    rc = N.ctn_dpt_tail_fwd(y.data_ptr(), w.data_ptr(), *[p[k].data_ptr() for k in R.DPT_TAIL_ORDER], out.data_ptr(), None, what.data_ptr(),
                            B, Nb, Bc, n_src, frames, pitch, L, stride, 0, T, 1, N.MATH_NAMES["fp32"], base, nb, st())
    assert rc == N.CTN_EUNSUPPORTED
    assert N.ctn_total_launch_count() == n0


# ---- ctn_sfm_segment_fwd / ctn_sfm_overlap_add_fwd ----------------------------------------------------------------------------------
def _ola_cases():
    cases = []
    for K, P in ((16, 8), (16, 16), (16, 5), (16, 24)):
        cases += [(K, P, K + j) for j in range(P)]
    return cases + [(100, 30, f) for f in (100, 101, 115, 129, 250)] + [(250, 125, f) for f in (250, 251, 374, 1000)]


@pytest.mark.parametrize("K,P,frames", _ola_cases())
def test_sfm_segment_and_overlap_add_exact(K, P, frames):
    """segmentation is a copy: bit for bit; the overlap-add is the fp32 sum of the covering chunks in ascending s, from 0, which a
    CPU fp32 loop in the same order reproduces bit for bit"""
    B, Fc = 2, 8
    pitch = N.ctn_pitch(frames)
    pl, pr, S = R.segment_geometry(frames, K, P)
    zp = N.ctn_pitch(S * K)
    x = R.pitched(B, Fc, frames, pitch, frames, pad="random")    # the pad columns of x must not reach Z
    xd = dev(x)
    (Z,), n = twice(lambda o, base, nb: N.ctn_sfm_segment_fwd(xd.data_ptr(), o[0].data_ptr(), B, Fc, frames, pitch, K, P, pl, pr, zp, st()),
                    [(B, Fc, zp)], 0)
    assert n == 1
    assert torch.equal(Z, R.sfm_segment(x[..., :frames], K, P, pl, pr, zp))
    Zin = torch.randn(B, Fc, zp, generator=torch.Generator().manual_seed(K + P))
    Zin[..., S * K:] = float("nan")                              # past the chunks: must not be read
    Zd = dev(Zin)
    (y,), n = twice(lambda o, base, nb: N.ctn_sfm_overlap_add_fwd(Zd.data_ptr(), o[0].data_ptr(), B, Fc, S, K, P, zp, pl, frames, pitch,
                                                                  st()), [(B, Fc, pitch)], 0)
    assert n == 1
    assert torch.equal(y, R.sfm_overlap_add(Zin, S, K, P, pl, frames, pitch))


# ---- ctn_sfm_pos_enc_fwd ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("intra", [1, 0])
@pytest.mark.parametrize("S,C", [(3, 16), (1, 1), (2, 250), (5000, 1), (1, 5000), (7, 3)])
def test_sfm_pos_enc_exact(S, C, intra):
    B, Fc = 2, 32
    pitch = N.ctn_pitch(S * C)
    pe = sepformer_ref.positional_encoding(Fc)
    X = R.pitched(B, Fc, S * C, pitch, S + C)
    Xd, ped = dev(X), dev(pe)
    (out,), n = twice(lambda o, base, nb: N.ctn_sfm_pos_enc_fwd(Xd.data_ptr(), ped.data_ptr(), o[0].data_ptr(), B, Fc, S, C, pitch, intra,
                                                                st()), [(B, Fc, pitch)], 0)
    assert n == 1
    assert torch.equal(out, R.sfm_pos_enc(X, pe, S, C, intra))
    if (C if intra else S) == 5000:                              # the buffer's last row is read
        x = X[..., S * C - 1]
        assert torch.equal(out[..., S * C - 1], x + (x + pe[4999, 0]))


def test_sfm_pos_enc_refuses_past_the_buffer():
    B, Fc = 1, 32
    pe = dev(sepformer_ref.positional_encoding(Fc))
    for S, C, intra in ((1, 5001, 1), (5001, 1, 0)):
        pitch = N.ctn_pitch(S * C)
        X, out = torch.zeros(B, Fc, pitch, device=DEV), torch.zeros(B, Fc, pitch, device=DEV)
        torch.cuda.synchronize()
        n0 = N.ctn_total_launch_count()
        assert N.ctn_sfm_pos_enc_fwd(X.data_ptr(), pe.data_ptr(), out.data_ptr(), B, Fc, S, C, pitch, intra, st()) == N.CTN_EINVAL
        assert N.ctn_total_launch_count() == n0


# ---- ctn_sfm_transformer_fwd --------------------------------------------------------------------------------------------------------
# (B, F, heads, d_ff, layers, S, C, intra, mode)
TRANSFORMER = [
    (2, 64, 8, 100, 1, 3, 16, 1, "fp32"), (2, 64, 8, 100, 1, 3, 16, 0, "tf32x3"),
    (1, 64, 1, 96, 3, 5, 7, 1, "f16x3"), (3, 64, 1, 96, 3, 5, 7, 0, "fp32"),
    (2, 32, 4, 48, 3, 1, 9, 1, "tf32"), (2, 32, 4, 48, 3, 1, 9, 0, "f16x3"),       # S = 1
    (2, 32, 4, 48, 3, 9, 1, 1, "tf32x3"), (2, 32, 4, 48, 3, 9, 1, 0, "tf32"),      # C = 1
    (1, 32, 4, 48, 65, 2, 3, 1, "tf32x3"), (1, 32, 4, 48, 65, 2, 3, 0, "f16x3"),   # past the 64-layer batch of weight images
    (1, 32, 4, 48, 65, 2, 3, 1, "fp32"),
    (1, 32, 1, 64, 1, 5000, 2, 0, "tf32x3"),                                        # an inter sequence of exactly 5000 chunks
]


@pytest.mark.parametrize("B,F,heads,d_ff,layers,S,C,intra,mode", TRANSFORMER)
def test_sfm_transformer_against_fp64(B, F, heads, d_ff, layers, S, C, intra, mode):
    sd = R.transformer_sd(F, d_ff, layers, F + layers + S)
    ptr_keys = [k for k, _ in R.transformer_keys(F, d_ff, layers)]
    w = {k: dev(v) for k, v in sd.items()}
    ptrs = (N._fp * len(ptr_keys))(*[w[k].data_ptr() for k in ptr_keys])
    pitch = N.ctn_pitch(S * C)
    X = R.pitched(B, F, S * C, pitch, S * C + layers)
    Xd = dev(X)
    math_ = N.MATH_NAMES[mode]
    run = lambda o, base, nb: N.ctn_sfm_transformer_fwd(Xd.data_ptr(), o[0].data_ptr(), ptrs, B, F, heads, d_ff, layers, S, C, pitch,  # noqa: E731
                                                        intra, EPS, math_, base, nb, st())
    (out,), n = twice(run, [(B, F, pitch)], N.ctn_sfm_transformer_workspace_bytes(B, F, d_ff, layers, pitch, math_))
    # the weight images go in batches of up to 64 layers, 48 images per launch
    imgs = 0 if mode == "fp32" else sum(-(-4 * min(64, layers - l0) // 48) for l0 in range(0, layers, 64))
    assert n == 7 * layers + 2 + imgs
    assert torch.equal(Xd.cpu(), X)                              # the outer residual is read, never written
    assert not out[..., S * C:].any()
    ref = R.sfm_transformer(X, sd, S, C, layers, heads, EPS, intra)
    R.check(R.sequences(out, S, C, intra), R.sequences(ref, S, C, intra), 2, R.rel_of(mode))


# ---- ctn_tas_tail_fwd ---------------------------------------------------------------------------------------------------------------
TAS = [(n_src, 1, mode) for n_src in (1, 2, 3, 4) for mode in MODES] + [(2, 0, mode) for mode in MODES]


@pytest.mark.parametrize("n_src,softmax,mode", TAS)
def test_tas_tail_against_fp64(n_src, softmax, mode):
    """logits near 90 (expf overflows without the max subtraction), except in the single-pass tf32 mode, whose logit error at that
    size is not inside any useful bound"""
    B, Nb, Hd, frames, L, stride, crop = 2, 32, 32, 37, 4, 2, 1
    pitch = N.ctn_pitch(frames)
    T = (frames - 1) * stride + L - 3
    skip = R.pitched(B, Hd, frames, pitch, 12)
    w = R.pitched(B, Nb, frames, pitch, 9 + n_src, pad="random")
    p = R.tas_tail_params(Nb, Hd, n_src, L, 13, logit_scale=1.0 if mode == "tf32" else 30.0)
    d = {k: dev(v) for k, v in p.items()}
    sd_, wd = dev(skip), dev(w)
    run = lambda o, base, nb: N.ctn_tas_tail_fwd(sd_.data_ptr(), wd.data_ptr(), d["fc_w"].data_ptr(), d["fc_b"].data_ptr(),  # noqa: E731
                                                 d["dec_w"].data_ptr(), o[0].data_ptr(), o[2].data_ptr(), o[1].data_ptr(), B, Nb, Hd,
                                                 n_src, frames, pitch, L, stride, crop, T, softmax, N.MATH_NAMES[mode], base, nb, st())
    outs, _ = twice(run, [(B, n_src, T), (B, n_src * Nb, pitch), (B, n_src, Nb, frames)],
                    N.ctn_tas_tail_workspace_bytes(Nb, Hd, n_src, N.MATH_NAMES[mode]))
    what = outs[1].reshape(B, n_src, Nb, pitch)
    assert not what[..., frames:].any()
    assert torch.equal(outs[2], what[..., :frames])
    if softmax and n_src == 1:                                   # a softmax over one source is exactly 1
        assert torch.equal(what[:, 0, :, :frames], w[..., :frames])
    ref_out, ref_what = R.tas_tail(skip, w, p["fc_w"], p["fc_b"], p["dec_w"], n_src, softmax, stride, crop, T, frames)
    rel = R.rel_of(mode)
    R.check(what, ref_what, 2, rel)
    R.check(outs[0], ref_out, 2, rel)


# ---- the attention past 65535 sequences ---------------------------------------------------------------------------------------------
def test_mha_past_65535_sequences():
    NSEQ, T, F, heads = 70001, 3, 32, 4
    w = {k: dev(v) for k, v in dptnet_ref.synth_state_dict([("in_proj_weight", (3 * F, F)), ("in_proj_bias", (3 * F,)),
                                                            ("out_proj.weight", (F, F)), ("out_proj.bias", (F,))], 5).items()}
    z = torch.randn(NSEQ, T, F, generator=torch.Generator().manual_seed(6))
    zd = dev(z)
    run = lambda o, base, nb: N.ctn_mha_fwd(zd.data_ptr(), NSEQ, T, F, heads, w["in_proj_weight"].data_ptr(), w["in_proj_bias"].data_ptr(),  # noqa: E731
                                            w["out_proj.weight"].data_ptr(), w["out_proj.bias"].data_ptr(), o[0].data_ptr(), base, nb, st())
    (y,), n = twice(run, [(NSEQ, T, F)], N.ctn_mha_workspace_bytes(NSEQ, T, F))
    assert n == 3
    ref = dptnet_ref.mha(z.double(), {k: v.cpu() for k, v in w.items()}, "", heads)
    R.check(y, ref, 1)


def test_galr_inter_block_past_the_old_limit():
    """B Q = 65568 attention sequences, B <= 65535"""
    B, S, K, Q, F, heads = 2049, 2, 40, 32, 32, 4
    keys = [("fc_map.weight", (Q, K)), ("fc_map.bias", (Q,)), ("norm2d_in.norm.weight", (F,)), ("norm2d_in.norm.bias", (F,)),
            ("multihead_attn.in_proj_weight", (3 * F, F)), ("multihead_attn.in_proj_bias", (3 * F,)),
            ("multihead_attn.out_proj.weight", (F, F)), ("multihead_attn.out_proj.bias", (F,)), ("norm2d_out.norm.weight", (F,)),
            ("norm2d_out.norm.bias", (F,)), ("fc_inv.weight", (K, Q)), ("fc_inv.bias", (K,))]
    sd = galrnet_ref.synth_state_dict(keys, 3)
    w = {k: dev(v) for k, v in sd.items()}
    div = (10000 ** (torch.arange(F // 2) / F)).to(DEV)
    x = torch.randn(B, S, K, F, generator=torch.Generator().manual_seed(7))
    xd = dev(x)
    ptrs = [w[k].data_ptr() for k, _ in keys]

    def run(o, base, nb):
        return N.ctn_galr_inter_fwd(xd.data_ptr(), *ptrs[:4], div.data_ptr(), heads, *ptrs[4:], o[0].data_ptr(), B, S, K, Q, F, EPS, EPS,
                                    base, nb, st())
    (out,), n = twice(run, [(B, S, K, F)], N.ctn_galr_inter_workspace_bytes(B, S, K, Q, F))
    assert n == 6
    ref = galrnet_ref.inter_block(x.double(), sd, "", heads, Q, EPS, pe=galrnet_ref.pe_table(S * Q, F))
    R.check(out, ref, 1)


# ---- whole models -------------------------------------------------------------------------------------------------------------------
def dptnet_of(case, **over):
    g = DPT_GOLD[case]
    c = dict(g["cfg"], **over)
    m = DPTNet(c["n_basis"], c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable",
               enc_nonlinear=c["enc_nonlinear"], sep_bottleneck_channels=c["sep_bottleneck_channels"],
               sep_hidden_channels=c["sep_hidden_channels"], sep_chunk_size=c["sep_chunk_size"], sep_hop_size=c["sep_hop_size"],
               sep_num_blocks=c["sep_num_blocks"], sep_num_heads=c["sep_num_heads"], mask_nonlinear=c["mask_nonlinear"], causal=False,
               n_sources=c["n_sources"], eps=c["eps"])
    sd = dptnet_ref.synth_state_dict(g["keys_shapes"], c["seed"])
    m.load_state_dict(sd)
    return m.to(DEV).eval(), sd, c, dptnet_ref.dptnet_fwd


def sepformer_of(case, **over):
    g = SFM_GOLD[case]
    c = dict(g["cfg"], **over)
    m = SepFormer(c["n_basis"], c["kernel_size"], enc_basis="trainable", dec_basis="trainable", causal=False,
                  **{k: c[k] for k in ("stride", "enc_nonlinear", "sep_bottleneck_channels", "sep_chunk_size", "sep_hop_size", "sep_num_blocks",
                                       "sep_num_layers_intra", "sep_num_layers_inter", "sep_num_heads_intra", "sep_num_heads_inter",
                                       "sep_d_ff_intra", "sep_d_ff_inter", "mask_nonlinear", "n_sources", "eps")})
    sd = sepformer_ref.synth_state_dict(g["keys_shapes"], c["seed"])
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval(), sd, c, sepformer_ref.sepformer_fwd


MODELS = {"dptnet": dptnet_of, "sepformer": sepformer_of}


def samples_for(c, frames):
    return (frames - 1) * c["stride"] + c["kernel_size"]


def run_model(m, x):
    with torch.no_grad():
        out = m(x.to(DEV))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("math", [None, "fp32", "tf32x3"])
@pytest.mark.parametrize("r", range(8))
@pytest.mark.parametrize("model", sorted(MODELS))
def test_tiny_model_every_padding_remainder(model, r, math):
    """tiny config, chunk 16, hop 8: 100 + r frames give every padding remainder of the segmentation"""
    m, sd, c, fwd = MODELS[model]("tiny")
    m.math = math
    x = torch.randn(2, 1, samples_for(c, 100 + r), generator=torch.Generator().manual_seed(r))
    R.check(run_model(m, x), fwd(x, sd, c), 2)


@pytest.mark.parametrize("hop,frames", [(16, 50), (16, 63), (4, 50), (4, 63), (6, 50), (6, 63)])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_tiny_model_other_hops(model, hop, frames):
    """sep_hop_size equal to the chunk of 16, a quarter of it, and 6, which does not divide it"""
    m, sd, c, fwd = MODELS[model]("tiny", sep_hop_size=hop)
    x = torch.randn(2, 1, samples_for(c, frames), generator=torch.Generator().manual_seed(hop + frames))
    R.check(run_model(m, x), fwd(x, sd, c), 2)


@pytest.mark.parametrize("case", ["tiny", "recipe_2spk"])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_model_silence_is_exactly_zero(model, case):
    """w = 0 makes every output 0 unless a NaN arose in the separator (NaN * 0 = NaN)"""
    m, _, c, _ = MODELS[model](case)
    out = run_model(m, torch.zeros(2, 1, samples_for(c, 700)))
    assert torch.equal(out, torch.zeros_like(out))


def test_dptnet_cuda_graph_replay_matches_eager():
    m, sd, c, _ = dptnet_of("tiny")
    x = torch.randn(2, 1, 401, generator=torch.Generator().manual_seed(4)).to(DEV)
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.no_grad(), torch.cuda.stream(s):
        eager = m(x)  # warm-up on the capture stream: the workspaces exist before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = m(x)
    torch.cuda.current_stream(DEV).wait_stream(s)
    x.copy_(torch.randn(2, 1, 401, generator=torch.Generator().manual_seed(5)).to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = m(x)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    assert not torch.equal(out, eager)
    R.check(out, dptnet_ref.dptnet_fwd(x.cpu(), sd, c), 2)


def test_dptnet_reference_checkpoint_loads(tmp_path):
    """a checkpoint as the reference's trainer writes it: its get_config() keys plus the state_dict, through build_model"""
    g = DPT_GOLD["tiny"]
    c = g["cfg"]
    sd = dptnet_ref.synth_state_dict(g["keys_shapes"], c["seed"])
    ckpt = {"n_basis": c["n_basis"], "kernel_size": c["kernel_size"], "stride": c["stride"], "enc_basis": "trainable",
            "dec_basis": "trainable", "enc_nonlinear": c["enc_nonlinear"], "window_fn": None, "enc_onesided": None,
            "enc_return_complex": None, "sep_hidden_channels": c["sep_hidden_channels"],
            "sep_bottleneck_channels": c["sep_bottleneck_channels"], "sep_chunk_size": c["sep_chunk_size"],
            "sep_hop_size": c["sep_hop_size"], "sep_num_blocks": c["sep_num_blocks"], "sep_num_heads": c["sep_num_heads"],
            "sep_norm": True, "sep_nonlinear": "relu", "sep_dropout": 0.1, "mask_nonlinear": c["mask_nonlinear"], "causal": False,
            "n_sources": c["n_sources"], "eps": c["eps"], "state_dict": sd}
    path = str(tmp_path / "best.pth")
    torch.save(ckpt, path)
    m = DPTNet.build_model(path, load_state_dict=True).to(DEV).eval()
    R.check(run_model(m, g["x"]), dptnet_ref.dptnet_fwd(g["x"], sd, c), 2)


def test_dptnet_past_65535_attention_sequences():
    """B = 4097, 24 frames: 2 chunks of 16, so the inter path attends over B * 16 = 65552 sequences; samples are independent, so
    the fp64 reference runs on the first and the last"""
    m, sd, c, _ = dptnet_of("tiny")
    B, frames = 4097, 24
    assert B * c["sep_chunk_size"] > 65535 and R.segment_geometry(frames, c["sep_chunk_size"], c["sep_hop_size"])[2] == 2
    x = torch.randn(B, 1, samples_for(c, frames), generator=torch.Generator().manual_seed(8))
    out = run_model(m, x)
    ends = [0, B - 1]
    R.check(out[ends], dptnet_ref.dptnet_fwd(x[ends], sd, c), 2)


def test_sepformer_at_the_encodings_length():
    """5000 chunks (the positional encoding's rows) run and stay finite; 5001 raise ValueError before any launch"""
    m, _, c, _ = sepformer_of("tiny")
    K, P = c["sep_chunk_size"], c["sep_hop_size"]
    frames = 4999 * P + K
    assert R.segment_geometry(frames, K, P)[2] == 5000
    x = torch.randn(1, 1, samples_for(c, frames), generator=torch.Generator().manual_seed(1))
    out = run_model(m, x)
    assert torch.isfinite(out).all() and out.abs().max() > 0
    x = torch.randn(1, 1, samples_for(c, frames + P)).to(DEV)
    torch.cuda.synchronize()
    n0 = N.ctn_total_launch_count()
    with torch.no_grad(), pytest.raises(ValueError):
        m(x)
    assert N.ctn_total_launch_count() == n0
