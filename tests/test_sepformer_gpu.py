"""SepFormer on the GPU against fp64 (tests/sepformer_ref.py) and the reference's goldens: the attention, token LayerNorm,
per-sequence norm + residual and tail entries on their own (outputs and workspaces pre-filled with NaN), the whole model in every
1x1 numeric mode; edge lengths, every head dimension, B = 1 and 3, a single chunk, inputs scaled by 1e-3 and 1e3; a reference
checkpoint through build_model; a repeated call bit for bit; the launches each call makes; one CUDA-graph capture."""
import math
import os

import pytest
import torch
import torch.nn.functional as F_

import sepformer_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.sepformer import SepFormer

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sepformer.pt"), weights_only=False)
DEV = torch.device("cuda", 0)


def nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device=DEV)


def nan_ws(nbytes):
    buf = torch.full(((int(nbytes) + 512) // 4 + 1,), float("nan"), dtype=torch.float32, device=DEV).view(torch.uint8)
    return N.aligned(buf), buf


def st():
    return N.stream_ptr(DEV)


def check(out, ref):
    err = float((out.double().cpu() - ref).abs().max())
    assert err <= R.bound(ref), (err, R.bound(ref))


def seqs(X, S, C, intra):
    """(B, F, pitch) -> (B * nseq, len, F) sequences of the path, in fp64 on the CPU"""
    B, F, _ = X.shape
    z = X[:, :, :S * C].double().cpu().reshape(B, F, S, C)
    return z.permute(0, 2, 3, 1).reshape(B * S, C, F) if intra else z.permute(0, 3, 2, 1).reshape(B * C, S, F)


def unseqs(x, B, F, S, C, intra):
    return (x.reshape(B, S, C, F).permute(0, 3, 1, 2) if intra else x.reshape(B, C, S, F).permute(0, 3, 2, 1)).reshape(B, F, S * C)


@pytest.mark.parametrize("intra", [1, 0])
@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 127, 128, 129, 250, 640, 2000])
@pytest.mark.parametrize("F,heads", [(64, 8), (64, 4), (64, 2), (64, 1), (256, 8)])
def test_attention_against_fp64(T, F, heads, intra):
    if T >= 640 and (F, heads) not in ((64, 4), (256, 8)):
        pytest.skip("long sequences at the recipe's and one other head dimension")
    B, other = (2, 3) if T < 640 else (1, 2)
    S, C = (other, T) if intra else (T, other)
    pitch = N.ctn_pitch(S * C)
    g = torch.Generator().manual_seed(T + heads)
    qkv = torch.randn(B, 3 * F, pitch, generator=g).to(DEV)
    in_b = (0.1 * torch.randn(3 * F, generator=g)).to(DEV)
    outs = []
    for _ in range(2):
        O = nan(B, F, pitch)
        N.check(N.ctn_sfm_attn_fwd(qkv.data_ptr(), in_b.data_ptr(), O.data_ptr(), B, F, heads, S, C, pitch, intra, st()), "ctn_sfm_attn_fwd")
        assert N.ctn_last_launch_count() == 1
        outs.append(O)
    torch.cuda.synchronize()
    assert torch.equal(outs[0][:, :, :S * C], outs[1][:, :, :S * C])
    qkvb = (qkv + in_b.view(1, -1, 1)).double().cpu()
    q, k, v = (seqs(qkvb[:, i * F:(i + 1) * F], S, C, intra) for i in range(3))
    n, L, _ = q.shape
    d = F // heads
    q, k, v = (t.reshape(n, L, heads, d).transpose(1, 2) for t in (q, k, v))
    o = torch.softmax((q / math.sqrt(d)) @ k.transpose(-1, -2), dim=-1) @ v
    ref = unseqs(o.transpose(1, 2).reshape(n, L, F), B, F, S, C, intra)
    check(outs[0][:, :, :S * C], ref)


@pytest.mark.parametrize("scale", [1.0, 1e-3, 1e3])
@pytest.mark.parametrize("F", [32, 256])
def test_token_layer_norm_against_fp64(F, scale):
    B, ntok = 2, 300
    pitch = N.ctn_pitch(ntok)
    g = torch.Generator().manual_seed(F)
    X = (torch.randn(B, F, pitch, generator=g) * scale).to(DEV)
    Y = (torch.randn(B, F, pitch, generator=g) * scale).to(DEV)
    bias, gamma, beta = (torch.randn(F, generator=g).to(DEV) for _ in range(3))
    X[:, :, 7] = 0.5 * scale  # tokens whose features are all equal: exactly beta
    Y[:, :, 7] = 0.25 * scale
    X[1, :, 9] = 3.0 * scale
    outs = []
    for _ in range(2):
        out = nan(B, F, pitch)
        N.check(N.ctn_sfm_token_ln_fwd(X.data_ptr(), Y.data_ptr(), None, gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), B, F, ntok,
                                       pitch, 1e-12, st()), "ctn_sfm_token_ln_fwd")
        assert N.ctn_last_launch_count() == 1
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0][:, :, ntok:], torch.zeros_like(outs[0][:, :, ntok:]))
    assert torch.equal(outs[0][:, :, 7], beta.view(1, -1).expand(B, F))
    x = (X + Y)[:, :, :ntok].double().cpu().transpose(1, 2)
    ref = R.layer_norm(x, gamma.double().cpu(), beta.double().cpu(), 1e-12).transpose(1, 2)
    check(outs[0][:, :, :ntok], ref)
    # with the bias, in place on X
    Xc = X.clone()
    N.check(N.ctn_sfm_token_ln_fwd(Xc.data_ptr(), Y.data_ptr(), bias.data_ptr(), gamma.data_ptr(), beta.data_ptr(), Xc.data_ptr(), B, F,
                                   ntok, pitch, 1e-12, st()), "ctn_sfm_token_ln_fwd")
    x = (X + (Y + bias.view(1, -1, 1)))[:, :, :ntok].double().cpu().transpose(1, 2)
    check(Xc[:, :, :ntok], R.layer_norm(x, gamma.double().cpu(), beta.double().cpu(), 1e-12).transpose(1, 2))


@pytest.mark.parametrize("intra", [1, 0])
@pytest.mark.parametrize("B,F,S,C", [(1, 32, 1, 1), (3, 64, 5, 250), (1, 256, 31, 250), (2, 32, 3, 2000)])
def test_seq_norm_residual_against_fp64(B, F, S, C, intra):
    pitch = N.ctn_pitch(S * C)
    g = torch.Generator().manual_seed(S * C)
    X, Rs = (torch.randn(B, F, pitch, generator=g).to(DEV) for _ in range(2))
    gamma, beta = (torch.randn(F, generator=g).to(DEV) for _ in range(2))
    outs = []
    for _ in range(2):
        out = nan(B, F, pitch)
        N.check(N.ctn_sfm_seq_norm_res_fwd(X.data_ptr(), Rs.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(), B, F, S, C, pitch,
                                           intra, 1e-12, st()), "ctn_sfm_seq_norm_res_fwd")
        assert N.ctn_last_launch_count() == 1
        outs.append(out)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    assert not outs[0][:, :, S * C:].any()
    ref = unseqs(R.gln_seq(seqs(X, S, C, intra), gamma.double().cpu(), beta.double().cpu(), 1e-12), B, F, S, C, intra) + \
        Rs[:, :, :S * C].double().cpu()
    check(outs[0][:, :, :S * C], ref)


@pytest.mark.parametrize("mask_relu,math_", [(1, "tf32x3"), (0, "fp32"), (1, "fp32")])
def test_tail_against_fp64(mask_relu, math_):
    B, Nb, Bc, S, frames, L, stride = 2, 256, 256, 3, 300, 16, 8
    pitch = N.ctn_pitch(frames)
    keys = [("prelu", (1,)), ("map_w", (S * Nb, Bc)), ("map_b", (S * Nb,)), ("gtu_w", (Nb, Nb)), ("gtu_b", (Nb,)), ("gate_w", (Nb, Nb)),
            ("gate_b", (Nb,)), ("out_w", (Nb, Nb)), ("out_b", (Nb,)), ("dec_w", (Nb, 1, L))]
    p = {k: v.to(DEV) for k, v in R.synth_state_dict(keys, 4).items()}
    g = torch.Generator().manual_seed(8)
    y = torch.randn(B, Bc, pitch, generator=g).to(DEV)
    w = torch.relu(torch.randn(B, Nb, pitch, generator=g)).to(DEV)
    T = (frames - 1) * stride + L - 6
    out, latent, what = nan(B, S, T), nan(B, S, Nb, frames), nan(B, S * Nb, pitch)
    (base, nbytes), keep = nan_ws(N.ctn_sfm_tail_workspace_bytes(B, Nb, Bc, S, pitch))
    N.check(N.ctn_sfm_tail_fwd(y.data_ptr(), w.data_ptr(), *[p[k].data_ptr() for k, _ in keys], out.data_ptr(), latent.data_ptr(),
                               what.data_ptr(), B, Nb, Bc, S, frames, pitch, L, stride, 3, T, mask_relu, _mode(math_), base, nbytes, st()),
            "ctn_sfm_tail_fwd")
    assert N.ctn_last_launch_count() == (1 if math_ != "fp32" else 0) + 6 + 1 + 1
    torch.cuda.synchronize()
    d = {k: v.double().cpu() for k, v in p.items()}
    yy = y[:, :, :frames].double().cpu()
    yy = torch.where(yy >= 0, yy, d["prelu"] * yy)
    m = (F_.conv1d(yy, d["map_w"].unsqueeze(-1), d["map_b"])).reshape(B * S, Nb, frames)
    u = torch.tanh(F_.conv1d(m, d["gtu_w"].unsqueeze(-1), d["gtu_b"])) * torch.sigmoid(F_.conv1d(m, d["gate_w"].unsqueeze(-1), d["gate_b"]))
    v = F_.conv1d(u, d["out_w"].unsqueeze(-1), d["out_b"])
    mk = torch.relu(v) if mask_relu else torch.sigmoid(v)
    wh = w[:, :, :frames].double().cpu().unsqueeze(1) * mk.reshape(B, S, Nb, frames)
    check(latent, wh)
    full = F_.conv_transpose1d(wh.reshape(B * S, Nb, frames), d["dec_w"], stride=stride).reshape(B, S, -1)
    check(out, full[..., 3:3 + T])


def _mode(name):
    from ctn_b200.models.tdcn import resolve_math
    return resolve_math(name)


def model_of(case, **over):
    g = GOLD[case]
    c = dict(g["cfg"], **over)
    m = SepFormer(c["n_basis"], c["kernel_size"], enc_basis="trainable", dec_basis="trainable", causal=False,
                  **{k: c[k] for k in ("stride", "enc_nonlinear", "sep_bottleneck_channels", "sep_chunk_size", "sep_hop_size", "sep_num_blocks",
                                       "sep_num_layers_intra", "sep_num_layers_inter", "sep_num_heads_intra", "sep_num_heads_inter",
                                       "sep_d_ff_intra", "sep_d_ff_inter", "mask_nonlinear", "n_sources", "eps")})
    keys_shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    sd = R.synth_state_dict(keys_shapes, c["seed"])
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval(), sd, c


@pytest.mark.parametrize("case", sorted(GOLD))
def test_model_against_golden_and_fp64(case):
    m, sd, c = model_of(case)
    g = GOLD[case]
    with torch.no_grad():
        out = m(g["x"].to(DEV))
        out2 = m(g["x"].to(DEV))
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    ref = R.sepformer_fwd(g["x"], sd, c)
    check(out, ref)
    gold = g["out"].double()
    assert float((out.double().cpu() - gold).abs().max()) <= R.bound(gold) + 2e-5 * float(gold.abs().max())


@pytest.mark.parametrize("case,B,T,math_", [("recipe_2spk", 1, 2008, None), ("recipe_2spk", 3, 4000, None), ("recipe_2spk", 1, 2008, "fp32"),
                                            ("recipe_2spk", 2, 6000, "tf32x3"), ("recipe_3spk", 1, 2008, None),
                                            ("recipe_3spk", 3, 3000, "fp32")])
def test_recipe_model_edges(case, B, T, math_):
    """T = 2008 samples: 250 frames, exactly one chunk; B = 1 and 3; both source counts; every 1x1 numeric mode"""
    m, sd, c = model_of(case)
    m.math = math_
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(T + B))
    with torch.no_grad():
        out, latent = m.extract_latent(x.to(DEV))
    torch.cuda.synchronize()
    frames = (T - 16) // 8 + 1
    assert torch.isfinite(out).all() and latent.shape == (B, c["n_sources"], 256, frames)
    check(out, R.sepformer_fwd(x, sd, c))


@pytest.mark.parametrize("scale", [1e-3, 1e3])
def test_model_scaled_inputs(scale):
    m, sd, c = model_of("tiny")
    x = torch.randn(2, 1, 900, generator=torch.Generator().manual_seed(9)) * scale
    with torch.no_grad():
        out = m(x.to(DEV))
    check(out, R.sepformer_fwd(x, sd, c))


def test_reference_checkpoint_loads(tmp_path):
    """a checkpoint the reference's trainer writes: its get_config() plus its state_dict (the seeded weights, reference keys)"""
    g = GOLD["tiny"]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    ckpt = dict(g["ref_config"])
    ckpt["state_dict"] = sd
    path = str(tmp_path / "best.pth")
    torch.save(ckpt, path)
    m = SepFormer.build_model(path, load_state_dict=True).to(DEV).eval()
    with torch.no_grad():
        out = m(g["x"].to(DEV))
    check(out, R.sepformer_fwd(g["x"], sd, g["cfg"]))


def test_model_launches():
    """per call: encoder 1; head: gLN fold 1 + its weight image (not in fp32) + 1x1 1; segment 1; per transformer of L layers
    positional encoding 1 + 7 L + final gLN 1 (+ 1 weight-image launch for its 4 L <= 48 images outside fp32); overlap-add 1;
    tail: PReLU, map, GTU contraction, GTU, bottleneck_conv1d_out, mask 6 + decoder 1 (+ 1 weight-image launch outside fp32)"""
    m, sd, c = model_of("recipe_2spk")
    x = torch.randn(1, 1, 4000, generator=torch.Generator().manual_seed(2)).to(DEV)
    L, nb = c["sep_num_layers_intra"], c["sep_num_blocks"]
    for math_, img in (("fp32", 0), ("tf32x3", 1), (None, 1)):
        m.math = math_
        with torch.no_grad():
            m(x)
            n0 = N.ctn_total_launch_count()
            m(x)
            n = N.ctn_total_launch_count() - n0
        expect = 1 + (2 + img) + 1 + 2 * nb * (7 * L + 2 + img) + 1 + (6 + 1 + img)
        assert n == expect, (math_, n, expect)


def test_cuda_graph_replay_matches_eager():
    m, sd, c = model_of("tiny")
    x = torch.randn(2, 1, 1203, generator=torch.Generator().manual_seed(4)).to(DEV)
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.no_grad(), torch.cuda.stream(s):
        eager = m(x)  # warm-up on the capture stream: the workspaces exist before the capture
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = m(x)
    torch.cuda.current_stream(DEV).wait_stream(s)
    x.copy_(torch.randn(2, 1, 1203, generator=torch.Generator().manual_seed(5)).to(DEV))
    graph.replay()
    torch.cuda.synchronize()
    with torch.no_grad():
        ref = m(x)
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    assert not torch.equal(out, eager)
