"""GALRNet on the GPU against fp64 (tests/galrnet_ref.py) and the reference's goldens: the globally attentive block
(``ctn_galr_inter_fwd``) and the separator head (``ctn_dpt_head_fwd`` without a bottleneck) on their own, with outputs and workspaces pre-filled with
NaN, across K, Q, S, F and B; digital silence; inputs scaled by 1e-3 and 1e3; the whole model in every 1x1 numeric mode at every
padding remainder of the hop; a repeated call bit for bit; a CUDA-graph replay; the launches each call makes."""
import os

import pytest
import torch

import galrnet_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.galrnet import GALRNet

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "galrnet.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
EPS = 1e-12


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


def inter_weights(F, K, Q, seed):
    keys = [("fc_map.weight", (Q, K)), ("fc_map.bias", (Q,)), ("norm2d_in.norm.weight", (F,)), ("norm2d_in.norm.bias", (F,)),
            ("multihead_attn.in_proj_weight", (3 * F, F)), ("multihead_attn.in_proj_bias", (3 * F,)),
            ("multihead_attn.out_proj.weight", (F, F)), ("multihead_attn.out_proj.bias", (F,)), ("norm2d_out.norm.weight", (F,)),
            ("norm2d_out.norm.bias", (F,)), ("fc_inv.weight", (K, Q)), ("fc_inv.bias", (K,))]
    return R.synth_state_dict(keys, seed)


def inter_call(x, sd, heads, Q):
    B, S, K, F = x.shape
    w = {k: v.to(DEV) for k, v in sd.items()}
    div = (10000 ** (torch.arange(F // 2) / F)).to(DEV)
    out = nan(B, S, K, F)
    (base, nbytes), keep = nan_ws(N.ctn_galr_inter_workspace_bytes(B, S, K, Q, F))
    N.check(N.ctn_galr_inter_fwd(x.data_ptr(), w["fc_map.weight"].data_ptr(), w["fc_map.bias"].data_ptr(), w["norm2d_in.norm.weight"].data_ptr(),
                                 w["norm2d_in.norm.bias"].data_ptr(), div.data_ptr(), heads, w["multihead_attn.in_proj_weight"].data_ptr(),
                                 w["multihead_attn.in_proj_bias"].data_ptr(), w["multihead_attn.out_proj.weight"].data_ptr(),
                                 w["multihead_attn.out_proj.bias"].data_ptr(), w["norm2d_out.norm.weight"].data_ptr(),
                                 w["norm2d_out.norm.bias"].data_ptr(), w["fc_inv.weight"].data_ptr(), w["fc_inv.bias"].data_ptr(),
                                 out.data_ptr(), B, S, K, Q, F, EPS, EPS, base, nbytes, st()), "ctn_galr_inter_fwd")
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    return out, n


def inter_ref(x, sd, heads, Q):
    B, S, K, F = x.shape
    return R.inter_block(x.double().cpu(), sd, "", heads, Q, EPS, pe=R.pe_table(S * Q, F))


# (B, S, K, Q, F, heads): K in {1, 16, 100, 250}, Q in {1, 32, K}, S in {1, 2, 79, 199}, F in {32, 64, 128}, B in {1, 3}
INTER = [(1, 1, 1, 1, 32, 4), (3, 2, 1, 1, 64, 8), (1, 2, 16, 1, 32, 4), (3, 79, 16, 16, 128, 8), (1, 199, 16, 16, 32, 4),
         (1, 79, 100, 32, 64, 8), (3, 79, 100, 32, 64, 8), (1, 199, 100, 32, 64, 8), (1, 2, 100, 100, 32, 4), (3, 1, 100, 32, 128, 8),
         (1, 79, 100, 1, 64, 8), (3, 2, 250, 250, 64, 8), (1, 79, 250, 32, 128, 8), (1, 1, 250, 1, 128, 16), (3, 199, 250, 32, 32, 4)]


@pytest.mark.parametrize("B,S,K,Q,F,heads", INTER)
def test_inter_block_against_fp64(B, S, K, Q, F, heads):
    sd = inter_weights(F, K, Q, B + S + K + Q + F)
    x = torch.randn(B, S, K, F, generator=torch.Generator().manual_seed(S * K + Q)).to(DEV)
    out, n = inter_call(x, sd, heads, Q)
    assert n == 6
    assert torch.isfinite(out).all()
    check(out, inter_ref(x, sd, heads, Q))
    out2, _ = inter_call(x, sd, heads, Q)
    assert torch.equal(out, out2)


def test_inter_block_in_place():
    B, S, K, Q, F, heads = 2, 79, 100, 32, 64, 8
    sd = inter_weights(F, K, Q, 4)
    x = torch.randn(B, S, K, F, generator=torch.Generator().manual_seed(4)).to(DEV)
    out, _ = inter_call(x, sd, heads, Q)
    w = {k: v.to(DEV) for k, v in sd.items()}
    div = (10000 ** (torch.arange(F // 2) / F)).to(DEV)
    y = x.clone()
    (base, nbytes), keep = nan_ws(N.ctn_galr_inter_workspace_bytes(B, S, K, Q, F))
    N.check(N.ctn_galr_inter_fwd(y.data_ptr(), *[w[k].data_ptr() for k in ("fc_map.weight", "fc_map.bias", "norm2d_in.norm.weight",
                                                                           "norm2d_in.norm.bias")], div.data_ptr(), heads,
                                 *[w[k].data_ptr() for k in ("multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias",
                                                             "multihead_attn.out_proj.weight", "multihead_attn.out_proj.bias",
                                                             "norm2d_out.norm.weight", "norm2d_out.norm.bias", "fc_inv.weight", "fc_inv.bias")],
                                 y.data_ptr(), B, S, K, Q, F, EPS, EPS, base, nbytes, st()), "ctn_galr_inter_fwd")
    torch.cuda.synchronize()
    assert torch.equal(out, y)


@pytest.mark.parametrize("scale", [0.0, 1e-3, 1e3])
def test_inter_block_silence_and_scaled_inputs(scale):
    """digital silence: every down-mapped token is fc_map's bias, the same for all channels, and its LayerNorm is exactly beta"""
    B, S, K, Q, F, heads = 2, 79, 100, 32, 64, 8
    sd = inter_weights(F, K, Q, 9)
    x = (torch.randn(B, S, K, F, generator=torch.Generator().manual_seed(3)) * scale).to(DEV)
    out, _ = inter_call(x, sd, heads, Q)
    assert torch.isfinite(out).all()
    check(out, inter_ref(x, sd, heads, Q))


def test_inter_block_grid_limit_refusals_before_launch():
    F, K, Q = 64, 100, 32
    sd = inter_weights(F, K, Q, 1)
    x = torch.randn(1, 3, K, F).to(DEV)
    w = {k: v.to(DEV) for k, v in sd.items()}
    div = torch.ones(F // 2, device=DEV)
    ws = torch.empty(N.ctn_galr_inter_workspace_bytes(1, 3, K, Q, F) + 256, dtype=torch.uint8, device=DEV)
    base, nbytes = N.aligned(ws)

    def call(B=1, S=3, K_=K, Q_=Q, heads=8, nb=nbytes):
        ptrs = [w[k].data_ptr() for k in ("fc_map.weight", "fc_map.bias", "norm2d_in.norm.weight", "norm2d_in.norm.bias")]
        ptrs2 = [w[k].data_ptr() for k in ("multihead_attn.in_proj_weight", "multihead_attn.in_proj_bias", "multihead_attn.out_proj.weight",
                                           "multihead_attn.out_proj.bias", "norm2d_out.norm.weight", "norm2d_out.norm.bias",
                                           "fc_inv.weight", "fc_inv.bias")]
        return N.ctn_galr_inter_fwd(x.data_ptr(), *ptrs, div.data_ptr(), heads, *ptrs2, x.data_ptr(), B, S, K_, Q_, F, EPS, EPS, base, nb, st())

    assert call(Q_=K + 1) == N.CTN_EUNSUPPORTED
    assert call(heads=16) == N.CTN_EUNSUPPORTED          # head dimension 4
    assert call(B=65536) == N.CTN_EUNSUPPORTED           # B > 65535: the grids of the down- and up-map
    assert call(S=65536) == N.CTN_EUNSUPPORTED           # S > 65535
    assert call(B=2049) == N.CTN_EWORKSPACE              # B Q = 65568 attention sequences are inside the envelope
    assert call(nb=nbytes // 2) == N.CTN_EWORKSPACE
    assert N.ctn_last_launch_count() == 0


@pytest.mark.parametrize("B,F,frames,K,P", [(1, 64, 499, 100, 50), (3, 32, 16, 16, 8), (1, 128, 3999, 100, 50), (3, 64, 1000, 250, 125),
                                            (2, 64, 101, 100, 50)])
def test_head_without_bottleneck_against_fp64(B, F, frames, K, P):
    pitch = N.ctn_pitch(frames)
    g = torch.Generator().manual_seed(frames)
    w = torch.zeros(B, F, pitch)
    w[..., :frames] = torch.randn(B, F, frames, generator=g)
    w = w.to(DEV)
    sd = {"separator.norm2d.norm.weight": 1 + 0.1 * torch.randn(F, generator=g), "separator.norm2d.norm.bias": 0.1 * torch.randn(F, generator=g)}
    cfg = {"sep_chunk_size": K, "sep_hop_size": P, "eps": EPS}
    pl, pr, S = R.segment_geometry(frames, K, P)
    gm, bt = (sd[k].to(DEV) for k in ("separator.norm2d.norm.weight", "separator.norm2d.norm.bias"))
    outs = []
    for _ in range(2):
        z = nan(B, S, K, F)
        (base, nbytes), keep = nan_ws(N.ctn_dpt_head_workspace_bytes(B, F, F, pitch, S, K))
        N.check(N.ctn_dpt_head_fwd(w.data_ptr(), None, None, gm.data_ptr(), bt.data_ptr(), z.data_ptr(), B, F, F, frames, pitch, K, P, pl, pr,
                                   EPS, N.MATH_NAMES["fp32"], base, nbytes, st()), "ctn_dpt_head_fwd")
        assert N.ctn_last_launch_count() == 3
        outs.append(z)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    check(outs[0], R.head(w[..., :frames].double().cpu(), sd, cfg))


def model_of(case):
    g = GOLD[case]
    c = g["cfg"]
    m = GALRNet(c["n_basis"], c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable",
                enc_nonlinear=c["enc_nonlinear"], sep_hidden_channels=c["sep_hidden_channels"], sep_chunk_size=c["sep_chunk_size"],
                sep_hop_size=c["sep_hop_size"], sep_down_chunk_size=c["sep_down_chunk_size"], sep_num_blocks=c["sep_num_blocks"],
                sep_num_heads=c["sep_num_heads"], sep_norm=True, sep_dropout=c["sep_dropout"], mask_nonlinear=c["mask_nonlinear"],
                low_dimension=True, causal=False, n_sources=c["n_sources"], eps=c["eps"])
    sd = R.synth_state_dict(g["keys_shapes"], c["seed"])
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).eval(), sd, c


@pytest.mark.parametrize("case", sorted(GOLD))
@pytest.mark.parametrize("math", [None, "fp32", "tf32x3"])
def test_model_against_golden_and_fp64(case, math):
    m, sd, c = model_of(case)
    m.math = math
    g = GOLD[case]
    with torch.no_grad():
        out = m(g["x"].to(DEV))
    torch.cuda.synchronize()
    check(out, R.galrnet_fwd(g["x"], sd, c))
    gold = g["out"].double()
    assert float((out.double().cpu() - gold).abs().max()) <= R.bound(gold) + 2e-5 * float(gold.abs().max())


@pytest.mark.parametrize("math", [None, "fp32", "tf32x3"])
@pytest.mark.parametrize("r", range(8))
def test_tiny_model_every_padding_remainder(r, math):
    """tiny config, hop 8: 100 + r frames give every padding remainder of the segmentation"""
    m, sd, c = model_of("tiny")
    m.math = math
    frames = 100 + r
    T = (frames - 1) * c["stride"] + c["kernel_size"]
    x = torch.randn(2, 1, T, generator=torch.Generator().manual_seed(r))
    with torch.no_grad():
        out, latent = m.extract_latent(x.to(DEV))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and latent.shape == (2, 2, c["n_basis"], frames)
    check(out, R.galrnet_fwd(x, sd, c))


@pytest.mark.parametrize("frames", [100, 101, 150, 175, 199])
def test_recipe_model_padding_remainders(frames):
    """recipe config, hop 50: a single chunk, and padding 49, 0, 25 and 1 frames"""
    m, sd, c = model_of("recipe_2spk")
    T = (frames - 1) * c["stride"] + c["kernel_size"]
    x = torch.randn(1, 1, T, generator=torch.Generator().manual_seed(frames))
    with torch.no_grad():
        out = m(x.to(DEV))
    check(out, R.galrnet_fwd(x, sd, c))


@pytest.mark.parametrize("scale", [0.0, 1e-3, 1e3])
def test_model_silence_and_scaled_inputs(scale):
    m, sd, c = model_of("recipe_3spk")
    x = torch.randn(2, 1, 2400, generator=torch.Generator().manual_seed(9)) * scale
    with torch.no_grad():
        out = m(x.to(DEV))
    assert torch.isfinite(out).all()
    check(out, R.galrnet_fwd(x, sd, c))


def test_reference_checkpoint_loads(tmp_path):
    """a wsj0-2mix checkpoint as the reference's trainer writes it: its get_config() plus its state_dict"""
    g = GOLD["recipe_2spk"]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    ckpt = dict(g["ref_config"])
    ckpt["state_dict"] = sd
    path = str(tmp_path / "best.pth")
    torch.save(ckpt, path)
    config = torch.load(path, map_location="cpu", weights_only=False)
    state = config.pop("state_dict")
    m = GALRNet(**config)
    m.load_state_dict(state, strict=True)
    m = m.to(DEV).eval()
    with torch.no_grad():
        out = m(g["x"].to(DEV))
    check(out, R.galrnet_fwd(g["x"], sd, g["cfg"]))


def test_repeated_call_is_bit_identical():
    m, _, _ = model_of("recipe_3spk")
    x = GOLD["recipe_3spk"]["x"].to(DEV)
    with torch.no_grad():
        a = m(x)
        b = m(x)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_model_launches_with_batched_tail_images():
    """per call: encoder 1; head 3; per block: intra bi-LSTM 2 + gLN and residual 2, inter 6; overlap-add 1; tail: (its two weight
    images in one launch outside fp32) PReLU 1, two 1x1, GTU + mask 1, decoder 1"""
    m, _, c = model_of("recipe_2spk")
    x = torch.randn(1, 1, 4000, generator=torch.Generator().manual_seed(2)).to(DEV)
    for math_, img in (("fp32", 0), ("tf32x3", 1)):
        m.math = math_
        with torch.no_grad():
            m(x)
            n0 = N.ctn_total_launch_count()
            m(x)
            n = N.ctn_total_launch_count() - n0
        expect = 1 + 3 + c["sep_num_blocks"] * (2 + 2 + 6) + 1 + (img + 1 + 2 + 1 + 1)
        assert n == expect, (math_, n, expect)


def test_cuda_graph_replay_matches_eager():
    m, sd, c = model_of("tiny")
    x = torch.randn(2, 1, 1203, generator=torch.Generator().manual_seed(4)).to(DEV)
    s = torch.cuda.Stream(DEV)
    s.wait_stream(torch.cuda.current_stream(DEV))
    with torch.no_grad(), torch.cuda.stream(s):
        eager = m(x)  # warm-up on the capture stream: the workspaces and the encoding's divisors exist before the capture
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
