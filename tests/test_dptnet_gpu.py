"""DPTNet on the GPU against fp64 (tests/dptnet_ref.py) and the reference's goldens: the attention, per-sequence norm and
ReLU-projection bi-LSTM entries on their own (outputs and workspaces pre-filled with NaN), the head and tail entries through the
whole model in every 1x1 numeric mode; edge lengths, every head dimension, B = 1 and 3, a single chunk, inputs scaled by 1e-3 and
1e3; a repeated call bit for bit; the launches each call makes."""
import os

import pytest
import torch

import dptnet_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.dptnet import DPTNet

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dptnet.pt"), weights_only=False)
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


def mha_call(z, heads, w):
    NSEQ, T, F = z.shape
    y = nan(NSEQ, T, F)
    (base, nbytes), keep = nan_ws(N.ctn_mha_workspace_bytes(NSEQ, T, F))
    N.check(N.ctn_mha_fwd(z.data_ptr(), NSEQ, T, F, heads, w["in_proj_weight"].data_ptr(), w["in_proj_bias"].data_ptr(),
                          w["out_proj.weight"].data_ptr(), w["out_proj.bias"].data_ptr(), y.data_ptr(), base, nbytes, st()), "ctn_mha_fwd")
    n = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    return y, n


def mha_weights(F, seed):
    return {k: v.to(DEV) for k, v in R.synth_state_dict([("in_proj_weight", (3 * F, F)), ("in_proj_bias", (3 * F,)),
                                                          ("out_proj.weight", (F, F)), ("out_proj.bias", (F,))], seed).items()}


@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 127, 128, 129, 640, 2000])
@pytest.mark.parametrize("F,heads", [(64, 4), (64, 8), (64, 2), (64, 1), (32, 4), (128, 8)])
def test_attention_against_fp64(T, F, heads):
    if T >= 640 and (F, heads) not in ((64, 4), (64, 1), (128, 8)):
        pytest.skip("long sequences at the recipe's and the extreme head dimensions")
    NSEQ = 3 if T < 640 else 2
    w = mha_weights(F, 100 + T)
    z = torch.randn(NSEQ, T, F, generator=torch.Generator().manual_seed(T)).to(DEV)
    with torch.no_grad():
        y, n = mha_call(z, heads, w)
        assert n == 3
        ref = R.mha(z.double().cpu(), {k: v.cpu() for k, v in w.items()}, "", heads)
        check(y, ref)
        y2, _ = mha_call(z, heads, w)
        assert torch.equal(y, y2)


@pytest.mark.parametrize("scale", [1e-3, 1e3])
def test_attention_saturating_inputs(scale):
    F, heads, T = 64, 4, 300
    w = mha_weights(F, 7)
    z = (torch.randn(2, T, F, generator=torch.Generator().manual_seed(3)) * scale).to(DEV)
    with torch.no_grad():
        y, _ = mha_call(z, heads, w)
    ref = R.mha(z.double().cpu(), {k: v.cpu() for k, v in w.items()}, "", heads)
    assert torch.isfinite(y).all()
    check(y, ref)


@pytest.mark.parametrize("swap", [0, 1])
@pytest.mark.parametrize("B,D1,D2,F", [(1, 1, 1, 64), (3, 5, 250, 64), (1, 250, 7, 32), (2, 3, 2000, 64)])
def test_seq_norm_against_fp64(B, D1, D2, F, swap):
    g = torch.Generator().manual_seed(D2)
    Y0, Y1, R_ = (torch.randn(B, D1, D2, F, generator=g).to(DEV) for _ in range(3))
    bias, gamma, beta = (torch.randn(F, generator=g).to(DEV) for _ in range(3))
    out = nan(*((B, D2, D1, F) if swap else (B, D1, D2, F)))
    args = lambda o: (Y0.data_ptr(), Y1.data_ptr(), bias.data_ptr(), R_.data_ptr(), gamma.data_ptr(), beta.data_ptr(), o.data_ptr(),  # noqa: E731
                      B, D1, D2, F, 1e-12, swap, st())
    N.check(N.ctn_seq_norm_fwd(*args(out)), "ctn_seq_norm_fwd")
    assert N.ctn_last_launch_count() == 1
    out2 = nan(*out.shape)
    N.check(N.ctn_seq_norm_fwd(*args(out2)), "ctn_seq_norm_fwd")
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    x = (Y0 + Y1 + bias + R_).double().cpu().reshape(B * D1, D2, F)
    ref = R.gln_seq(x, gamma.double().cpu(), beta.double().cpu(), 1e-12).reshape(B, D1, D2, F)
    if swap:
        ref = ref.transpose(1, 2)
    check(out, ref)


@pytest.mark.parametrize("NSEQ,T,F,H", [(3, 1, 64, 128), (3, 2, 64, 128), (70, 65, 64, 128), (5, 250, 32, 32), (2, 129, 128, 64)])
def test_relu_projection_lstm_against_fp64(NSEQ, T, F, H):
    keys = [("rnn.weight_ih_l0", (4 * H, F)), ("rnn.weight_hh_l0", (4 * H, H)), ("rnn.bias_ih_l0", (4 * H,)), ("rnn.bias_hh_l0", (4 * H,)),
            ("rnn.weight_ih_l0_reverse", (4 * H, F)), ("rnn.weight_hh_l0_reverse", (4 * H, H)), ("rnn.bias_ih_l0_reverse", (4 * H,)),
            ("rnn.bias_hh_l0_reverse", (4 * H,)), ("fc.weight", (F, 2 * H))]
    sd = R.synth_state_dict(keys, NSEQ + T)
    w = {k: v.to(DEV) for k, v in sd.items()}
    z = torch.randn(NSEQ, T, F, generator=torch.Generator().manual_seed(1)).to(DEV)
    ptrs = (N._fp * 8)(*[w[k].data_ptr() for k, _ in keys[:8]])
    (base, nbytes), keep = nan_ws(N.ctn_bilstm_workspace_bytes(F, H, F))
    outs = []
    for _ in range(2):
        P = nan(2, NSEQ, T, F)
        N.check(N.ctn_bilstm_relu_proj_fwd(z.data_ptr(), NSEQ, T, F, H, ptrs, w["fc.weight"].data_ptr(), F, P.data_ptr(), None, base, nbytes,
                                           st()), "ctn_bilstm_relu_proj_fwd")
        assert N.ctn_last_launch_count() == 2
        outs.append(P)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])
    h = R.bilstm(z.double().cpu(), sd, "rnn.")
    ref = torch.relu(h) @ sd["fc.weight"].double().t()
    check(outs[0][0] + outs[0][1], ref)


def model_of(case):
    g = GOLD[case]
    c = g["cfg"]
    m = DPTNet(c["n_basis"], c["kernel_size"], stride=c["stride"], enc_basis="trainable", dec_basis="trainable",
               enc_nonlinear=c["enc_nonlinear"], sep_bottleneck_channels=c["sep_bottleneck_channels"],
               sep_hidden_channels=c["sep_hidden_channels"], sep_chunk_size=c["sep_chunk_size"], sep_hop_size=c["sep_hop_size"],
               sep_num_blocks=c["sep_num_blocks"], sep_num_heads=c["sep_num_heads"], mask_nonlinear=c["mask_nonlinear"], causal=False,
               n_sources=c["n_sources"], eps=c["eps"])
    sd = R.synth_state_dict(g["keys_shapes"], c["seed"])
    m.load_state_dict(sd)
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
    ref = R.dptnet_fwd(g["x"], sd, c)
    check(out, ref)
    gold = g["out"].double()
    assert float((out.double().cpu() - gold).abs().max()) <= R.bound(gold) + 2e-5 * float(gold.abs().max())


@pytest.mark.parametrize("B,T,math", [(1, 251, None), (3, 600, None), (1, 251, "fp32"), (2, 800, "tf32x3")])
def test_recipe_model_edges(B, T, math):
    """T = 251 samples: 250 frames, exactly one chunk; B = 3; every 1x1 numeric mode"""
    m, sd, c = model_of("recipe_2spk")
    m.math = math
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(T + B))
    with torch.no_grad():
        out, latent = m.extract_latent(x.to(DEV))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all() and latent.shape == (B, 2, 64, T - 1)
    check(out, R.dptnet_fwd(x, sd, c))


@pytest.mark.parametrize("scale", [1e-3, 1e3])
def test_model_scaled_inputs(scale):
    m, sd, c = model_of("tiny")
    x = torch.randn(2, 1, 400, generator=torch.Generator().manual_seed(9)) * scale
    with torch.no_grad():
        out = m(x.to(DEV))
    check(out, R.dptnet_fwd(x, sd, c))


def test_model_launches_with_batched_tail_images():
    """per call: encoder 1; head 1x1 (+ its weight image outside fp32) + segment + 2; per block 2 x (3 + 1 + 2 + 1); overlap-add 1;
    tail: (its two weight images in one launch outside fp32) PReLU 1, two 1x1, GTU + mask 1, decoder 1"""
    m, sd, c = model_of("recipe_2spk")
    x = torch.randn(1, 1, 800, generator=torch.Generator().manual_seed(2)).to(DEV)
    for math, img in (("fp32", 0), ("tf32x3", 1)):
        m.math = math
        with torch.no_grad():
            m(x)
            n0 = N.ctn_total_launch_count()
            m(x)
            n = N.ctn_total_launch_count() - n0
        dec = 1
        expect = 1 + (img + 1 + 1 + 2) + c["sep_num_blocks"] * 14 + 1 + (img + 1 + 2 + 1 + dec)
        assert n == expect, (math, n, expect)
