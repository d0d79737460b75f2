"""LSTM-TasNet on the GPU against fp64 (tests/lstm_tasnet_ref.py) and the reference's goldens: the recurrence entry and the
encoder + frame norm entry on their own (outputs and workspaces pre-filled with NaN), the whole model in every 1x1 numeric mode at
B = 1 and 3, both source counts, causal, T = L and every padding remainder; a reference checkpoint through build_model; a repeated
call bit for bit; the launches each call makes; one CUDA-graph capture."""
import os

import pytest
import torch

import lstm_tasnet_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.tasnet import TasNet

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tasnet.pt"), weights_only=False)
DEV = torch.device("cuda", 0)
ARGS = ("kernel_size", "stride", "enc_basis", "enc_nonlinear", "sep_num_blocks", "sep_num_layers", "sep_hidden_channels", "causal",
        "mask_nonlinear", "n_sources", "eps")


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


def model_of(case, **over):
    g = GOLD[case]
    c = dict(g["cfg"], **over)
    m = TasNet(c["n_basis"], dec_basis="trainable", rnn_type="lstm", **{k: c[k] for k in ARGS})
    sd = R.synth_state_dict(g["keys_shapes"], c["seed"]) if not over else R.synth_state_dict(
        [(k, tuple(v.shape)) for k, v in m.state_dict().items()], c["seed"])
    m.load_state_dict(sd)
    return m.to(DEV).eval(), sd, c


def run_lstm(x, ws, B, F, H, dirs, T, math_, skip_in=None):
    pitch = N.ctn_pitch(T)
    xp = torch.zeros(B, F, pitch, device=DEV)
    xp[:, :, :T] = x.to(DEV)
    wd = [t.to(DEV).contiguous() for t in ws]
    out = nan(B, dirs * H, pitch)
    skip_out = nan(B, dirs * H, pitch) if skip_in is not None else None
    sk = None
    if skip_in is not None:
        sk = torch.zeros(B, dirs * H, pitch, device=DEV)
        sk[:, :, :T] = skip_in.to(DEV)
    (base, nbytes), keep = nan_ws(N.ctn_tas_lstm_workspace_bytes(B, F, H, dirs, pitch, N.MATH_NAMES[math_]))
    wp = (N._fp * len(wd))(*[t.data_ptr() for t in wd])
    N.check(N.ctn_tas_lstm_fwd(xp.data_ptr(), wp, out.data_ptr(), N.ptr(sk), N.ptr(skip_out), B, F, H, dirs, T, pitch, N.MATH_NAMES[math_],
                               base, nbytes, st()), "ctn_tas_lstm_fwd")
    launches = N.ctn_last_launch_count()
    torch.cuda.synchronize()
    assert torch.all(out[:, :, T:] == 0)
    return out, skip_out, launches


def lstm_weights(F, H, dirs, seed):
    g = torch.Generator().manual_seed(seed)
    k = H ** -0.5
    ws = []
    for _ in range(dirs):
        ws += [(torch.rand(4 * H, F, generator=g) * 2 - 1) * k, (torch.rand(4 * H, H, generator=g) * 2 - 1) * k,
               (torch.rand(4 * H, generator=g) * 2 - 1) * k, (torch.rand(4 * H, generator=g) * 2 - 1) * k]
    return ws


def test_envelope_from_device():
    for dirs in (1, 2):
        hmax = N.ctn_tas_lstm_max_hidden(dirs)
        assert hmax >= 500 * 1.5, hmax  # the recipe's H = 500 is well inside
        assert N.ctn_tas_lstm_supported(7, hmax, dirs) == 1
        assert N.ctn_tas_lstm_supported(7, hmax + 1, dirs) == 0
        assert N.ctn_tas_lstm_group(500, dirs) >= 1


LSTM_CASES = [  # (F, H, T, B, dirs, math)
    (24, 32, 1, 1, 2, "fp32"), (24, 32, 2, 3, 1, "f16x3"), (40, 100, 31, 3, 2, "fp32"), (40, 100, 32, 1, 2, "tf32x3"),
    (40, 100, 33, 2, 1, "f16x3"), (500, 500, 1599, 1, 2, "f16x3"), (1000, 500, 64, 3, 2, "fp32"), (16, 32, 5000, 1, 2, "fp32"),
    (500, 500, 200, 1, 1, "fp32"),
]


@pytest.mark.parametrize("F,H,T,B,dirs,math_", LSTM_CASES)
def test_lstm_entry_against_fp64(F, H, T, B, dirs, math_):
    ws = lstm_weights(F, H, dirs, F + H + T)
    x = torch.randn(B, F, T, generator=torch.Generator().manual_seed(T))
    out, _, launches = run_lstm(x, ws, B, F, H, dirs, T, math_)
    assert launches == 3 + (math_ != "fp32")
    check(out[:, :, :T], R.lstm_ref(x, ws, dirs))


@pytest.mark.parametrize("dirs", [2, 1])
def test_lstm_entry_envelope_maximum(dirs):
    H = N.ctn_tas_lstm_max_hidden(dirs)
    ws = lstm_weights(32, H, dirs, 5)
    x = torch.randn(1, 32, 40, generator=torch.Generator().manual_seed(5))
    out, _, _ = run_lstm(x, ws, 1, 32, H, dirs, 40, "fp32")
    check(out[:, :, :40], R.lstm_ref(x, ws, dirs))


@pytest.mark.parametrize("H,dirs", [(32, 2), (500, 2), (100, 1)])
def test_lstm_entry_past_a_sequence_group(H, dirs):
    """B = one more than a pass of the recurrence carries: the last sequence runs in a second pass from a zero state"""
    B = N.ctn_tas_lstm_group(H, dirs) + 1
    ws = lstm_weights(24, H, dirs, 7)
    x = torch.randn(B, 24, 37, generator=torch.Generator().manual_seed(7))
    skip = torch.randn(B, dirs * H, 37, generator=torch.Generator().manual_seed(8))
    out, skip_out, _ = run_lstm(x, ws, B, 24, H, dirs, 37, "fp32", skip_in=skip)
    ref = R.lstm_ref(x, ws, dirs)
    check(out[:, :, :37], ref)
    check(skip_out[:, :, :37], ref + skip.double())


def test_lstm_entry_saturating_and_repeatable():
    ws = lstm_weights(40, 100, 2, 9)
    x = torch.randn(2, 40, 50, generator=torch.Generator().manual_seed(9)) * 1e3
    out, _, _ = run_lstm(x, ws, 2, 40, 100, 2, 50, "fp32")
    assert torch.isfinite(out).all()
    check(out[:, :, :50], R.lstm_ref(x, ws, 2))
    again, _, _ = run_lstm(x, ws, 2, 40, 100, 2, 50, "fp32")
    assert torch.equal(out, again)


def run_enc(case, x):
    g = GOLD[case]
    c = g["cfg"]
    sd = R.synth_state_dict(g["keys_shapes"], c["seed"])
    B, _, T = x.shape
    frames, pl, pr = N.frames_of(T, c["kernel_size"], c["stride"])
    pitch = N.ctn_pitch(frames)
    w, xn = nan(B, c["n_basis"], pitch), nan(B, c["n_basis"], pitch)
    d = {k: v.to(DEV) for k, v in sd.items()}
    xd = x.to(DEV).contiguous()
    if c["enc_basis"] == "trainableGated":
        nrm = torch.full((B,), float("nan"), dtype=torch.float64, device=DEV)
        N.check(N.ctn_tas_enc_gated_fwd(xd.data_ptr(), d["encoder.conv1d_U.weight"].data_ptr(), d["encoder.conv1d_V.weight"].data_ptr(),
                                        d["separator.gamma"].data_ptr(), d["separator.beta"].data_ptr(), w.data_ptr(), xn.data_ptr(),
                                        nrm.data_ptr(), B, T, pl, pr, c["n_basis"], c["kernel_size"], c["stride"], pitch, 1e-12, c["eps"],
                                        st()), "ctn_tas_enc_gated_fwd")
        assert N.ctn_last_launch_count() == 2
    else:
        N.check(N.ctn_encoder_fwd(xd.data_ptr(), d["encoder.conv1d.weight"].data_ptr(), w.data_ptr(), B, T, pl, pr, c["n_basis"],
                                  c["kernel_size"], c["stride"], 1, pitch, None, st()), "ctn_encoder_fwd")
        N.check(N.ctn_tas_frame_norm_fwd(w.data_ptr(), d["separator.gamma"].data_ptr(), d["separator.beta"].data_ptr(), xn.data_ptr(), B,
                                         c["n_basis"], frames, pitch, c["eps"], st()), "ctn_tas_frame_norm_fwd")
        assert N.ctn_last_launch_count() == 1
    torch.cuda.synchronize()
    assert torch.all(w[:, :, frames:] == 0) and torch.all(xn[:, :, frames:] == 0)
    rw, rxn = R.enc_norm_ref(x, sd, c, pl, pr)
    return w[:, :, :frames], xn[:, :, :frames], rw, rxn, sd


@pytest.mark.parametrize("case", ["tiny_gated", "tiny_plain_softmax", "recipe_2spk"])
@pytest.mark.parametrize("scale", [1.0, 1e-3, 1e3])
def test_encoder_frame_norm_against_fp64(case, scale):
    x = torch.randn(2, 1, 3001, generator=torch.Generator().manual_seed(3)) * scale
    w, xn, rw, rxn, _ = run_enc(case, x)
    check(w, rw)
    check(xn, rxn)


@pytest.mark.parametrize("case", ["tiny_gated", "tiny_plain_softmax"])
def test_encoder_silence_gives_beta(case):
    x = torch.randn(2, 1, 2000, generator=torch.Generator().manual_seed(4))
    x[0] = 0  # an all-zero recording
    x[1, :, 500:1200] = 0  # digital silence inside a recording
    w, xn, rw, rxn, sd = run_enc(case, x)
    assert torch.isfinite(xn).all()
    beta = sd["separator.beta"].view(-1).to(DEV)
    assert torch.equal(xn[0], beta[:, None].expand_as(xn[0]))
    L, s = GOLD[case]["cfg"]["kernel_size"], GOLD[case]["cfg"]["stride"]
    silent = [t for t in range(xn.shape[2]) if t * s >= 500 + L and t * s + L <= 1200 - L]
    assert silent and torch.equal(xn[1][:, silent], beta[:, None].expand(-1, len(silent)))
    check(xn, rxn)


@pytest.mark.parametrize("case", sorted(GOLD))
@pytest.mark.parametrize("math_", ["fp32", "tf32x3", "f16x3"])
def test_model_against_goldens_and_fp64(case, math_):
    m, sd, c = model_of(case)
    m.math = math_
    g = GOLD[case]
    with torch.no_grad():
        out = m(g["x"].to(DEV))
    torch.cuda.synchronize()
    check(out, R.tasnet_fwd(g["x"], sd, c))
    gold = g["out"].double()
    assert float((out.double().cpu() - gold).abs().max()) <= R.bound(gold) + 2e-5 * float(gold.abs().max())


def test_model_tf32_single_pass():
    """the fast mode's single tf32 pass: a looser bound"""
    m, sd, c = model_of("tiny_gated")
    m.math = "tf32"
    g = GOLD["tiny_gated"]
    with torch.no_grad():
        out = m(g["x"].to(DEV))
    ref = R.tasnet_fwd(g["x"], sd, c)
    assert float((out.double().cpu() - ref).abs().max()) <= 1e-2 * float(ref.abs().max())


@pytest.mark.parametrize("case,B,T,math_", [("recipe_2spk", 1, 40, None), ("recipe_2spk", 3, 8001, None), ("recipe_3spk", 1, 4005, "fp32"),
                                            ("recipe_3spk", 3, 2019, "tf32x3"), ("tiny_causal", 1, 16, None), ("tiny_causal", 3, 1111, None),
                                            ("tiny_plain_softmax", 1, 8, "fp32"), ("tiny_plain_softmax", 3, 999, None)])
def test_model_edges(case, B, T, math_):
    """T = kernel_size (one frame); B = 1 and 3; both source counts; causal; softmax"""
    m, sd, c = model_of(case)
    m.math = math_
    x = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(T + B))
    with torch.no_grad():
        out, latent = m.extract_latent(x.to(DEV))
    torch.cuda.synchronize()
    frames = N.frames_of(T, c["kernel_size"], c["stride"])[0]
    assert torch.isfinite(out).all() and latent.shape == (B, c["n_sources"], c["n_basis"], frames)
    check(out, R.tasnet_fwd(x, sd, c))


@pytest.mark.parametrize("rem", range(8))
def test_model_every_padding_remainder(rem):
    m, sd, c = model_of("tiny_gated")
    T = 16 + 8 * 20 + rem
    x = torch.randn(2, 1, T, generator=torch.Generator().manual_seed(rem))
    with torch.no_grad():
        out = m(x.to(DEV))
    assert out.shape == (2, 2, T)
    check(out, R.tasnet_fwd(x, sd, c))


def test_model_refuses_hidden_past_envelope():
    H = N.ctn_tas_lstm_max_hidden(2) + 1
    m = TasNet(8, kernel_size=4, enc_basis="trainableGated", dec_basis="trainable", sep_num_blocks=1, sep_num_layers=1,
               sep_hidden_channels=H, mask_nonlinear="sigmoid").to(DEV).eval()
    with torch.no_grad(), pytest.raises(NotImplementedError, match="at most {}".format(H - 1)):
        m(torch.randn(1, 1, 100, device=DEV))


def test_reference_checkpoint_loads(tmp_path):
    """a wsj0-2mix checkpoint as the reference's trainer writes it: its get_config() plus its state_dict"""
    g = GOLD["recipe_2spk"]
    sd = R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
    ckpt = dict(g["ref_config"])
    ckpt["state_dict"] = sd
    path = str(tmp_path / "best.pth")
    torch.save(ckpt, path)
    m = TasNet.build_model(path, load_state_dict=True).to(DEV).eval()
    with torch.no_grad():
        out = m(g["x"].to(DEV))
    check(out, R.tasnet_fwd(g["x"], sd, g["cfg"]))


def test_repeated_call_is_bit_identical():
    m, _, _ = model_of("recipe_3spk")
    x = GOLD["recipe_3spk"]["x"].to(DEV)
    with torch.no_grad():
        a = m(x)
        b = m(x)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_model_launches():
    """per call: gated encoder + frame norm 2; per LSTM layer prep, input projection, recurrence 3 (+ 1 weight image outside
    fp32); tail fc 1 + decoder 1 (+ 1 weight image outside fp32)"""
    m, _, c = model_of("recipe_2spk")
    x = torch.randn(1, 1, 4000, generator=torch.Generator().manual_seed(2)).to(DEV)
    layers = c["sep_num_blocks"] * c["sep_num_layers"]
    for math_, img in (("fp32", 0), ("tf32x3", 1), (None, 1)):
        m.math = math_
        with torch.no_grad():
            m(x)
            n0 = N.ctn_total_launch_count()
            m(x)
            n = N.ctn_total_launch_count() - n0
        expect = 2 + layers * (3 + img) + (2 + img)
        assert n == expect, (math_, n, expect)


def test_cuda_graph_replay_matches_eager():
    m, sd, c = model_of("tiny_gated")
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
