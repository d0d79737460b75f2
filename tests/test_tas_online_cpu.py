"""Online LSTM-TasNet (ctn_tas_online_*, TasNet.online) without a GPU: the C ABI's refusals, which return before any CUDA call, the
state size, the Python envelope, and the fp64 chunked restatement (tests/tas_online_ref.py) against the whole-signal restatement,
the reference's goldens and five planted mistakes."""
import ctypes as C
import os

import pytest
import torch

import lstm_tasnet_ref as R
import tas_online_ref as O
from ctn_b200 import _native as N
from ctn_b200.models.tasnet import TasNet

FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced: every call below is refused before it would be
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tasnet_causal_plain.pt"), weights_only=False)
ARGS = ("kernel_size", "stride", "enc_basis", "enc_nonlinear", "sep_num_blocks", "sep_num_layers", "sep_hidden_channels", "causal",
        "mask_nonlinear", "n_sources", "eps")


def _cfg(**kw):
    base = dict(n_basis=64, kernel_size=16, stride=8, hidden=32, num_blocks=2, num_layers=2, n_sources=2, causal=1, gated=0, enc_relu=0,
                mask_softmax=0, math=0, eps=1e-12)
    base.update(kw)
    return N.TasConfig(**base)


def _params(layers=4):
    arr = (N._fp * (4 * layers))(*([FAKE] * (4 * layers)))
    p = N.TasParams(enc_w=FAKE, gamma=FAKE, beta=FAKE, lstm=C.cast(arr, C.POINTER(N._fp)), fc_w=FAKE, fc_b=FAKE, dec_w=FAKE)
    return p, arr


def _bytes(cfg, B=1, frames=32):
    need = C.c_size_t(0)
    return N.ctn_tas_online_state_bytes(C.byref(cfg), B, frames, C.byref(need)), need.value


def _all_entries(c, p):
    y = C.c_size_t(0)
    return [N.ctn_tas_online_state_bytes(C.byref(c), 1, 32, C.byref(y)),
            N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, 1 << 30, None),
            N.ctn_tas_online_reset(C.byref(c), FAKE, 1, None),
            N.ctn_tas_online_push(C.byref(c), C.byref(p), FAKE, FAKE, 1, 32, 8, FAKE, None),
            N.ctn_tas_online_flush(C.byref(c), FAKE, 1, FAKE, None)]


@pytest.mark.parametrize("kw", [dict(causal=0), dict(gated=1), dict(causal=0, gated=1)])
def test_non_causal_and_gated_are_unsupported(kw):
    p, _keep = _params()
    assert _all_entries(_cfg(**kw), p) == [N.CTN_EUNSUPPORTED] * 5


@pytest.mark.parametrize("kw", [dict(kernel_size=12), dict(n_basis=0), dict(hidden=0), dict(num_blocks=0), dict(num_layers=0),
                                dict(n_sources=0), dict(stride=0), dict(math=7)])
def test_bad_config_is_invalid(kw):
    p, _keep = _params()
    assert _all_entries(_cfg(**kw), p) == [N.CTN_EINVAL] * 5


def test_decoder_history_past_shared_memory_is_unsupported():
    """N (L/S - 1) floats of decoder history per row must fit the decoder's 48 KB"""
    p, _keep = _params()
    assert _all_entries(_cfg(n_basis=4097, kernel_size=32, stride=8), p) == [N.CTN_EUNSUPPORTED] * 5
    assert _bytes(_cfg(n_basis=4096, kernel_size=16, stride=4))[0] == N.CTN_OK  # 3 frames x 4096 = exactly 48 KB


@pytest.mark.parametrize("B,n", [(1, 12), (1, 0), (1, -8), (1, 264), (0, 8), (-1, 8)])
def test_push_rejects_bad_sizes(B, n):
    """n % stride != 0, n = 0, n > max_chunk (32 frames = 256 samples), B <= 0"""
    p, _keep = _params()
    assert N.ctn_tas_online_push(C.byref(_cfg()), C.byref(p), FAKE, FAKE, B, 32, n, FAKE, None) == N.CTN_EINVAL


def test_null_pointers_alignment_and_short_state():
    c = _cfg()
    p, _keep = _params()
    need = C.c_size_t(0)
    assert N.ctn_tas_online_state_bytes(None, 1, 32, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_tas_online_state_bytes(C.byref(c), 1, 32, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_state_bytes(C.byref(c), 0, 32, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_tas_online_state_bytes(C.byref(c), 1, 0, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_tas_online_init(C.byref(c), None, 1, 32, FAKE, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, None, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 0, 32, FAKE, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, 16, None) == N.CTN_EWORKSPACE
    st, nb = _bytes(c)
    assert st == N.CTN_OK
    assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, nb - 1, None) == N.CTN_EWORKSPACE
    assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, FAKE + 4, 1 << 30, None) == N.CTN_EALIGN
    assert N.ctn_tas_online_push(C.byref(c), C.byref(p), FAKE + 64, FAKE, 1, 32, 8, FAKE, None) == N.CTN_EALIGN
    assert N.ctn_tas_online_reset(C.byref(c), FAKE + 16, 1, None) == N.CTN_EALIGN
    assert N.ctn_tas_online_flush(C.byref(c), FAKE + 8, 1, FAKE, None) == N.CTN_EALIGN
    assert N.ctn_tas_online_reset(C.byref(c), None, 1, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_reset(C.byref(c), FAKE, 0, None) == N.CTN_EINVAL
    for args in ((None, FAKE, 1, 32, 8, FAKE), (FAKE, None, 1, 32, 8, FAKE), (FAKE, FAKE, 1, 32, 8, None), (FAKE, FAKE, 1, 0, 8, FAKE)):
        assert N.ctn_tas_online_push(C.byref(c), C.byref(p), *args, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_push(C.byref(c), None, FAKE, FAKE, 1, 32, 8, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_flush(C.byref(c), None, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_flush(C.byref(c), FAKE, 1, None, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_flush(C.byref(c), FAKE, 0, FAKE, None) == N.CTN_EINVAL


@pytest.mark.parametrize("field", ["enc_w", "gamma", "beta", "fc_w", "fc_b", "lstm"])
def test_null_parameters_are_invalid(field):
    c = _cfg()
    p, _keep = _params()
    setattr(p, field, None)
    assert N.ctn_tas_online_push(C.byref(c), C.byref(p), FAKE, FAKE, 1, 32, 8, FAKE, None) == N.CTN_EINVAL
    if field in ("fc_w", "lstm"):
        assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, 1 << 30, None) == N.CTN_EINVAL


@pytest.mark.parametrize("slot", [0, 5, 15])
def test_a_null_lstm_tensor_is_invalid(slot):
    c = _cfg()
    p, arr = _params()
    arr[slot] = None
    assert N.ctn_tas_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_tas_online_push(C.byref(c), C.byref(p), FAKE, FAKE, 1, 32, 8, FAKE, None) == N.CTN_EINVAL


def test_zero_delay_flush_takes_a_null_tail():
    """kernel_size == stride: the tail is empty, so a null y_tail is not refused by the pointer checks (the state alignment is)"""
    c = _cfg(kernel_size=8, stride=8)
    assert N.ctn_tas_online_flush(C.byref(c), FAKE + 4, 1, None, None) == N.CTN_EALIGN


@pytest.mark.parametrize("B", [1, 3])
def test_recurrent_state_is_16_kb_per_stream_at_the_recipe_size(B):
    """(h, c) of X R = 4 layers at H = 500: 4 * 2 * 500 * 4 bytes = 16000 bytes per stream, on top of the other carried state"""
    rec = dict(n_basis=500, kernel_size=40, stride=20, hidden=500, num_blocks=2, num_layers=2)
    _, one = _bytes(_cfg(**rec), B)
    _, more = _bytes(_cfg(**dict(rec, num_blocks=3)), B)
    st, two = _bytes(_cfg(**rec), 2 * B)
    assert st == N.CTN_OK
    assert more - one >= 2 * B * 2 * 500 * 4  # two more layers: their (h, c) and more
    assert two - one >= B * 16000


# ---- Python envelope ---------------------------------------------------------------------------------------------------------------
def _model(**kw):
    c = dict(n_basis=32, kernel_size=16, stride=8, enc_basis="trainable", enc_nonlinear=None, sep_num_blocks=1, sep_num_layers=1,
             sep_hidden_channels=16, causal=True, mask_nonlinear="sigmoid", n_sources=2)
    c.update(kw)
    return TasNet(c.pop("n_basis"), dec_basis="trainable", **c)


@pytest.mark.parametrize("kw,what", [(dict(enc_basis="trainableGated"), "norm"), (dict(causal=False), "bidirectional"),
                                     (dict(rnn_type="gru"), "rnn_type"), (dict(in_channels=2), "monaural")])
def test_online_envelope_refusals(kw, what):
    with pytest.raises(NotImplementedError, match=what):
        _model(**kw).online(batch_size=1, max_chunk=320)


@pytest.mark.parametrize("B,chunk", [(0, 320), (1, 0), (1, 12), (1, 321)])
def test_online_rejects_bad_geometry(B, chunk):
    with pytest.raises(ValueError):
        _model().online(batch_size=B, max_chunk=chunk)


def test_online_has_no_cpu_fallback():
    with pytest.raises(RuntimeError):
        _model().online(batch_size=1, max_chunk=320)


def test_shim_models_have_online():
    from models.tasnet import TasNet as Shim
    from models.lstm_tasnet import LSTMTasNet
    assert Shim.online is TasNet.online and LSTMTasNet.online is TasNet.online


# ---- fp64 chunked restatement ----------------------------------------------------------------------------------------------------
def _gold(case):
    g = GOLD[case]
    return g, R.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"]), g["cfg"]


def _mix(total, S, pattern):
    out, i = [], 0
    while sum(out) < total:
        out.append(min(pattern[i % len(pattern)] * S, total - sum(out)))
        i += 1
    return out


@pytest.mark.parametrize("case", sorted(GOLD))
def test_whole_signal_restatement_matches_the_golden(case):
    g, sd, cfg = _gold(case)
    ref = R.tasnet_fwd(g["x"], sd, cfg)
    assert float((ref - g["out"].double()).abs().max()) <= R.bound(ref)


@pytest.mark.parametrize("case", sorted(GOLD))
@pytest.mark.parametrize("pattern", [(1,), (1, 5, 128, 300, 2, 129), (3,), (7, 2)])
def test_chunked_restatement_equals_the_whole_signal(case, pattern):
    g, sd, cfg = _gold(case)
    x = g["x"]
    ref = R.tasnet_fwd(x, sd, cfg)
    got = O.stream_fwd(x, sd, cfg, _mix(x.shape[-1], cfg["stride"], pattern))
    assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    assert float((got - g["out"].double()).abs().max()) <= R.bound(ref)


def test_zero_delay_restatement_has_an_empty_flush():
    g, sd, cfg = _gold("causal_plain_sigmoid")
    cfg = dict(cfg, kernel_size=8, stride=8)
    m = _model(kernel_size=8, stride=8, sep_num_blocks=2, sep_num_layers=2, sep_hidden_channels=24)
    sd = R.synth_state_dict([(k, tuple(v.shape)) for k, v in m.state_dict().items()], 3)
    x = g["x"]
    st = O.Stream(sd, cfg, x.shape[0])
    y = torch.cat([st.push(x[..., i:i + 40]) for i in range(0, 800, 40)], dim=2)
    assert st.flush().shape[-1] == 0
    assert float((y - R.tasnet_fwd(x, sd, cfg)).abs().max()) <= 1e-12 * float(y.abs().max())


@pytest.mark.parametrize("defect", O.DEFECTS)
def test_bound_rejects_planted_mistakes(defect):
    """each mistake of a streaming implementation leaves the whole-signal restatement by more than the fp64 bound, and the
    stream-vs-offline bound"""
    g, sd, cfg = _gold("causal_plain_sigmoid")
    x = g["x"]
    ref = R.tasnet_fwd(x, sd, cfg)
    got = O.stream_fwd(x, sd, cfg, _mix(x.shape[-1], cfg["stride"], (1, 5, 3, 2)), defect=defect)
    assert float((got - ref).abs().max()) > R.bound(ref), defect
    assert bool(((got - ref).abs() > O.stream_bound(ref)).any()), defect


def test_early_pushes_complete_no_frame():
    """with L = 2S the first push of one stride completes nothing; its output is the delay's zeros and the state is untouched"""
    g, sd, cfg = _gold("causal_plain_sigmoid")
    st = O.Stream(sd, cfg, 2)
    y = st.push(g["x"][..., :8])
    assert torch.all(y == 0) and all(torch.all(h == 0) and torch.all(c == 0) for h, c in st.hc.values())
    with pytest.raises(ValueError):
        st.flush()
