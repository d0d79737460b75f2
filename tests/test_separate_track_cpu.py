"""ConvTasNet.separate_track without a GPU: the exported symbols, the segment plan (ctn_track_plan) against its restatement, the
C ABI's refusals (each returns before any CUDA call), the workspace formula, the fp64 restatement against the reference golden,
and the Python envelope."""
import ctypes as C
import os

import pytest
import torch

import separate_long_ref as SL
import separate_track_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet, TRACK_CHUNK_BATCH

FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced: every call below is refused before it would be
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_stereo_track.pt")
NAMES = ("ctn_track_plan", "ctn_track_stats_scratch_bytes", "ctn_track_stats", "ctn_track_gather", "ctn_track_overlap_add",
         "ctn_separate_track_workspace_bytes", "ctn_convtasnet_separate_track")


def _cfg(**kw):
    c = N.Config()
    base = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2,
                num_layers=4, n_sources=2, causal=0, enc_relu=0, mask_softmax=0, math=0, eps=1e-12, eps_tcn=1e-12, in_channels=2)
    base.update(kw)
    for k, v in base.items():
        setattr(c, k, v)
    return c


def _recipe_cfg(**kw):
    return _cfg(**dict(dict(n_basis=256, kernel_size=20, stride=10, bottleneck=256, hidden=512, skip=128, num_blocks=4, num_layers=10,
                            n_sources=4, math=3), **kw))


def _params():
    blocks = (N.BlockParams * 64)()
    for b in blocks:
        for name in N.BLOCK_FIELDS:
            setattr(b, name, FAKE)
    p = N.Params()
    for name, _ in N.Params._fields_:
        if name != "blocks":
            setattr(p, name, FAKE)
    p.blocks = blocks
    return p, blocks


def _plan(T, segment, hop):
    K = N.ctn_track_plan(T, segment, hop, None, 0)
    if K < 0:
        return K, None
    starts = (C.c_int * K)()
    assert N.ctn_track_plan(T, segment, hop, starts, K) == K
    return K, list(starts)


def test_symbols_exported():
    for name in NAMES:
        assert hasattr(N.lib, name) and name in N.EXPORTED


# the tester's layout: T < segment, T == segment, T == k segment, T == k segment + 1, the recipe's 240 s track
TESTER = [(50, 100), (100, 100), (300, 100), (301, 100), (2137, 400), (1, 7), (240 * 44100, 8 * 44100), (240 * 44100 + 1, 8 * 44100)]
# the cross-faded layout, including an odd segment with hop = segment // 2
CROSS = [(50, 100, 50), (100, 100, 50), (300, 100, 50), (301, 100, 100), (2137, 400, 300), (977, 101, 50), (12345, 333, 166),
         (240 * 44100, 8 * 44100, 4 * 44100)]


@pytest.mark.parametrize("T,segment", TESTER)
def test_tester_plan_matches_restatement(T, segment):
    K, starts = _plan(T, segment, 0)
    ref, Lc = R.plan(T, segment, None)
    assert Lc == segment and K == len(ref) and starts == ref
    assert K == -(-T // segment)
    assert all(b - a == segment for a, b in zip(starts, starts[1:]))    # neighbours share no samples and leave no gap
    assert starts[-1] < T <= starts[-1] + segment                      # the last segment holds the end of the track


@pytest.mark.parametrize("T,segment,hop", CROSS)
def test_crossfaded_plan_is_the_chunk_plan(T, segment, hop):
    K, starts = _plan(T, segment, hop)
    ref, Lc = R.plan(T, segment, hop)
    assert K == len(ref) and starts == ref
    assert (K, starts) == (N.ctn_chunk_plan(T, segment, hop, None, 0), SL.plan(T, segment, hop)[0])
    assert starts[-1] + Lc == T


@pytest.mark.parametrize("T,segment,hop", [(1000, 100, 49), (1000, 100, 101), (1000, 101, 49), (1000, 0, 0), (1000, -4, 0), (1000, 100, -1),
                                           (0, 100, 0), (-5, 100, 0), (0, 100, 50)])
def test_plan_rejects(T, segment, hop):
    assert N.ctn_track_plan(T, segment, hop, None, 0) == N.CTN_EINVAL


def test_plan_capacity():
    starts = (C.c_int * 3)()
    assert N.ctn_track_plan(301, 100, 0, starts, 3) == N.CTN_EINVAL   # four segments
    assert N.ctn_track_plan(300, 100, 0, starts, 3) == 3


def _call(c, p, x=FAKE, B=1, T=100000, segment=4000, hop=0, cb=4, out=FAKE, ws=FAKE, ws_bytes=1 << 40):
    return N.ctn_convtasnet_separate_track(C.byref(c) if c is not None else None, C.byref(p) if p is not None else None, x, B, T,
                                           segment, hop, cb, out, ws, ws_bytes, None)


def _ws(c, B, T, segment, hop, cb):
    need = C.c_size_t(0)
    assert N.ctn_separate_track_workspace_bytes(C.byref(c), B, T, segment, hop, cb, C.byref(need)) == N.CTN_OK
    return need.value


def test_argument_errors():
    c = _cfg()
    p, _keep = _params()
    need = _ws(c, 1, 100000, 4000, 0, 4)
    for kw in (dict(hop=1999), dict(hop=4001), dict(hop=-1), dict(segment=0), dict(segment=-8), dict(B=0), dict(T=0), dict(cb=0),
               dict(segment=8, hop=0)):                                 # the last: a segment shorter than the encoder kernel
        assert _call(c, p, **kw) == N.CTN_EINVAL, kw
    assert _call(None, p) == N.CTN_EINVAL
    assert _call(c, None) == N.CTN_EINVAL
    for kw in (dict(x=None), dict(out=None), dict(ws=None)):
        assert _call(c, p, **kw) == N.CTN_EINVAL, kw
    assert _call(_cfg(in_channels=65), p) == N.CTN_EINVAL
    assert _call(c, p, ws=FAKE + 4) == N.CTN_EALIGN
    assert _call(c, p, ws_bytes=need - 1) == N.CTN_EWORKSPACE
    assert _call(c, p, ws_bytes=16) == N.CTN_EWORKSPACE
    assert _call(c, p, B=40000) == N.CTN_EUNSUPPORTED                   # B * C = 80000 (track, channel) rows on gridDim.y
    assert N.ctn_separate_track_workspace_bytes(C.byref(c), 1, 100000, 4000, 0, 4, None) == N.CTN_EINVAL
    assert N.ctn_separate_track_workspace_bytes(C.byref(c), 1, 100000, 4000, 1000, 4, C.byref(C.c_size_t())) == N.CTN_EINVAL
    # the whole envelope of the forward: monaural, causal, softmax, 64 channels, every math mode
    for kw in (dict(in_channels=1), dict(in_channels=0), dict(causal=1), dict(mask_softmax=1), dict(in_channels=64), dict(math=1),
               dict(math=3)):
        assert _ws(_cfg(**kw), 1, 100000, 4000, 0, 4) > 0, kw


def test_step_entry_errors():
    big = 1 << 30
    assert N.ctn_track_stats_scratch_bytes(1, 2, 1000, 100, 49) == 0
    assert N.ctn_track_stats_scratch_bytes(1, 2, 1000, 1, 0) == 0                 # one sample: no unbiased std
    assert N.ctn_track_stats_scratch_bytes(1, 2, 1000, 100, 0) == 8 * 2 * 10 * 2  # (sum, sum of squares) per row, one CTA per row
    assert N.ctn_track_stats_scratch_bytes(1, 2, 240 * 44100, 8 * 44100, 0) == 8 * 2 * 30 * 2 * 44   # 44 CTAs per 8 s row
    assert N.ctn_track_stats(None, 1, 2, 1000, 100, 0, FAKE, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_track_stats(FAKE, 1, 2, 1000, 100, 0, None, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_track_stats(FAKE, 1, 2, 1000, 100, 0, FAKE, None, big, None) == N.CTN_EINVAL
    assert N.ctn_track_stats(FAKE, 1, 0, 1000, 100, 0, FAKE, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_track_stats(FAKE, 1, 65, 1000, 100, 0, FAKE, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_track_stats(FAKE, 1, 2, 1000, 100, 49, FAKE, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_track_stats(FAKE, 1, 2, 1000, 100, 0, FAKE + 4, FAKE, big, None) == N.CTN_EALIGN
    assert N.ctn_track_stats(FAKE, 1, 2, 1000, 100, 0, FAKE, FAKE + 4, big, None) == N.CTN_EALIGN
    assert N.ctn_track_stats(FAKE, 1, 2, 1000, 100, 0, FAKE, FAKE, 8 * 2 * 20 - 1, None) == N.CTN_EWORKSPACE
    assert N.ctn_track_gather(None, FAKE, 1, 2, 1000, 100, 0, 1e-12, 0, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_gather(FAKE, None, 1, 2, 1000, 100, 0, 1e-12, 0, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_gather(FAKE, FAKE, 1, 2, 1000, 100, 0, 1e-12, 0, 1, None, None) == N.CTN_EINVAL
    assert N.ctn_track_gather(FAKE, FAKE, 1, 2, 1000, 100, 0, 1e-12, 9, 2, FAKE, None) == N.CTN_EINVAL    # K = 10: chunks 9, 10
    assert N.ctn_track_gather(FAKE, FAKE, 1, 2, 1000, 100, 0, 1e-12, -1, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_gather(FAKE, FAKE, 1, 2, 1000, 100, 0, -1.0, 0, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_gather(FAKE, FAKE, 1, 2, 1000, 100, 0, float("nan"), 0, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_gather(FAKE, FAKE + 4, 1, 2, 1000, 100, 0, 1e-12, 0, 1, FAKE, None) == N.CTN_EALIGN
    assert N.ctn_track_gather(FAKE, FAKE, 1, 2, 100000 * 40, 100, 0, 1e-12, 0, 40000, FAKE, None) == N.CTN_EUNSUPPORTED
    assert N.ctn_track_overlap_add(None, FAKE, 1, 2, 2, 1000, 100, 0, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_overlap_add(FAKE, None, 1, 2, 2, 1000, 100, 0, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_overlap_add(FAKE, FAKE, 1, 2, 2, 1000, 100, 0, None, None) == N.CTN_EINVAL
    assert N.ctn_track_overlap_add(FAKE, FAKE, 1, 0, 2, 1000, 100, 0, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_overlap_add(FAKE, FAKE, 1, 2, 2, 1000, 100, 101, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_track_overlap_add(FAKE, FAKE + 4, 1, 2, 2, 1000, 100, 0, FAKE, None) == N.CTN_EALIGN
    assert N.ctn_track_overlap_add(FAKE, FAKE, 40000, 2, 2, 1000, 100, 0, FAKE, None) == N.CTN_EUNSUPPORTED


def _r256(n):
    return (n + 255) // 256 * 256


@pytest.mark.parametrize("B,C_,S,segment,hop", [(1, 2, 4, 8 * 44100, 0), (1, 2, 4, 8 * 44100, 4 * 44100), (3, 2, 2, 4000, 0),
                                                (2, 1, 3, 4000, 2500), (1, 3, 2, 9000, 0)])
def test_workspace_grows_with_T_by_the_estimates_and_statistics_only(B, C_, S, segment, hop):
    """beyond chunk_batch chunks, bytes(T) = const + [statistics] + [their partials] + [chunk estimates], each rounded up to 256"""
    c = _cfg(n_basis=256, kernel_size=20, stride=10, bottleneck=128, hidden=256, skip=128, n_sources=S, in_channels=C_)
    split = min(64, -(-segment // 8192))

    def grows(T):
        K = N.ctn_track_plan(T, segment, hop, None, 0)
        rows = B * K * C_
        return _r256(16 * rows) + _r256(16 * rows * split) + _r256(4 * B * K * S * C_ * segment)

    T1, T2 = 40 * segment, 40 * segment + 1234567
    b1, b2 = _ws(c, B, T1, segment, hop, 4), _ws(c, B, T2, segment, hop, 4)
    assert b2 - b1 == grows(T2) - grows(T1)
    # the rest is one chunk batch of the forward's workspace and one standardised batch
    fwd = C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(c), 4, segment, C.byref(fwd)) == N.CTN_OK
    rest = b1 - grows(T1)
    assert fwd.value <= rest <= fwd.value + _r256(4 * 4 * C_ * segment) + 1024
    whole = C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(c), B, T2, C.byref(whole)) == N.CTN_OK
    assert b2 < whole.value


def test_default_chunk_batch_fits_the_stated_workspace():
    """the docstring's figures: one batch of model workspace under 8 GB at the recipe size, 8.2 GB for the whole call on 240 s"""
    c = _recipe_cfg()
    seg = 8 * 44100
    fwd, more = C.c_size_t(0), C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(c), TRACK_CHUNK_BATCH, seg, C.byref(fwd)) == N.CTN_OK
    assert N.ctn_workspace_bytes(C.byref(c), TRACK_CHUNK_BATCH + 1, seg, C.byref(more)) == N.CTN_OK
    assert fwd.value < 8e9 < more.value
    assert _ws(c, 1, 240 * 44100, seg, 0, TRACK_CHUNK_BATCH) < 8.3e9


# ---- the restatement against the reference golden ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.mark.parametrize("layout", ["tester", "crossfaded"])
def test_restatement_matches_reference_golden(golden, layout):
    r = golden[layout]
    hop = None if layout == "tester" else golden["hop"]
    x = golden["mixture"][:, 0]                                     # (B, C, T)
    B, Cn, T = x.shape
    seg = golden["segment"]
    starts, Lc = R.plan(T, seg, hop)
    assert starts == r["starts"]
    K = len(starts)
    xc = R.chunks(x, starts, Lc)
    st = R.stats(xc)
    # statistics and standardised chunks: fp64 rounding apart (the reference sums in a different order)
    ref_st = torch.stack([r["mean64"], r["std64"]], -1).reshape(B * K, Cn, 2)
    assert bool(((st - ref_st).abs() <= 1e-13 * (1 + ref_st.abs())).all())
    z = R.standardise(xc, st, golden["eps"])
    torch.testing.assert_close(z, R.standardise(xc, ref_st, golden["eps"]), rtol=1e-12, atol=1e-12)
    # the all-zero segment standardises to exact zeros, the DC segment to unit variance
    if layout == "tester":
        assert bool((z[1] == 0).all()) and bool((st[1] == 0).all())
        assert abs(float(z[3].std(-1).max()) - 1.0) < 1e-10     # std / (std + eps)
    # the de-standardising overlap-add of the reference's own fp64 chunk estimates
    out = R.separate(x, r["est64"], seg, hop)
    torch.testing.assert_close(out, r["out64"], rtol=1e-12, atol=1e-12)
    # and the fp32 record within its own fp32-vs-fp64 spread
    assert float((out - r["out"].double()).abs().max()) <= 1.5 * r["fp32_vs_fp64_maxabs"] + 1e-12


# ---- Python envelope ---------------------------------------------------------------------------------------------------------
def _model(**kw):
    return ConvTasNet(64, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=32,
                      sep_bottleneck_channels=16, sep_skip_channels=16, sep_num_blocks=1, sep_num_layers=2, causal=False, **kw)


def test_python_envelope():
    stereo, mono = _model(in_channels=2), _model()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            stereo.separate_track(torch.zeros(1, 1, 2, 1000), 400)
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            mono.separate_track(torch.zeros(1, 1, 1000), 400)
        with pytest.raises(ValueError, match="takes the 4-D input"):
            stereo.separate_track(torch.zeros(1, 1, 1000), 400)
        with pytest.raises(ValueError, match="does not match in_channels"):
            stereo.separate_track(torch.zeros(1, 1, 3, 1000), 400)
        with pytest.raises(ValueError, match="expected"):
            stereo.separate_track(torch.zeros(1, 2, 2, 1000), 400)
        with pytest.raises(ValueError, match="expected"):
            mono.separate_track(torch.zeros(1, 2, 1000), 400)
        with pytest.raises(ValueError, match="dimension"):
            mono.separate_track(torch.zeros(1000), 400)
    with pytest.raises(NotImplementedError, match="inference-only"):
        stereo.separate_track(torch.zeros(1, 1, 2, 1000), 400)      # autograd on, parameters require grad
    with pytest.raises(NotImplementedError):
        with torch.no_grad():
            mono.separate_long(torch.zeros(1, 1, 2, 1000), 400)     # separate_long still takes monaural input only


def test_shim_model_has_separate_track():
    from models.conv_tasnet import ConvTasNet as Shim
    assert Shim.separate_track is ConvTasNet.separate_track
