"""ConvTasNet.separate_track on the GPU (``-m gpu``).

Each step runs on its own against float64 (separate_track_ref.py): the statistics within a bound derived from their double
summation, the standardising gather within one fp32 rounding of the fp64 value computed from the kernel's own statistics, and
the de-standardising overlap-add within one fp32 rounding of fp64.  The whole call is compared with the same steps run one
segment at a time through ``model(...)`` and de-standardised in fp64, and with the reference golden minted from the recipe's
tester steps (tests/golden/make_golden_stereo_track.py)."""
import ctypes as C

import pytest
import torch

import convtasnet_oracle as O
import separate_track_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet
from test_parity_gpu import MODES

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 2e-5   # test_parity_gpu.py's stereo forward against the reference golden


def _stream():
    return N.stream_ptr(torch.device("cuda", torch.cuda.current_device()))


def _hop(hop):
    return 0 if hop is None else hop


def _stats(x, segment, hop):
    B, Cn, T = x.shape
    K = N.ctn_track_plan(T, segment, _hop(hop), None, 0)
    st = torch.full((B, K, Cn, 2), float("nan"), dtype=torch.float64, device="cuda")
    nbytes = N.ctn_track_stats_scratch_bytes(B, Cn, T, segment, _hop(hop))
    scratch = torch.full((nbytes // 8 + 1,), float("nan"), dtype=torch.float64, device="cuda")
    N.check(N.ctn_track_stats(x.data_ptr(), B, Cn, T, segment, _hop(hop), st.data_ptr(), scratch.data_ptr(), nbytes, _stream()),
            "ctn_track_stats")
    return st


def _gather(x, st, segment, hop, first, n, eps=1e-12):
    B, Cn, T = x.shape
    _, Lc = R.plan(T, segment, hop)
    xc = torch.full((n, Cn, Lc), float("nan"), device="cuda")
    N.check(N.ctn_track_gather(x.data_ptr(), st.data_ptr(), B, Cn, T, segment, _hop(hop), eps, first, n, xc.data_ptr(), _stream()),
            "ctn_track_gather")
    return xc


def _ola(est, st, B, T, segment, hop):
    S, Cn = est.shape[1], est.shape[2]
    out = torch.full((B, S, Cn, T), float("nan"), device="cuda")
    N.check(N.ctn_track_overlap_add(est.data_ptr(), st.data_ptr(), B, S, Cn, T, segment, _hop(hop), out.data_ptr(), _stream()),
            "ctn_track_overlap_add")
    return out


def _track(B, Cn, T, segment, seed, dc=True):
    """a seeded track with an all-zero segment (segment 1) and a large DC offset (segment 3) in track 0"""
    g = torch.Generator().manual_seed(seed)
    x = 0.3 * torch.randn(B, Cn, T, generator=g)
    if T > 2 * segment:
        x[0, :, segment:2 * segment] = 0.0
    if dc and T > 4 * segment:
        x[0, :, 3 * segment:4 * segment] += 500.0
    return x


# (T, segment, hop): several statistics CTAs per row (segment > 8192), odd T, T < segment, T a multiple of the segment
GEOMS = [(50021, 20000, None), (50021, 20000, 10001), (30011, 9000, None), (30011, 9000, 4500), (977, 101, None), (977, 101, 50),
         (5000, 8192 * 3 + 5, None), (4000, 1000, None), (4000, 1000, 1000)]


@pytest.mark.parametrize("T,segment,hop", GEOMS)
@pytest.mark.parametrize("Cn", [1, 2, 3])
def test_stats_vs_fp64(Cn, T, segment, hop):
    B = 2
    x = _track(B, Cn, T, segment, seed=T + Cn)
    # a base that is only 4-byte aligned, so no row starts on a 16-byte boundary
    xd = torch.empty(B * Cn * T + 1, device="cuda")[1:].reshape(B, Cn, T)
    xd.copy_(x)
    st = _stats(xd, segment, hop).cpu()
    starts, Lc = R.plan(T, segment, hop)
    xc = R.chunks(x.double(), starts, Lc)
    ref = R.stats(xc).reshape(st.shape)
    bound = R.stats_bounds(xc).reshape(st.shape)
    err = (st - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    if T > 2 * segment and hop is None:
        assert bool((st[0, 1] == 0).all())                       # the all-zero segment: mean 0, std 0 exactly
    assert torch.equal(_stats(xd, segment, hop).cpu(), st)       # no atomics: the same bits twice


@pytest.mark.parametrize("T,segment,hop", GEOMS)
@pytest.mark.parametrize("Cn", [1, 2])
def test_gather_vs_fp64(Cn, T, segment, hop):
    B = 2
    x = _track(B, Cn, T, segment, seed=3 * T + Cn)
    xd = x.cuda()
    st = _stats(xd, segment, hop)
    starts, Lc = R.plan(T, segment, hop)
    K = len(starts)
    xc = _gather(xd, st, segment, hop, 0, B * K).cpu()
    x64 = R.chunks(x.double(), starts, Lc)
    st_k = st.cpu().reshape(B * K, Cn, 2)
    want = R.standardise(x64, st_k)
    assert bool(((xc.double() - want).abs() <= R.gather_bound(x64, st_k)).all())
    assert bool(torch.isfinite(xc).all())
    if T > 2 * segment and hop is None:
        assert bool((xc[1] == 0).all())                          # the all-zero segment gives exact zeros, not NaN
    if T > 4 * segment and hop is None:
        # the DC segment: against the exact statistics, the statistics' own error propagated through 1 / (std + eps)
        ref_st = R.stats(x64[3:4])
        dmean, dstd = R.stats_bounds(x64[3:4]).unbind(-1)
        y = R.standardise(x64[3:4], ref_st)
        prop = (dmean[..., None] + y.abs() * dstd[..., None]) / (ref_st[..., 1:] + 1e-12)
        assert bool(((xc[3:4].double() - y).abs() <= R.gather_bound(x64[3:4], ref_st) + prop).all())
    # a slice of the chunks
    if B * K > 2:
        assert torch.equal(_gather(xd, st, segment, hop, 1, B * K - 2).cpu(), xc[1:-1])


@pytest.mark.parametrize("T,segment,hop", GEOMS)
@pytest.mark.parametrize("S,Cn", [(1, 1), (4, 2), (2, 3)])
def test_overlap_add_vs_fp64(S, Cn, T, segment, hop):
    B = 2
    g = torch.Generator().manual_seed(11 * T + S)
    starts, Lc = R.plan(T, segment, hop)
    K = len(starts)
    est = torch.randn(B * K, S, Cn, Lc, generator=g)
    st = torch.stack([torch.randn(B, K, Cn, generator=g, dtype=torch.float64) * 30,
                      torch.rand(B, K, Cn, generator=g, dtype=torch.float64) * 5], -1)
    out = _ola(est.cuda(), st.cuda(), B, T, segment, hop).cpu()
    for b in range(B):
        ref, mag = R.overlap_add(est[b * K:(b + 1) * K], st[b], starts, Lc, T, hop is not None, magnitude=True)
        assert bool(((out[b].double() - ref).abs() <= R.ola_bound(ref, mag)).all())
    if hop is None:
        # unit statistics: the tester's concatenate-and-crop, bit for bit
        unit = torch.zeros(B, K, Cn, 2, dtype=torch.float64)
        unit[..., 1] = 1.0
        out = _ola(est.cuda(), unit.cuda(), B, T, segment, hop).cpu()
        cat = est.reshape(B, K, S, Cn, Lc).permute(0, 2, 3, 1, 4).reshape(B, S, Cn, K * Lc)[..., :T]
        assert torch.equal(out, cat)


# ---- the whole call -------------------------------------------------------------------------------------------------------------
SMALL = dict(n_basis=64, kernel_size=16, sep_hidden_channels=128, sep_bottleneck_channels=32, sep_skip_channels=32, sep_num_blocks=2,
             sep_num_layers=3, n_sources=4)
CONFIGS = {
    "stereo_gln": dict(SMALL, causal=False, in_channels=2),
    "stereo_cln": dict(SMALL, causal=True, in_channels=2),
    "stereo_softmax": dict(SMALL, causal=False, in_channels=2, mask_nonlinear="softmax"),
    "mono_gln": dict(SMALL, causal=False, in_channels=1),
}


def _build(cfg, sd, math=None):
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, stride=cfg.stride, enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg.enc_nonlinear, sep_hidden_channels=cfg.sep_hidden_channels,
                   sep_bottleneck_channels=cfg.sep_bottleneck_channels, sep_skip_channels=cfg.sep_skip_channels,
                   sep_kernel_size=cfg.sep_kernel_size, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers,
                   mask_nonlinear=cfg.mask_nonlinear, causal=cfg.causal, n_sources=cfg.n_sources, eps=cfg.eps,
                   in_channels=cfg.in_channels)
    m.load_state_dict(sd, strict=True)
    m.math = math
    return m.cuda().eval()


def _model(name, mode="fp32", seed=51):
    cfg = O.OracleConfig(**CONFIGS[name])
    return cfg, _build(cfg, O.synth_state_dict(cfg, seed=seed), math=mode)


def _input(x, model):
    """(B, C, T) -> the model's input form"""
    return x.unsqueeze(1) if model.in_channels > 1 else x


def _steps(model, x, segment, hop):
    """the kernel's statistics and standardised chunks, ``model(...)`` one segment at a time, de-standardised in fp64 ->
    (ref (B, S, C, T) float64, mag)"""
    B, Cn, T = x.shape
    starts, Lc = R.plan(T, segment, hop)
    K = len(starts)
    st = _stats(x, segment, hop)
    xc = _gather(x, st, segment, hop, 0, B * K, eps=model.eps)
    with torch.no_grad():
        est = torch.stack([model(_input(xc[i:i + 1], model))[0].reshape(model.n_sources, Cn, Lc) for i in range(B * K)])
    st, est = st.cpu(), est.cpu()
    outs = [R.overlap_add(est[b * K:(b + 1) * K], st[b], starts, Lc, T, hop is not None, magnitude=True) for b in range(B)]
    return torch.stack([o[0] for o in outs]), torch.stack([o[1] for o in outs])


def _call(model, x, segment, hop=None, chunk_batch=3):
    with torch.no_grad():
        out = model.separate_track(_input(x, model), segment, hop=hop, chunk_batch=chunk_batch)
    return out if model.in_channels > 1 else out.unsqueeze(2)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_whole_call_vs_steps(name, mode):
    cfg, model = _model(name, mode)
    B, T, segment = 2, 14321, 3000
    x = _track(B, max(cfg.in_channels, 1), T, segment, seed=52).cuda()
    for hop in (None, 2000):
        ref, mag = _steps(model, x, segment, hop)
        out = _call(model, x, segment, hop).cpu().double()
        assert out.shape == ref.shape
        assert bool(((out - ref).abs() <= R.ola_bound(ref, mag)).all()), float((out - ref).abs().max())
    assert model.last_launches > 0


def test_chunk_batch_does_not_change_a_bit():
    cfg, model = _model("stereo_gln", "f16x3" if "f16x3" in MODES else "fp32")
    x = _track(2, 2, 21000, 3000, seed=53).cuda()
    for hop in (None, 1700):
        base = _call(model, x, 3000, hop, chunk_batch=4)
        for cb in (1, 3, 1000):
            assert torch.equal(_call(model, x, 3000, hop, chunk_batch=cb), base)


def test_tracks_of_a_batch_do_not_interact():
    cfg, model = _model("stereo_gln")
    x = _track(3, 2, 15000, 3000, seed=54).cuda()
    out = _call(model, x, 3000, chunk_batch=4)
    for b in range(3):
        torch.testing.assert_close(_call(model, x[b:b + 1].clone(), 3000, chunk_batch=4)[0], out[b], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("mode", MODES)
def test_second_call_gives_the_same_bits(mode):
    cfg, model = _model("stereo_gln", mode)
    x = _track(2, 2, 15000, 3000, seed=55).cuda()
    for hop in (None, 2000):
        assert torch.equal(_call(model, x, 3000, hop), _call(model, x, 3000, hop))


def test_call_is_cuda_graph_capturable():
    """every launch on the caller's stream, nothing read back: capture once, replay on new input"""
    cfg, model = _model("stereo_gln")
    x1 = _track(2, 2, 15000, 3000, seed=56).unsqueeze(1).cuda()
    x2 = _track(2, 2, 15000, 3000, seed=57).unsqueeze(1).cuda()
    xs = x1.clone()
    side = torch.cuda.Stream()
    with torch.no_grad():
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                model.separate_track(xs, 3000)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            out_g = model.separate_track(xs, 3000)
        for x in (x2, x1):
            xs.copy_(x)
            g.replay()
            torch.cuda.synchronize()
            assert torch.equal(out_g, model.separate_track(x, 3000))


@pytest.mark.parametrize("mode", MODES)
def test_against_reference_golden(golden_dir, mode):
    import os
    r = torch.load(os.path.join(golden_dir, "tiny_stereo_track.pt"), weights_only=False)
    cfg = O.OracleConfig(**r["cfg"])
    model = _build(cfg, O.synth_state_dict(cfg, seed=r["wseed"]), math=mode)
    x = r["mixture"].cuda()
    for layout, hop in (("tester", None), ("crossfaded", r["hop"])):
        with torch.no_grad():
            out = model.separate_track(x, r["segment"], hop=hop)
        assert out.shape == r[layout]["out64"].shape
        torch.testing.assert_close(out.cpu().double(), r[layout]["out64"], rtol=RTOL, atol=ATOL)


def test_recipe_size_track():
    """one 240 s stereo track at 44.1 kHz through the recipe's separator on 8 s segments"""
    cfg = O.OracleConfig(n_basis=256, kernel_size=20, sep_hidden_channels=512, sep_bottleneck_channels=256, sep_skip_channels=128,
                         sep_num_blocks=4, sep_num_layers=10, causal=False, n_sources=4, in_channels=2)
    model = _build(cfg, O.synth_state_dict(cfg, seed=58), math="f16x3" if "f16x3" in MODES else "fp32")
    sr, segment = 44100, 8 * 44100
    T = 240 * sr + 1234
    x = _track(1, 2, T, segment, seed=59).cuda()
    c = model.native_config()
    need, fwd = C.c_size_t(0), C.c_size_t(0)
    N.check(N.ctn_separate_track_workspace_bytes(C.byref(c), 1, T, segment, 0, 3, C.byref(need)))
    N.check(N.ctn_workspace_bytes(C.byref(c), 3, segment, C.byref(fwd)))
    assert fwd.value < 8e9 and need.value < 8.3e9                   # the figures of separate_track's docstring
    out = _call(model, x, segment)
    assert out.shape == (1, 4, 2, T) and bool(torch.isfinite(out).all())
    ref, mag = _steps(model, x, segment, None)
    err = (out.cpu().double() - ref).abs()
    assert bool((err <= R.ola_bound(ref, mag)).all()), float(err.max())
