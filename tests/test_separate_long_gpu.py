"""ConvTasNet.separate_long on the GPU (``-m gpu``).

The three post-processing entry points (ctn_chunk_gather / ctn_chunk_align / ctn_chunk_overlap_add) run on synthetic chunk
estimates against slicing, planted permutations and the float64 restatement (separate_long_ref.py).  The whole call is
compared with that restatement fed with the estimates the existing forward gives for the same chunks, at the forward's own
tolerance (rtol 1e-4 / atol 2e-5), with identical permutations."""
import ctypes as C

import pytest
import torch

import convtasnet_oracle as O
import separate_long_ref as R
from ctn_b200 import _native as N
from test_parity_gpu import MODES, build_model

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 2e-5


def _stream():
    return N.stream_ptr(torch.device("cuda", torch.cuda.current_device()))


def _gather(x, chunk, hop, first, n):
    B, _, T = x.shape
    xc = torch.full((n, 1, min(chunk, T)), float("nan"), device="cuda")
    N.check(N.ctn_chunk_gather(x.data_ptr(), B, T, chunk, hop, first, n, xc.data_ptr(), _stream()), "ctn_chunk_gather")
    return xc


def _align(est, B, T, chunk, hop):
    S = est.shape[1]
    K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
    perms = torch.full((B, K, S), -1, dtype=torch.int32, device="cuda")
    nbytes = N.ctn_chunk_align_scratch_bytes(B, S, T, chunk, hop)
    scratch = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device="cuda")
    N.check(N.ctn_chunk_align(est.data_ptr(), B, S, T, chunk, hop, perms.data_ptr(), scratch.data_ptr(), nbytes, _stream()), "ctn_chunk_align")
    return perms


def _ola(est, perms, B, T, chunk, hop):
    S = est.shape[1]
    out = torch.full((B, S, T), float("nan"), device="cuda")
    N.check(N.ctn_chunk_overlap_add(est.data_ptr(), N.ptr(perms), B, S, T, chunk, hop, out.data_ptr(), _stream()), "ctn_chunk_overlap_add")
    return out


def _cut(sig, chunk, hop):
    """sig (B, S, T) -> (B*K, S, Lc), chunk index b*K + k"""
    starts, Lc = R.plan(sig.shape[-1], chunk, hop)
    return torch.stack([sig[b, :, s0:s0 + Lc] for b in range(sig.shape[0]) for s0 in starts]).contiguous()


# (T, chunk, hop): regular; odd sizes and an uneven last overlap; 16-byte aligned rows; several scoring CTAs per pair (chunk >
# 4096); three chunks over one sample (the last chunk reaches back past chunk K-2's start); T < chunk; hop == chunk
GEOMS = [(1000, 100, 50), (977, 101, 77), (4096 + 512, 1024, 512), (30011, 9000, 4500), (1130, 100, 50), (50, 100, 50)]


@pytest.mark.parametrize("T,chunk,hop", GEOMS + [(1000, 100, 100)])
@pytest.mark.parametrize("B", [1, 3])
def test_gather_is_slicing(B, T, chunk, hop):
    x = torch.randn(B, 1, T, device="cuda")
    starts, Lc = R.plan(T, chunk, hop)
    ref = _cut(x, chunk, hop)
    K = len(starts)
    assert torch.equal(_gather(x, chunk, hop, 0, B * K), ref)
    if B * K > 2:
        assert torch.equal(_gather(x, chunk, hop, 1, B * K - 2), ref[1:-1])
    # a base that is only 4-byte aligned
    y = torch.randn(B * T + 1, device="cuda")[1:].reshape(B, 1, T)
    assert torch.equal(_gather(y, chunk, hop, 0, B * K), _cut(y, chunk, hop))


@pytest.mark.parametrize("T,chunk,hop", GEOMS)
@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6])
def test_align_recovers_planted_permutations(S, T, chunk, hop):
    B = 2
    g = torch.Generator().manual_seed(1000 * S + T)
    src = torch.randn(B, S, T, generator=g)
    starts, Lc = R.plan(T, chunk, hop)
    K = len(starts)
    est = torch.empty(B * K, S, Lc)
    want = torch.empty(B, K, S, dtype=torch.int32)
    for b in range(B):
        q0 = None
        for k, s0 in enumerate(starts):
            q = torch.randperm(S, generator=g)                   # row r of this chunk carries source q[r]
            est[b * K + k] = src[b, q, s0:s0 + Lc]
            q0 = q if k == 0 else q0
            inv = torch.argsort(q)
            want[b, k] = inv[q0].to(torch.int32)                 # output source s = what row s of chunk 0 carries
    est = est.cuda()
    perms = _align(est, B, T, chunk, hop)
    assert torch.equal(perms.cpu(), want)
    ref_out, ref_perms = R.separate(est.cpu(), B, T, chunk, hop)
    assert torch.equal(perms.cpu().long(), ref_perms)
    # and the aligned chunks reassemble the sources in chunk 0's order
    out = _ola(est, perms, B, T, chunk, hop).cpu()
    for b in range(B):
        assert torch.equal(out[b, :, :8], est[b * K, :, :8].cpu())
    torch.testing.assert_close(out.double(), ref_out, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("S", [2, 3, 6])
def test_align_ties_take_the_first_permutation(S):
    T, chunk, hop, B = 1000, 100, 50, 2
    one = torch.randn(B, 1, T, device="cuda").expand(B, S, T).contiguous()     # every source the same: every permutation ties
    K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
    ident = torch.arange(S, dtype=torch.int32).expand(B, K, S)
    assert torch.equal(_align(_cut(one, chunk, hop), B, T, chunk, hop).cpu(), ident)
    assert torch.equal(_align(torch.zeros(B * K, S, chunk, device="cuda"), B, T, chunk, hop).cpu(), ident)
    # sources 0 and 1 the same, the rest distinct and swapped in every odd chunk: the tie between rows 0 and 1 keeps their order
    if S == 6:
        sig = torch.randn(B, S, T, device="cuda")
        sig[:, 1] = sig[:, 0]
        est = _cut(sig, chunk, hop).reshape(B, K, S, chunk)
        odd = list(range(S))
        odd[-1], odd[-2] = odd[-2], odd[-1]
        est[:, 1::2] = est[:, 1::2][:, :, odd]
        perms = _align(est.reshape(B * K, S, chunk).contiguous(), B, T, chunk, hop).cpu()
        for k in range(K):
            want = odd if k % 2 else list(range(S))
            assert perms[0, k].tolist() == want and perms[1, k].tolist() == want


@pytest.mark.parametrize("T,chunk,hop", GEOMS + [(1000, 100, 100), (1001, 100, 100), (9, 3, 1)])
@pytest.mark.parametrize("S", [1, 2, 7])
def test_overlap_add_vs_fp64(S, T, chunk, hop):
    B = 2
    g = torch.Generator().manual_seed(7 * T + S)
    starts, Lc = R.plan(T, chunk, hop)
    K = len(starts)
    est = torch.randn(B * K, S, Lc, generator=g)
    perms = torch.stack([torch.randperm(S, generator=g) for _ in range(B * K)]).reshape(B, K, S)
    out = _ola(est.cuda(), perms.to(torch.int32).cuda(), B, T, chunk, hop).cpu()
    out_id = _ola(est.cuda(), None, B, T, chunk, hop).cpu()
    for b in range(B):
        e = est[b * K:(b + 1) * K]
        ref = R.overlap_add(e, [tuple(p.tolist()) for p in perms[b]], starts, Lc, T)
        torch.testing.assert_close(out[b].double(), ref, rtol=1e-6, atol=1e-6 * float(ref.abs().max()))
        ref = R.overlap_add(e, None, starts, Lc, T)
        torch.testing.assert_close(out_id[b].double(), ref, rtol=1e-6, atol=1e-6 * float(ref.abs().max()))
    # where one chunk covers a sample its weight is exactly one: both ends of the recording are copies
    head = min(hop, T) if K > 1 else T
    assert torch.equal(out_id[0, :, :1], est[0, :, :1])
    if K > 1 and hop == chunk:
        assert torch.equal(out_id[0, :, :head], est[0, :, :head])
    assert torch.equal(out_id[:, :, -1], torch.stack([est[b * K + K - 1, :, -1] for b in range(B)]))


@pytest.mark.parametrize("T,chunk,hop", GEOMS + [(1001, 100, 100), (9, 3, 1)])
def test_chunks_of_one_signal_reassemble_it(T, chunk, hop):
    """the weights over every sample sum to one, also where three chunks cover it"""
    B, S = 2, 2
    sig = torch.randn(B, S, T, device="cuda") * 3.0 + 0.5
    out = _ola(_cut(sig, chunk, hop), None, B, T, chunk, hop)
    assert bool(((out - sig).abs() <= 2e-7 * sig.abs()).all())
    starts, Lc = R.plan(T, chunk, hop)
    cover = (R.weights(starts, Lc, T) > 0).sum(0)
    assert int(cover.min()) >= 1
    if (T, chunk, hop) == (1130, 100, 50):
        assert int(cover.max()) == 3


def test_steps_are_deterministic():
    B, S, T, chunk, hop = 2, 3, 30011, 9000, 4500
    K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
    est = torch.randn(B * K, S, chunk, device="cuda")
    p1, p2 = _align(est, B, T, chunk, hop), _align(est, B, T, chunk, hop)
    assert torch.equal(p1, p2)
    assert torch.equal(_ola(est, p1, B, T, chunk, hop), _ola(est, p2, B, T, chunk, hop))


# ---- the whole call -------------------------------------------------------------------------------------------------------------
SMALL = dict(n_basis=64, kernel_size=16, sep_hidden_channels=128, sep_bottleneck_channels=32, sep_skip_channels=32, sep_num_blocks=2,
             sep_num_layers=3)
CONFIGS = {
    "small_gln": dict(SMALL, causal=False, n_sources=2),
    "small_gln_3spk": dict(SMALL, causal=False, n_sources=3, enc_nonlinear="relu"),
    "small_cln": dict(SMALL, causal=True, n_sources=2),
    "small_softmax": dict(SMALL, causal=False, n_sources=2, mask_nonlinear="softmax"),
    "paper": dict(causal=False, n_sources=2),       # N = 512, B = 128, H = 512, Sc = 128, P = 3, X = 8, R = 3
}


def _reference(model, x, chunk, hop, align=True):
    """the restatement fed with the estimates the plain forward gives for the same chunks"""
    B, _, T = x.shape
    with torch.no_grad():
        est = model(_cut(x, chunk, hop))
    return R.separate(est.cpu(), B, T, chunk, hop, do_align=align)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(CONFIGS))
def test_whole_call_vs_restatement(name, mode):
    cfg = O.OracleConfig(**CONFIGS[name])
    model = build_model(cfg, O.synth_state_dict(cfg, seed=41), math=mode)
    B, T, chunk, hop = 2, 14321, 4000, 2000
    x = O.synth_batch(B, cfg.n_sources, T, seed=42)[0].cuda()
    ref, ref_perms = _reference(model, x, chunk, hop)
    with torch.no_grad():
        out = model.separate_long(x, chunk, chunk_batch=5)
    assert out.shape == (B, cfg.n_sources, T)
    assert torch.equal(model.last_chunk_perms.cpu().long(), ref_perms)
    torch.testing.assert_close(out.cpu().double(), ref, rtol=RTOL, atol=ATOL)
    assert model.last_launches > 0
    # an uneven hop, no alignment
    ref, ref_perms = _reference(model, x, chunk, 3100, align=False)
    with torch.no_grad():
        out = model.separate_long(x, chunk, hop=3100, align=False)
    assert torch.equal(model.last_chunk_perms.cpu().long(), ref_perms)
    torch.testing.assert_close(out.cpu().double(), ref, rtol=RTOL, atol=ATOL)


def _small(mode="fp32", **kw):
    cfg = O.OracleConfig(**dict(CONFIGS["small_gln"], **kw))
    return cfg, build_model(cfg, O.synth_state_dict(cfg, seed=43), math=mode)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("T", [4000, 3999, 1234])
def test_short_input_is_the_plain_forward(mode, T):
    cfg, model = _small(mode)
    x = O.synth_batch(3, 2, T, seed=T)[0].cuda()
    with torch.no_grad():
        want = model(x)
        assert torch.equal(model.separate_long(x, 4000), want)
        assert torch.equal(model.last_chunk_perms.cpu(), torch.arange(2, dtype=torch.int32).expand(3, 1, 2))
        assert torch.equal(model.separate_long(x, 4000, hop=4000, align=False), want)


def test_chunk_batch_does_not_change_the_result():
    cfg, model = _small()
    x = O.synth_batch(2, 2, 21000, seed=5)[0].cuda()
    with torch.no_grad():
        base = model.separate_long(x, 4000, chunk_batch=16)
        perms = model.last_chunk_perms.clone()
        for cb in (1, 3, 1000):
            out = model.separate_long(x, 4000, chunk_batch=cb)
            assert torch.equal(model.last_chunk_perms, perms)
            torch.testing.assert_close(out, base, rtol=RTOL, atol=ATOL)


def test_recordings_of_a_batch_do_not_interact():
    cfg, model = _small()
    x = O.synth_batch(3, 2, 15000, seed=6)[0].cuda()
    with torch.no_grad():
        out = model.separate_long(x, 4000, chunk_batch=4)
        perms = model.last_chunk_perms.clone()
        for b in range(3):
            alone = model.separate_long(x[b:b + 1].clone(), 4000, chunk_batch=4)
            assert torch.equal(model.last_chunk_perms[0], perms[b])
            torch.testing.assert_close(alone[0], out[b], rtol=RTOL, atol=ATOL)


@pytest.mark.parametrize("mode", MODES)
def test_second_call_gives_the_same_bits(mode):
    cfg, model = _small(mode)
    x = O.synth_batch(2, 2, 15000, seed=7)[0].cuda()
    with torch.no_grad():
        a = model.separate_long(x, 4000)
        pa = model.last_chunk_perms
        b = model.separate_long(x, 4000)
    assert torch.equal(a, b) and torch.equal(pa, model.last_chunk_perms)


def test_enhancement_model_skips_alignment():
    cfg, model = _small(n_sources=1)
    x = O.synth_batch(2, 1, 15000, seed=8)[0].cuda()
    ref, _ = _reference(model, x, 4000, 2000)
    with torch.no_grad():
        a = model.separate_long(x, 4000)
        b = model.separate_long(x, 4000, align=False)
    assert torch.equal(a, b)
    torch.testing.assert_close(a.cpu().double(), ref, rtol=RTOL, atol=ATOL)


def test_call_is_cuda_graph_capturable():
    """every launch on the caller's stream, nothing read back: capture once, replay on new input"""
    cfg, model = _small()
    x1 = O.synth_batch(2, 2, 15000, seed=9)[0].cuda()
    x2 = O.synth_batch(2, 2, 15000, seed=10)[0].cuda()
    xs = x1.clone()
    side = torch.cuda.Stream()
    with torch.no_grad():
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                model.separate_long(xs, 4000)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side):
            out_g = model.separate_long(xs, 4000)
            perms_g = model.last_chunk_perms
        for x in (x2, x1):
            xs.copy_(x)
            g.replay()
            torch.cuda.synchronize()
            out_e = model.separate_long(x, 4000)
            assert torch.equal(perms_g, model.last_chunk_perms)
            torch.testing.assert_close(out_g, out_e, rtol=0, atol=1e-6)


def test_ten_minutes_at_paper_size():
    cfg = O.OracleConfig(causal=False, n_sources=2)
    model = build_model(cfg, O.synth_state_dict(cfg, seed=111))
    B, T, chunk, hop, cb = 1, 600 * 8000, 32000, 16000, 16
    x = O.synth_batch(B, 2, T, seed=11)[0].cuda()
    with torch.no_grad():
        out = model.separate_long(x, chunk, hop, chunk_batch=cb)
    assert out.shape == (B, 2, T) and bool(torch.isfinite(out).all())
    K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
    assert K == 299 and model.last_chunk_perms.shape == (B, K, 2)
    c = model.native_config()
    need, fwd, whole = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    N.check(N.ctn_separate_long_workspace_bytes(C.byref(c), B, T, chunk, hop, cb, C.byref(need)))
    N.check(N.ctn_workspace_bytes(C.byref(c), cb, chunk, C.byref(fwd)))
    N.check(N.ctn_workspace_bytes(C.byref(c), B, T, C.byref(whole)))
    # one batch of chunks of model workspace + the chunk estimates, against a workspace that grows with every frame of T
    assert need.value <= fwd.value + 4 * (cb * chunk + B * K * 2 * chunk) + (1 << 20)
    assert whole.value > 0.9 * fwd.value * T / (cb * chunk)
    assert need.value * 8 < whole.value


def test_error_paths():
    cfg, model = _small()
    x = O.synth_batch(1, 2, 9000, seed=12)[0]
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            model.separate_long(x, 4000)
        with pytest.raises(NotImplementedError):
            model.separate_long(x.cuda().unsqueeze(2), 4000)
        for kw in (dict(hop=1999), dict(hop=4001), dict(hop=4000)):     # the last: alignment needs chunks that share samples
            with pytest.raises(ValueError):
                model.separate_long(x.cuda(), 4000, **kw)
        with pytest.raises(ValueError):
            model.separate_long(x.cuda(), 0)
    with pytest.raises(NotImplementedError):
        model.separate_long(x.cuda(), 4000)                                 # autograd on, parameters require grad
    cfg7 = O.OracleConfig(**dict(CONFIGS["small_gln"], n_sources=7))
    m7 = build_model(cfg7, O.synth_state_dict(cfg7, seed=3), math="fp32")
    x7 = O.synth_batch(1, 7, 9000, seed=13)[0].cuda()
    with torch.no_grad():
        with pytest.raises(NotImplementedError):
            m7.separate_long(x7, 4000)
        out = m7.separate_long(x7, 4000, align=False)                       # overlap-add alone takes any number of sources
    assert out.shape == (1, 7, 9000) and bool(torch.isfinite(out).all())
