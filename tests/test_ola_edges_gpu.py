"""separate_long's and separate_track's chunk steps at their edges on the GPU (``-m gpu``), against float64 (ola_edges_ref.py).

The step entries run directly with NaN-filled outputs.  Every row stays within its bound of fp64 (permutations exactly), repeats
bit for bit on a second call and launches the count the routing predicts; one past each grid limit is refused before any launch.
Rows: alignment across compose tiles (K - 1 up to 21845 at B = 3: 65535 scoring pairs), every scoring split with planted, last-
slice-only, tied and near-tied permutations, the overlap-add where the most chunks meet and in short plans, the statistics at
every split under a DC offset, a first-sample outlier, silence and a one-sample last segment, one alignment + overlap-add whose
chunk estimates pass 2^31 elements, and whole calls at the chunk-batch caps with a tiny model in every math mode.  Each test
prints its worst error / bound and the branch its row names."""

import pytest
import torch

import convtasnet_oracle as O
import gln_forward_edges_ref as GR
import ola_edges_ref as R
import separate_track_ref as ST
import test_separate_long_gpu as LG
import test_separate_track_gpu as TG
from ctn_b200 import _native as N
from test_parity_gpu import build_model

pytestmark = pytest.mark.gpu

MODES = ["fp32"] + (["tf32x3", "f16x3", "tf32"] if N.ctn_has_tcgen05() else [])


def _report(family, row, worst, reaches):
    print("[ola edges {}] {}: {:.3g} of bound ({})".format(family, row, worst, reaches))


def _launches():
    return N.ctn_last_launch_count()


def _align(est, B, T, chunk, hop):
    perms = LG._align(est, B, T, chunk, hop)
    return perms, _launches()


def _ola_long(est, perms, B, T, chunk, hop):
    out = LG._ola(est, perms, B, T, chunk, hop)
    return out, _launches()


# ---- 1. alignment across compose tiles ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ALIGN))
def test_align_across_tiles(name):
    r = R.ALIGN[name]
    K, Lc, starts = R.chunk_plan(r.T, r.chunk, r.hop)
    g = torch.Generator().manual_seed(K * 10 + r.S)
    est = torch.empty(r.B * K, r.S, Lc)
    want = torch.empty(r.B, K, r.S, dtype=torch.int64)
    for b in range(r.B):
        src = torch.randn(r.S, r.T, generator=g)
        q = R.plant_perms(K, r.S, seed=100 * b + r.S)
        est[b * K:(b + 1) * K] = R.planted_est(src, q, starts, Lc)
        want[b] = R.planted_want(q)
    ed = est.cuda()
    perms, n = _align(ed, r.B, r.T, r.chunk, r.hop)
    assert n == R.align_launches(r.S, K)
    assert torch.equal(perms.cpu().long(), want)
    assert torch.equal(_align(ed, r.B, r.T, r.chunk, r.hop)[0], perms)
    out, n = _ola_long(ed, perms, r.B, r.T, r.chunk, r.hop)
    assert n == R.OLA_LAUNCHES
    assert torch.equal(_ola_long(ed, perms, r.B, r.T, r.chunk, r.hop)[0], out)
    out = out.cpu().double()
    worst = 0.0
    for b in range(r.B):
        ref, mag = R.overlap_add(est[b * K:(b + 1) * K], want[b], starts, Lc, r.hop, r.T)
        worst = max(worst, R.share((out[b] - ref).abs(), ST.ola_bound(ref, mag)))
    assert worst <= 1.0
    _report("align", name, worst, r.reaches)


# ---- 2. every scoring split -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.SCORE))
def test_scoring_splits(name):
    r = R.SCORE[name]
    K, Lc, starts = R.chunk_plan(r.T, r.chunk, r.hop)
    g = torch.Generator().manual_seed(Lc + r.S)
    src = torch.randn(r.S, r.T, generator=g)
    q = R.plant_perms(K, r.S, seed=Lc + r.S)
    want = R.planted_want(q)
    cases = {"planted": R.planted_est(src, q, starts, Lc),
             "last slice decides": R.planted_est(R.last_slice_decides(src, starts, Lc), q, starts, Lc)}
    # near tie: rows 0 and 1 differ by 1e-3 (relative 1e-6 of the scores); exact tie: every source the same
    near = src.clone()
    near[1] = near[0] + 1e-3 * torch.randn(r.T, generator=g)
    cases["near tie"] = R.planted_est(near, q, starts, Lc)
    same = src[:1].expand(r.S, r.T)
    cases["exact tie"] = R.planted_est(same, q, starts, Lc)
    for case, est in cases.items():
        ed = est.cuda()
        perms, n = _align(ed, 1, r.T, r.chunk, r.hop)
        assert n == 2
        got = perms.cpu()[0].long()
        expect = torch.arange(r.S).expand(K, r.S) if case == "exact tie" else want
        assert torch.equal(got, expect), case
        assert torch.equal(got, R.align(est, starts, Lc)), case
        assert torch.equal(_align(ed, 1, r.T, r.chunk, r.hop)[0], perms)
    _report("score", name, 0.0, r.reaches + "; permutations exact")


# ---- 3. one past each grid limit: refused with zero launches ---------------------------------------------------------------------
def _refuse(entry, a):
    dummy = torch.zeros(1024, device="cuda")
    d64 = torch.zeros(1024, dtype=torch.float64, device="cuda")
    st = LG._stream()
    if entry == "ctn_chunk_align":
        nbytes = N.ctn_chunk_align_scratch_bytes(a["B"], min(a["S"], 6), a["T"], a["chunk"], a["hop"])
        scratch = torch.empty(nbytes // 8 + 1, dtype=torch.float64, device="cuda")
        perms = torch.empty(8, dtype=torch.int32, device="cuda")
        return N.ctn_chunk_align(dummy.data_ptr(), a["B"], a["S"], a["T"], a["chunk"], a["hop"], perms.data_ptr(),
                                 scratch.data_ptr(), nbytes, st)
    if entry == "ctn_chunk_gather":
        return N.ctn_chunk_gather(dummy.data_ptr(), a["B"], a["T"], a["chunk"], a["hop"], 0, a["n"], dummy.data_ptr(), st)
    if entry == "ctn_track_stats":
        return N.ctn_track_stats(dummy.data_ptr(), a["B"], a["C"], a["T"], a["segment"], a["hop"], d64.data_ptr(), d64.data_ptr(),
                                 1 << 30, st)
    if entry == "ctn_track_gather":
        return N.ctn_track_gather(dummy.data_ptr(), d64.data_ptr(), a["B"], a["C"], a["T"], a["segment"], a["hop"], 1e-12, 0, a["n"],
                                  dummy.data_ptr(), st)
    return N.ctn_track_overlap_add(dummy.data_ptr(), d64.data_ptr(), a["B"], a["S"], a["C"], a["T"], a["segment"], a["hop"],
                                   dummy.data_ptr(), st)


@pytest.mark.parametrize("name", list(R.REFUSE))
def test_refused_before_any_launch(name):
    r = R.REFUSE[name]
    rc = _refuse(r.entry, r.args)
    assert rc == getattr(N, "CTN_" + r.code), (name, rc)
    assert _launches() == 0
    _report("refuse", name, 0.0, r.reaches)


def test_grid_limits_themselves_are_accepted():
    """the last accepted size of each limit runs and is right: a 65535-chunk gather, n C = 65535 track rows, B C = 65535"""
    T, chunk, hop = 32 + 16 * 65535, 32, 16
    x = torch.randn(1, 1, T, device="cuda")
    xc = LG._gather(x, chunk, hop, 1, 65535)
    assert _launches() == R.GATHER_LAUNCHES
    starts = R.chunk_plan(T, chunk, hop)[2]
    idx = torch.tensor(starts[1:65536], device="cuda")[:, None] + torch.arange(chunk, device="cuda")
    assert torch.equal(xc[:, 0], x[0, 0][idx])
    # n C = 65535 (C = 3, n = 21845) and B C = 65535 (B = 21845, C = 3), tester layout
    Cn, seg = 3, 4
    xt = torch.randn(1, Cn, seg * 21845, device="cuda")
    st = TG._stats(xt, seg, None)
    g = TG._gather(xt, st, seg, None, 0, 21845)
    assert _launches() == R.GATHER_LAUNCHES
    x64 = xt.cpu().double().reshape(Cn, 21845, seg).transpose(0, 1)
    st64 = st.cpu()[0]
    want = ST.standardise(x64, st64)
    assert bool(((g.cpu().double() - want).abs() <= ST.gather_bound(x64, st64)).all())
    Bt = 21845
    est = torch.randn(Bt, 1, Cn, seg, device="cuda")
    sts = torch.stack([torch.randn(Bt, 1, Cn, dtype=torch.float64), torch.rand(Bt, 1, Cn, dtype=torch.float64) * 3], -1).cuda()
    out = TG._ola(est, sts, Bt, seg, seg, None)
    assert _launches() == R.OLA_LAUNCHES
    ref = sts[..., 1].cpu()[:, 0, None, :, None] * est.cpu().double() + sts[..., 0].cpu()[:, 0, None, :, None]
    mag = (sts[..., 1].cpu()[:, 0, None, :, None] * est.cpu().double()).abs() + sts[..., 0].cpu()[:, 0, None, :, None].abs()
    assert bool(((out.cpu().double() - ref).abs() <= ST.ola_bound(ref, mag)).all())


# ---- 4. the overlap-add where the most chunks meet, and short plans ------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.OLA))
@pytest.mark.parametrize("S", R.OLA_S)
def test_overlap_add_edges(name, S):
    r = R.OLA[name]
    K, Lc, starts = R.chunk_plan(r.T, r.chunk, r.hop)
    B = 2
    g = torch.Generator().manual_seed(r.T + S)
    est = torch.randn(B * K, S, Lc, generator=g)
    perms = torch.stack([torch.randperm(S, generator=g) for _ in range(B * K)]).reshape(B, K, S)
    ed, pd = est.cuda(), perms.to(torch.int32).cuda()
    worst = 0.0
    for p in (pd, None):
        out, n = _ola_long(ed, p, B, r.T, r.chunk, r.hop)
        assert n == R.OLA_LAUNCHES
        assert torch.equal(_ola_long(ed, p, B, r.T, r.chunk, r.hop)[0], out)
        out = out.cpu().double()
        for b in range(B):
            ref, mag = R.overlap_add(est[b * K:(b + 1) * K], None if p is None else perms[b], starts, Lc, r.hop, r.T)
            worst = max(worst, R.share((out[b] - ref).abs(), ST.ola_bound(ref, mag)))
    assert worst <= 1.0
    _report("ola", "{} S={}".format(name, S), worst, r.reaches)


# ---- 5. statistics at every split -------------------------------------------------------------------------------------------------
def _stats_track(r, seed):
    """(1, C, 3 segment + 1): segment 0 a DC of 1e4 with std 1e-2, segment 1 unit noise whose first sample is 1e3, segment 2
    silent, segment 3 one valid sample (then segment - 1 zeros of padding); the last channel silent throughout when C > 1"""
    g = torch.Generator().manual_seed(seed)
    seg = r.segment
    x = torch.empty(1, r.C, r.T)
    x[:, :, :seg] = 1e4 + 1e-2 * torch.randn(1, r.C, seg, generator=g)
    x[:, :, seg:2 * seg] = torch.randn(1, r.C, seg, generator=g)
    x[:, :, seg] = 1e3
    x[:, :, 2 * seg:3 * seg] = 0.0
    x[:, :, 3 * seg] = 0.7
    if r.C > 1:
        x[:, -1] = 0.0
    return x


@pytest.mark.parametrize("name", list(R.STATS))
def test_stats_edges(name):
    r = R.STATS[name]
    K, Lc, starts = R.track_plan(r.T, r.segment, 0)
    x = _stats_track(r, seed=r.segment + r.C)
    xd = x.cuda()
    st = TG._stats(xd, r.segment, None)
    assert _launches() == R.TRACK_STATS_LAUNCHES
    assert torch.equal(TG._stats(xd, r.segment, None), st)
    xc = TG._gather(xd, st, r.segment, None, 0, K)
    assert _launches() == R.GATHER_LAUNCHES
    assert torch.equal(TG._gather(xd, st, r.segment, None, 0, K), xc)
    S = 1 if r.C == 64 else 2
    g = torch.Generator().manual_seed(r.C)
    est = torch.randn(K, S, r.C, Lc, generator=g)
    out = TG._ola(est.cuda(), st, 1, r.T, r.segment, None)
    assert _launches() == R.OLA_LAUNCHES
    assert torch.equal(TG._ola(est.cuda(), st, 1, r.T, r.segment, None), out)
    st, xc, out = st.cpu()[0], xc.cpu(), out.cpu()[0]
    w_stats = w_gather = w_ola = 0.0
    for c in range(r.C):
        x64 = ST.chunks(x[:, c:c + 1].double(), starts, Lc)                   # (K, 1, Lc)
        ref = R.stats64(x64)
        bound = ST.stats_bounds(x64)
        w_stats = max(w_stats, R.share((st[:, c:c + 1] - ref).abs(), bound))
        y = ST.standardise(x64, st[:, c:c + 1])
        w_gather = max(w_gather, R.share((xc[:, c:c + 1].double() - y).abs(), ST.gather_bound(x64, st[:, c:c + 1])))
        o64, mag = ST.overlap_add(est[:, :, c:c + 1], st[:, c:c + 1], starts, Lc, r.T, False, magnitude=True)
        w_ola = max(w_ola, R.share((out[:, c:c + 1].double() - o64).abs(), ST.ola_bound(o64, mag)))
    # silence: mean and std exactly 0, the gather exact zeros, the overlap-add the mean (0) exactly
    assert bool((st[2] == 0).all()) and bool((xc[2] == 0).all()) and bool((out[:, :, 2 * r.segment:3 * r.segment] == 0).all())
    if r.C > 1:
        assert bool((st[:, -1] == 0).all()) and bool((xc[:, -1] == 0).all()) and bool((out[:, -1] == 0).all())
    assert max(w_stats, w_gather, w_ola) <= 1.0, (w_stats, w_gather, w_ola)
    _report("stats", name, w_stats, r.reaches + "; gather {:.3g}, overlap-add {:.3g}".format(w_gather, w_ola))


# ---- 6. chunk estimates past 2^31 elements ----------------------------------------------------------------------------------------
def test_estimates_past_2_31_elements():
    fig = R.big_figures()
    S, T, chunk, hop = R.BIG["S"], R.BIG["T"], R.BIG["chunk"], R.BIG["hop"]
    K, Lc, starts = fig["K"], fig["Lc"], fig["starts"]
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    gen = torch.Generator(device="cuda").manual_seed(61)
    src = torch.randn(S, T, device="cuda", generator=gen)
    q = R.plant_perms(K, S, seed=61)
    want = R.planted_want(q)
    est = torch.empty(K, S, Lc, device="cuda")
    U = src.unfold(1, Lc, hop)                                           # (S, regular starts, Lc) view
    qd = q.cuda()
    for k0 in range(0, K - 1, 512):
        k1 = min(K - 1, k0 + 512)
        est[k0:k1] = U[qd[k0:k1], torch.arange(k0, k1, device="cuda")[:, None]]
    est[K - 1] = src[qd[K - 1], T - Lc:]
    perms, n = _align(est, 1, T, chunk, hop)
    assert n == 2
    assert torch.equal(perms.cpu()[0].long(), want)
    out, n = _ola_long(est, perms, 1, T, chunk, hop)
    assert n == R.OLA_LAUNCHES
    peak = torch.cuda.max_memory_allocated()
    kc = fig["k_cross"]
    windows = {"start": (0, 40000), "end": (T - 40000, T),
               "chunk {} (offset 2^31)".format(kc): (starts[kc] - 20000, starts[kc] + Lc + 20000)}
    P = perms.cpu()[0].long()
    worst = 0.0
    for wname, (t0, t1) in windows.items():
        ref, mag = R.overlap_add_window(lambda k: est[k].cpu(), P, starts, Lc, T, t0, t1)
        got = out[0, :, t0:t1].cpu().double()
        worst = max(worst, R.share((got - ref).abs(), ST.ola_bound(ref, mag)))
        # planted copies of one source: the aligned output is chunk 0's row order of src
        assert bool(((got - src[qd[0], t0:t1].cpu().double()).abs() <= 4e-7 * ref.abs() + 1e-30).all()), wname
    assert worst <= 1.0
    print("[ola edges big] K = {}, estimates {:.3g} elements ({:.2f} GB), output {:.2f} GB, source {:.2f} GB computed; torch "
          "peak allocation {:.2f} GB".format(K, fig["est_elems"], fig["est_bytes"] / 1e9, fig["out_bytes"] / 1e9,
                                            fig["src_bytes"] / 1e9, peak / 1e9))
    _report("big", "S=6 T={}".format(T), worst, "estimate offsets past 2^31 at chunk {}".format(kc))
    del est, out, src, U
    torch.cuda.empty_cache()


# ---- 7. whole calls at the chunk-batch caps ---------------------------------------------------------------------------------------
TINY = dict(n_basis=32, kernel_size=16, sep_hidden_channels=32, sep_bottleneck_channels=16, sep_skip_channels=16, sep_num_blocks=1,
            sep_num_layers=2, causal=False)


def _tol_share(got, ref, mode):
    rtol, atol = GR.tol(mode)
    if mode == "tf32":
        atol *= max(1.0, float(ref.abs().max()))
    return GR.share(got, ref, rtol, atol)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("S,align", [(1, True), (2, False)])
def test_separate_long_past_65535_chunks(mode, S, align):
    cfg = O.OracleConfig(**dict(TINY, n_sources=S))
    sd = O.synth_state_dict(cfg, seed=71)
    model = build_model(cfg, sd, math=mode)
    chunk, hop = 32, 16
    T = chunk + hop * 65535 + 5
    K, Lc, starts = R.chunk_plan(T, chunk, hop)
    assert K == 65537
    x = O.synth_batch(1, S, T, seed=72)[0].cuda()
    with torch.no_grad():
        big = model.separate_long(x, chunk, hop, chunk_batch=100000, align=align)
        n_big = model.last_launches
        small = model.separate_long(x, chunk, hop, chunk_batch=4096, align=align)
        n_small = model.last_launches
    assert torch.equal(big, small)
    assert torch.equal(model.last_chunk_perms.cpu(), torch.arange(S, dtype=torch.int32).expand(1, K, S))
    assert n_big < n_small
    sd64 = {k: v.double() for k, v in sd.items()}
    xc = x.cpu().double()[0, 0]
    worst = 0.0
    for t0, t1 in ((0, 64), (starts[65533], starts[65536] + Lc), (T - 64, T)):
        ks = [k for k, s0 in enumerate(starts) if s0 < t1 and s0 + Lc > t0]
        chunks = torch.stack([xc[starts[k]:starts[k] + Lc] for k in ks])[:, None]
        with torch.no_grad():
            e64 = O.conv_tasnet_fwd(chunks, sd64, cfg)[0]
        ref, _ = R.overlap_add_window(lambda k: e64[ks.index(k)], torch.arange(S).expand(K, S), starts, Lc, T, t0, t1)
        worst = max(worst, _tol_share(big[0, :, t0:t1].cpu(), ref, mode))
    assert worst <= 1.0
    nb = 65535 // S
    _report("whole long", "{} S={} align={}".format(mode, S, align), worst,
            "K = 65537: batches of {} chunks (chunk_batch 100000 capped at 65535 / S) and a short last one of {}".format(
                nb, K % nb))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("Cn,S", [(3, 2), (2, 4)])
def test_separate_track_at_the_batch_cap(mode, Cn, S):
    """the chunk batch is capped at 65535 / max(C, S): the gather's (chunk, channel) rows and the decoder's (chunk, source)
    rows both ride on gridDim.y"""
    cfg = O.OracleConfig(**dict(TINY, n_sources=S, in_channels=Cn))
    sd = O.synth_state_dict(cfg, seed=73)
    model = TG._build(cfg, sd, math=mode)
    seg = 32
    nb = 65535 // max(Cn, S)
    T = seg * (nb + 1) + 7
    K = R.track_plan(T, seg, 0)[0]
    assert K == nb + 2
    x = TG._track(1, Cn, T, seg, seed=74, dc=False).cuda()
    big = TG._call(model, x, seg, None, chunk_batch=100000)
    n_big = model.last_launches
    small = TG._call(model, x, seg, None, chunk_batch=4096)
    assert torch.equal(big, small)
    assert n_big < model.last_launches
    sd64 = {k: v.double() for k, v in sd.items()}
    worst = 0.0
    for k in (0, nb - 1, nb, nb + 1):
        x64 = ST.chunks(x[:, :, k * seg:(k + 1) * seg].cpu().double(), [0], seg)          # (1, C, seg), zeros past T
        st = ST.stats(x64)
        with torch.no_grad():
            e64 = O.conv_tasnet_fwd(ST.standardise(x64, st, cfg.eps)[:, None], sd64, cfg)[0][0]   # (S, C, seg)
        ref = st[0, :, 1][None, :, None] * e64 + st[0, :, 0][None, :, None]
        n = min(seg, T - k * seg)
        worst = max(worst, _tol_share(big[0, :, :, k * seg:k * seg + n].cpu(), ref[..., :n], mode))
    assert worst <= 1.0
    _report("whole track", "{} C={} S={}".format(mode, Cn, S), worst,
            "K = {}: a {}-segment batch (65535 / max(C, S)) and a batch of 2".format(K, nb))
