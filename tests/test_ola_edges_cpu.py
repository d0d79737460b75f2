"""The rows of tests/test_ola_edges_gpu.py without a GPU: each reaches the branch its `reaches` text names by the restated routing
(ola_edges_ref.py), the kernel-order restatements agree with separate_long_ref.py / separate_track_ref.py, and each check rejects
a planted defect: compose losing its carry across tiles, the scoring dropping its last partial, the statistics losing their
shift or dividing by n, the ramps losing their half-sample offset, and the overlap-add skipping a covering chunk."""
import pytest
import torch

import ola_edges_ref as R
import separate_long_ref as SL
import separate_track_ref as ST


# ---- routing -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ALIGN))
def test_align_row_reaches(name):
    r = R.ALIGN[name]
    K, _, _ = R.chunk_plan(r.T, r.chunk, r.hop)
    got = R.reached_align(r)
    assert r.B * (K - 1) <= R.GRID_Y
    pairs = int(name.split("_")[0][1:])
    assert K - 1 == pairs
    if pairs > 256:
        assert "r loop past 256" in got
    if pairs > R.OLA_TILE:
        assert "tiles={}".format(R.ceil_div(pairs, R.OLA_TILE)) in got and "short last tile" in got
    if "65535" in r.reaches:
        assert "grid y = 65535" in got


def test_align_rows_cover_every_tile_count():
    tiles = set().union(*(R.reached_align(r) for r in R.ALIGN.values()))
    assert {"tiles=1", "tiles=2", "tiles=3", "tiles=22", "r loop past 256", "short last tile", "grid y = 65535"} <= tiles
    assert {r.S for r in R.ALIGN.values()} == {2, 3, 4, 5, 6}


@pytest.mark.parametrize("name", list(R.SCORE))
def test_score_row_reaches(name):
    r = R.SCORE[name]
    assert R.chunk_plan(r.T, r.chunk, r.hop) is not None
    got = R.reached_score(r)
    assert "G={}".format(int(r.reaches.split("G = ")[1].split()[0].rstrip(","))) in got
    assert "ov > G 256" in got
    if name.endswith("_edge") and R.score_split(r.chunk) > 1:
        assert "short last slice" in got


def test_score_rows_cover_every_split():
    got = set().union(*(R.reached_score(r) for r in R.SCORE.values()))
    assert {"G=1", "G=2", "G=8", "G=16", "short last slice", "slice > 4096"} <= got
    assert R.score_split(61440) == 15 and R.score_split(61441) == 16 and R.score_split(10 ** 6) == 16


@pytest.mark.parametrize("name", list(R.STATS))
def test_stats_row_reaches(name):
    r = R.STATS[name]
    K, Lc, starts = R.track_plan(r.T, r.segment, 0)
    assert K == 4 and r.T - starts[-1] == 1                       # the last segment: one valid sample, segment - 1 zeros
    G = R.stats_split(Lc)
    assert "G = {}".format(G) in r.reaches
    assert R.ceil_div(Lc, G) > R.TRACK_SLICE if G == R.TRACK_MAX_SPLIT else True
    assert 1 <= r.C <= R.TRACK_MAX_C


def test_stats_rows_cover_every_split():
    assert {R.stats_split(r.segment) for r in R.STATS.values()} == {1, 2, 44, 64}
    assert {r.C for r in R.STATS.values()} == {1, 2, 3, 64}


def test_three_chunks_is_the_most_over_one_sample():
    """exhaustively over small plans: k_overlap_add's ks[4] never holds a fourth chunk, and its walk visits exactly the chunks
    that cover t; three is reached (odd chunk, hop = chunk / 2)"""
    most = 0
    for chunk in range(2, 26):
        for hop in range(max(chunk // 2, 1), chunk + 1):
            for T in range(1, 6 * chunk):
                K, Lc, starts = R.chunk_plan(T, chunk, hop)
                m = R.max_cover(starts, Lc, T)
                most = max(most, m)
                assert m <= 3, (T, chunk, hop)
                for t in range(0, T, max(1, T // 40)):
                    assert R.covering(starts, Lc, hop, T, t) == [k for k, s0 in enumerate(starts) if s0 <= t < s0 + Lc]
    assert most == 3


@pytest.mark.parametrize("name", list(R.OLA))
def test_ola_row_reaches(name):
    r = R.OLA[name]
    K, Lc, starts = R.chunk_plan(r.T, r.chunk, r.hop)
    m = R.max_cover(starts, Lc, r.T)
    if "three" in r.reaches:
        assert m == 3 and r.chunk % 2 == 1 and r.hop == r.chunk // 2
    if name == "t_chunk_plus_1":
        assert K == 2 and R.overlaps(starts, Lc) == [r.chunk - 1]
    if name == "t_chunk_minus_1":
        assert K == 1 and Lc == r.T
    if name == "last_reaches_back":
        assert R.overlaps(starts, Lc)[-1] > r.chunk - r.hop


def test_refusal_rows_are_one_past_their_limit():
    f = R.REFUSE
    K, _, _ = R.chunk_plan(**{k: f["align_pairs_65536"].args[k] for k in ("T", "chunk", "hop")})
    assert f["align_pairs_65536"].args["B"] * (K - 1) == R.GRID_Y + 1
    K, _, _ = R.chunk_plan(**{k: f["align_b2_pairs_65536"].args[k] for k in ("T", "chunk", "hop")})
    assert f["align_b2_pairs_65536"].args["B"] * (K - 1) == R.GRID_Y + 1
    a = f["chunk_gather_65536"].args
    assert R.chunk_plan(a["T"], a["chunk"], a["hop"])[0] >= a["n"] == R.GRID_Y + 1
    a = f["track_gather_nc_65536"].args
    assert a["n"] * a["C"] == R.GRID_Y + 1 and R.track_plan(a["T"], a["segment"], 0)[0] >= a["n"]
    a = f["track_ola_bc_65536"].args
    assert a["B"] * a["C"] == R.GRID_Y + 1
    assert f["align_s7"].args["S"] == R.OLA_MAX_S + 1
    assert f["track_stats_c65"].args["C"] == R.TRACK_MAX_C + 1


def test_big_row_crosses_2_31():
    fig = R.big_figures()
    assert fig["est_elems"] > 2 ** 31 and fig["K"] > fig["k_cross"] + 2
    assert R.BIG["B"] * (fig["K"] - 1) <= R.GRID_Y and R.score_split(fig["Lc"]) == 8
    assert 8.0e9 < fig["est_bytes"] < 9.0e9 and 4.0e9 < fig["out_bytes"] < 4.5e9
    # the output offsets stay below 2^31; the estimate offsets of chunk k_cross straddle it
    assert R.BIG["S"] * R.BIG["T"] < 2 ** 31
    lo = (fig["k_cross"] * R.BIG["S"]) * fig["Lc"]
    assert lo <= 2 ** 31 < lo + R.BIG["S"] * fig["Lc"]


# ---- restatements agree --------------------------------------------------------------------------------------------------------
def _planted(S, T, chunk, hop, seed):
    K, Lc, starts = R.chunk_plan(T, chunk, hop)
    g = torch.Generator().manual_seed(seed)
    src = torch.randn(S, T, generator=g, dtype=torch.float64)
    q = R.plant_perms(K, S, seed)
    return src, q, starts, Lc


@pytest.mark.parametrize("S", [2, 3])
def test_align_restatement_finds_planted(S):
    src, q, starts, Lc = _planted(S, 1130, 100, 50, seed=S)
    est = R.planted_est(src, q, starts, Lc)
    want = R.planted_want(q)
    assert torch.equal(R.align(est, starts, Lc), want)
    assert torch.equal(torch.tensor(SL.align(est, starts, Lc)), want)


def test_planted_perms_change_every_chunk():
    for S in range(2, 7):
        q = R.plant_perms(2 * R.OLA_TILE + 2, S, seed=S)
        want = R.planted_want(q)
        ident = torch.arange(S)
        changes = (q[1:] != q[:-1]).any(1)
        assert int(changes.sum()) >= len(q) - 2
        assert not torch.equal(want[R.OLA_TILE], ident) and not torch.equal(want[2 * R.OLA_TILE], ident)


@pytest.mark.parametrize("name", ["odd_3cover", "last_reaches_back", "t_chunk_plus_1", "hop_eq_chunk"])
def test_ola_restatement_equals_separate_long_ref(name):
    r = R.OLA[name]
    K, Lc, starts = R.chunk_plan(r.T, r.chunk, r.hop)
    g = torch.Generator().manual_seed(3)
    est = torch.randn(K, 3, Lc, generator=g)
    perms = torch.stack([torch.randperm(3, generator=g) for _ in range(K)])
    out, _ = R.overlap_add(est, perms, starts, Lc, r.hop, r.T)
    ref = SL.overlap_add(est, [tuple(p.tolist()) for p in perms], starts, Lc, r.T)
    torch.testing.assert_close(out, ref, rtol=1e-13, atol=1e-13)
    w = SL.weights(starts, Lc, r.T)
    for k in range(K):
        assert torch.equal(R.chunk_weights(starts, Lc, k), w[k, starts[k]:starts[k] + Lc])
    w, m = R.overlap_add_window(lambda k: est[k], perms, starts, Lc, r.T, 3, min(r.T, 300))
    torch.testing.assert_close(w, ref[:, 3:min(r.T, 300)], rtol=1e-13, atol=1e-13)


def test_stats_restatements_equal_separate_track_ref():
    g = torch.Generator().manual_seed(4)
    xc = (torch.randn(3, 2, 777, generator=g) * 2 + 5).float().double()
    ref = ST.stats(xc)
    torch.testing.assert_close(R.stats64(xc), ref, rtol=1e-14, atol=1e-14)
    torch.testing.assert_close(R.stats_kernel(xc.reshape(6, 777)), ref.reshape(6, 2), rtol=1e-12, atol=1e-12)


# ---- each check rejects its planted defect ------------------------------------------------------------------------------------------
def test_compose_tile_reset_is_caught():
    """pairs past 1024: a compose that restarts from the identity at each tile scrambles every source after pair 1024"""
    for S in (2, 3, 6):
        q = R.plant_perms(R.OLA_TILE + 2, S, seed=10 + S)
        want = R.planted_want(q)
        inv = torch.argsort(q, dim=1)
        local = [tuple(int(v) for v in inv[k + 1][q[k]]) for k in range(len(q) - 1)]   # pi_k: row of k -> row of k + 1
        assert torch.equal(R.compose(local, S), want)
        bad = R.compose(local, S, mut="tile_reset")
        assert torch.equal(bad[:R.OLA_TILE + 1], want[:R.OLA_TILE + 1])
        assert not torch.equal(bad[R.OLA_TILE + 1:], want[R.OLA_TILE + 1:])


@pytest.mark.parametrize("Lc", [4097, 32000])
def test_scoring_drop_last_partial_is_caught(Lc):
    """estimates that differ only in the last CTA's slice: without that partial every permutation ties and the identity wins"""
    S, hop = 3, Lc - Lc // 2
    T = Lc + 2 * hop
    src, q, starts, _ = _planted(S, T, Lc, hop, seed=Lc)
    est = R.planted_est(R.last_slice_decides(src, starts, Lc), q, starts, Lc)
    want = R.planted_want(q)
    assert torch.equal(R.align(est, starts, Lc), want)
    bad = R.align(est, starts, Lc, mut="drop_last")
    assert not torch.equal(bad, want)


def _stats_share(xc, mut):
    ref = R.stats64(xc)
    bound = ST.stats_bounds(xc)
    got = R.stats_kernel(xc.reshape(-1, xc.shape[-1]), mut).reshape(ref.shape)
    return R.share((got - ref).abs(), bound)


def test_stats_bound_accepts_the_kernel_order():
    g = torch.Generator().manual_seed(5)
    x = (1e4 + 1e-2 * torch.randn(2, 3, 352800, generator=g, dtype=torch.float64)).float().double()
    assert _stats_share(x, None) <= 1.0


def test_stats_no_shift_is_caught():
    """a DC offset of 1e4 with std 1e-2 over the recipe segment: unshifted squares lose the variance"""
    g = torch.Generator().manual_seed(6)
    x = (1e4 + 1e-2 * torch.randn(1, 2, 352800, generator=g, dtype=torch.float64)).float().double()
    assert _stats_share(x, "no_shift") > R.REJECT


@pytest.mark.parametrize("n", [2, 5000, 600000])
def test_stats_biased_is_caught(n):
    g = torch.Generator().manual_seed(7)
    x = torch.randn(1, 2, n, generator=g, dtype=torch.float64).float().double()
    assert _stats_share(x, "biased") > R.REJECT


def _ola_share(name, mut, S=2):
    r = R.OLA[name]
    K, Lc, starts = R.chunk_plan(r.T, r.chunk, r.hop)
    g = torch.Generator().manual_seed(8)
    est = torch.randn(K, S, Lc, generator=g)
    ref, mag = R.overlap_add(est, None, starts, Lc, r.hop, r.T)
    bad, _ = R.overlap_add(est, None, starts, Lc, r.hop, r.T, mut=mut)
    return R.share((bad - ref).abs(), ST.ola_bound(ref, mag))


def test_ramps_without_half_sample_are_caught():
    for name in ("odd_3cover", "t_chunk_plus_1"):
        assert _ola_share(name, "no_half") > R.REJECT


def test_overlap_add_skipping_a_covering_chunk_is_caught():
    """the most chunks the plan puts over a sample is three: a walk that keeps two regular chunks and the last loses the third"""
    assert _ola_share("odd_3cover", "drop_third") > R.REJECT
    assert _ola_share("odd_3cover", None) == 0.0
