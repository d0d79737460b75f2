"""Rows, routing facts, kernel-order restatements, planted inputs and bounds of tests/test_ola_edges_gpu.py (test infrastructure
only): the chunk steps of ConvTasNet.separate_long (ctn_chunk_gather / ctn_chunk_align / ctn_chunk_overlap_add) and of
ConvTasNet.separate_track (ctn_track_stats / ctn_track_gather / ctn_track_overlap_add), all in csrc/ctn_ola.cu, at their edges.

Plain torch, no import of the native library: test_ola_edges_cpu.py shows without a GPU that every row reaches the branch its
`reaches` text names and that each check rejects a planted defect.  The fp64 restatements of the operations themselves are
separate_long_ref.py (SL) and separate_track_ref.py (ST); this file adds what the edges need on top of them.

Routing facts restated from ctn_ola.cu:
  * chunk_plan: Lc = min(chunk, T); K = 1 if T <= chunk, else ceil((T - chunk) / hop) + 1; chunk k starts at k hop, the last at
    T - Lc.  Alignment scores B (K - 1) pairs on gridDim.y: at most 65535, else CTN_EUNSUPPORTED before any launch.
  * score_split(Lc) = ceil(Lc / 4096) CTAs per pair, at most 16; CTA g sums the overlap's slice [g s, min(ov, (g + 1) s)),
    s = ceil(ov / G); k_compose_perms adds the G partials in CTA order.
  * k_compose_perms composes the per-pair permutations in tiles of OLA_TILE = 1024 pairs; a thread per pair (strided by 256
    threads, so n > 256 pairs of a tile loop), and the running permutation `cur` of thread s carries from tile to tile.
  * k_overlap_add: the chunks covering t are the regular ones k_lo .. k_hi (at most K - 2) and the last, in ks[4].  The last
    chunk starts after (K - 2) hop (K is the least count that reaches T), and three regular chunks meet only at t = m hop with
    m <= K - 2 (odd chunk, hop = chunk / 2), so at most THREE chunks cover a sample: the fourth slot is never used.
    test_ola_edges_cpu.py shows this exhaustively over small plans; the rows reach three.
  * track_plan: hop = 0 is the tester layout (K = ceil(T / segment), zeros past T); otherwise chunk_plan.  stats_split(Lc) =
    ceil(Lc / 8192) CTAs per row, at most 64 (slices longer than 8192 past that); the track gather puts n C rows and the track
    overlap-add B C rows on gridDim.y (at most 65535 each); the whole call's chunk batch is at most 65535 / max(C, S).

Bounds (u32 = 2^-24, u64 = 2^-53):
  * statistics: ST.stats_bounds, derived from the double shifted sums (Higham's (n - 1) u sum|terms| for any order of sums).
  * overlap-add: one fp32 rounding of the fp64 value plus 32 u64 of the weighted magnitude (ST.ola_bound): the weights in double
    (sinpi / cospi), two fused roundings per chunk, at most three chunks, the reciprocal and the product.
  * gather: ST.gather_bound, one fp32 rounding plus the double subtraction and division.
"""
import collections
import itertools
import math

import torch

import separate_long_ref as SL
import separate_track_ref as ST

OLA_TILE = 1024
OLA_MAX_S = 6
OLA_MAX_SPLIT = 16
SCORE_SLICE = 4096
TRACK_SLICE = 8192
TRACK_MAX_SPLIT = 64
GRID_Y = 65535
TRACK_MAX_C = 64
REJECT = 4.0        # a planted defect must land this many times past its bound


def ceil_div(a, b):
    return -(-a // b)


# ---- routing restated ---------------------------------------------------------------------------------------------------------
def chunk_plan(T, chunk, hop):
    """-> (K, Lc, starts); None where ctn_chunk_plan refuses"""
    if T <= 0 or chunk <= 0 or hop <= 0 or hop < chunk // 2 or hop > chunk:
        return None
    Lc = min(chunk, T)
    K = 1 if T <= chunk else ceil_div(T - chunk, hop) + 1
    starts = [T - Lc if k == K - 1 else k * hop for k in range(K)]
    assert (starts, Lc) == tuple(SL.plan(T, chunk, hop))
    return K, Lc, starts


def score_split(Lc):
    return min(max(ceil_div(Lc, SCORE_SLICE), 1), OLA_MAX_SPLIT)


def stats_split(Lc):
    return min(max(ceil_div(Lc, TRACK_SLICE), 1), TRACK_MAX_SPLIT)


def track_plan(T, segment, hop):
    """-> (K, Lc, starts) of ctn_track_plan (hop 0: the tester layout)"""
    if hop:
        return chunk_plan(T, segment, hop)
    K = ceil_div(T, segment)
    return K, segment, [k * segment for k in range(K)]


def overlaps(starts, Lc):
    return [max(starts[k] + Lc - starts[k + 1], 0) for k in range(len(starts) - 1)]


def covering(starts, Lc, hop, T, t):
    """the chunks k_overlap_add visits for sample t, in its order: regular k_lo .. k_hi, then the last"""
    K = len(starts)
    k_lo = (t - Lc) // hop + 1 if t >= Lc else 0
    k_hi = min(t // hop, K - 2)
    ks = list(range(k_lo, k_hi + 1))
    if t >= starts[-1]:
        ks.append(K - 1)
    return ks


def max_cover(starts, Lc, T):
    """most chunks over one sample (from the chunk extents, not from the kernel's walk)"""
    d = [0] * (T + 1)
    for s0 in starts:
        d[s0] += 1
        d[s0 + Lc] -= 1
    run, best = 0, 0
    for v in d[:T]:
        run += v
        best = max(best, run)
    return best


# ---- kernel-order restatements, each with its planted defect -------------------------------------------------------------------
def pair_scores(a, b, G, mut=None):
    """a, b (S, ov) float64: c[i][j] = sum over the G CTA slices of <a_i, b_j>, slices added in CTA order.
    mut='drop_last': the last CTA's partial is left out"""
    ov = a.shape[1]
    sl = ceil_div(ov, G)
    c = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float64)
    for g in range(G - 1 if mut == "drop_last" else G):
        q0, q1 = g * sl, min(ov, (g + 1) * sl)
        if q0 < q1:
            c += a[:, q0:q1] @ b[:, q0:q1].t()
    return c


def best_perm(c):
    """first maximum of sum_i c[i][pi(i)] over itertools.permutations order"""
    S = c.shape[0]
    best, best_v = None, None
    for pi in itertools.permutations(range(S)):
        v = sum(float(c[i, pi[i]]) for i in range(S))
        if best is None or v > best_v:
            best, best_v = pi, v
    return best


def align(est, starts, Lc, mut=None):
    """est (K, S, Lc) of one recording -> perms (K, S) int64 through pair_scores / best_perm / compose"""
    ov = overlaps(starts, Lc)
    G = score_split(Lc)
    e = est.double()
    local = [best_perm(pair_scores(e[k, :, Lc - ov[k]:], e[k + 1, :, :ov[k]], G, mut)) for k in range(len(starts) - 1)]
    return compose(local, est.shape[1], mut)


def compose(local, S, mut=None):
    """per-pair permutations -> P (K, S): P_0 = id, P_{k+1}(s) = pi_k(P_k(s)), in tiles of OLA_TILE pairs.
    mut='tile_reset': every tile starts again from the identity (the carry of `cur` lost)"""
    P = [list(range(S))]
    cur = list(range(S))
    for k0 in range(0, len(local), OLA_TILE):
        if mut == "tile_reset":
            cur = list(range(S))
        for r, pi in enumerate(local[k0:k0 + OLA_TILE]):
            cur = [pi[c] for c in cur]
            P.append(list(cur))
    return torch.tensor(P, dtype=torch.int64)


def chunk_weights(starts, Lc, k, mut=None):
    """(Lc,) float64 w_k of SL.weights for chunk k alone (the dense (K, T) table does not fit the long rows).
    mut='no_half': the ramps sample at r / a instead of (r + 1/2) / a"""
    half = 0.0 if mut == "no_half" else 0.5
    K, s0 = len(starts), starts[k]
    wk = torch.ones(Lc, dtype=torch.float64)
    if k > 0:
        a = max(starts[k - 1] + Lc - s0, 0)
        if a > 0:
            wk[:a] *= torch.sin(0.5 * math.pi * (torch.arange(a, dtype=torch.float64) + half) / a) ** 2
    if k < K - 1:
        n = max(s0 + Lc - starts[k + 1], 0)
        if n > 0:
            wk[Lc - n:] *= torch.cos(0.5 * math.pi * (torch.arange(n, dtype=torch.float64) + half) / n) ** 2
    return wk


def overlap_add(est, perms, starts, Lc, hop, T, mut=None):
    """est (K, S, Lc) of one recording, perms (K, S) or None -> (out (S, T), mag (S, T)) float64, the kernel's walk over the
    covering chunks.  mut='drop_third': ks holds two regular chunks, a third regular one is skipped; 'no_half': see
    chunk_weights"""
    K, S, _ = est.shape
    num = torch.zeros(S, T, dtype=torch.float64)
    mag = torch.zeros(S, T, dtype=torch.float64)
    den = torch.zeros(T, dtype=torch.float64)
    for k, s0 in enumerate(starts):
        wk = chunk_weights(starts, Lc, k, mut)
        if mut == "drop_third":
            for t in range(s0, s0 + Lc):
                ks = covering(starts, Lc, hop, T, t)
                if k != K - 1 and len([j for j in ks if j != K - 1]) >= 3 and ks.index(k) == 2:
                    wk[t - s0] = 0.0
        e = est[k].double() if perms is None else est[k, perms[k]].double()
        num[:, s0:s0 + Lc] += wk * e
        mag[:, s0:s0 + Lc] += wk * e.abs()
        den[s0:s0 + Lc] += wk
    return num / den, mag / den


def overlap_add_window(chunk_est, perms, starts, Lc, T, t0, t1):
    """out[:, t0:t1] of one recording in float64 from only the chunks that cover the window: chunk_est(k) -> (S, Lc), perms
    (K, S) -> ((S, t1 - t0), mag)"""
    num = mag = den = 0.0
    for k, s0 in enumerate(starts):
        if s0 >= t1 or s0 + Lc <= t0:
            continue
        e = chunk_est(k).double()[perms[k]]
        wk = chunk_weights(starts, Lc, k)
        lo, hi = max(t0, s0), min(t1, s0 + Lc)
        ek = torch.zeros(e.shape[0], t1 - t0, dtype=torch.float64)
        w = torch.zeros(t1 - t0, dtype=torch.float64)
        ek[:, lo - t0:hi - t0] = e[:, lo - s0:hi - s0]
        w[lo - t0:hi - t0] = wk[lo - s0:hi - s0]
        num = num + w * ek
        mag = mag + w * ek.abs()
        den = den + w
    return num / den, mag / den


def stats_kernel(xc, mut=None):
    """xc (R, Lc) float64 rows (zeros past T included) -> (R, 2) mean and std the way k_track_stats / _combine form them.
    mut='no_shift': sums of x and x^2 (no shift by the first sample); 'biased': the variance divided by n"""
    n = xc.shape[-1]
    s = torch.zeros_like(xc[:, :1]) if mut == "no_shift" else xc[:, :1]
    d = xc - s
    S1, S2 = d.sum(-1), (d * d).sum(-1)
    var = (S2 - S1 * (S1 / n)).clamp_min(0) / (n if mut == "biased" else n - 1)
    return torch.stack([s[:, 0] + S1 / n, var.sqrt()], -1)


def stats64(xc):
    """xc (..., Lc) float64 -> (..., 2): mean and unbiased std, each sum taken about an accurate centre (shift by the first sample,
    then a correction pass) so the reference's own error is a few u64 of the row's spread, far inside ST.stats_bounds"""
    n = xc.shape[-1]
    m = xc[..., :1] + (xc - xc[..., :1]).sum(-1, keepdim=True) / n
    m = m + (xc - m).sum(-1, keepdim=True) / n
    var = ((xc - m) ** 2).sum(-1) / (n - 1)
    return torch.stack([m[..., 0], var.sqrt()], -1)


def share(err, bound):
    return float((err / bound).max())


# ---- planted inputs --------------------------------------------------------------------------------------------------------------
def plant_perms(K, S, seed):
    """q (K, S): row r of chunk k carries source q[k][r].  q changes at every chunk (S = 2: at every chunk but the second, so the
    permutation P_k is not the identity at the tile boundaries k = 1024, 2048), and q[k] != q[0] at every tile boundary"""
    g = torch.Generator().manual_seed(seed)
    allp = [list(p) for p in itertools.permutations(range(S))]
    q = [allp[int(torch.randint(len(allp), (1,), generator=g))]]
    for k in range(1, K):
        if S == 2:
            q.append(q[-1] if k == 1 else q[-1][::-1])
            continue
        cand = [p for p in allp if p != q[-1] and (k % OLA_TILE or p != q[0])]
        q.append(cand[int(torch.randint(len(cand), (1,), generator=g))])
    return torch.tensor(q, dtype=torch.int64)


def planted_want(q):
    """the permutations alignment must find for planted q: P_k(s) = the row of chunk k that carries what row s of chunk 0 does"""
    inv = torch.argsort(q, dim=1)
    return inv[:, q[0]]


def planted_est(src, q, starts, Lc):
    """src (S, T) one recording -> est (K, S, Lc): est[k][r] = src[q[k][r], starts[k]:+Lc]"""
    return torch.stack([src[q[k], s0:s0 + Lc] for k, s0 in enumerate(starts)])


def last_slice_decides(src, starts, Lc):
    """src (S, T) -> a copy that is zero over every overlap except its last scoring CTA's slice: planted estimates of it differ
    only there, so only that slice tells the permutations apart (all others tie, and a tie keeps the identity).  The overlaps
    must not share samples (hop >= Lc / 2, regular starts)"""
    src = src.clone()
    G = score_split(Lc)
    ov = overlaps(starts, Lc)
    for k in range(len(starts) - 1):
        assert k == 0 or starts[k + 1] >= starts[k - 1] + Lc
        src[:, starts[k + 1]:starts[k + 1] + (G - 1) * ceil_div(ov[k], G)] = 0.0
    return src


# ---- rows --------------------------------------------------------------------------------------------------------------------------
Align = collections.namedtuple("Align", "B S T chunk hop reaches")
Score = collections.namedtuple("Score", "S T chunk hop reaches")
Ola = collections.namedtuple("Ola", "T chunk hop reaches")
Stats = collections.namedtuple("Stats", "C segment T reaches")
Refuse = collections.namedtuple("Refuse", "entry args code reaches")


def _align_T(pairs, chunk=64, hop=32, tail=17):
    """T with K - 1 = pairs and a last chunk that moves left by hop - tail samples (an uneven last overlap)"""
    return chunk + hop * (pairs - 1) + tail


ALIGN = {}
for _p in (257, 1024, 1025, 2049):
    for _S in range(2, 7):
        ALIGN["p{}_s{}".format(_p, _S)] = Align(2, _S, _align_T(_p), 64, 32,
                                                "K - 1 = {}: {}".format(_p, {257: "a tile of 257 pairs, the r loop past 256",
                                                                            1024: "exactly one full tile",
                                                                            1025: "a second tile of one pair: cur carried",
                                                                            2049: "three tiles, the last of one pair"}[_p]))
for _S in (2, 6):
    ALIGN["p21845_b3_s{}".format(_S)] = Align(3, _S, _align_T(21845), 64, 32, "B (K - 1) = 65535: the scoring grid's last row")

SCORE = {}
for _Lc, _tag in ((4096, "G = 1"), (4097, "G = 2"), (32000, "G = 8"), (61441, "G = 16 (the cap reached)"),
                  (140001, "G = 16 (capped: slices past 4096)")):
    _G = score_split(_Lc)
    for _S in range(2, 7):
        # overlap Lc - hop = Lc // 2 (> G 256) and, second, G m + 1 (one sample past whole slices: a short last slice)
        SCORE["lc{}_s{}".format(_Lc, _S)] = Score(_S, _Lc + 2 * (_Lc - _Lc // 2), _Lc, _Lc - _Lc // 2, _tag + ", overlap Lc/2")
        _ov = _G * ((_Lc // 2 - 2) // _G) + 1
        SCORE["lc{}_s{}_edge".format(_Lc, _S)] = Score(_S, _Lc + 2 * (_Lc - _ov), _Lc, _Lc - _ov, _tag + ", overlap G m + 1")

OLA = {
    "odd_3cover": Ola(977, 101, 50, "odd chunk, hop = chunk / 2: three chunks over t = m hop (the most the plan allows)"),
    "odd_3cover_long": Ola(20011, 1001, 500, "odd chunk, hop = chunk / 2, 39 chunks, three over every t = m hop"),
    "last_reaches_back": Ola(1130, 100, 50, "the last chunk overlaps its predecessor by more than chunk - hop"),
    "t_chunk_plus_1": Ola(102, 101, 50, "T = chunk + 1: K = 2, overlap chunk - 1"),
    "t_chunk_minus_1": Ola(100, 101, 50, "T = chunk - 1: K = 1, Lc = T, a copy"),
    "hop_eq_chunk": Ola(1001, 100, 100, "hop = chunk: no overlap but the last chunk's"),
}
OLA_S = (1, 2, 7)

# C = 1, 2, 3 and 64 at every split; tester layout with K = 4 segments: DC, first-sample outlier, silence, one valid sample
STATS = {}
for _seg, _tag in ((5000, "G = 1"), (8193, "G = 2"), (8 * 44100, "G = 44 (the recipe's 8 s segment)"),
                   (600000, "G = 64 (capped: slices of 9375 > 8192)")):
    for _C in (1, 2, 3, 64):
        STATS["seg{}_c{}".format(_seg, _C)] = Stats(_C, _seg, 3 * _seg + 1,
                                                    _tag + "; DC 1e4, outlier first sample, silent segment, one valid sample")

# one past each grid limit: refused before any launch
REFUSE = {
    "align_pairs_65536": Refuse("ctn_chunk_align", dict(B=1, S=2, T=_align_T(65536), chunk=64, hop=32), "EUNSUPPORTED",
                                "B (K - 1) = 65536 scoring pairs"),
    "align_b2_pairs_65536": Refuse("ctn_chunk_align", dict(B=2, S=3, T=_align_T(32768), chunk=64, hop=32), "EUNSUPPORTED",
                                   "B = 2, K - 1 = 32768: B (K - 1) = 65536"),
    "align_s7": Refuse("ctn_chunk_align", dict(B=1, S=7, T=1000, chunk=100, hop=50), "EUNSUPPORTED", "S = 7 > OLA_MAX_S"),
    "chunk_gather_65536": Refuse("ctn_chunk_gather", dict(B=1, T=32 + 16 * 65536, chunk=32, hop=16, n=65536), "EUNSUPPORTED",
                                 "a chunk batch of 65536 on gridDim.y"),
    "track_gather_nc_65536": Refuse("ctn_track_gather", dict(B=1, C=2, T=65536, segment=2, hop=0, n=32768), "EUNSUPPORTED",
                                    "n C = 65536 rows on gridDim.y"),
    "track_ola_bc_65536": Refuse("ctn_track_overlap_add", dict(B=32768, C=2, S=1, T=4, segment=2, hop=0), "EUNSUPPORTED",
                                 "B C = 65536 rows on gridDim.y"),
    "track_stats_c65": Refuse("ctn_track_stats", dict(B=1, C=65, T=100, segment=50, hop=0), "EINVAL", "C = 65 > 64"),
    "track_gather_c65": Refuse("ctn_track_gather", dict(B=1, C=65, T=100, segment=50, hop=0, n=1), "EINVAL", "C = 65 > 64"),
    "track_ola_c65": Refuse("ctn_track_overlap_add", dict(B=1, C=65, S=1, T=100, segment=50, hop=0), "EINVAL", "C = 65 > 64"),
}

# ---- the launch counts ----------------------------------------------------------------------------------------------------------
def align_launches(S, K):
    """identity compose alone (S = 1 or K = 1), else the scores and the compose"""
    return 1 if (S == 1 or K == 1) else 2


GATHER_LAUNCHES, OLA_LAUNCHES, TRACK_STATS_LAUNCHES = 1, 1, 2

# ---- past 2^31 elements (row 6) --------------------------------------------------------------------------------------------------
BIG = dict(S=6, B=1, chunk=32000, hop=16000, T=180_000_017)


def big_figures():
    """the row's element counts and bytes, and the chunk whose estimate offset (k S + r) Lc first crosses 2^31"""
    K, Lc, starts = chunk_plan(BIG["T"], BIG["chunk"], BIG["hop"])
    S = BIG["S"]
    est = K * S * Lc
    k_cross = (2 ** 31) // (S * Lc)
    return dict(K=K, Lc=Lc, starts=starts, est_elems=est, est_bytes=4 * est, out_bytes=4 * S * BIG["T"],
                src_bytes=4 * S * BIG["T"], k_cross=k_cross)


# ---- every row with the branches it reaches, from the restated routing ------------------------------------------------------------
def reached_align(r):
    K, Lc, starts = chunk_plan(r.T, r.chunk, r.hop)
    got = {"tiles={}".format(ceil_div(K - 1, OLA_TILE))}
    if (K - 1) % OLA_TILE and K - 1 > OLA_TILE:
        got.add("short last tile")
    if min(K - 1, OLA_TILE) > 256:
        got.add("r loop past 256")
    if r.B * (K - 1) == GRID_Y:
        got.add("grid y = 65535")
    return got


def reached_score(r):
    K, Lc, starts = chunk_plan(r.T, r.chunk, r.hop)
    G = score_split(Lc)
    got = {"G={}".format(G)}
    for ov in overlaps(starts, Lc):
        if ov > G * 256:
            got.add("ov > G 256")
        sl = ceil_div(ov, G)
        if ov % sl and G > 1:
            got.add("short last slice")
        if sl > SCORE_SLICE:
            got.add("slice > 4096")
    return got
