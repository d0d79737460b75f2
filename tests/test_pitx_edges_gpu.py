"""Edge cases of ORPIT and Sinkhorn PIT over SI-SDR (csrc/ctn_pitx.cu through ctn_b200/criterion/pit.py and the C ABI), ``-m gpu``,
against float64 references of the same operations on the same fp32 inputs.  Each row names in `reaches` the branch it selects and
the constant that selects it: PITX_C = 256 (the T-chunk), PITX_CTAS = 528 (the stats grid target: one CTA per sample from B = 528),
the KS lanes-per-pair ladder (KS = 32 halved while KS * pairs > 256), the pair backward's gx <= 64, gridDim.y <= 65535 (samples past
it loop) and PITX_MAX = 16.

References.  ORPIT: the candidate scores of tests/pit_variants_oracle.py ``orpit`` written out over the batch in float64 (``_orpit64``,
checked against ``PO.orpit`` on the first samples of every row).  The rests r_i = sum_{j < n_b, j != i} t_j are formed in fp32 in
ascending j (``_rests``), as the kernel forms them and as the reference does on fp32 tensors, and given to the float64 SI-SDR: kernel
and reference score bit-equal rows, so no rest-rounding term enters the value bound.  SinkPIT: ``PO.sinkpit`` in float64 for the input
gradient, and its Sinkhorn tail restated on an S x S leaf table (``_sinkhorn64``, checked against ``PO.sinkpit``) for loss_b, P, dL
and the Jacobians below.  Gradients come from float64 autograd driven by uneven per-sample weights w_b = 1 + b mod 7 on loss_b (and
weights on P where the row drives P), so a kernel that used one sample's weight for another would fail.

Bounds.  k_pitx_stats has the numerics of k_pit_pass1/2 (fp32 runs of at most four, double across them, alpha in fp32), so a pair's
SI-SDR is held to ``_sisdr_bound`` and a pair's gradient to ``_grad_bound`` of tests/test_loss_optim_edges_gpu.py, derived there (u =
2^-24).  On top of those:
  * ORPIT value.  Candidate i scores v = s0 + s1 / (n_b - 1), s0 = SI-SDR(e0, t_i), s1 = SI-SDR(e1, r_i), each computed in double,
    cast to fp32, then an fp32 divide and add: |v - v64| <= b0 + b1 / (n_b - 1) + u (|s0| + 2 |s1| / (n_b - 1) + |v|).
  * ORPIT gradient.  Row e0: ``_grad_bound`` of (e0, t_sel).  Row e1: ``_grad_bound`` of (e1, r_sel) plus
    2 n_b u (sum_{j != sel} |ct1 t_j| + |cx1 e1|): k_pitx_pair_bwd expands ct1 r_sel into n_b - 1 fmas over the t_j after the
    product cx1 e1, each rounded relative to a partial sum no larger than that sum, and r_sel was itself rounded n_b - 2 times.
  * SinkPIT loss_b, P and dL.  The per-pair table bound dL_ij (``_sisdr_bound``) is propagated to first order through the float64
    Jacobian of loss_b, P and dL with respect to the S x S table L (autograd on the leaf table; a double backward for dL), times 2
    for second-order terms; plus the fp32 rounding of the output (u |.|, and 2^-149 for P's underflow); plus (2K + 2) 2^-44 times
    the magnitude of the summands, for the double arithmetic of the K iterations and of their walk-back Z_before = Z_after + lse.
    The last term matters only where an output cancels to ~0, e.g. loss_b at K = 0 (L + Z / c = 0).  The Jacobian grows with
    coldness by itself, so no coldness is excluded as ill-conditioned.
  * SinkPIT input gradient, row i: the sum over j of the pair bound ``_grad_bound`` with weight -dL_ij, the coefficient error
    |ddL_ij| (|ct_ij t_j| + |cx_ij e_i|), and the fp32 accumulation S u (|W_ij t_j| + |cx_ij dL_ij e_i|) of the fma chain and of cx_i.
  * The pair table of ctn_sinkpit_fwd (``pair_sisdr``) is held to ``_sisdr_bound`` + u |v|, and dL of ctn_sinkpit_bwd to its bound
    above: together they separate the Sinkhorn backward from the pair backward.
Indices (ORPIT) and patterns (SinkPIT, argmax of P) equal the fp64 ones wherever the fp64 margin exceeds both bounds; otherwise the
kernel's choice must be optimal within them, and the gradient is checked through the choice the kernel made.  Exact ties are built at
T <= 256, where each sample's statistics come from one CTA, so the tied scores are bit-equal (the tied ORPIT targets are multiples of
1/64 below 8 in magnitude, so every rest sum is exact in any order), and the first index is asserted directly.
"""
import collections

import pytest
import torch

import convtasnet_oracle as O
import pit_variants_oracle as PO
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import ORPIT, SinkPIT, sinkpit
from ctn_b200.criterion.sdr import NegSISDR, SISDR
from test_loss_optim_edges_gpu import EPS, U, _grad_bound, _grad_coef, _place, _sisdr_bound, _stats

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
F64 = torch.float64
CRITS = {"NegSISDR": (NegSISDR, False), "SISDR": (SISDR, True)}
PITX_C, PITX_CTAS = 256, 528
T_BIG = PITX_CTAS * PITX_C + 1   # 529 chunks: at B = 1 the stats grid is 528 CTAs, so CTA 0 also takes the last chunk
FWD_LAUNCHES, BWD_LAUNCHES = 3, 2


def _weights(B):
    return (1 + torch.arange(B) % 7).float()


def _put(x, layout):
    """GPU tensor equal to x: 'slice1' is x[1:] of a batch one sample larger (a base at a float offset of one sample), the rest as
    test_loss_optim_edges_gpu._place ('contig', 'offK', 'transposed')"""
    if layout != "slice1":
        return _place(x, layout)
    big = torch.zeros((x.shape[0] + 1,) + tuple(x.shape[1:]), device=DEV)
    big[1:].copy_(x)
    return big[1:]


def _share(key, err, bound):
    bad = ~(err <= bound)  # a NaN counts as over the bound
    assert not bool(bad.any()), "{}: {} entries over the bound, worst {:.3e} (bound there {:.3e})".format(
        key, int(bad.sum()), float(err[bad].max()) if bool(torch.isfinite(err[bad]).all()) else float("nan"),
        float(bound[bad][0]))
    return float((err / bound.clamp_min(1e-300)).max())


def _tail(x, k=300.0):
    """the last sample of every row times k, so that the last chunk carries a large share of every statistic"""
    x = x.clone()
    x[..., -1] *= k
    return x


# ---- ORPIT ---------------------------------------------------------------------------------------------------------------------

def _orpit_gen(lens, T, seed, snr_db=5.0):
    """targets of unequal levels (zero past n_b); estimate 0 = target k_b + noise, estimate 1 = the others' sum + noise"""
    g = torch.Generator().manual_seed(seed)
    B, n = len(lens), max(lens)
    nb = torch.tensor(lens)
    lev = torch.logspace(-0.4, 0.4, n, dtype=F64)[torch.randperm(n, generator=g)]
    t = torch.randn(B, n, T, generator=g, dtype=F64) * lev.view(1, n, 1)
    t = t * (torch.arange(n).view(1, n, 1) < nb.view(B, 1, 1))
    k = (torch.rand(B, generator=g, dtype=F64) * nb).long()
    one = t[torch.arange(B), k]
    e = torch.stack([one, t.sum(1) - one], 1)
    noise = torch.randn(B, 2, T, generator=g, dtype=F64)
    noise = noise * e.norm(dim=-1, keepdim=True) / noise.norm(dim=-1, keepdim=True).clamp_min(1e-300) * 10 ** (-snr_db / 20)
    return (e + noise).float(), t.float()


def _orpit_mod(kind, lens, T, seed, **kw):
    e, t = _orpit_gen(lens, T, seed, **kw)
    if kind == "x1e4":
        t = t * 1e4
    elif kind == "x1e-6":
        t = t * 1e-6
    elif kind == "dc1e3":
        e, t = e + 1e3, t + 1e3
    elif kind == "silent_est":
        e[0, 1], e[1, 0] = 0, 0
    elif kind == "silent_tgt":
        t[1, 1] = 0
    elif kind == "silent_rest":
        t[:, 2] = -t[:, 1]                                      # r_0 = t_1 + t_2 = 0 exactly
    elif kind == "scaled":
        e[:, 0] = 2 * t[:, 0]                                   # e0 = 2 t_0: alpha = 2, the residual is exactly 0
    elif kind == "tail":
        e, t = _tail(e), _tail(t)
    return e, t, lens


def _orpit_tie(n, T, i, k, seed):
    """targets t_i == t_k bit-equal, multiples of 1/64 below 8: estimate 0 follows t_i, so candidates i and k tie exactly"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(-511, 512, (1, n, T), generator=g).float() / 64
    t[0, k] = t[0, i]
    rest = t[0].sum(0) - t[0, i]
    e0 = t[0, i] + 0.3 * t[0, i].std() * torch.randn(T, generator=g)
    e1 = rest + 0.3 * rest.std() * torch.randn(T, generator=g)
    return torch.stack([e0, e1]).unsqueeze(0), t, [n]


ORow = collections.namedtuple("ORow", "make packed crit layout reaches")


def _o(lens, T, seed, kind=None, packed=False, crit="NegSISDR", layout="contig", reaches="", **kw):
    return ORow(lambda: _orpit_mod(kind, lens, T, seed, **kw), packed, crit, layout, reaches)


ORPIT_ROWS = {
    "T1": _o([3] * 3, 1, 1, reaches="T = 1: one partial chunk of one sample; eps decides every score"),
    "T255": _o([3] * 3, 255, 2, crit="SISDR", reaches="T = PITX_C - 1: one partial chunk"),
    "T256": _o([3] * 3, 256, 3, reaches="T = PITX_C: exactly one chunk"),
    "T257": _o([3] * 3, 257, 4, reaches="T = PITX_C + 1: a second chunk of one sample"),
    "B1_Tbig": _o([4], T_BIG, 5, kind="tail", reaches="B = 1, 529 chunks > gx = PITX_CTAS = 528: CTA 0 grid-strides to the last "
                  "chunk (which carries a large share of every statistic); pair backward gx = 133 clamped to 64"),
    "B528": _o([3] * 528, 700, 6, reaches="B = PITX_CTAS: gx = 1, one CTA walks all 3 chunks of its sample"),
    "B600": _o([3] * 600, 300, 7, crit="SISDR", reaches="B = 600 > PITX_CTAS: gx = 1 over 2 chunks"),
    "B70000": _o([3] * 70000, 9, 8, reaches="B = 70000 > 65535: the stats and pair backward loop samples over gridDim.y"),
    "n2": _o([2] * 4, 1001, 9, reaches="n = 2: the rest is the other target; g1 = g0"),
    "n4": _o([4] * 3, 1001, 10, crit="SISDR", reaches="n = 4: 8 pairs, KS = 32"),
    "n8": _o([8] * 3, 1001, 11, reaches="n = 8: 16 pairs, KS = 16"),
    "n16": _o([16] * 3, 1001, 12, reaches="n = PITX_MAX = 16: 32 pairs, KS = 8, 34 staged rows"),
    "packed16": _o([2, 16, 2, 2, 3, 2, 2, 2], 777, 13, packed=True,
                   reaches="packed n = 16 with most n_b = 2: inactive pairs p % nt >= n_b; g1 = g0 / (n_b - 1) per sample"),
    "packed_unsorted": _o([4, 2, 5, 3], 1603, 14, packed=True, crit="SISDR",
                          reaches="enforce_sorted=False with unsorted lengths: n_b per sample through pad_packed_sequence"),
    "x1e4": _o([3] * 3, 1000, 15, kind="x1e4", reaches="targets x 1e4: alpha ~ 1e-4, fp32 runs of 4 at |x t| ~ 1e4"),
    "x1e-6_T3": _o([3] * 3, 3, 16, kind="x1e-6", reaches="targets x 1e-6 at T = 3: tt ~ 3e-12 ~ eps decides alpha"),
    "dc1e3": _o([3] * 3, 1000, 17, kind="dc1e3", reaches="DC offset 1e3: kappa ~ 1, |x| / |r| ~ 1e3"),
    "silent_est": _o([3] * 3, 1001, 18, kind="silent_est", reaches="e1 = 0 (sample 0), e0 = 0 (sample 1): den = 0, gradient 0"),
    "silent_tgt": _o([3] * 3, 1001, 19, kind="silent_tgt", reaches="t_1 = 0 in sample 1: tt = 0, alpha = 0 / eps"),
    "silent_rest": _o([3] * 3, 1001, 20, kind="silent_rest", crit="SISDR",
                      reaches="t_2 = -t_1 exactly: r_0 = 0, tt = 0 and <e1, r_0> = 0 for candidate 0"),
    "scaled": _o([3] * 3, 1001, 21, kind="scaled", reaches="e0 = 2 t_0: residual 0, den + eps = eps"),
    **{f"snr{d}": _o([3] * 3, 4001, 22 + d, snr_db=float(d), reaches=f"SI-SDR ~ {d} dB: the explicit residual carries the score")
       for d in (40, 60, 80)},
    "slice1_T1001": _o([3] * 3, 1001, 25, layout="slice1",
                       reaches="est[1:], tgt[1:] of larger batches: the target base at an odd float offset (3 * 1001), scalar loads"),
    "transposed": _o([3] * 3, 1000, 26, layout="transposed", crit="SISDR",
                     reaches="transposed estimate: ORPIT's contiguous() copy"),
}


def _rests(t, lens):
    """r_i = sum_{j < n_b, j != i} t_j in t's dtype, ascending j from 0, as k_pitx_stats forms it (0 for i >= n_b)"""
    B, n, T = t.shape
    live = (torch.arange(n).view(1, n) < torch.tensor(lens).view(B, 1)).unsqueeze(-1)
    zero = torch.zeros((), dtype=t.dtype)
    r = torch.zeros_like(t)
    for i in range(n):
        acc = torch.zeros(B, T, dtype=t.dtype)
        for j in range(n):
            if j != i:
                acc = acc + torch.where(live[:, j], t[:, j], zero)
        r[:, i] = torch.where(live[:, i], acc, zero)
    return r


def _orpit64(est, tgt, lens, rest_dtype=torch.float32):
    """(v (B, n) float64 candidate scores, -inf past n_b; their bounds; the rests as float64)"""
    B, n, T = tgt.shape
    x, t = est.double(), tgt.double()
    r = _rests(tgt.to(rest_dtype), lens).double()
    nb1 = (torch.tensor(lens, dtype=F64) - 1).view(B, 1)
    s0 = O.sisdr(x[:, :1].expand(B, n, T), t, eps=EPS)
    s1 = O.sisdr(x[:, 1:].expand(B, n, T), r, eps=EPS)
    v = s0 + s1 / nb1
    bound = _sisdr_bound(_stats(x[:, :1], t), s0) + _sisdr_bound(_stats(x[:, 1:], r), s1) / nb1 \
        + U * (s0.abs() + 2 * (s1 / nb1).abs() + v.abs())
    live = torch.arange(n).view(1, n) < torch.tensor(lens).view(B, 1)
    return v.masked_fill(~live, -float("inf")), bound, r


def _orpit_check(name, row):
    est, tgt, lens = row.make()
    B, n, T = tgt.shape
    cls, maximize = CRITS[row.crit]
    sign = 1.0 if maximize else -1.0
    v, vb, r = _orpit64(est, tgt, lens)
    # the batched reference against the oracle's per-sample loop (float64 rests there, so here too)
    m = min(B, 3)
    vd, _, _ = _orpit64(est[:m], tgt[:m], lens[:m], rest_dtype=F64)
    lo, io = PO.orpit(est[:m].double(), tgt[:m].double(), lens[:m], maximize=maximize, batch_mean=False)
    best = vd.max(1).values
    assert bool(((lo - sign * best).abs() <= 1e-9 * (1 + best.abs())).all()), (lo, sign * best)
    assert bool((vd.gather(1, io.view(m, 1)).squeeze(1) >= best - 1e-9 * (1 + best.abs())).all())
    # the kernel, through ORPIT with uneven weights on loss_b
    x = _put(est, row.layout).requires_grad_(True)
    tg = _put(tgt, "slice1" if row.layout == "slice1" else "contig")
    target = torch.nn.utils.rnn.pack_padded_sequence(tg, torch.tensor(lens), batch_first=True, enforce_sorted=False) \
        if row.packed else tg
    w = _weights(B)
    loss_b, idx = ORPIT(cls())(x, target, batch_mean=False)
    (loss_b * w.to(DEV)).sum().backward()
    idx, loss_b, grad = idx.cpu(), loss_b.detach().cpu().double(), x.grad.cpu().double()
    assert idx.dtype == torch.int64
    ar = torch.arange(B)
    # index: the fp64 best wherever it leads the runner-up by more than both bounds, optimal within the bounds everywhere
    top = v.topk(2, dim=1)
    i0, i1 = top.indices[:, 0], top.indices[:, 1]
    sep = (top.values[:, 0] - top.values[:, 1]) > vb[ar, i0] + vb[ar, i1]
    assert torch.equal(idx[sep], i0[sep]), (name, int((idx[sep] != i0[sep]).sum()))
    assert bool((v[ar, i0] - v[ar, idx] <= vb[ar, i0] + vb[ar, idx]).all()), (name, "not optimal within the bound")
    # value through the chosen candidate
    s_val = _share(name + " loss_b", (loss_b - sign * v[ar, idx]).abs(), vb[ar, idx])
    # gradient through the chosen candidate
    xd, td = est.double(), tgt.double()
    tsel, rsel = td[ar, idx], r[ar, idx]
    nb = torch.tensor(lens, dtype=F64)
    x64 = xd.clone().requires_grad_(True)
    lb64 = sign * (O.sisdr(x64[:, 0], tsel, eps=EPS) + O.sisdr(x64[:, 1], rsel, eps=EPS) / (nb - 1))
    (lb64 * w.double()).sum().backward()
    st0, st1 = _stats(xd[:, 0], tsel), _stats(xd[:, 1], rsel)
    g0 = sign * w.double()
    g1 = g0 / (nb - 1)
    ct0, cx0 = _grad_coef(st0)
    ct1, cx1 = _grad_coef(st1)
    live = (torch.arange(n).view(1, n) < nb.view(B, 1)).unsqueeze(-1)
    abs_others = (td.abs() * live).sum(1) - tsel.abs()
    gb0 = _grad_bound(st0, tsel, xd[:, 0], ct0 * g0, cx0 * g0)
    gb1 = _grad_bound(st1, rsel, xd[:, 1], ct1 * g1, cx1 * g1) + 2 * nb.view(B, 1) * U * (
        (ct1 * g1).abs().unsqueeze(-1) * abs_others + (cx1 * g1).abs().unsqueeze(-1) * xd[:, 1].abs())
    s_grad = _share(name + " gradient", (grad - x64.grad).abs(), torch.stack([gb0, gb1], 1))
    return idx, v, vb, s_val, s_grad, int((~sep).sum())


@pytest.mark.parametrize("name", list(ORPIT_ROWS))
def test_orpit_vs_fp64(name):
    """ORPIT(NegSISDR | SISDR): loss_b, indices and the input gradient of sum_b w_b loss_b against float64"""
    *_, s_val, s_grad, amb = _orpit_check(name, ORPIT_ROWS[name])
    print("[orpit {}] worst share of the bound: value {:.3f}, gradient {:.3f}{} -- {}".format(
        name, s_val, s_grad, " ({} samples optimal within the bound)".format(amb) if amb else "", ORPIT_ROWS[name].reaches))


ORPIT_TIES = {  # name: (n, T, i, k) -- k_orpit_finalize resolves the tie at shuffle distance 2^floor(log2(i ^ k))
    "tie_0_1_n3": (3, 256, 0, 1),
    "tie_1_2_n16": (16, 200, 1, 2),
    "tie_3_4_n16": (16, 128, 3, 4),
    "tie_7_8_n16": (16, 256, 7, 8),
    "tie_0_15_n16": (16, 64, 0, 15),
}


@pytest.mark.parametrize("name", list(ORPIT_TIES))
def test_orpit_exact_tie_takes_the_first_candidate(name):
    """t_i == t_k: candidates i and k score bit-equal (one CTA per sample at T <= 256); the first, i, is taken (torch.min / max)"""
    n, T, i, k = ORPIT_TIES[name]
    row = ORow(lambda: _orpit_tie(n, T, i, k, 40 + n + i + k), False, "NegSISDR", "contig", "")
    idx, v, vb, *_ = _orpit_check(name, row)
    assert float(v[0, i]) == float(v[0, k])
    others = [j for j in range(n) if j not in (i, k)]
    assert float(v[0, i] - v[0, others].max()) > float(vb[0, i] + vb[0, others].max()), "the tied pair must be the clear best"
    assert int(idx[0]) == i, (name, int(idx[0]))
    print("[orpit {}] kernel index {} (tied with {}), resolved at shuffle distance {}".format(name, int(idx[0]), k,
                                                                                            1 << ((i ^ k).bit_length() - 1)))


def test_orpit_launch_counts_past_65535_samples():
    """ctn_orpit_fwd / ctn_orpit_bwd called directly at B = 70000 (counts are per host thread): 3 forward, 2 backward"""
    B, n, T = 70000, 3, 9
    est, tgt = _orpit_gen([n] * B, T, 50)
    x, t = est.to(DEV), tgt.to(DEV)
    st = N.stream_ptr(DEV)
    lb, idx, dx = torch.empty(B, device=DEV), torch.empty(B, dtype=torch.int64, device=DEV), torch.empty_like(x)
    scratch = torch.empty(N.ctn_orpit_scratch_bytes(B, n) // 8 + 1, dtype=F64, device=DEV)
    N.check(N.ctn_orpit_fwd(x.data_ptr(), t.data_ptr(), None, B, n, T, EPS, 0, lb.data_ptr(), idx.data_ptr(), scratch.data_ptr(), st),
            "ctn_orpit_fwd")
    assert N.ctn_last_launch_count() == FWD_LAUNCHES
    N.check(N.ctn_orpit_bwd(x.data_ptr(), t.data_ptr(), None, idx.data_ptr(), B, n, T, EPS, 0, scratch.data_ptr(), None, dx.data_ptr(),
                            st), "ctn_orpit_bwd")
    assert N.ctn_last_launch_count() == BWD_LAUNCHES
    torch.cuda.synchronize()
    assert bool(torch.isfinite(lb).all()) and bool(torch.isfinite(dx).all())


# ---- SinkPIT -------------------------------------------------------------------------------------------------------------------

def _sink_gen(B, S, T, seed, snr_db=5.0):
    """estimates = targets of unequal levels permuted per sample + noise; w = weights of <P, w>"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(B, S, T, generator=g, dtype=F64) * torch.logspace(-0.3, 0.3, S, dtype=F64).view(1, S, 1)
    perm = torch.argsort(torch.rand(B, S, generator=g), dim=1)
    clean = torch.gather(t, 1, perm.unsqueeze(-1).expand(B, S, T))
    noise = torch.randn(B, S, T, generator=g, dtype=F64)
    noise = noise * clean.norm(dim=-1, keepdim=True) / noise.norm(dim=-1, keepdim=True).clamp_min(1e-300) * 10 ** (-snr_db / 20)
    w = torch.randn(B, S, S, generator=g)
    return (clean + noise).float(), t.float(), w


def _sink_mod(kind, B, S, T, seed, **kw):
    e, t, w = _sink_gen(B, S, T, seed, **kw)
    if kind == "x1e4":
        t = t * 1e4
    elif kind == "x1e-6":
        t = t * 1e-6
    elif kind == "dc1e3":
        e, t = e + 1e3, t + 1e3
    elif kind == "silent_tgt":
        t[:, 1] = 0                                             # column 1 of L: 10 log10(eps / (|e_i|^2 + eps)), tt = 0
    elif kind == "dup_tgt":
        t[:, 2] = t[:, 1]                                       # columns 1 and 2 of L bit-equal
        e = torch.stack([t[b, torch.tensor([1, 0, 3, 2])] for b in range(B)])
        e = e + 0.3 * torch.randn(e.shape, generator=torch.Generator().manual_seed(seed + 1))
    elif kind == "scaled":
        e = 2 * t[:, torch.arange(S).flip(0)]                   # est = 2 tgt (reversed): residual 0 on the matching pairs
    elif kind == "tail":
        e, t = _tail(e), _tail(t)
    return e, t, w


SRow = collections.namedtuple("SRow", "make K c crit layout drive reaches")


def _s(B, S, T, seed, kind=None, K=10, c=1.0, crit="NegSISDR", layout="contig", drive="both", reaches="", **kw):
    return SRow(lambda: _sink_mod(kind, B, S, T, seed, **kw), K, c, crit, layout, drive, reaches)


SINK_ROWS = {
    "T1": _s(3, 3, 1, 101, reaches="T = 1: one partial chunk of one sample"),
    "T255": _s(3, 3, 255, 102, crit="SISDR", drive="loss", reaches="T = PITX_C - 1"),
    "T256": _s(3, 3, 256, 103, drive="P", reaches="T = PITX_C: exactly one chunk"),
    "T257": _s(3, 3, 257, 104, reaches="T = PITX_C + 1: a second chunk of one sample"),
    "B1_Tbig": _s(1, 2, T_BIG, 105, kind="tail", reaches="B = 1, 529 chunks > gx = 528: stats grid stride to the last chunk; "
                  "pair backward gx = 64 < 133 (grid stride)"),
    **{f"S{S}": _s(2, S, 301 + S, 110 + S, crit="SISDR" if S % 3 == 0 else "NegSISDR",
                   drive=("loss", "P", "both")[S % 3], reaches=f"S = {S}: {S * S} pairs, KS = {ks}")
       for S, ks in ((1, 32), (2, 32), (4, 16), (5, 8), (8, 4), (9, 2), (12, 1), (16, 1))},
    "B528": _s(528, 2, 700, 130, reaches="B = PITX_CTAS: gx = 1, one CTA walks all 3 chunks"),
    "B600": _s(600, 2, 300, 131, drive="loss", reaches="B = 600: gx = 1 over 2 chunks"),
    "B70000": _s(70000, 2, 9, 132, reaches="B = 70000 > 65535: stats and pair backward loop samples over gridDim.y"),
    "x1e4": _s(3, 3, 1000, 140, kind="x1e4", reaches="targets x 1e4: alpha ~ 1e-4"),
    "x1e-6_T3": _s(3, 3, 3, 141, kind="x1e-6", reaches="targets x 1e-6 at T = 3: tt ~ eps"),
    "dc1e3": _s(3, 3, 1000, 142, kind="dc1e3", reaches="DC offset 1e3: every pair ~60 dB, P near uniform"),
    "silent_tgt": _s(3, 3, 1001, 143, kind="silent_tgt", reaches="t_1 = 0: tt = 0 for a whole column of L"),
    "scaled": _s(3, 3, 1001, 144, kind="scaled", crit="SISDR", reaches="est = 2 tgt: den = 0 on the matching pairs"),
    "K0_c1": _s(3, 3, 501, 150, K=0, c=1.0, drive="P", reaches="K = 0: P = exp(c SI-SDR) (< 1e5 here, fits fp32), loss = 0"),
    "K0_c1e-3": _s(3, 3, 501, 151, K=0, c=1e-3, reaches="K = 0 at coldness 1e-3: P ~ 1"),
    "K1": _s(3, 4, 501, 152, K=1, reaches="K = 1: one half-step pair each way"),
    "K1000": _s(2, 3, 501, 153, K=1000, reaches="K = 1000: the walk-back over 2000 half-steps"),
    "c1e-3": _s(3, 4, 501, 154, c=1e-3, reaches="coldness 1e-3: P ~ 1/S, Z / c ~ 1e3"),
    "c100_K100": _s(3, 4, 501, 155, K=100, c=100.0, snr_db=15.0, drive="P", reaches="coldness 100: P near a hard permutation"),
    "c1e3": _s(3, 4, 501, 156, c=1e3, snr_db=15.0, reaches="coldness 1e3: P a hard permutation, |Z| ~ 1e4"),
    "slice1_T1001": _s(3, 3, 1001, 160, layout="slice1",
                       reaches="est[1:], tgt[1:] of larger batches: bases at an odd float offset (3 * 1001), scalar loads"),
    "transposed": _s(3, 3, 1000, 161, layout="transposed", drive="P", reaches="transposed estimate: sinkpit's contiguous() copy"),
}


def _sinkhorn64(L, c, K, maximize):
    """PO.sinkpit's tail (pit.py:180-191) on the table L = -SI-SDR (B, S, S): (loss_b, P, Z)"""
    Z = -c * L
    for _ in range(K):
        Z = Z - torch.logsumexp(Z, dim=1, keepdim=True)
        Z = Z - torch.logsumexp(Z, dim=2, keepdim=True)
    P = torch.exp(Z)
    loss = torch.sum((L + Z / c) * P, dim=(1, 2))
    return (-loss if maximize else loss), P, Z


def _propagate(y, L, dLt):
    """sum_kl |d y_ij / d L_kl| dLt_kl for a (B, S, S) function y of the (B, S, S) leaf L (samples are independent)"""
    S = y.shape[1]
    out = torch.zeros_like(y, dtype=F64).detach()
    for i in range(S):
        for j in range(S):
            (J,) = torch.autograd.grad(y[:, i, j].sum(), L, retain_graph=True, allow_unused=True)
            if J is not None:
                out[:, i, j] = (J.abs() * dLt).sum((1, 2))
    return out


class _SinkRef:
    """float64 reference of one SinkPIT row: table, its bound, loss_b, P with their bounds, and dL / input gradient per driver"""

    def __init__(self, est, tgt, K, c, maximize):
        self.est, self.tgt, self.K, self.c, self.maximize = est, tgt, K, c, maximize
        x, t = est.double(), tgt.double()
        self.st = _stats(x.unsqueeze(2), t.unsqueeze(1))
        self.v = O.sisdr(x.unsqueeze(2), t.unsqueeze(1), eps=EPS)
        self.dLt = _sisdr_bound(self.st, self.v)
        self.L = (-self.v).requires_grad_(True)
        self.loss, self.P, Z = _sinkhorn64(self.L, c, K, maximize)
        Pd, Ld, self.Z = self.P.detach(), self.L.detach(), Z.detach()
        self.D = (2 * K + 2) * 2.0 ** -44 * (1 + self.Z.abs().amax((1, 2), keepdim=True))
        (gl,) = torch.autograd.grad(self.loss.sum(), self.L, retain_graph=True)
        self.b_loss = 2 * (gl.abs() * self.dLt).sum((1, 2)) + U * self.loss.detach().abs() \
            + self.D.view(-1) * ((Ld.abs() + self.Z.abs() / c + 1 / c) * Pd).sum((1, 2))
        self.b_P = 2 * _propagate(self.P, self.L, self.dLt) + (U + self.D) * Pd + 2.0 ** -149
        B = est.shape[0]
        m = min(B, 4)
        lo, Po = PO.sinkpit(x[:m], t[:m], coldness=c, iteration=K, maximize=maximize, batch_mean=False)
        assert bool(((lo - self.loss[:m].detach()).abs() <= 1e-3 * self.b_loss[:m]).all()), "restated Sinkhorn vs PO.sinkpit"
        assert bool(((Po - Pd[:m]).abs() <= 1e-3 * self.b_P[:m]).all()), "restated Sinkhorn vs PO.sinkpit"
        self._grads = {}

    def grads(self, key, wl, wp):
        """(dL64, its bound, input gradient64, its bound) of sum_b wl_b loss_b + sum wp * P, cached under key"""
        if key in self._grads:
            return self._grads[key]
        c, S = self.c, self.est.shape[1]
        wpd = torch.zeros_like(self.P) if wp is None else wp.double()
        total = (self.loss * wl.double()).sum() + (self.P * wpd).sum()
        (dL,) = torch.autograd.grad(total, self.L, create_graph=True)
        g = (wl.double() * (-1.0 if self.maximize else 1.0)).view(-1, 1, 1)
        Pd, Ld = self.P.detach(), self.L.detach()
        M = g.abs() * (Pd / c + (Ld.abs() + self.Z.abs() / c) * Pd) + wpd.abs() * Pd
        b_dL = 2 * _propagate(dL, self.L, self.dLt) + U * dL.detach().abs() \
            + self.D * (g.abs() * Pd + c * S * M.amax((1, 2), keepdim=True))
        dL = dL.detach()
        x, t = self.est.double(), self.tgt.double()
        xg = x.clone().requires_grad_(True)
        lo, Po = PO.sinkpit(xg, t, coldness=c, iteration=self.K, maximize=self.maximize, batch_mean=False)
        ((lo * wl.double()).sum() + (Po * wpd).sum()).backward()
        ct, cx = _grad_coef(self.st)
        wgt = -dL
        tt_, xx_ = t.unsqueeze(1), x.unsqueeze(2)
        a_t, a_x = ((ct * wgt).unsqueeze(-1) * tt_).abs(), ((cx * wgt).unsqueeze(-1) * xx_).abs()
        gb = _grad_bound(self.st, tt_, xx_, ct * wgt, cx * wgt) \
            + b_dL.unsqueeze(-1) * ((ct.unsqueeze(-1) * tt_).abs() + (cx.unsqueeze(-1) * xx_).abs()) + S * U * (a_t + a_x)
        self._grads[key] = (dL, b_dL, xg.grad, gb.sum(2))
        return self._grads[key]


def _pattern_check(name, pattern, ref):
    P64, bP = ref.P.detach(), ref.b_P
    S = P64.shape[-1]
    if S == 1:
        assert bool((pattern == 0).all())
        return 0
    top = P64.topk(2, dim=2)
    j0, j1 = top.indices[..., 0], top.indices[..., 1]
    g = lambda a, j: a.gather(2, j.unsqueeze(-1)).squeeze(-1)
    sep = (top.values[..., 0] - top.values[..., 1]) > g(bP, j0) + g(bP, j1)
    assert torch.equal(pattern[sep], j0[sep]), (name, "pattern")
    assert bool((g(P64, j0) - g(P64, pattern) <= g(bP, j0) + g(bP, pattern)).all()), (name, "pattern not optimal within the bound")
    return int((~sep).sum())


def _sink_check(name, row):
    est, tgt, gw = row.make()
    B, S, T = est.shape
    K, c = row.K, row.c
    cls, maximize = CRITS[row.crit]
    ref = _SinkRef(est, tgt, K, c, maximize)
    w = _weights(B)
    sh = {}
    xd, td = _put(est, row.layout), _put(tgt, "slice1" if row.layout == "slice1" else "contig")
    # C ABI: pair table, loss_b, P, then dL and d_est; grad_loss_b null means 1 per sample, grad_P null means none
    xc, tc = xd.contiguous(), td.contiguous()
    stp = N.stream_ptr(DEV)
    lb, P, pair = torch.empty(B, device=DEV), torch.empty(B, S, S, device=DEV), torch.empty(B, S, S, device=DEV)
    scratch = torch.empty(N.ctn_sinkpit_scratch_bytes(B, S, K) // 8 + 1, dtype=F64, device=DEV)
    N.check(N.ctn_sinkpit_fwd(xc.data_ptr(), tc.data_ptr(), B, S, T, K, float(c), EPS, int(maximize), lb.data_ptr(), P.data_ptr(),
                              pair.data_ptr(), scratch.data_ptr(), stp), "ctn_sinkpit_fwd")
    assert N.ctn_last_launch_count() == FWD_LAUNCHES
    use_l, use_p = row.drive in ("loss", "both"), row.drive in ("P", "both")
    gl_c, gp_c = (w.to(DEV) if use_l else None), (gw.to(DEV) if use_p else None)
    dL, dx = torch.empty(B, S, S, device=DEV), torch.empty_like(xc)
    N.check(N.ctn_sinkpit_bwd(xc.data_ptr(), tc.data_ptr(), B, S, T, K, float(c), EPS, int(maximize), scratch.data_ptr(), N.ptr(gl_c),
                              N.ptr(gp_c), dL.data_ptr(), dx.data_ptr(), stp), "ctn_sinkpit_bwd")
    assert N.ctn_last_launch_count() == BWD_LAUNCHES
    sh["pair"] = _share(name + " pair_sisdr", (pair.cpu().double() - ref.v).abs(), ref.dLt + U * ref.v.abs())
    sh["value"] = _share(name + " loss_b (C ABI)", (lb.cpu().double() - ref.loss.detach()).abs(), ref.b_loss)
    sh["P"] = _share(name + " P (C ABI)", (P.cpu().double() - ref.P.detach()).abs(), ref.b_P)
    dL64, b_dL, g64, gb = ref.grads(("w" if use_l else "ones", use_p), w if use_l else torch.ones(B), gw if use_p else None)
    sh["dL"] = _share(name + " dL (C ABI)", (dL.cpu().double() - dL64).abs(), b_dL)
    sh["gradient"] = _share(name + " d_est (C ABI)", (dx.cpu().double() - g64).abs(), gb)
    # Python: sinkpit() under autograd (an unused output passes no gradient: grad_loss_b = zeros, grad_P = null), SinkPIT's pattern
    x = _put(est, row.layout).requires_grad_(True)
    loss_p, P_p = sinkpit(cls(), x, td, coldness=c, iteration=K, batch_mean=False)
    total = (loss_p * w.to(DEV)).sum() if use_l else 0.0
    if use_p:
        total = total + (P_p * gw.to(DEV)).sum()
    total.backward()
    sh["value"] = max(sh["value"], _share(name + " loss_b", (loss_p.detach().cpu().double() - ref.loss.detach()).abs(), ref.b_loss))
    sh["P"] = max(sh["P"], _share(name + " P", (P_p.detach().cpu().double() - ref.P.detach()).abs(), ref.b_P))
    _, _, g64p, gbp = ref.grads(("w" if use_l else "zeros", use_p), w if use_l else torch.zeros(B), gw if use_p else None)
    sh["gradient"] = max(sh["gradient"], _share(name + " input gradient", (x.grad.cpu().double() - g64p).abs(), gbp))
    with torch.no_grad():
        _, pattern = SinkPIT(cls(), n_sources=S, coldness=c, iteration=K)(xd, td, batch_mean=False)
    pattern = pattern.cpu()
    assert pattern.dtype == torch.int64
    amb = _pattern_check(name, pattern, ref)
    return sh, amb, pattern, P.cpu(), ref


@pytest.mark.parametrize("name", list(SINK_ROWS))
def test_sinkpit_vs_fp64(name):
    """ctn_sinkpit_fwd / _bwd (pair table, loss_b, P, dL, d_est) and sinkpit() / SinkPIT (loss_b, P, pattern, input gradient)
    against float64, driven through loss_b, P or both as the row says"""
    sh, amb, *_ = _sink_check(name, SINK_ROWS[name])
    print("[sinkpit {}] worst share of the bound: {}{} -- {}".format(
        name, ", ".join("{} {:.3f}".format(k, v) for k, v in sh.items()),
        " ({} rows of P optimal within the bound)".format(amb) if amb else "", SINK_ROWS[name].reaches))


@pytest.mark.parametrize("T", [64, 256])
def test_sinkpit_equal_targets_take_the_first_column(T):
    """t_1 == t_2 bit-equal at T <= 256: columns 1 and 2 of the kernel's P are bit-equal, and the rows whose best target is the
    duplicated one take column 1 (torch.argmax's first maximum)"""
    row = _s(3, 4, T, 170 + T, kind="dup_tgt", K=50, c=10.0)
    _, _, pattern, P, ref = _sink_check(f"dup_tgt_T{T}", row)
    assert torch.equal(P[:, :, 1], P[:, :, 2])
    P64 = ref.P.detach()
    tied = (P64[:, :, 1] == P64[:, :, 2]) & (P64[:, :, 1] == P64.max(dim=2).values)
    assert int(tied.sum()) >= 3
    assert bool((pattern[tied] == 1).all()), pattern
