"""Edge cases of the SI-SDR / PIT loss (csrc/ctn_loss.cu) and of the native clip + Adam step (csrc/ctn_optim.cu, ctn_b200/optim.py),
``-m gpu``, against plain float64 references of the same operations on the same fp32 inputs.

Loss.  The reference is oracle/convtasnet_oracle.py (``sisdr``, ``sdr``, ``neg_sisdr``, ``pit_neg_sisdr``) in float64; gradients
come from float64 autograd driven by non-uniform per-sample weights on ``loss_b``.  Each LOSS_ROWS row names in `reaches` the
branch it selects and the constant that selects it.  The bound follows the kernel's arithmetic (``_sisdr_bound``):
  * <x,t> and |t|^2 are fp32 products summed in runs of at most four, then in double: relative error <= 4u kappa and 4u, with
    u = 2^-24 and kappa = sum|x t| / |sum x t| (the conditioning of the dot product);
  * alpha = <x,t> / (|t|^2 + eps) in fp32 (two casts, an add, a divide): eps_a = (4 kappa + 8) u;
  * the residual alpha t - x and its squares in fp32: alpha's own error cancels to first order in |alpha t - x|^2 (alpha is the
    minimiser), what is left is 2 u |r| |alpha t| (one rounding per element) plus eps_a^2 |alpha t|^2 and 2 eps_a |alpha <r,t>|
    (<r,t> != 0 only through eps); all over Q = |r|^2 + eps.  When |r|^2 >> eps the first term is the 2u |x| / |r| that makes a
    60 dB row legitimately worse than a 0 dB one;
  * num = alpha^2 |t|^2 (2 eps_a + 5u), the quotient (3u), and 10 log10f in fp32 (3u |v|).
  |v - v64| <= 2 * [4.343 (dnum / (num + eps) + dden / Q + 3u) + 3u |v64|]; the factor 2 covers the roundings of the double sums,
  the casts of the double statistics to fp32, and second-order terms.  The gradient of a pair, ct t + cx x with ct, cx from the
  double statistics, is held per element to 16 u (1 + kappa + |x| |r| / Q) (|ct64 t| + |cx64 x|) plus the fp32 rounding of
  both products: the coefficients inherit the relative error of the statistics.
Permutations must equal the fp64 oracle's wherever the best and second-best fp64 losses are further apart than their bounds;
where they are not (T = 1: every pair scores ~10 log10(x^2 / eps) whatever the target), the chosen permutation must be optimal
within the bound, and the gradient is checked through the permutation the kernel chose.  Exact ties are built so that the tied
permutations have bit-equal statistics (duplicated rows, T <= 256 so that each pass runs one CTA per sample), and the
lexicographically first one is asserted directly: the fp64 oracle's sum over sources is not order-symmetric.

Optimizer.  The reference is clip_grad_norm_ + Adam written out in float64 below (``_Adam64``), fed the same fp32 gradients and
the fp32-rounded beta1, beta2, eps and lr that the kernel receives.  Bound per element after k steps:
  sum_s C_ADAM u (|p64_s| + lr_s |D64_s| (1 + 1 / (2 (1 - beta2^t)) + 1 / (1 - beta1^t))),  D = m_hat / (sqrt(v_hat) + eps),
where the bias-correction terms are powf's rounding relative to 1 - beta^t (the kernel computes them in fp32), and C_ADAM = 32
covers the ~10 roundings of one update and the error the moments carry from step to step.  The reported norm is held to 2u.
"""
import collections
import ctypes as C
import itertools
import math

import pytest
import torch

import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import PIT1d
from ctn_b200.criterion.sdr import NegSISDR, SISDR, sdr, sisdr
from ctn_b200.optim import FlatClipAdam

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS = 1e-12
K10 = 10.0 / math.log(10.0)
C_GRAD = 16.0
C_ADAM = 32.0
DEV = torch.device("cuda")


# ---- loss: float64 statistics and bounds ----------------------------------------------------------------------------------

def _stats(x, t):
    """x, t float64 (..., T) -> dict of per-row float64 statistics"""
    xt, tt = (x * t).sum(-1), (t * t).sum(-1)
    axt = (x * t).abs().sum(-1)
    alpha = xt / (tt + EPS)
    r = alpha.unsqueeze(-1) * t - x
    den = (r * r).sum(-1)
    at2 = alpha * alpha * tt
    kappa = torch.where(axt == 0, torch.ones_like(axt), axt / xt.abs().clamp_min(1e-300))
    return dict(xt=xt, tt=tt, alpha=alpha, den=den, at2=at2, kappa=kappa, rt=(r * t).sum(-1), xn=x.norm(dim=-1),
                rn=den.sqrt())


def _sisdr_bound(st, v64):
    """per-row bound on |SI-SDR - SI-SDR64| (see the module docstring)"""
    ea = U * (4 * st["kappa"] + 8)
    Q = st["den"] + EPS
    dden = 3 * U * st["den"] + 2 * U * st["rn"] * st["at2"].sqrt() + (ea * ea + 2 * U * ea + 2 * U * U) * st["at2"] \
        + 2 * ea * (st["alpha"] * st["rt"]).abs()
    dnum = (2 * ea + 5 * U) * st["at2"]
    return 2 * (K10 * (dnum / (st["at2"] + EPS) + dden / Q + 3 * U) + 3 * U * v64.abs())


def _grad_coef(st):
    """(ct, cx) of sisdr_grad_coef in float64 from float64 statistics: dSI-SDR/dx = ct t + cx x"""
    xt, tt, den, alpha = st["xt"], st["tt"], st["den"], st["alpha"]
    P, Q = alpha * alpha * tt + EPS, den + EPS
    ct = K10 * (2 * alpha * tt / ((tt + EPS) * P) - (2 * (alpha * tt - xt) / (tt + EPS) - 2 * alpha) / Q)
    return ct, K10 * (-2.0 / Q)


def _grad_bound(st, t, x, ct, cx):
    """per-element bound on the gradient of one SI-SDR pair (rows of x, t) with coefficients ct, cx (already weighted)"""
    rel = C_GRAD * U * (1 + st["kappa"] + st["xn"] * st["rn"] / (st["den"] + EPS))
    a = (ct.unsqueeze(-1) * t).abs() + (cx.unsqueeze(-1) * x).abs()
    return rel.unsqueeze(-1) * a + 2 * U * a


def _pairs(x, t):
    """(B,S,T) -> pair statistics of (x_i, t_j) as (B,S,S) tensors and the (B,S,S) fp64 SI-SDR table"""
    B, S, _ = x.shape
    st = {k: v.expand(B, S, S) for k, v in _stats(x.unsqueeze(2), t.unsqueeze(1)).items()}
    return st, O.sisdr(x.unsqueeze(2), t.unsqueeze(1), eps=EPS)


PERMS = {S: torch.tensor(list(itertools.permutations(range(S))), dtype=torch.long) for S in range(1, 7)}


def _perm_losses(table, bound, S):
    """loss and bound of every permutation (B, S!): loss = -mean_i v[i, p(i)]; the fp32 sum over sources adds u sum|v|"""
    P = PERMS[S]
    ar = torch.arange(S)
    vals = table[:, ar.unsqueeze(0), P]                                # (B, S!, S)
    return -vals.mean(-1), bound[:, ar.unsqueeze(0), P].mean(-1) + U * vals.abs().sum(-1)


LEX = {S: {tuple(p): i for i, p in enumerate(P.tolist())} for S, P in PERMS.items()}


def _lex_index(perm):
    return LEX[len(perm)][tuple(perm)]


# ---- loss: inputs --------------------------------------------------------------------------------------------------------

def _gen(B, S, T, seed, snr_db=5.0):
    """targets ~ N(0, 1); estimate i = target pi_b(i) (a random permutation per sample) plus noise at snr_db"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(B, S, T, generator=g, dtype=torch.float64)
    pi = torch.stack([torch.randperm(S, generator=g) for _ in range(B)])
    n = torch.randn(B, S, T, generator=g, dtype=torch.float64)
    clean = torch.gather(t, 1, pi.unsqueeze(-1).expand(B, S, T))
    scale = clean.norm(dim=-1, keepdim=True) / n.norm(dim=-1, keepdim=True).clamp_min(1e-300) * 10 ** (-snr_db / 20)
    return (clean + n * scale).float(), t.float()


def _tie(S, T, seed, pi, dup_tgt=None, dup_est=None):
    """estimate i = target pi[i] + noise, with two target rows (dup_tgt) or two estimate rows (dup_est) made bit-equal, so that
    pi and pi with the duplicated pair exchanged score bit-equal losses"""
    g = torch.Generator().manual_seed(seed)
    t = torch.randn(1, S, T, generator=g)
    if dup_tgt:
        t[0, dup_tgt[1]] = t[0, dup_tgt[0]]
    e = t[0, list(pi)] + 0.3 * torch.randn(S, T, generator=g)
    if dup_est:
        a, b = dup_est
        e[a] = 0.5 * (t[0, pi[a]] + t[0, pi[b]]) + 0.3 * torch.randn(T, generator=g)
        e[b] = e[a]
    return e.unsqueeze(0).contiguous(), t


def _degenerate(kind, T, seed):
    e, t = _gen(3, 2, T, seed)
    if kind == "silent_tgt":
        t[1, 0] = 0
    elif kind == "silent_est":
        e[1, 1] = 0
    elif kind == "both_silent":
        e[2], t[2] = 0, 0
    elif kind == "scaled":
        e = 2.0 * t[:, [1, 0]]                                          # est = c tgt exactly: alpha = 2, residual 0
    return e, t


Row = collections.namedtuple("Row", "make layout reaches")


def _T_row(T, B=3):
    return lambda: _gen(B, 2, T, 1000 + T % 9973)


LOSS_ROWS = {
    **{f"T{T}": Row(_T_row(T), "contig", "T % 4 != 0: k_pit_pass1's scalar loop (nvec = 0)") for T in (1, 2, 3, 5, 7)},
    **{f"T{T}": Row(_T_row(T), "contig", "T % 4 == 0: k_pit_pass1's float4 loop, no scalar tail") for T in (4, 8, 1024)},
    "T1023": Row(_T_row(1023), "contig", "T % 4 == 3: scalar loop, pass 1 at gx = 1 over 1023 samples"),
    "T1025": Row(_T_row(1025), "contig", "T % 4 == 1: scalar loop, pass 2 at gx2 = 5 CTAs"),
    "T32772": Row(_T_row(32772, 2), "contig", "T/4 = 8193: pass 1 wants 33 CTAs, clamped to 32; pass 2 clamped to 64"),
    "T65537": Row(_T_row(65537, 2), "contig", "backward gx = 65 clamped to 64 (grid-stride over T), scalar pass 1 at 32"),
    "T2M": Row(_T_row(2 ** 21 + 1, 1), "contig", "T = 2^21 + 1: every grid clamp, ~256 samples per thread in pass 1"),
    **{f"S{S}": Row((lambda S=S: _gen(3, S, 4001, 2000 + S)), "contig",
                    f"S = {S}: {math.factorial(S)} permutations = {-(-math.factorial(S) // 32)} warp(s) in k_pit_finalize")
       for S in range(1, 7)},
    "x1e4": Row(lambda: (lambda e, t: (e, t * 1e4))(*_gen(3, 2, 4000, 31)), "contig", "targets x 1e4: alpha ~ 1e-4"),
    "tiny_T3": Row(lambda: (lambda e, t: (e, t * 1e-6))(*_gen(3, 2, 3, 32)), "contig",
                   "targets x 1e-6 at T = 3: |t|^2 ~ 3e-12 ~ eps, eps decides alpha, num and den"),
    "tiny_T8": Row(lambda: (lambda e, t: (e * 1e-6, t * 1e-6))(*_gen(3, 2, 8, 33)), "contig",
                   "both x 1e-6 at T = 8 (float4): |t|^2 ~ 8e-12"),
    "dc1e3": Row(lambda: (lambda e, t: (e + 1e3, t + 1e3))(*_gen(3, 2, 4000, 34)), "contig",
                 "DC offset 1e3 on both: kappa ~ 1, |x| / |r| ~ 1e3"),
    "silent_tgt": Row(lambda: _degenerate("silent_tgt", 1001, 35), "contig", "|t|^2 = 0: alpha = 0 / eps, num = 0"),
    "silent_est": Row(lambda: _degenerate("silent_est", 1001, 36), "contig", "x = 0: den = 0, SI-SDR = 0, gradient exactly 0"),
    "both_silent": Row(lambda: _degenerate("both_silent", 1000, 37), "contig", "x = t = 0: every statistic 0, SI-SDR 0"),
    "scaled": Row(lambda: _degenerate("scaled", 4001, 38), "contig", "est = 2 tgt exactly: residual 0, den + eps = eps"),
    **{f"snr{d}": Row((lambda d=d: _gen(3, 2, 4001, 40 + d, snr_db=d)), "contig",
                      f"SI-SDR ~ {d} dB: |x| / |r| ~ 10^{d // 20}, the residual carries the result") for d in (40, 60, 80)},
    **{f"off{k}_T{T}": Row(_T_row(T), f"off{k}", f"contiguous view at a {4 * k}-byte offset, T % 4 = {T % 4}"
                           + (": the float4 gate must refuse misaligned rows" if T % 4 == 0 else ": scalar loads"))
       for k in (1, 2, 3) for T in (1000, 1001)},
    "transposed": Row(_T_row(1000), "transposed", "non-contiguous (transposed storage): .contiguous() copies"),
    "B40000": Row(lambda: _gen(40000, 2, 16, 72), "contig", "B = 40000 > 65535 / 2: the backward's B S = 80000 rows loop over gridDim.y"),
}


def _place(x, layout):
    """GPU tensor equal to x in the given memory layout"""
    if layout == "contig":
        return x.to(DEV)
    if layout.startswith("off"):
        k = int(layout[3:])
        buf = torch.empty(x.numel() + k, device=DEV)
        v = buf[k:].view(x.shape)
        v.copy_(x)
        assert v.is_contiguous() and v.data_ptr() % 16 == 4 * k
        return v
    y = torch.empty(x.shape[0], x.shape[2], x.shape[1], device=DEV)
    y.copy_(x.transpose(1, 2))
    v = y.transpose(1, 2)
    assert not v.is_contiguous()
    return v


_REF = {}


def _reference(name):
    """(est, tgt, pair stats, fp64 table, pair bounds, oracle loss_b, oracle perm), cached per row"""
    if name not in _REF:
        e, t = LOSS_ROWS[name].make()
        x64, t64 = e.double(), t.double()
        st, table = _pairs(x64, t64)
        bound = _sisdr_bound(st, table)
        loss64, perm64 = O.pit_neg_sisdr(x64, t64, batch_mean=False)
        _REF[name] = (e, t, st, table, bound, loss64, perm64)
    return _REF[name]


def _weights(B, seed=5):
    return (0.5 + torch.rand(B, generator=torch.Generator().manual_seed(seed))).float()


def _grad64(x, t, perm, w):
    """fp64 autograd of sum_b w_b (-mean_i SI-SDR(x_i, t_perm[i])) through the given permutation"""
    x64 = x.detach().double().requires_grad_(True)
    tp = torch.gather(t.double(), 1, perm.unsqueeze(-1).expand_as(x64))
    loss_b = -O.sisdr(x64, tp, eps=EPS).mean(-1)
    (loss_b * w.double()).sum().backward()
    return x64.grad


def _check_pit(name):
    e, t, st, table, bound, loss64, perm64 = _reference(name)
    B, S, T = e.shape
    x, tg = _place(e, LOSS_ROWS[name].layout).requires_grad_(True), _place(t, LOSS_ROWS[name].layout)
    loss_b, perm = PIT1d(NegSISDR(), S)(x, tg, batch_mean=False)
    w = _weights(B)
    (loss_b * w.to(DEV)).sum().backward()
    perm, loss_b = perm.cpu(), loss_b.detach().cpu().double()
    # permutation: the oracle's wherever the fp64 optimum is separated from the runner-up by more than both bounds
    pl, pb = _perm_losses(table, bound, S)
    order = pl.argsort(dim=1, stable=True)
    ill = []
    for b in range(B):
        ours = _lex_index(perm[b].tolist())
        if S > 1 and pl[b, order[b, 1]] - pl[b, order[b, 0]] <= pb[b, order[b, 0]] + pb[b, order[b, 1]]:
            ill.append(b)
            assert pl[b, ours] - pl[b, order[b, 0]] <= pb[b, ours] + pb[b, order[b, 0]], (name, b, "not optimal within the bound")
        else:
            assert torch.equal(perm[b], perm64[b]), (name, b, perm[b], perm64[b])
    # value: loss of the chosen permutation vs fp64
    idx = torch.tensor([_lex_index(p) for p in perm.tolist()])
    ar = torch.arange(B)
    err = (loss_b - pl[ar, idx]).abs()
    lb = pb[ar, idx]
    assert bool((err <= lb).all()), "{}: loss error {} over bound {}".format(name, err.tolist(), lb.tolist())
    share = float((err / lb).max())
    d64 = _grad64(e, t, perm, w)
    ct, cx = _grad_coef(st)
    sel = lambda a: torch.gather(a, 2, perm.unsqueeze(-1)).squeeze(-1)          # (B,S) at j = perm[b, i]
    stp = {k: sel(v) for k, v in st.items()}
    coef = (w.double() * (-1.0 / S)).unsqueeze(-1)
    tp = torch.gather(t.double(), 1, perm.unsqueeze(-1).expand(B, S, T))
    gb = _grad_bound(stp, tp, e.double(), sel(ct) * coef, sel(cx) * coef)
    gerr = (x.grad.cpu().double() - d64).abs()
    bad = ~(gerr <= gb)  # a NaN counts as over the bound
    assert not bool(bad.any()), "{}: {} gradient entries over the bound, worst {:.3e} (bound {:.3e})".format(
        name, int(bad.sum()), float(gerr.max()), float(gb[gerr == gerr.max()][0]))
    return share, float((gerr / gb.clamp_min(1e-300)).max()), ill


@pytest.mark.parametrize("name", list(LOSS_ROWS))
def test_pit_vs_fp64(name):
    """PIT1d(NegSISDR) forward (loss_b, permutation) and backward (weighted loss_b) against the fp64 oracle on each LOSS_ROWS row"""
    share, gshare, ill = _check_pit(name)
    print("[{}] worst |loss - loss64| / bound {:.3f}, worst |grad - grad64| / bound {:.3f}{} -- {}".format(
        name, share, gshare, " (ill-conditioned permutation in samples {}: optimal within the bound)".format(ill) if ill else "",
        LOSS_ROWS[name].reaches))


# ---- ties -------------------------------------------------------------------------------------------------------------------

TIE_ROWS = {
    # name: (S, T, pi, dup_tgt, dup_est, reaches)
    "est01_S6": (6, 200, (0, 1, 2, 3, 4, 5), None, (0, 1), "est[0] == est[1]: indices 0 (warp 0) and 120 (warp 3) tie"),
    "hi_cross_S6": (6, 256, (5, 0, 2, 1, 3, 4), (0, 3), None, "minimum at index 606 (warp 18) ties with 686 (warp 21)"),
    "in_warp_S6": (6, 128, (2, 0, 1, 3, 5, 4), (4, 5), None, "tie of two neighbouring indices inside one warp (shuffle step)"),
    "in_warp_S3": (3, 17, (2, 0, 1), (0, 1), None, "S = 3: tie inside the single warp, scalar path"),
}


@pytest.mark.parametrize("name", list(TIE_ROWS))
def test_exact_ties_take_the_first_minimum(name):
    """Two permutations with bit-equal losses: the lexicographically first wins (torch.min's first minimum, pit.py:39)"""
    S, T, pi, dup_tgt, dup_est, reaches = TIE_ROWS[name]
    e, t = _tie(S, T, 77, pi, dup_tgt, dup_est)
    other = list(pi)
    if dup_tgt:
        a, b = dup_tgt
        other = [b if j == a else a if j == b else j for j in pi]
    else:
        a, b = dup_est
        other[a], other[b] = other[b], other[a]
    first = min(_lex_index(pi), _lex_index(other))
    loss_b, perm = PIT1d(NegSISDR(), S)(e.to(DEV), t.to(DEV), batch_mean=False)
    got = _lex_index(perm[0].tolist())
    assert got == first, (name, got, sorted((_lex_index(pi), _lex_index(other))))
    st, table = _pairs(e.double(), t.double())
    pl, pb = _perm_losses(table, _sisdr_bound(st, table), S)
    assert abs(float(loss_b[0]) - float(pl[0, first])) <= float(pb[0, first])
    # the tied pair is the optimum, every other permutation is clearly worse
    assert float(pl[0].sort().values[2]) > float(pl[0, first]) + 1.0
    print("[{}] kernel index {} (warp {}), tied with {} (warp {}) -- {}".format(
        name, got, got // 32, max(_lex_index(pi), _lex_index(other)), max(_lex_index(pi), _lex_index(other)) // 32, reaches))


# ---- sisdr() / sdr() rows, the criterion API, large batches ----------------------------------------------------------------

def _row_check(v, v64, bound, what):
    err = (v.detach().cpu().double() - v64).abs()
    assert bool((err <= bound).all()), "{}: {} rows over the bound, worst {:.3e}".format(what, int((err > bound).sum()), float(err.max()))
    return float((err / bound).max())


SISDR_ROWS = {
    "T5": (lambda: _gen(4, 3, 5, 51), "contig", "scalar path, S = 1 kernels with B = rows"),
    "T4096": (lambda: _gen(4, 3, 4096, 52), "contig", "float4 path"),
    "off1_T4000": (lambda: _gen(4, 3, 4000, 53), "off1", "misaligned base with T % 4 == 0: the float4 gate"),
    "off3_T4001": (lambda: _gen(4, 3, 4001, 54), "off3", "12-byte offset view, scalar loads"),
    "snr60": (lambda: _gen(4, 3, 4001, 55, snr_db=60), "contig", "60 dB rows"),
    "rows70000": (lambda: _gen(35000, 2, 12, 56), "contig", "70000 rows > 65535: the row loop over gridDim.y"),
}


@pytest.mark.parametrize("name", list(SISDR_ROWS))
def test_sisdr_rows_vs_fp64(name):
    """sisdr() no-grad (ctn_sisdr_fwd) and autograd (the S = 1 PIT pair), value and gradient against fp64 per row"""
    make, layout, reaches = SISDR_ROWS[name]
    e, t = make()
    x64, t64 = e.double(), t.double()
    st = _stats(x64, t64)
    v64 = O.sisdr(x64, t64, eps=EPS)
    bound = _sisdr_bound(st, v64)
    x, tg = _place(e, layout), _place(t, layout)
    with torch.no_grad():
        s1 = _row_check(sisdr(x, tg), v64, bound, name + " no-grad")
    xg = x.detach().clone().requires_grad_(True) if layout == "contig" else _place(e, layout).requires_grad_(True)
    v = sisdr(xg, tg)
    W = _weights(v.numel()).view(v.shape)
    (v * W.to(DEV)).sum().backward()
    s2 = _row_check(v, v64, bound, name + " autograd")
    xr = x64.clone().requires_grad_(True)
    (O.sisdr(xr, t64, eps=EPS) * W.double()).sum().backward()
    ct, cx = _grad_coef(st)
    gb = _grad_bound(st, t64, x64, ct * W.double(), cx * W.double())
    gerr = (xg.grad.cpu().double() - xr.grad).abs()
    assert bool((gerr <= gb).all()), "{}: {} gradient entries over the bound".format(name, int((gerr > gb).sum()))
    print("[sisdr {}] worst share: no-grad {:.3f}, autograd {:.3f}, gradient {:.3f} -- {}".format(
        name, s1, s2, float((gerr / gb.clamp_min(1e-300)).max()), reaches))


def _sdr_bound(x64, t64, v64):
    """|t|^2 in fp32 runs of <= 4 squares; the residual t - x rounded once, relative to itself, so its squares carry 2u more;
    casts, eps adds, quotient (5u each side); 10 log10f (3u |v|); factor 2 as for SI-SDR"""
    tt = (t64 * t64).sum(-1)
    ee = ((t64 - x64) ** 2).sum(-1)
    return 2 * (K10 * (5 * U * tt / (tt + EPS) + 7 * U * ee / (ee + EPS) + 3 * U) + 3 * U * v64.abs())


SDR_ROWS = {
    "T5": (lambda: _gen(3, 2, 5, 61), "contig", "T % 4 = 1: the scalar tail only"),
    "T1023": (lambda: _gen(3, 2, 1023, 62), "contig", "T % 4 = 3: odd rows start misaligned, scalar loop for those rows"),
    "T4100": (lambda: _gen(3, 2, 4100, 63), "contig", "aligned rows, float4 loop over 1025 vectors, gx = 2"),
    "off2_T4000": (lambda: _gen(3, 2, 4000, 64), "off2", "8-byte offset view: every row misaligned"),
    "snr70": (lambda: _gen(3, 2, 4001, 65, snr_db=70), "contig", "70 dB: the explicit residual t - x"),
    "rows70000": (lambda: _gen(35000, 2, 9, 66), "contig", "70000 rows > 65535: the row loop over gridDim.y"),
}


@pytest.mark.parametrize("name", list(SDR_ROWS))
def test_sdr_rows_vs_fp64(name):
    make, layout, reaches = SDR_ROWS[name]
    e, t = make()
    v64 = O.sdr(e.double(), t.double(), eps=EPS)
    with torch.no_grad():
        s = _row_check(sdr(_place(e, layout), _place(t, layout)), v64, _sdr_bound(e.double(), t.double(), v64), name)
    print("[sdr {}] worst share {:.3f} -- {}".format(name, s, reaches))


def test_4d_input_past_65535_rows():
    """(B, S, M, T) = (17000, 2, 2, 9): 68000 rows through sisdr() (no-grad and autograd) and NegSISDR's 4-D reduction"""
    e, t = _gen(34000, 2, 9, 71)
    e, t = e.view(17000, 2, 2, 9), t.view(17000, 2, 2, 9)
    x64, t64 = e.double(), t.double()
    v64 = O.sisdr(x64, t64, eps=EPS)
    bound = _sisdr_bound(_stats(x64, t64), v64)
    with torch.no_grad():
        s1 = _row_check(sisdr(e.to(DEV), t.to(DEV)), v64, bound, "4-D no-grad")
        loss = NegSISDR()(e.to(DEV), t.to(DEV), batch_mean=False)
    ref = O.neg_sisdr(x64, t64, batch_mean=False)
    assert bool(((loss.cpu().double() - ref).abs() <= bound.mean(dim=(1, 2)) + 4 * U * v64.abs().sum(dim=(1, 2))).all())
    xg = e.to(DEV).requires_grad_(True)
    v = sisdr(xg, t.to(DEV))
    v.sum().backward()
    s2 = _row_check(v, v64, bound, "4-D autograd")
    assert torch.isfinite(xg.grad).all()
    print("[4-D 68000 rows] worst share no-grad {:.3f}, autograd {:.3f}".format(s1, s2))


@pytest.mark.parametrize("cls", [NegSISDR, SISDR])
@pytest.mark.parametrize("reduction", ["mean", "sum"])
@pytest.mark.parametrize("batch_mean", [True, False])
def test_criterion_api_vs_reference_semantics(cls, reduction, batch_mean):
    """NegSISDR / SISDR x reduction x batch_mean on (B,S,T) directly and through PIT1d, against the reference's reductions"""
    e, t = _gen(5, 3, 1001, 81)
    x64, t64 = e.double(), t.double()
    sign = -1.0 if cls is NegSISDR else 1.0
    v64 = O.sisdr(x64, t64, eps=EPS)
    vb = _sisdr_bound(_stats(x64, t64), v64)
    red = (lambda a: a.mean(1)) if reduction == "mean" else (lambda a: a.sum(1))
    ref = red(sign * v64)
    bound = red(vb) + 3 * U * v64.abs().sum(1)
    if batch_mean:
        ref, bound = ref.mean(0), bound.mean(0) + 5 * U * ref.abs().sum()
    with torch.no_grad():
        got = cls(reduction=reduction)(e.to(DEV), t.to(DEV), batch_mean=batch_mean).cpu().double()
    assert bool(((got - ref).abs() <= bound).all()), (got, ref)
    # PIT over the same criterion: the reference's pit() applies the criterion per permutation and takes min (max for SISDR)
    pl64, perm64 = O.pit_neg_sisdr(x64, t64, batch_mean=False, reduction=reduction)
    with torch.no_grad():
        loss, perm = PIT1d(cls(reduction=reduction), 3)(e.to(DEV), t.to(DEV), batch_mean=batch_mean)
    assert torch.equal(perm.cpu(), perm64)
    want = -sign * pl64
    if batch_mean:
        want = want.mean(0)
    scale = 3.0 if reduction == "sum" else 1.0
    assert bool(((loss.cpu().double() - want).abs() <= scale * (vb.max() + 4 * U * v64.abs().max())).all()), (loss, want)


def test_launch_counts_are_constant():
    """per C call on this thread: PIT forward 3 (+1 with the batch mean), backward 1, sisdr 3, sdr 2, whatever B, S and T"""
    st = N.stream_ptr(DEV)
    for B, S, T in [(1, 1, 1), (3, 2, 4001), (70000, 1, 12), (40000, 2, 16), (2, 6, 32772), (1, 2, 65537)]:
        e, t = _gen(B, S, T, 91)
        x, tg = e.to(DEV), t.to(DEV)
        loss_b, lm = torch.empty(B, device=DEV), torch.empty(1, device=DEV)
        perm, d = torch.empty(B, S, dtype=torch.int64, device=DEV), torch.empty_like(x)
        scratch = torch.empty(N.ctn_sisdr_pit_scratch_bytes(B, S) // 8, dtype=torch.float64, device=DEV)
        for mean, want in ((None, 3), (lm.data_ptr(), 4)):
            N.check(N.ctn_sisdr_pit_fwd(x.data_ptr(), tg.data_ptr(), B, S, T, EPS, loss_b.data_ptr(), perm.data_ptr(), mean, None,
                                        scratch.data_ptr(), st))
            assert N.ctn_last_launch_count() == want, (B, S, T, mean)
        N.check(N.ctn_sisdr_pit_bwd(x.data_ptr(), tg.data_ptr(), perm.data_ptr(), B, S, T, EPS, scratch.data_ptr(), None, -1.0 / S,
                                    d.data_ptr(), st))
        assert N.ctn_last_launch_count() == 1
        rows = B * S
        out = torch.empty(rows, device=DEV)
        sc = torch.empty(N.ctn_sisdr_pit_scratch_bytes(rows, 1) // 8, dtype=torch.float64, device=DEV)
        N.check(N.ctn_sisdr_fwd(x.data_ptr(), tg.data_ptr(), rows, T, EPS, out.data_ptr(), sc.data_ptr(), st))
        assert N.ctn_last_launch_count() == 3
        N.check(N.ctn_sdr_fwd(x.data_ptr(), tg.data_ptr(), rows, T, EPS, out.data_ptr(), sc.data_ptr(), st))
        assert N.ctn_last_launch_count() == 2
    torch.cuda.synchronize()


# ---- optimizer ----------------------------------------------------------------------------------------------------------------

f32 = lambda a: float(torch.tensor(a, dtype=torch.float32))


class _Adam64:
    """clip_grad_norm_ + torch.optim.Adam (amsgrad off) in float64 over a list of tensors, with the fp32-rounded hyper-parameters
    the kernel receives; tracks the per-element error budget of the fp32 kernel"""

    def __init__(self, params, betas=(0.9, 0.999), eps=1e-8, wd=0.0, max_norm=0.0, step=0, m=None, v=None):
        self.p = [p.detach().double().clone() for p in params]
        self.m = [torch.zeros_like(p) for p in self.p] if m is None else [a.double().clone() for a in m]
        self.v = [torch.zeros_like(p) for p in self.p] if v is None else [a.double().clone() for a in v]
        self.b1, self.b2, self.eps, self.wd, self.max_norm = f32(betas[0]), f32(betas[1]), f32(eps), f32(wd), f32(max_norm)
        self.t = step
        self.budget = [torch.zeros_like(p) for p in self.p]

    def step(self, grads, lr):
        lr = f32(lr)
        g = [a.double() for a in grads]
        norm = math.sqrt(sum(float((a * a).sum()) for a in g))
        clip = min(1.0, self.max_norm / (norm + f32(1e-6))) if self.max_norm > 0 else 1.0
        self.t += 1
        bc1, bc2 = 1 - self.b1 ** self.t, 1 - self.b2 ** self.t
        for k, (p, gk) in enumerate(zip(self.p, g)):
            gk = gk * clip
            if self.wd != 0:
                gk = gk + self.wd * p
            self.m[k] = self.b1 * self.m[k] + (1 - self.b1) * gk
            self.v[k] = self.b2 * self.v[k] + (1 - self.b2) * gk * gk
            D = (self.m[k] / bc1) / ((self.v[k] / bc2).sqrt() + self.eps)
            p -= lr * D
            self.budget[k] += C_ADAM * U * (p.abs() + lr * D.abs() * (1 + 1 / (2 * bc2) + 1 / bc1))
        return norm


def _adam_check(got, ref, what):
    worst = 0.0
    for k, (a, r, b) in enumerate(zip(got, ref.p, ref.budget)):
        err = (a.detach().double() - r).abs()
        bad = ~(err <= b)  # a NaN counts as over the bound
        assert not bool(bad.any()), "{} tensor {}: {} entries over the bound, worst {:.3e} vs {:.3e}".format(
            what, k, int(bad.sum()), float(err.max()), float(b[err == err.max()][0]))
        worst = max(worst, float((err / b.clamp_min(1e-300)).max()))
    return worst


def _norm_check(tn, norm64):
    assert abs(float(tn) - norm64) <= 2 * U * norm64 + 1e-30, (float(tn), norm64)


class _Bucket(torch.nn.Module):
    """parameters whose .grad are views of one flat buffer at the given offsets, the layout the native backward produces"""

    def __init__(self, numels, offs, flat_len, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ps = torch.nn.ParameterList([torch.nn.Parameter((torch.randn(n, generator=g) * 0.1).to(DEV)) for n in numels])
        self.last_flat_grad = torch.zeros(flat_len, device=DEV)
        self.offs = offs
        for p, o in zip(self.ps, offs):
            p.grad = self.last_flat_grad[o:o + p.numel()]

    def fill(self, grads, pad=None):
        if pad is not None:
            self.last_flat_grad.copy_(pad)
        for g, o in zip(grads, self.offs):
            self.last_flat_grad[o:o + g.numel()].copy_(g)


def _grads(numels, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(n, generator=g, device=DEV) * scale for n in numels]


ABI_NUMELS = [1, 3, 2047, 2048, 2049, 6144, 6145, 100003]


def _abi_layout():
    """offsets that are not multiples of 64 (nor of 4), a gap of 5..11 floats after each tensor, flat length % 4 == 3"""
    offs, o = [], 7
    for k, n in enumerate(ABI_NUMELS):
        offs.append(o)
        o += n + 5 + k % 7
    o += (3 - o % 4) % 4
    assert o % 4 == 3 and all(x % 64 for x in offs)
    return offs, o


def test_clip_adam_c_abi_layout():
    """ctn_clip_adam_step through ctypes on the chunk-table edges (numel 1 .. 100003 around CHUNK = 2048), unaligned offsets, a
    flat length % 4 == 3 and NON-ZERO padding, which must stay out of the norm and untouched in m and v; 6 steps, clip active"""
    offs, L = _abi_layout()
    n = len(ABI_NUMELS)
    gen = torch.Generator(device=DEV).manual_seed(11)
    params = [torch.randn(k, generator=gen, device=DEV) * 0.1 for k in ABI_NUMELS]
    ref = _Adam64(params, max_norm=1.0)
    flat = torch.randn(L, generator=gen, device=DEV) * 3.0                       # padding: non-zero
    m, v = torch.full((L,), 7.0, device=DEV), torch.full((L,), 9.0, device=DEV)  # padding of the state: must stay as it is
    for k in range(n):
        m[offs[k]:offs[k] + ABI_NUMELS[k]] = 0
        v[offs[k]:offs[k] + ABI_NUMELS[k]] = 0
    numel_c = (C.c_int * n)(*ABI_NUMELS)
    nch = N.ctn_clip_adam_chunks(numel_c, n, None, None, 0)
    ct, co = (C.c_int * nch)(), (C.c_int * nch)()
    N.ctn_clip_adam_chunks(numel_c, n, ct, co, nch)
    table = torch.tensor([[ct[i], co[i]] for i in range(nch)], dtype=torch.int32, device=DEV)
    ptrs = torch.tensor([p.data_ptr() for p in params], dtype=torch.int64, device=DEV)
    offs_d = torch.tensor(offs, dtype=torch.int64, device=DEV)
    numel_d = torch.tensor(ABI_NUMELS, dtype=torch.int32, device=DEV)
    lr, step = torch.full((1,), 1e-3, device=DEV), torch.zeros(1, dtype=torch.int64, device=DEV)
    sumsq, tn = torch.zeros(1, dtype=torch.float64, device=DEV), torch.zeros(1, device=DEV)
    pad_mask = torch.ones(L, dtype=torch.bool, device=DEV)
    for k in range(n):
        pad_mask[offs[k]:offs[k] + ABI_NUMELS[k]] = False
    pad0 = flat[pad_mask].clone()
    for s in range(6):
        grads = _grads(ABI_NUMELS, 100 + s, scale=0.01 * (s + 1))
        for g, o in zip(grads, offs):
            flat[o:o + g.numel()] = g
        N.check(N.ctn_clip_adam_step(table.data_ptr(), nch, ptrs.data_ptr(), offs_d.data_ptr(), numel_d.data_ptr(), n, flat.data_ptr(),
                                     L, m.data_ptr(), v.data_ptr(), sumsq.data_ptr(), lr.data_ptr(), step.data_ptr(), 0.9, 0.999, 1e-8,
                                     0.0, 1.0, tn.data_ptr(), N.stream_ptr(DEV)), "ctn_clip_adam_step")
        assert N.ctn_last_launch_count() == 3
        norm64 = ref.step(grads, 1e-3)
        _norm_check(tn[0], norm64)
    assert norm64 > 1.0                                                       # the clip is active
    assert torch.equal(m[pad_mask], torch.full_like(pad0, 7.0)) and torch.equal(v[pad_mask], torch.full_like(pad0, 9.0))
    assert int(step[0]) == 6
    print("[C ABI] worst parameter error / bound {:.3f}".format(_adam_check(params, ref, "C ABI")))


@pytest.mark.parametrize("case", ["clip_lo", "clip_hi", "wd_clip", "betas_eps", "norm1e8", "norm1e-12"])
def test_clip_adam_hyper_parameters(case):
    """max_norm at the norm x (1 -/+ 1e-3) (clip active / inactive), weight decay 1e-2 with the clip, non-default betas and eps,
    gradient norms of 1e8 and 1e-12; 5 steps of FlatClipAdam on a bucket of 6 tensors"""
    numels = [5, 2048, 3001, 64, 2049, 777]
    offs, o = [], 0
    for k in numels:
        offs.append(o)
        o += (k + 63) // 64 * 64
    model = _Bucket(numels, offs, o, seed=21)
    scale = {"norm1e8": 1e8 / 60, "norm1e-12": 1e-12 / 60}.get(case, 1.0)
    grads = [_grads(numels, 200 + s, scale) for s in range(5)]
    norms = [math.sqrt(sum(float((g.double() ** 2).sum()) for g in gs)) for gs in grads]
    kw = dict(max_norm=norms[0] * (1 - 1e-3) if case == "clip_lo" else norms[0] * (1 + 1e-3) if case == "clip_hi" else 1.0)
    if case == "wd_clip":
        kw.update(weight_decay=1e-2)
    if case == "betas_eps":
        kw.update(betas=(0.8, 0.95), eps=1e-6, max_norm=0.0)
    if case.startswith("norm"):
        kw.update(max_norm=1.0, eps=1e-8)
    opt = FlatClipAdam(model, lr=1e-3, **kw)
    ref = _Adam64(list(model.ps), betas=kw.get("betas", (0.9, 0.999)), eps=kw.get("eps", 1e-8), wd=kw.get("weight_decay", 0.0),
                  max_norm=kw["max_norm"])
    for s in range(5):
        model.fill(grads[s])
        tn = opt.step()
        norm64 = ref.step(grads[s], 1e-3)
        _norm_check(tn[0], norm64)
    worst = _adam_check(list(model.ps), ref, case)
    print("[{}] worst parameter error / bound {:.3f}".format(case, worst))


def test_clip_adam_long_run_and_lr_halving():
    """1000 steps on a small bucket, lr halved through set_lr at steps 300 and 600: bias correction at large t, the step counter"""
    numels = [3, 2048, 1000]
    model = _Bucket(numels, [0, 64, 2112], 3136, seed=31)
    opt = FlatClipAdam(model, lr=1e-3, max_norm=2.0)
    ref = _Adam64(list(model.ps), max_norm=2.0)
    lr = 1e-3
    for s in range(1000):
        if s in (300, 600):
            lr /= 2
            opt.set_lr(lr)
        gs = _grads(numels, 1000 + s, scale=0.05)
        model.fill(gs)
        opt.step()
        ref.step(gs, lr)
    assert int(opt.step_count[0]) == 1000
    print("[1000 steps] worst parameter error / bound {:.3f}".format(_adam_check(list(model.ps), ref, "long run")))


def test_clip_adam_resume_at_a_large_step():
    """step_count = 100000 with preloaded m, v (as after loading a checkpoint): 1 - beta^t ~ 1, the moments dominate"""
    numels = [2049, 5]
    model = _Bucket(numels, [0, 2112], 2176, seed=41)
    opt = FlatClipAdam(model, lr=1e-3, max_norm=5.0)
    model.fill(_grads(numels, 400))
    lay = opt._bind(model.last_flat_grad)
    gen = torch.Generator(device=DEV).manual_seed(42)
    m0 = torch.randn(2176, generator=gen, device=DEV) * 1e-2
    v0 = torch.rand(2176, generator=gen, device=DEV) * 1e-4
    lay["m"].copy_(m0)
    lay["v"].copy_(v0)
    opt.step_count.fill_(100000)
    ref = _Adam64(list(model.ps), max_norm=5.0, step=100000, m=[m0[0:2049], m0[2112:2117]], v=[v0[0:2049], v0[2112:2117]])
    for s in range(3):
        gs = _grads(numels, 410 + s)
        model.fill(gs)
        opt.step()
        ref.step(gs, 1e-3)
    assert int(opt.step_count[0]) == 100003
    print("[resume] worst parameter error / bound {:.3f}".format(_adam_check(list(model.ps), ref, "resume")))


def _small_model():
    from test_parity_gpu import build_model
    cfg = O.OracleConfig(n_basis=32, kernel_size=16, sep_hidden_channels=64, sep_bottleneck_channels=32, sep_skip_channels=32,
                         sep_num_blocks=2, sep_num_layers=3, causal=False, n_sources=2)
    return build_model(cfg, O.synth_state_dict(cfg, seed=3)).train()


def test_clip_adam_frozen_parameter():
    """encoder.conv1d.weight frozen (fine-tuning): the native backward still writes its gradient into the flat bucket, but the norm
    is that of the trainable tensors only (what clip_grad_norm_(model.parameters()) sees), the frozen weight stays bit-unchanged
    and every other tensor matches the fp64 reference"""
    model = _small_model()
    frozen = model.encoder.conv1d.weight
    frozen.requires_grad_(False)
    w0 = frozen.detach().clone()
    opt = FlatClipAdam(model, lr=1e-3, max_norm=0.05)
    trainable = [p for p in model.parameters() if p.requires_grad]
    ref = _Adam64(trainable, max_norm=0.05)
    mixture, sources = O.synth_batch(2, 2, 2000, seed=8)
    for _ in range(3):
        opt.zero_grad()
        loss, _ = PIT1d(NegSISDR(), 2)(model(mixture.cuda()), sources.cuda())
        loss.backward()
        gs = [p.grad.detach().clone() for p in trainable]
        assert float(model.last_flat_grad.abs().sum()) > sum(float(g.abs().sum()) for g in gs)  # the frozen gradient is in the bucket
        tn = opt.step()
        _norm_check(tn[0], ref.step(gs, 1e-3))
    assert torch.equal(frozen.detach(), w0)
    print("[frozen encoder] worst parameter error / bound {:.3f}".format(_adam_check(trainable, ref, "frozen")))


def test_clip_adam_paper_size_bucket():
    """the paper-size bucket (N=512 L=16 B=128 H=512 Sc=128 X=8 R=3, 2 speakers) with the gradients of one native backward, 10 steps
    of that gradient scaled per step, with the clip active"""
    from test_parity_gpu import build_model
    cfg = O.OracleConfig(causal=False, n_sources=2, n_basis=512, kernel_size=16, sep_hidden_channels=512, sep_bottleneck_channels=128,
                         sep_skip_channels=128, sep_num_blocks=3, sep_num_layers=8)
    model = build_model(cfg, O.synth_state_dict(cfg, seed=113)).train()
    mixture, sources = O.synth_batch(1, 2, 800, seed=114)
    loss, _ = PIT1d(NegSISDR(), 2)(model(mixture.cuda()), sources.cuda())
    loss.backward()
    params = list(model.parameters())
    g0 = [p.grad.detach().clone() for p in params]
    norm0 = math.sqrt(sum(float((g.double() ** 2).sum()) for g in g0))
    opt = FlatClipAdam(model, lr=1e-3, max_norm=0.5 * norm0)
    ref = _Adam64(params, max_norm=0.5 * norm0)
    for s in range(10):
        gs = [g * (1.0 + 0.1 * s) for g in g0]
        for p, g in zip(params, gs):
            p.grad.copy_(g)
        tn = opt.step()
        _norm_check(tn[0], ref.step(gs, 1e-3))
    assert opt.launches_per_step == 3 and int(opt.step_count[0]) == 10
    print("[paper size, {} tensors, {} parameters] worst parameter error / bound {:.3f}".format(
        len(params), sum(p.numel() for p in params), _adam_check(params, ref, "paper")))


def test_clip_adam_graph_replay():
    """opt.step() captured in a CUDA graph after a warm-up step, replayed 5 times with new gradients copied into the captured flat
    buffer and set_lr between replays: equal to the same sequence run eagerly within the optimizer bound (not bitwise: k_sumsq adds
    its double partials with atomics in no fixed order), step counter advanced by 5 by the replays"""
    numels = [3, 2049, 700, 4096]
    offs = [0, 64, 2176, 2944]
    runs = {}
    for mode in ("eager", "graph"):
        model = _Bucket(numels, offs, 7040, seed=51)
        opt = FlatClipAdam(model, lr=1e-3, max_norm=1.0)
        model.fill(_grads(numels, 500))
        opt.step()                                                            # warm-up: binds the layout
        if mode == "graph":
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, capture_error_mode="relaxed"):
                opt.step()
            assert int(opt.step_count[0]) == 1                                 # capture runs nothing
        for k in range(5):
            model.fill(_grads(numels, 510 + k))
            opt.set_lr(1e-3 / (k + 1))
            if mode == "graph":
                graph.replay()
            else:
                opt.step()
        torch.cuda.synchronize()
        assert int(opt.step_count[0]) == 6, mode
        runs[mode] = [p.detach().clone() for p in model.ps]
    ref = _Adam64([p for p in _Bucket(numels, offs, 7040, seed=51).ps], max_norm=1.0)
    ref.step(_grads(numels, 500), 1e-3)
    for k in range(5):
        ref.step(_grads(numels, 510 + k), 1e-3 / (k + 1))
    w1, w2 = _adam_check(runs["eager"], ref, "eager"), _adam_check(runs["graph"], ref, "graph")
    for a, b, bud in zip(runs["graph"], runs["eager"], ref.budget):
        assert bool(((a - b).double().abs() <= 2 * bud).all())
    print("[graph replay] worst parameter error / bound: eager {:.3f}, replayed {:.3f}".format(w1, w2))
