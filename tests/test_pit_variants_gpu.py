"""ORPIT and Sinkhorn PIT on the GPU (``-m gpu``): ctn_orpit_* / ctn_sinkpit_* through ``ORPIT`` / ``sinkpit`` / ``SinkPIT``
against the oracle (tests/pit_variants_oracle.py ``orpit`` / ``sinkpit``) run in FLOAT64 with torch autograd, which is
pinned to the reference by tests/test_pit_variants_cpu.py.

Bounds: loss within 2e-4 dB (ORPIT) and 1e-4 * S dB (SinkPIT), P within 1e-5, indices and patterns exact, input gradients
within rtol 1e-4 + 1e-5 * max|g64| (the bound of test_sisdr_autograd_matches_oracle).  Each case also checks that its inputs
are well conditioned: the fp32 run of the oracle sits 10x inside every bound, and the best candidate (ORPIT) or every row's
argmax of P (SinkPIT) leads by a stated margin, so an exact index comparison is meaningful.
"""
import pytest
import torch

import convtasnet_oracle as O
import pit_variants_oracle as PO
from ctn_b200 import _native as N
from ctn_b200.criterion.pit import ORPIT, PIT1d, SinkPIT, sinkpit
from ctn_b200.criterion.sdr import NegSISDR, SISDR
from test_parity_gpu import build_model
from test_train_edges_gpu import MODES, _assert_well_conditioned, _check_grads

pytestmark = pytest.mark.gpu

CRITS = {"NegSISDR": (NegSISDR, False), "SISDR": (SISDR, True)}
ORPIT_LOSS_TOL = 2e-4
P_TOL = 1e-5
G_RTOL, G_ATOL = 1e-4, 1e-5
ORPIT_MARGIN = 1e-2   # dB between the best and the second-best candidate
P_MARGIN = 1e-3       # between the largest and the second-largest entry of every row of P (100x P_TOL)
FWD_LAUNCHES, BWD_LAUNCHES = 3, 2  # pass 1, pass 2, finalize / Sinkhorn; coefficients / Sinkhorn backward, pair backward


def _grad_err(g, g64):
    """max over entries of |g - g64| / (rtol |g64| + atol max|g64|): <= 1 passes"""
    return float(((g.double() - g64).abs() / (G_RTOL * g64.abs() + G_ATOL * float(g64.abs().max()) + 1e-30)).max())


# ---- ORPIT ---------------------------------------------------------------------------------------------------------------

def orpit_inputs(lens, T, seed, dup=False):
    """targets of unequal levels; estimate 0 = one target + noise, estimate 1 = the others' sum + noise.  dup: target 1 is a copy
    of target 0 and estimate 0 follows it, so candidates 0 and 1 tie exactly"""
    g = torch.Generator().manual_seed(seed)
    B, n = len(lens), max(lens)
    est, tgt = torch.zeros(B, 2, T), torch.zeros(B, n, T)
    for b, nb in enumerate(lens):
        t = torch.randn(nb, T, generator=g) * torch.logspace(-0.4, 0.4, nb)[torch.randperm(nb, generator=g)].unsqueeze(1)
        if dup:
            t[1] = t[0]
        k = 0 if dup else int(torch.randint(nb, (1,), generator=g))
        rest = t.sum(dim=0) - t[k]
        est[b, 0] = t[k] + 0.4 * t[k].std() * torch.randn(T, generator=g)
        est[b, 1] = rest + 0.4 * rest.std() * torch.randn(T, generator=g)
        tgt[b, :nb] = t
    return est, tgt


def orpit_margins(est, tgt, lens):
    """per sample: fp64 gap between the best and the second-best candidate score, and the index of the best"""
    out = []
    for b, nb in enumerate(lens):
        t = tgt[b, :nb].double()
        v = torch.stack([O.sisdr(est[b, 0].double(), t[i]) + O.sisdr(est[b, 1].double(), t.sum(0) - t[i]) / (nb - 1)
                         for i in range(nb)])
        s = torch.sort(v, descending=True).values
        out.append(float(s[0] - s[1]))
    return out


def orpit_reference(est, tgt, lens, maximize):
    """(loss_b64, idx64, grad64 of the batch mean, fp32 oracle's loss_b, idx, grad)"""
    res = []
    for dt in (torch.float64, torch.float32):
        x = est.to(dt).clone().requires_grad_(True)
        loss, idx = PO.orpit(x, tgt.to(dt), lens, maximize=maximize, batch_mean=False)
        loss.mean().backward()
        res.append((loss.detach(), idx, x.grad))
    return res


ORPIT_CASES = {  # name: (lens, T, seed, dup, packed)
    "n2_T1001_B4": ([2] * 4, 1001, 1, False, False),
    "n3_T1603_B8": ([3] * 8, 1603, 2, False, False),
    "n5_T32000_B4": ([5] * 4, 32000, 3, False, False),
    "n16_T1001_B3": ([16] * 3, 1001, 4, False, False),
    "n3_T128000_B2": ([3] * 2, 128000, 5, False, False),
    "n2_T32000_B64": ([2] * 64, 32000, 6, False, False),
    "packed_T1603": ([3, 2, 5, 2, 4, 16, 3], 1603, 7, False, True),
    "packed_T32000": ([2, 3, 3, 2], 32000, 8, False, True),
    # T <= 256: one chunk, so each sample's statistics come from one CTA and the tied candidates' scores are bit-equal
    "dup_tie_T256": ([3, 4, 2], 256, 9, True, True),
}


def _orpit_target(tgt, lens, packed):
    if not packed:
        return tgt.cuda()
    return torch.nn.utils.rnn.pack_padded_sequence(tgt.cuda(), torch.tensor(lens), batch_first=True, enforce_sorted=False)


@pytest.mark.parametrize("crit", list(CRITS))
@pytest.mark.parametrize("case", list(ORPIT_CASES))
def test_orpit_matches_fp64_oracle(case, crit):
    lens, T, seed, dup, packed = ORPIT_CASES[case]
    cls, maximize = CRITS[crit]
    est, tgt = orpit_inputs(lens, T, seed, dup)
    margins = orpit_margins(est, tgt, lens)
    (l64, i64, g64), (l32, i32, g32) = orpit_reference(est, tgt, lens, maximize)
    if dup:
        assert min(margins) == 0.0 and torch.equal(i64, torch.zeros_like(i64)), "the duplicated targets must tie at index 0"
    else:
        assert min(margins) >= ORPIT_MARGIN, f"ill-conditioned case: candidate margin {min(margins):.2e} dB"
    assert torch.equal(i32, i64)
    assert float((l32.double() - l64).abs().max()) <= ORPIT_LOSS_TOL / 10, "ill-conditioned case: fp32 oracle loss"
    assert _grad_err(g32, g64) <= 0.1, "ill-conditioned case: fp32 oracle gradient"
    x = est.cuda().requires_grad_(True)
    crit_m = ORPIT(cls())
    loss, idx = crit_m(x, _orpit_target(tgt, lens, packed), batch_mean=True)
    assert N.ctn_last_launch_count() == FWD_LAUNCHES
    loss.backward()
    with torch.no_grad():
        loss_b, _ = crit_m(est.cuda(), _orpit_target(tgt, lens, packed), batch_mean=False)
    assert idx.dtype == torch.int64 and torch.equal(idx.cpu(), i64)
    err = float((loss_b.cpu().double() - l64).abs().max())
    assert err <= ORPIT_LOSS_TOL, f"loss_b off by {err:.2e} dB"
    assert abs(float(loss.detach()) - float(l64.mean())) <= ORPIT_LOSS_TOL
    ge = _grad_err(x.grad.cpu(), g64)
    assert ge <= 1.0, f"input gradient error {ge:.2f} of the bound"
    print(f"[orpit {case} {crit}] loss {err:.2e} dB, gradient {ge:.3f} of bound, margin {min(margins):.3f} dB")


def test_orpit_n17_takes_the_generic_path():
    lens = [17, 17]
    est, tgt = orpit_inputs(lens, 203, 10)
    (l64, i64, g64), _ = orpit_reference(est, tgt, lens, False)
    x = est.cuda().requires_grad_(True)
    loss, idx = ORPIT(NegSISDR())(x, tgt.cuda(), batch_mean=False)
    loss.sum().backward()
    assert torch.equal(idx.cpu(), i64)
    assert float((loss.detach().cpu().double() - l64).abs().max()) <= ORPIT_LOSS_TOL
    assert _grad_err(x.grad.cpu() / 2, g64) <= 1.0


def test_orpit_rejects_one_target():
    est, tgt = orpit_inputs([3, 3], 203, 11)
    packed = torch.nn.utils.rnn.pack_sequence([tgt[0].cuda(), tgt[1, :1].cuda()], enforce_sorted=False)
    with pytest.raises(ValueError):
        ORPIT(NegSISDR())(est.cuda(), packed)
    with pytest.raises(ValueError):
        ORPIT(NegSISDR())(est.cuda(), tgt[:, :1].cuda())
    with pytest.raises(NotImplementedError):
        ORPIT(NegSISDR())(est.cuda().requires_grad_(True), tgt.cuda().requires_grad_(True))


# ---- SinkPIT -------------------------------------------------------------------------------------------------------------

# (S, K, coldness, crit) -> seed for the cases whose default seed 100 + S is ill-conditioned (all at coldness 0.1: there the fp32
# oracle's input gradient was up to 3.8x the bound away from fp64 on one sample's rows)
SINK_SEEDS = {
    (2, 200, 0.1, 'NegSISDR'): 1, (2, 200, 0.1, 'SISDR'): 1, (3, 200, 0.1, 'NegSISDR'): 14,
    (3, 200, 0.1, 'SISDR'): 11, (5, 200, 0.1, 'NegSISDR'): 2, (5, 200, 0.1, 'SISDR'): 2,
    (7, 1, 0.1, 'NegSISDR'): 1, (7, 1, 0.1, 'SISDR'): 1, (7, 10, 0.1, 'NegSISDR'): 1,
    (7, 10, 0.1, 'SISDR'): 1, (7, 200, 0.1, 'NegSISDR'): 1, (7, 200, 0.1, 'SISDR'): 1,
    (10, 1, 0.1, 'SISDR'): 1, (10, 10, 0.1, 'NegSISDR'): 1, (10, 10, 0.1, 'SISDR'): 1,
    (10, 200, 0.1, 'NegSISDR'): 1, (10, 200, 0.1, 'SISDR'): 1, (16, 1, 0.1, 'NegSISDR'): 4,
    (16, 1, 0.1, 'SISDR'): 4, (16, 10, 0.1, 'NegSISDR'): 4, (16, 10, 0.1, 'SISDR'): 4,
    (16, 200, 0.1, 'NegSISDR'): 4, (16, 200, 0.1, 'SISDR'): 4,
}


def sink_inputs(B, S, T, seed):
    """estimates = permuted targets of unequal levels + noise (SI-SDR about +5 dB on the matching pairs)"""
    g = torch.Generator().manual_seed(seed)
    tgt = torch.randn(B, S, T, generator=g) * torch.logspace(-0.3, 0.3, S).unsqueeze(-1)
    est = torch.stack([tgt[b, torch.randperm(S, generator=g)] for b in range(B)])
    est = est + 0.5 * est.std(dim=-1, keepdim=True) * torch.randn(B, S, T, generator=g)
    w = torch.randn(B, S, S, generator=g)  # weights of the extra loss term <P, w> that drives the d_P path
    return est, tgt, w


def sink_reference(est, tgt, w, K, c, maximize):
    """per dtype: (loss_b, P, grad of the batch-mean loss, grad of the batch-mean loss + <P, w>)"""
    res = []
    for dt in (torch.float64, torch.float32):
        out = []
        for use_p in (False, True):
            x = est.to(dt).clone().requires_grad_(True)
            loss, P = PO.sinkpit(x, tgt.to(dt), coldness=c, iteration=K, maximize=maximize, batch_mean=False)
            total = loss.mean() + ((P * w.to(dt)).sum() if use_p else 0.0)
            total.backward()
            out.append(x.grad)
        res.append((loss.detach(), P.detach(), out[0], out[1]))
    return res


def p_margin(P):
    s = torch.sort(P, dim=2, descending=True).values
    return float((s[..., 0] - s[..., 1]).min()) if P.shape[-1] > 1 else 1.0


SINK_CASES = [(S, K, c, crit) for S in (1, 2, 3, 5, 6, 7, 10, 16) for K in (1, 10, 200) for c in (0.1, 1.0, 10.0)
              for crit in CRITS]


@pytest.mark.parametrize("S,K,c,crit", SINK_CASES)
def test_sinkpit_matches_fp64_oracle(S, K, c, crit):
    cls, maximize = CRITS[crit]
    B, T = 3, 1001 + S
    est, tgt, w = sink_inputs(B, S, T, SINK_SEEDS.get((S, K, c, crit), 100 + S))
    (l64, P64, g64, gp64), (l32, P32, g32, gp32) = sink_reference(est, tgt, w, K, c, maximize)
    loss_tol = 1e-4 * S
    assert float((l32.double() - l64).abs().max()) <= loss_tol / 10, "ill-conditioned case: fp32 oracle loss"
    assert float((P32.double() - P64).abs().max()) <= P_TOL / 10, "ill-conditioned case: fp32 oracle P"
    assert max(_grad_err(g32, g64), _grad_err(gp32, gp64)) <= 0.1, "ill-conditioned case: fp32 oracle gradient"
    margin = p_margin(P64)
    assert margin >= P_MARGIN, f"argmax margin {margin:.2e}"
    crit_m = SinkPIT(cls(), n_sources=S, coldness=c, iteration=K)
    x = est.cuda().requires_grad_(True)
    loss_b, pattern = crit_m(x, tgt.cuda(), batch_mean=False)
    assert N.ctn_last_launch_count() == FWD_LAUNCHES
    loss_b.mean().backward()
    err = float((loss_b.detach().cpu().double() - l64).abs().max())
    assert err <= loss_tol, f"loss off by {err:.2e} dB"
    assert pattern.dtype == torch.int64 and torch.equal(pattern.cpu(), torch.argmax(P64, dim=2))
    ge = _grad_err(x.grad.cpu(), g64)
    assert ge <= 1.0, f"input gradient error {ge:.2f} of the bound"
    # P carries gradient: loss + <P, w>
    x2 = est.cuda().requires_grad_(True)
    loss2, P = sinkpit(cls(), x2, tgt.cuda(), coldness=c, iteration=K, batch_mean=True)
    perr = float((P.detach().cpu().double() - P64).abs().max())
    assert perr <= P_TOL, f"P off by {perr:.2e}"
    (loss2 + (P * w.cuda()).sum()).backward()
    gpe = _grad_err(x2.grad.cpu(), gp64)
    assert gpe <= 1.0, f"input gradient through P: error {gpe:.2f} of the bound"
    print(f"[sinkpit S={S} K={K} c={c} {crit}] loss {err:.2e} dB, P {perr:.1e}, grads {ge:.3f} / {gpe:.3f} of bound, "
          f"margin {margin:.2e}")


def test_sinkpit_generic_paths():
    """S = 17 and 4-D (multi-mic) inputs take the generic path with the reference's arithmetic.  For a 4-D input that is the
    reference's failure: its expand(-1, -1, n_sources, -1) names four sizes for a 5-D tensor (pit.py:169)."""
    est, tgt, _ = sink_inputs(2, 17, 203, 7)
    (l64, P64, _, _), _ = sink_reference(est, tgt, torch.zeros(2, 17, 17), 10, 1.0, False)
    loss, P = sinkpit(NegSISDR(), est.cuda(), tgt.cuda(), coldness=1.0, iteration=10, batch_mean=False)
    assert float((loss.cpu().double() - l64).abs().max()) <= 1e-4 * 17
    assert float((P.cpu().double() - P64).abs().max()) <= P_TOL
    est, tgt, _ = sink_inputs(2, 3, 203, 8)
    with pytest.raises(RuntimeError, match="number of sizes"):
        sinkpit(NegSISDR(), est.unsqueeze(2).cuda(), tgt.unsqueeze(2).cuda(), coldness=1.0, iteration=10)


# ---- cross-checks against the PIT kernels --------------------------------------------------------------------------------

@pytest.mark.parametrize("T", [1001, 32000])
@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6])
def test_pair_table_matches_pit_kernel(S, T):
    """SI-SDR(e_i, t_j) of ctn_sinkpit_fwd against ctn_sisdr_pit_fwd's pair_sisdr: within 1e-5 dB on the matching pairs
    (SI-SDR >= 0 dB).  A mismatched pair's <e, t> is a sum of T terms that nearly cancel, so any two fp32 accumulation orders
    differ there by up to ~1e-4 dB (both kernels do, on either side of fp64).  Every pair must sit within 1e-5 dB plus the
    fp32 accumulation bound of fp64: d(dB) = 20/ln 10 * d<e,t>/<e,t>, d<e,t> <= 4 eps32 sum_k |e_k t_k|."""
    est, tgt, _ = sink_inputs(4, S, T, 200 + S)
    x, t = est.cuda(), tgt.cuda()
    B, dev, st = 4, x.device, N.stream_ptr(x.device)
    ours, theirs = torch.empty(B, S, S, device=dev), torch.empty(B, S, S, device=dev)
    scratch = torch.empty(N.ctn_sinkpit_scratch_bytes(B, S, 1) // 8, dtype=torch.float64, device=dev)
    lb, P = torch.empty(B, device=dev), torch.empty(B, S, S, device=dev)
    N.check(N.ctn_sinkpit_fwd(x.data_ptr(), t.data_ptr(), B, S, T, 1, 1.0, 1e-12, 0, lb.data_ptr(), P.data_ptr(), ours.data_ptr(),
                              scratch.data_ptr(), st))
    sc2 = torch.empty(N.ctn_sisdr_pit_scratch_bytes(B, S) // 8, dtype=torch.float64, device=dev)
    perm = torch.empty(B, S, dtype=torch.int64, device=dev)
    N.check(N.ctn_sisdr_pit_fwd(x.data_ptr(), t.data_ptr(), B, S, T, 1e-12, lb.data_ptr(), perm.data_ptr(), None,
                                theirs.data_ptr(), sc2.data_ptr(), st))
    ref = O.sisdr(est.double().unsqueeze(2).expand(B, S, S, T), tgt.double().unsqueeze(1).expand(B, S, S, T))
    ours, theirs = ours.cpu().double(), theirs.cpu().double()
    good = ref >= 0
    assert good.sum() >= B * S
    assert float((ours - theirs)[good].abs().max()) <= 1e-5
    e64, t64 = est.double().unsqueeze(2), tgt.double().unsqueeze(1)
    cond = (e64 * t64).abs().sum(-1) / (e64 * t64).sum(-1).abs()
    tol = 1e-5 + 8.686 * 4 * 2 ** -24 * cond
    assert bool(((ours - ref).abs() <= tol).all()), float(((ours - ref).abs() / tol).max())


@pytest.mark.parametrize("S", [2, 3, 4, 5, 6])
def test_cold_sinkpit_pattern_equals_pit(S):
    est, tgt, _ = sink_inputs(6, S, 4000, 300 + S)
    loss, perm = PIT1d(NegSISDR(), S)(est.cuda(), tgt.cuda())
    _, pattern = SinkPIT(NegSISDR(), coldness=100.0, iteration=200)(est.cuda(), tgt.cuda())
    assert torch.equal(pattern, perm)


@pytest.mark.parametrize("B,S,K", [(1, 2, 0), (2, 3, 1), (8, 16, 200), (64, 5, 10)])
def test_launch_counts_are_constant(B, S, K):
    """ctn_last_launch_count after each C call (counts are per host thread, and autograd runs backward on its own thread, so
    the entries are called directly here): 3 forward, 2 backward, whatever B, S, n or K"""
    dev = torch.device("cuda")
    st, eps = N.stream_ptr(dev), 1e-12
    est, tgt, _ = sink_inputs(B, S, 333, 5)
    x, t = est.cuda(), tgt.cuda()
    lb, P, dL, dx = (torch.empty(B, device=dev), torch.empty(B, S, S, device=dev), torch.empty(B, S, S, device=dev),
                     torch.empty_like(x))
    scratch = torch.empty(N.ctn_sinkpit_scratch_bytes(B, S, K) // 8, dtype=torch.float64, device=dev)
    N.check(N.ctn_sinkpit_fwd(x.data_ptr(), t.data_ptr(), B, S, 333, K, 1.0, eps, 0, lb.data_ptr(), P.data_ptr(), None,
                              scratch.data_ptr(), st))
    assert N.ctn_last_launch_count() == FWD_LAUNCHES
    N.check(N.ctn_sinkpit_bwd(x.data_ptr(), t.data_ptr(), B, S, 333, K, 1.0, eps, 0, scratch.data_ptr(), None, P.data_ptr(),
                              dL.data_ptr(), dx.data_ptr(), st))
    assert N.ctn_last_launch_count() == BWD_LAUNCHES
    n = max(2, S)
    lens = [2 + b % (n - 1) for b in range(B)]
    est, tgt = orpit_inputs(lens, 333, 6)
    x, t = est.cuda(), tgt.cuda()
    n_b = torch.tensor(lens, dtype=torch.int32, device=dev)
    idx, dx = torch.empty(B, dtype=torch.int64, device=dev), torch.empty_like(x)
    scratch = torch.empty(N.ctn_orpit_scratch_bytes(B, n) // 8 + 1, dtype=torch.float64, device=dev)
    N.check(N.ctn_orpit_fwd(x.data_ptr(), t.data_ptr(), n_b.data_ptr(), B, n, 333, eps, 1, lb.data_ptr(), idx.data_ptr(),
                            scratch.data_ptr(), st))
    assert N.ctn_last_launch_count() == FWD_LAUNCHES
    N.check(N.ctn_orpit_bwd(x.data_ptr(), t.data_ptr(), n_b.data_ptr(), idx.data_ptr(), B, n, 333, eps, 1, scratch.data_ptr(),
                            None, dx.data_ptr(), st))
    assert N.ctn_last_launch_count() == BWD_LAUNCHES
    torch.cuda.synchronize()


# ---- training through the native node ------------------------------------------------------------------------------------

TRAIN_CFG = dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16,
                 sep_kernel_size=3, sep_num_blocks=1, sep_num_layers=3)


def _train_reference(cfg, sd, mixture, loss_fn):
    """(loss64, aux64, {key: grad64}, {key: fp32 oracle's distance to grad64})"""
    res = []
    for dt in (torch.float64, torch.float32):
        sdv = {k: v.to(dt).clone().requires_grad_(True) for k, v in sd.items()}
        out, _ = O.conv_tasnet_fwd(mixture.to(dt), sdv, cfg)
        loss, aux = loss_fn(out, dt)
        loss.backward()
        res.append((loss.detach(), aux, {k: v.grad for k, v in sdv.items()}))
    (l64, a64, g64), (_, _, g32) = res
    return l64, a64, g64, {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}


@pytest.mark.parametrize("mode", sorted({"fp32", MODES[-1]}))
def test_orpit_training_gradients_vs_fp64(mode):
    cfg = O.OracleConfig(causal=False, n_sources=2, **TRAIN_CFG)
    sd = O.synth_state_dict(cfg, seed=501)
    lens = [2, 3, 3, 2]
    mixture, sources = O.synth_batch(len(lens), 3, 1603, seed=502)
    for b, nb in enumerate(lens):
        sources[b, nb:] = 0
    l64, i64, g64, noise32 = _train_reference(cfg, sd, mixture,
                                              lambda out, dt: PO.orpit(out, sources.to(dt), lens, batch_mean=True))
    _assert_well_conditioned(g64, noise32)
    model = build_model(cfg, sd, math=mode).train()
    target = _orpit_target(sources, lens, True)
    loss, idx = ORPIT(NegSISDR())(model(mixture.cuda()), target)
    loss.backward()
    assert torch.equal(idx.cpu(), i64)
    assert abs(float(loss.detach()) - float(l64)) <= ORPIT_LOSS_TOL
    worst = _check_grads(model, g64, noise32)
    print(f"[orpit train {mode}] worst gradient error / role scale {worst[0]:.2e} ({worst[1]})")


@pytest.mark.parametrize("mode", sorted({"fp32", MODES[-1]}))
def test_sinkpit_training_gradients_vs_fp64(mode):
    cfg = O.OracleConfig(causal=False, n_sources=4, **TRAIN_CFG)
    sd = O.synth_state_dict(cfg, seed=511)
    mixture, sources = O.synth_batch(2, 4, 1603, seed=512)
    l64, _, g64, noise32 = _train_reference(cfg, sd, mixture,
                                            lambda out, dt: PO.sinkpit(out, sources.to(dt), coldness=1.0, iteration=10))
    _assert_well_conditioned(g64, noise32)
    model = build_model(cfg, sd, math=mode).train()
    loss, _ = SinkPIT(NegSISDR(), n_sources=4, coldness=1.0, iteration=10)(model(mixture.cuda()), sources.cuda())
    loss.backward()
    assert abs(float(loss.detach()) - float(l64)) <= 1e-4 * 4
    worst = _check_grads(model, g64, noise32)
    print(f"[sinkpit train {mode}] worst gradient error / role scale {worst[0]:.2e} ({worst[1]})")


def test_adam_steps_lower_the_orpit_loss():
    cfg = O.OracleConfig(causal=False, n_sources=2, **TRAIN_CFG)
    model = build_model(cfg, O.synth_state_dict(cfg, seed=521)).train()
    lens = [3, 2, 3]
    mixture, sources = O.synth_batch(len(lens), 3, 1603, seed=522)
    for b, nb in enumerate(lens):
        sources[b, nb:] = 0
    target = _orpit_target(sources, lens, True)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    crit = ORPIT(NegSISDR())
    losses = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        loss, _ = crit(model(mixture.cuda()), target)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses
