"""BSS Eval on the GPU (ctn_bss_eval_sources) against the fp64 oracle of tests/bss_ref.py: every SDR / SIR / SAR within 1e-4 dB,
the permutation wherever the oracle's best mean SIR is clear of the second by more than 1e-6 dB, the repeated mixture (the
tester's second call), projections that must and must not be forgiven, scale invariance, determinism, the refusals and the
reference-signature wrapper."""
import numpy as np
import pytest
import torch

import bss_ref as R

pytestmark = pytest.mark.gpu

TOL_DB = 1e-4


def _bss():
    from ctn_b200.utils import bss
    return bss


def _batch(seed, B, K, S, T, coloured):
    """ref (B, S, T), est (B, K, S, T) float32: set 0 the shuffled estimates of make_item, set 1 the mixture repeated S times"""
    rng = np.random.default_rng(seed)
    refs, ests = zip(*(R.make_item(rng, S, T, coloured) for _ in range(B)))
    ref = np.stack(refs)
    sets = [np.stack(ests)]
    if K > 1:
        sets.append(np.repeat(ref.sum(1, keepdims=True), S, axis=1))
    for _ in range(2, K):
        sets.append(np.stack([R.make_item(rng, S, T, coloured)[1] for _ in range(B)]))
    return torch.from_numpy(ref), torch.from_numpy(np.stack(sets, 1))


# (S, T, B, K, compute_permutation, coloured): every S, T, B, K and both settings appear with several of the others.  S L > T + L - 1
# makes the Gram matrix singular (test_singular_gram_is_reported), so S = 3 and 4 start at T = 4001.
ROWS = [(1, 600, 1, 1, True, False), (1, 40000, 5, 2, False, True), (1, 120000, 1, 2, True, False),
        (2, 600, 5, 2, True, False), (2, 4001, 1, 2, True, True), (2, 40000, 1, 2, True, True), (2, 40000, 5, 1, True, False),
        (2, 120000, 1, 1, False, False), (3, 4001, 5, 1, True, True), (3, 40000, 1, 2, False, False),
        (3, 120000, 1, 2, True, True), (4, 4001, 1, 1, True, True), (4, 40000, 5, 2, True, False), (4, 120000, 1, 1, False, False)]


@pytest.mark.parametrize("S,T,B,K,perm_on,coloured", ROWS)
def test_against_oracle(S, T, B, K, perm_on, coloured):
    bss = _bss()
    ref, est = _batch(1000 * S + T + B + K, B, K, S, T, coloured)
    sdr, sir, sar, perm = bss.bss_eval_sources_batch(ref.cuda(), est.cuda(), compute_permutation=perm_on)
    sdr, sir, sar, perm = (t.cpu().numpy() for t in (sdr, sir, sar, perm))
    worst = {"sdr": 0.0, "sir": 0.0, "sar": 0.0}
    checked = 0
    for b in range(B):
        for k in range(K):
            mixture = K > 1 and k == 1
            o_sdr, o_sir, o_sar, o_perm, margin = R.bss_eval_sources(ref[b].numpy(), est[b, k].numpy(), perm_on, return_margin=True)
            if margin > 1e-6:
                assert list(perm[b, k]) == list(o_perm), (b, k, perm[b, k], o_perm, margin)
                checked += 1
            elif not perm_on:
                assert list(perm[b, k]) == list(range(S))
            # compare the tables at the oracle's permutation, so that a near-tie cannot mix two estimates up
            g_sdr, g_sir, g_sar = sdr[b, k], sir[b, k], sar[b, k]
            if not np.array_equal(perm[b, k], o_perm):
                tab = bss.bss_eval_sources_batch(ref[b:b + 1].cuda(), est[b:b + 1, k:k + 1, list(o_perm)].cuda(), False)
                g_sdr, g_sir, g_sar = (t[0, 0].cpu().numpy() for t in tab[:3])
            # the residual behind the mixture's SAR is rounding noise on both sides, and with S = 1 so is the one behind its SDR
            # (the mixture is the reference): those are bounded below instead
            noise = {"sar"} | ({"sdr"} if S == 1 else set()) if mixture else set()
            pairs = [p for p in [("sdr", g_sdr, o_sdr), ("sir", g_sir, o_sir), ("sar", g_sar, o_sar)] if p[0] not in noise]
            for name, g in (("sdr", g_sdr), ("sar", g_sar)):
                if name in noise:
                    assert not np.isnan(g).any() and np.all(g >= 80.0), (name, g)
            for name, g, o in pairs:
                fin = np.isfinite(o)
                assert np.array_equal(np.isfinite(g), fin) and not np.isnan(g).any(), (name, g, o)
                assert np.array_equal(g[~fin], o[~fin]), (name, g, o)
                if fin.any():
                    err = float(np.max(np.abs(g[fin] - o[fin])))
                    worst[name] = max(worst[name], err)
                    assert err <= TOL_DB, (name, b, k, g, o)
            if S == 1:
                assert np.isposinf(g_sir).all()
    print("bss S={} T={} B={} K={} perm={} {}: worst |dSDR| {:.2e} |dSIR| {:.2e} |dSAR| {:.2e} dB, {} permutations checked".format(
        S, T, B, K, perm_on, "coloured" if coloured else "white", worst["sdr"], worst["sir"], worst["sar"], checked))


def _white(seed, S, T):
    return np.random.default_rng(seed).standard_normal((S, T)).astype(np.float32)


def test_filtered_reference_is_forgiven_and_a_long_delay_is_not():
    """e = r_j through a 512-tap FIR lies in the span of the delayed references: SDR >= 100 dB.  Delayed by 600 samples it does
    not (the filters stop at 511 samples of delay)."""
    bss = _bss()
    S, T = 2, 20000
    r = _white(7, S, T)
    r[:, T - 511:] = 0  # so that the whole filtered reference fits in T samples (the estimate is zero beyond T)
    rng = np.random.default_rng(8)
    fir = np.stack([np.convolve(r[j], rng.standard_normal(512) * np.exp(-np.arange(512) / 100.0))[:T] for j in range(S)])
    sdr, _, _, perm = bss.bss_eval_sources(torch.from_numpy(r), torch.from_numpy(fir.astype(np.float32)))
    print("bss 512-tap FIR: SDR", sdr.tolist())
    assert perm.tolist() == [0, 1] and bool((sdr >= 100.0).all())
    late = np.zeros_like(r)
    late[:, 600:] = r[:, :-600]
    sdr, _, _, _ = bss.bss_eval_sources(torch.from_numpy(r), torch.from_numpy(late), compute_permutation=False)
    print("bss 600-sample delay: SDR", sdr.tolist())
    assert bool((sdr < -10.0).all())


def test_scale_invariance_and_repeat_bits():
    bss = _bss()
    ref, est = _batch(21, 2, 2, 3, 8000, True)
    ref, est = ref.cuda(), est.cuda()
    a = bss.bss_eval_sources_batch(ref, est)
    b = bss.bss_eval_sources_batch(ref, est)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    # powers of two scale every product and sum exactly: the same bits
    p = bss.bss_eval_sources_batch(ref * 4.0, est * 0.125)
    assert all(torch.equal(x, y) for x, y in zip(a, p))
    # other scales round differently: within the bound against the oracle (coloured references)
    c = bss.bss_eval_sources_batch(ref * 5.3, est * 0.37)
    assert torch.equal(a[3], c[3])
    for x, y in zip(a[:2], c[:2]):
        assert float((x - y).abs().max()) <= TOL_DB
    assert float((a[2][:, 0] - c[2][:, 0]).abs().max()) <= TOL_DB  # SAR of the mixture set (k = 1) is rounding noise


def test_singular_gram_is_reported():
    """S L > T + L - 1: the S L delayed references cannot be independent; mir_eval would fall back to lstsq, this path says so"""
    bss = _bss()
    ref, est = _batch(5, 1, 1, 3, 600, False)
    with pytest.raises(ValueError, match="positive definite"):
        bss.bss_eval_sources_batch(ref.cuda(), est.cuda())


def test_refusals():
    bss = _bss()
    r, e = _white(1, 2, 3000), _white(2, 2, 3000)
    silent = r.copy()
    silent[1] = 0
    with pytest.raises(ValueError, match="reference source is silent"):
        bss.bss_eval_sources(torch.from_numpy(silent), torch.from_numpy(e))
    with pytest.raises(ValueError, match="estimated source is silent"):
        bss.bss_eval_sources(torch.from_numpy(r), torch.from_numpy(silent))
    with pytest.raises(ValueError, match="item 1"):
        ref = torch.from_numpy(np.stack([r, silent])).cuda()
        bss.bss_eval_sources_batch(ref, torch.from_numpy(np.stack([e, e]))[:, None].cuda())
    with pytest.raises(ValueError):
        bss.bss_eval_sources(torch.from_numpy(r), torch.from_numpy(e[:, :2999]))
    with pytest.raises(NotImplementedError):
        bss.bss_eval_sources(torch.from_numpy(_white(3, 5, 3000)), torch.from_numpy(_white(4, 5, 3000)))


def test_reference_signature():
    """the reference tester's call: CPU float32 (n_sources, T) or (T,) in, CPU float64 / int64 (n_sources,) out"""
    from utils.bss import bss_eval_sources  # the drop-in shim
    r, e = _white(11, 2, 5000), _white(12, 2, 5000)
    e = (e * 0.3 + r[::-1]).astype(np.float32)
    sdr, sir, sar, perm = bss_eval_sources(reference_sources=torch.from_numpy(r), estimated_sources=torch.from_numpy(e))
    for t in (sdr, sir, sar):
        assert t.dtype == torch.float64 and t.shape == (2,) and t.device.type == "cpu"
    assert perm.dtype == torch.int64 and perm.shape == (2,) and perm.tolist() == [1, 0]
    o = R.bss_eval_sources(r, e)
    for g, x in zip((sdr, sir, sar), o[:3]):
        assert np.max(np.abs(g.numpy() - x)) <= TOL_DB
    one = bss_eval_sources(torch.from_numpy(r[0]), torch.from_numpy(e[1]))
    assert [tuple(t.shape) for t in one] == [(1,)] * 4 and one[3].tolist() == [0] and np.isposinf(one[1].item())
    dev = bss_eval_sources(torch.from_numpy(r).cuda(), torch.from_numpy(e).cuda())
    assert all(t.is_cuda for t in dev) and torch.equal(dev[0].cpu(), sdr)
