"""Training with the SDR criterion on the GPU (``-m gpu``): the row backward ctn_sdr_bwd behind the SDR / NegSDR modules, the fused
PIT over SDR (ctn_sdr_pit_fwd / ctn_sdr_pit_bwd) behind PIT1d(NegSDR()), and the three recipes' training steps built on them.

Criterion: every value and every gradient element within the per-row bounds of tests/sdr_train_ref.py, which follow the kernels'
arithmetic, against float64 restatements on the same fp32 inputs.  Permutations equal the float64 ones wherever the best and the
second-best permutation are further apart than their bounds, and are optimal within the bounds elsewhere.  The model steps hold
every parameter gradient to 2e-4 of its role scale of fp64 autograd over the oracle (test_train_edges_gpu.py's criterion)."""
import os

import pytest
import torch

import convtasnet_oracle as O
import sdr_train_ref as R
from ctn_b200 import _native as N
from ctn_b200.criterion import pit as P
from ctn_b200.criterion.pit import ORPIT, PIT1d, SinkPIT
from ctn_b200.criterion.sdr import SDR, NegSDR
from test_parity_gpu import build_model
from test_train_edges_gpu import MODES, OUT_ATOL, OUT_RTOL, _assert_well_conditioned, _check_grads

pytestmark = pytest.mark.gpu

U = R.U
DEV = torch.device("cuda")


def _rand(shape, seed, scale=1.0):
    return scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))


def _assert_within(got, want, bound, what):
    err = (got.double().cpu() - want).abs()
    bad = ~(err <= bound)
    assert not bool(bad.any()), "{}: {} element(s) over the bound, worst |err| / bound = {:.3g} at {}".format(
        what, int(bad.sum()), float((err / bound).max()), tuple(int(i) for i in torch.nonzero(bad)[0]))
    return float((err / bound).max())


# ---- row SDR and its backward -----------------------------------------------------------------------------------------------

def _row_case(x, t, G, what):
    """SDR(reduction=None) rows under autograd, driven by the weights G (the row gradient is G itself, exact in fp32)"""
    xg = x.cuda().requires_grad_(True)
    v = SDR(reduction=None)(xg, t.cuda(), batch_mean=False)
    assert v.shape == x.shape[:-1] and v.requires_grad
    (v * G.cuda()).sum().backward()
    r1 = _assert_within(v.detach(), R.sdr64(x, t), R.sdr_bound(x, t), what + " value")
    r2 = _assert_within(xg.grad, R.sdr_grad64(x, t, G.double()), R.sdr_grad_bound(x, t, G.double()), what + " gradient")
    assert bool(torch.isfinite(xg.grad).all())
    print("[{}] worst error / bound: value {:.3f}, gradient {:.3f}".format(what, r1, r2))


@pytest.mark.parametrize("T", [1, 2, 3, 5, 4001, 160000, 352800])
def test_row_backward_vs_fp64(T):
    """(B, S, T) rows at T = 1, 2, 3 (no 128-bit body), 5 and 4001 (ragged rows: every row past the first unaligned), 160000 and
    352800 (20 s at 8 kHz, 8 s at 44.1 kHz: many chunks per row)"""
    B, S = (2, 2) if T > 10000 else (3, 4)
    t = _rand((B, S, T), 10 + T % 97)
    x = t + _rand((B, S, T), 11, 0.3) * torch.logspace(-3, 0, S).view(1, S, 1)
    G = _rand((B, S), 12)
    _row_case(x, t, G, "T={}".format(T))


@pytest.mark.parametrize("T", [4, 400, 4001])
@pytest.mark.parametrize("offset", [1, 2, 3])
def test_row_backward_offset_views(T, offset):
    """estimate and target as views starting `offset` floats into their storage: no 128-bit access is legal"""
    rows, n = 6, 6 * T
    tb = _rand((n + 4,), 20)
    xb = tb + _rand((n + 4,), 21, 0.1)
    t, x = tb[offset:offset + n].view(rows, T), xb[offset:offset + n].view(rows, T)
    tc, xv = tb.cuda()[offset:offset + n].view(rows, T), xb.cuda()[offset:offset + n].view(rows, T)
    assert xv.data_ptr() % 16 != 0 and tc.data_ptr() % 16 != 0
    xv.requires_grad_(True)
    G = _rand((rows,), 22)
    v = SDR(reduction=None)(xv, tc, batch_mean=False)
    (v * G.cuda()).sum().backward()
    _assert_within(v.detach(), R.sdr64(x, t), R.sdr_bound(x, t), "offset value")
    _assert_within(xv.grad, R.sdr_grad64(x, t, G.double()), R.sdr_grad_bound(x, t, G.double()), "offset gradient")


@pytest.mark.parametrize("T", [4, 5])
def test_row_backward_4d_past_65535_rows(T):
    """(2, 3, 11000, T): 66000 rows, past the 65535 rows one grid dimension holds"""
    t = _rand((2, 3, 11000, T), 30)
    x = t + _rand((2, 3, 11000, T), 31, 0.2)
    _row_case(x, t, _rand((2, 3, 11000), 32), "4-D, 66000 rows, T={}".format(T))


def test_row_backward_c_entry():
    """ctn_sdr_bwd with a null upstream gradient (= 1) and coef -0.5 on the scratch ctn_sdr_fwd left; one launch"""
    t = _rand((5, 1001), 40)
    x = t + _rand((5, 1001), 41, 0.5)
    xc, tc = x.cuda(), t.cuda()
    out = torch.empty(5, device=DEV)
    scratch = torch.empty(10, dtype=torch.float64, device=DEV)
    d = torch.empty_like(xc)
    N.check(N.ctn_sdr_fwd(xc.data_ptr(), tc.data_ptr(), 5, 1001, 1e-12, out.data_ptr(), scratch.data_ptr(), N.stream_ptr(DEV)), "fwd")
    N.check(N.ctn_sdr_bwd(xc.data_ptr(), tc.data_ptr(), 5, 1001, 1e-12, scratch.data_ptr(), None, -0.5, d.data_ptr(), N.stream_ptr(DEV)), "bwd")
    assert N.ctn_last_launch_count() == 1
    g = torch.full((5,), -0.5, dtype=torch.float64)
    _assert_within(d, R.sdr_grad64(x, t, g), R.sdr_grad_bound(x, t, g), "C entry gradient")


@pytest.mark.parametrize("kind", ["equal", "zero-target", "zero-estimate", "both-zero"])
def test_degenerate_rows(kind):
    """estimate == target: 10 log10((|t|^2 + eps) / eps) and a zero gradient; an all-zero target or estimate; both zero"""
    t = _rand((3, 2, 1001), 50)
    x = t + _rand((3, 2, 1001), 51, 0.1)
    if kind == "equal":
        x = t.clone()
    elif kind == "zero-target":
        t = torch.zeros_like(t)
    elif kind == "zero-estimate":
        x = torch.zeros_like(x)
    else:
        x, t = torch.zeros_like(x), torch.zeros_like(t)
    G = _rand((3, 2), 52)
    _row_case(x, t, G, kind)
    if kind == "equal":
        tt = (t.double() ** 2).sum(-1)
        torch.testing.assert_close(R.sdr64(x, t), 10 * torch.log10((tt + R.EPS) / R.EPS), rtol=1e-15, atol=0)
        xg = x.cuda().requires_grad_(True)
        NegSDR()(xg, t.cuda()).backward()
        assert float(xg.grad.abs().max()) == 0.0


# ---- fused PIT over SDR -----------------------------------------------------------------------------------------------------

def _pit_batch(B, S, T, seed, tie=None):
    """targets and estimates near a random permutation of them, the distortion spread over 0..60 dB across the batch.
    tie='exact': target 1 duplicates target 0; 'near': it differs from target 0 by 1e-7 relative."""
    t = _rand((B, S, T), seed)
    if tie == "exact":
        t[:, 1] = t[:, 0]
    elif tie == "near":
        t[:, 1] = t[:, 0] * (1 + 1e-7 * _rand((B, T), seed + 3))
    g = torch.Generator().manual_seed(seed + 1)
    perm = torch.stack([torch.randperm(S, generator=g) for _ in range(B)])
    sig = torch.logspace(-3, 0, B).view(B, 1, 1)
    x = torch.gather(t, 1, perm.unsqueeze(-1).expand(B, S, T)) + sig * _rand((B, S, T), seed + 2)
    return x, t


def _pit_call(x, t, mean=True, pair=True):
    B, S, T = x.shape
    xc, tc = x.cuda(), t.cuda()
    loss_b = torch.empty(B, device=DEV)
    perm = torch.empty(B, S, dtype=torch.int64, device=DEV)
    loss_mean = torch.empty(1, device=DEV) if mean else None
    pair_t = torch.empty(B, S, S, device=DEV) if pair else None
    scratch = torch.empty(N.ctn_sdr_pit_scratch_bytes(B, S) // 8, dtype=torch.float64, device=DEV)
    N.check(N.ctn_sdr_pit_fwd(xc.data_ptr(), tc.data_ptr(), B, S, T, 1e-12, loss_b.data_ptr(), perm.data_ptr(), N.ptr(loss_mean),
                              N.ptr(pair_t), scratch.data_ptr(), N.stream_ptr(DEV)), "ctn_sdr_pit_fwd")
    launches = N.ctn_last_launch_count()
    return dict(loss_b=loss_b.cpu(), perm=perm.cpu(), mean=None if loss_mean is None else loss_mean.cpu(),
                pair=None if pair_t is None else pair_t.cpu(), launches=launches, scratch=scratch, xc=xc, tc=tc, perm_dev=perm)


def _check_pit(got_loss_b, got_perm, ref, what):
    """loss_b within the bound of the float64 loss of the permutation the kernel chose; that permutation equal to the float64 one
    where the best is separated, optimal within the bounds elsewhere"""
    B, S = got_perm.shape
    place = S ** torch.arange(S - 1, -1, -1)   # itertools order is ascending in these codes
    chosen = torch.searchsorted((torch.tensor(R.perms(S), dtype=torch.long) * place).sum(1), (got_perm * place).sum(1))
    ar = torch.arange(B)
    _assert_within(got_loss_b, ref["all"][ar, chosen], ref["all_bound"][ar, chosen], what + " loss_b")
    sep = R.separated(ref)
    assert torch.equal(got_perm[sep], ref["perm"][sep]), what + ": permutation differs from fp64 on a separated sample"
    slack = ref["all"][ar, chosen] - ref["loss_b"] - ref["all_bound"][ar, chosen] - ref["bound"]
    assert bool((slack <= 0).all()), what + ": a permutation worse than the best beyond the bounds"
    return sep


@pytest.mark.parametrize("T", [200, 4000, 4001])
@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6])
def test_fused_pit_vs_fp64(S, T):
    """the C entry at every S: pair table (catches a transposed residual table), loss_b, permutation, batch mean, 3 launches;
    T = 200: one CTA per sample, 4000: 128-bit loads over several CTAs, 4001: element loads"""
    x, t = _pit_batch(6, S, T, 100 + S)
    ref = R.pit64(x, t)
    r = _pit_call(x, t)
    _assert_within(r["pair"], ref["v"], ref["v_bound"], "pair table")
    sep = _check_pit(r["loss_b"], r["perm"], ref, "S={} T={}".format(S, T))
    assert bool(sep.all())
    _assert_within(r["mean"][0:1], ref["loss_b"].mean().view(1), ref["bound"].mean().view(1) + 8 * U * ref["loss_b"].abs().mean(),
                   "batch mean")
    assert r["launches"] == 3


@pytest.mark.parametrize("S", [2, 3, 4, 5, 6])
def test_exact_ties_take_the_first_permutation(S):
    """target 1 duplicates target 0 (T = 200: one CTA per sample, so the tied pair statistics are bit-equal): the permutations that
    swap them tie exactly, and the lexicographically first one is taken"""
    x, t = _pit_batch(5, S, 200, 200 + S, tie="exact")
    ref = R.pit64(x, t)
    r = _pit_call(x, t)
    v = r["pair"]
    assert torch.equal(v[:, :, 0], v[:, :, 1])
    assert bool(R.separated(ref).all())
    assert torch.equal(r["perm"], ref["perm"])
    for b in range(5):   # the kernel's choice is the first of the exact ties
        p = r["perm"][b].tolist()
        assert p.index(0) < p.index(1), p


@pytest.mark.parametrize("S", [2, 3, 6])
def test_near_ties(S):
    """target 1 within 1e-7 of target 0: the two permutations are closer than their bounds, and the one chosen is optimal within them"""
    x, t = _pit_batch(5, S, 4001, 300 + S, tie="near")
    ref = R.pit64(x, t)
    r = _pit_call(x, t, pair=False)
    _check_pit(r["loss_b"], r["perm"], ref, "near ties S={}".format(S))


CRITERIA = [(cls, red, bm) for cls in (NegSDR, SDR) for red in ("mean", "sum") for bm in (True, False)]


@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6])
@pytest.mark.parametrize("crit", CRITERIA, ids=lambda c: "{}-{}-{}".format(c[0].__name__, c[1], "bm" if c[2] else "nobm"))
def test_pit_module_value_and_gradient(S, crit):
    """PIT1d(SDR | NegSDR, reduction mean | sum)(x, t, batch_mean) under autograd: the fused node; value = scale * loss_b (SDR
    negates, 'sum' multiplies by S); the gradient of non-uniform weights on loss_b through the selected permutation"""
    cls, red, bm = crit
    B, T = 5, 1001
    x, t = _pit_batch(B, S, T, 400 + S)
    ref = R.pit64(x, t)
    scale = (S if red == "sum" else 1) * (-1.0 if cls is SDR else 1.0)
    xg = x.cuda().requires_grad_(True)
    loss, perm = PIT1d(cls(reduction=red), S)(xg, t.cuda(), batch_mean=bm)
    assert torch.equal(perm.cpu(), ref["perm"])
    w = torch.linspace(0.5, 2.0, B)
    if bm:
        _assert_within(loss.detach().view(1) / scale, ref["loss_b"].mean().view(1),
                       ref["bound"].mean().view(1) + 8 * U * ref["loss_b"].abs().mean(), "loss")
        loss.backward()
        g = torch.full((B,), scale / B, dtype=torch.float64)
    else:
        _assert_within(loss.detach() / scale, ref["loss_b"], ref["bound"], "loss_b")
        (loss * w.cuda()).sum().backward()
        g = w.double() * scale
    _assert_within(xg.grad, R.pit_grad64(x, t, ref["perm"], g), R.pit_grad_bound(x, t, ref["perm"], g, g_rel=3 * U), "gradient")
    with torch.no_grad():
        loss_ng, perm_ng = PIT1d(cls(reduction=red), S)(x.cuda(), t.cuda(), batch_mean=bm)
    assert torch.equal(perm_ng, perm)


def test_pit_past_65535_samples():
    """B = 66000 samples: the pass and the backward loop over the grid's 65535 rows"""
    B, S, T = 66000, 2, 8
    x, t = _pit_batch(B, S, T, 500)
    ref = R.pit64(x, t)
    xg = x.cuda().requires_grad_(True)
    loss_b, perm = PIT1d(NegSDR(), S)(xg, t.cuda(), batch_mean=False)
    _check_pit(loss_b.detach().cpu(), perm.cpu(), ref, "B=66000")
    w = torch.linspace(0.5, 2.0, B)
    (loss_b * w.cuda()).sum().backward()
    pc = perm.cpu()
    _assert_within(xg.grad, R.pit_grad64(x, t, pc, w.double()), R.pit_grad_bound(x, t, pc, w.double(), g_rel=U), "gradient")


@pytest.mark.parametrize("S", [1, 2, 3, 4, 5, 6])
def test_fused_matches_the_generic_loop(S):
    """no grad: the fused PIT1d(NegSDR) and the reference's loop over the permutations (which evaluates NegSDR S! times) agree
    within the two bounds, with the same permutation wherever the best two are separated"""
    x, t = _pit_batch(4, S, 1001, 600 + S)
    ref = R.pit64(x, t)
    with torch.no_grad():
        fl, fp = PIT1d(NegSDR(), S)(x.cuda(), t.cuda(), batch_mean=False)
        gl, gp = P._pit_generic(NegSDR(), x.cuda(), t.cuda(), batch_mean=False)
    sep = R.separated(ref)
    assert torch.equal(fp.cpu()[sep], gp.cpu()[sep])
    _assert_within(fl.cpu(), gl.cpu().double(), 2 * ref["all_bound"].max(dim=1).values, "fused vs generic")


# ---- launches and graph capture -----------------------------------------------------------------------------------------------

def test_launch_counts_do_not_depend_on_the_shape():
    """forward: pass + finalize (+ batch mean); backward: one kernel; the row backward: one kernel -- at every B, S, T"""
    seen = set()
    for B in (1, 3, 70000):
        for S in (1, 3, 6):
            for T in (1, 5, 4001):
                if B * S * T > 3e7:
                    continue
                x, t = _pit_batch(B, S, T, 700) if B < 70000 else (_rand((B, S, T), 701), _rand((B, S, T), 702))
                for mean in (True, False):
                    r = _pit_call(x, t, mean=mean, pair=False)
                    seen.add(("fwd", mean, r["launches"]))
                d = torch.empty_like(r["xc"])
                N.check(N.ctn_sdr_pit_bwd(r["xc"].data_ptr(), r["tc"].data_ptr(), r["perm_dev"].data_ptr(), B, S, T, 1e-12,
                                          r["scratch"].data_ptr(), None, -1.0 / S, d.data_ptr(), N.stream_ptr(DEV)), "bwd")
                seen.add(("bwd", N.ctn_last_launch_count()))
                rows, row = B * S, torch.empty(B * S, device=DEV)
                row_scratch = torch.empty(2 * rows, dtype=torch.float64, device=DEV)
                N.check(N.ctn_sdr_fwd(r["xc"].data_ptr(), r["tc"].data_ptr(), rows, T, 1e-12, row.data_ptr(), row_scratch.data_ptr(),
                                      N.stream_ptr(DEV)), "row fwd")
                N.check(N.ctn_sdr_bwd(r["xc"].data_ptr(), r["tc"].data_ptr(), rows, T, 1e-12, row_scratch.data_ptr(), None, 1.0,
                                      d.data_ptr(), N.stream_ptr(DEV)), "row bwd")
                seen.add(("row bwd", N.ctn_last_launch_count()))
    assert seen == {("fwd", True, 3), ("fwd", False, 2), ("bwd", 1), ("row bwd", 1)}, seen


def test_graph_capture_replays_equal_to_eager():
    """ctn_sdr_pit_fwd + ctn_sdr_pit_bwd and ctn_sdr_fwd + ctn_sdr_bwd captured in one CUDA graph replay bit-equal to eager
    (T = 1000: one CTA per sample, so the double sums are order-deterministic)"""
    B, S, T = 4, 3, 1000
    x, t = _pit_batch(B, S, T, 800)
    xc, tc = x.cuda(), t.cuda()
    g = torch.linspace(0.5, 2.0, B, device=DEV)
    bufs = dict(loss_b=torch.empty(B, device=DEV), perm=torch.empty(B, S, dtype=torch.int64, device=DEV),
                mean=torch.empty(1, device=DEV), scratch=torch.empty(N.ctn_sdr_pit_scratch_bytes(B, S) // 8, dtype=torch.float64, device=DEV),
                d=torch.empty_like(xc), row=torch.empty(B * S, device=DEV), row_scratch=torch.empty(2 * B * S, dtype=torch.float64, device=DEV),
                row_d=torch.empty_like(xc))

    def run():
        st = N.stream_ptr(DEV)
        N.check(N.ctn_sdr_pit_fwd(xc.data_ptr(), tc.data_ptr(), B, S, T, 1e-12, bufs["loss_b"].data_ptr(), bufs["perm"].data_ptr(),
                                  bufs["mean"].data_ptr(), None, bufs["scratch"].data_ptr(), st), "fwd")
        N.check(N.ctn_sdr_pit_bwd(xc.data_ptr(), tc.data_ptr(), bufs["perm"].data_ptr(), B, S, T, 1e-12, bufs["scratch"].data_ptr(),
                                  g.data_ptr(), -1.0 / S, bufs["d"].data_ptr(), st), "bwd")
        N.check(N.ctn_sdr_fwd(xc.data_ptr(), tc.data_ptr(), B * S, T, 1e-12, bufs["row"].data_ptr(), bufs["row_scratch"].data_ptr(), st),
                "row fwd")
        N.check(N.ctn_sdr_bwd(xc.data_ptr(), tc.data_ptr(), B * S, T, 1e-12, bufs["row_scratch"].data_ptr(), None, 1.0,
                              bufs["row_d"].data_ptr(), st), "row bwd")

    run()
    torch.cuda.synchronize()
    eager = {k: v.clone() for k, v in bufs.items() if k not in ("scratch", "row_scratch")}
    for v in bufs.values():
        v.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, capture_error_mode="relaxed"):
        run()
    graph.replay()
    torch.cuda.synchronize()
    for k, v in eager.items():
        assert torch.equal(bufs[k], v), k


# ---- end to end: the recipes' training steps ------------------------------------------------------------------------------------

SMALL = dict(n_basis=32, kernel_size=16, sep_bottleneck_channels=16, sep_hidden_channels=32, sep_skip_channels=16, sep_kernel_size=3,
             sep_num_blocks=1, sep_num_layers=3, n_sources=2)


def _oracle_pit_grads(cfg, sd, mixture, sources, dtype):
    sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    out, _ = O.conv_tasnet_fwd(mixture.to(dtype), sdv, cfg)
    loss, perm = R.pit_neg_sdr_autograd(out, sources.to(dtype))
    loss.backward()
    return out.detach(), perm, {k: v.grad for k, v in sdv.items()}


@pytest.mark.parametrize("causal", [False, True], ids=["gLN", "cLN"])
def test_pit_neg_sdr_step_vs_fp64(causal):
    """the WHAM recipe's step, PIT1d(NegSDR(), 2)(model(mixture), sources).backward(), through the gLN step and the cLN step
    (causal_training): permutation and every parameter gradient against fp64 autograd over the oracle"""
    cfg = O.OracleConfig(causal=causal, **SMALL)
    sd = O.synth_state_dict(cfg, seed=901)
    mixture, sources = O.synth_batch(3, cfg.n_sources, 1037, seed=902)
    out64, perm64, g64 = _oracle_pit_grads(cfg, sd, mixture, sources, torch.float64)
    _, perm32, g32 = _oracle_pit_grads(cfg, sd, mixture, sources, torch.float32)
    assert torch.equal(perm32, perm64)
    noise32 = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
    _assert_well_conditioned(g64, noise32)
    model = build_model(cfg, sd, math=MODES[-1]).train()
    model.causal_training = causal
    out = model(mixture.cuda())
    loss, perm = PIT1d(NegSDR(), cfg.n_sources)(out, sources.cuda())
    torch.testing.assert_close(out.detach().cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    assert torch.equal(perm.cpu(), perm64)
    loss.backward()
    worst = _check_grads(model, g64, noise32)
    print("[{} PIT1d(NegSDR)] worst gradient error / role scale {:.2e} ({})".format("cLN" if causal else "gLN", *worst))


def test_pit_neg_sdr_step_vs_reference_golden(golden_dir):
    """sdr_grad.pt, minted from the unmodified reference: the tiny gLN model's permutation, loss and every parameter gradient under
    PIT1d(NegSDR())"""
    r = torch.load(os.path.join(golden_dir, "sdr_grad.pt"), weights_only=False)["model"]
    cfg = O.OracleConfig(**r["cfg"])
    sd = O.synth_state_dict(cfg, seed=r["wseed"])
    mixture, sources = O.synth_batch(r["batch"], cfg.n_sources, r["T"], seed=r["xseed"])
    g64 = {k: v["sample64"].view(v["shape"]) for k, v in r["grads"].items()}
    noise32 = {k: v["fp32_vs_fp64_maxabs"] for k, v in r["grads"].items()}
    for mode in MODES:
        model = build_model(cfg, sd, math=mode).train()
        out = model(mixture.cuda())
        loss, perm = PIT1d(NegSDR(), cfg.n_sources)(out, sources.cuda())
        assert torch.equal(perm.cpu(), r["perm"])
        # the loss of this estimate, within the kernels' bound of its fp64 value; and that value near the reference's
        ref = R.pit64(out.detach().cpu(), sources)
        _assert_within(loss.detach().view(1), ref["loss_b"].mean().view(1),
                       ref["bound"].mean().view(1) + 8 * U * ref["loss_b"].abs().mean(), "loss")
        assert abs(float(ref["loss_b"].mean()) - r["loss64"]) <= 5e-4 * (1 + abs(r["loss64"]))
        loss.backward()
        worst = _check_grads(model, g64, noise32)
        print("[golden {}] worst gradient error / role scale {:.2e} ({})".format(mode, *worst))


def test_musdb_neg_sdr_step_vs_fp64():
    """the MUSDB18 recipe's step with criterion 'sdr': a stereo model with multichannel_training, the mixture and sources standardised
    by the mixture's mean and std over time, NegSDR()(model(mixture), sources).backward() against fp64 autograd over the oracle"""
    from test_multichannel_train_gpu import _build, _inputs
    cfg = O.OracleConfig(causal=False, in_channels=2, **dict(SMALL, n_sources=3))
    sd = O.synth_state_dict(cfg, seed=911)
    mixture, sources, _ = _inputs(cfg, 2, 1037, 912)
    mean, std = mixture.mean(dim=-1, keepdim=True), mixture.std(dim=-1, keepdim=True)
    mix_s, src_s = (mixture - mean) / (std + R.EPS), (sources - mean) / (std + R.EPS)

    def oracle(dtype):
        sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
        out, _ = O.conv_tasnet_fwd(mix_s.to(dtype), sdv, cfg)
        (-R.sdr_autograd(out, src_s.to(dtype)).mean()).backward()
        return out.detach(), {k: v.grad for k, v in sdv.items()}

    out64, g64 = oracle(torch.float64)
    _, g32 = oracle(torch.float32)
    noise32 = {k: float((g32[k].double() - g64[k]).abs().max()) for k in g64}
    _assert_well_conditioned(g64, noise32)
    model = _build(cfg, sd, MODES[-1])
    out = model(mix_s.cuda())
    torch.testing.assert_close(out.detach().cpu(), out64.float(), rtol=OUT_RTOL, atol=OUT_ATOL)
    NegSDR()(out, src_s.cuda()).backward()
    worst = _check_grads(model, g64, noise32)
    print("[MUSDB18 NegSDR] worst gradient error / role scale {:.2e} ({})".format(*worst))


def test_wham_and_musdb_loops_lower_the_loss():
    """a few Adam steps on one batch: PIT1d(NegSDR(), 2) on a gLN model, NegSDR() on a standardised stereo model; the loss falls"""
    from test_multichannel_train_gpu import _build, _inputs
    cfg = O.OracleConfig(causal=False, **SMALL)
    model = build_model(cfg, O.synth_state_dict(cfg, seed=921), math=MODES[-1]).train()
    mixture, sources = O.synth_batch(2, 2, 2000, seed=922)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    losses = []
    for _ in range(6):
        opt.zero_grad()
        loss, _ = PIT1d(NegSDR(), 2)(model(mixture.cuda()), sources.cuda())
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert losses[-1] < losses[0], losses
    mcfg = O.OracleConfig(causal=False, in_channels=2, **SMALL)
    mm = _build(mcfg, O.synth_state_dict(mcfg, seed=923), MODES[-1])
    mix, src, _ = _inputs(mcfg, 2, 2000, 924)
    mean, std = mix.mean(dim=-1, keepdim=True), mix.std(dim=-1, keepdim=True)
    mix_s, src_s = ((mix - mean) / (std + R.EPS)).cuda(), ((src - mean) / (std + R.EPS)).cuda()
    opt = torch.optim.Adam(mm.parameters(), lr=1e-3)
    mlosses = []
    for _ in range(6):
        opt.zero_grad()
        loss = NegSDR()(mm(mix_s), src_s)
        loss.backward()
        opt.step()
        mlosses.append(float(loss.detach()))
    assert mlosses[-1] < mlosses[0], mlosses


# ---- ORPIT and Sinkhorn PIT over NegSDR (the generic loops through the differentiable module) ----------------------------------

def test_orpit_neg_sdr_vs_fp64():
    """ORPIT(NegSDR()) runs the reference's per-sample loop; the float64 restatement is fed the 'rest' target the loop forms in fp32,
    so every row is held to the kernels' bounds: value, selected index, and the gradient of the batch mean"""
    B, n, T = 3, 3, 1001
    t = _rand((B, n, T), 950)
    x = torch.stack([t[:, 0], t[:, 1:].sum(1)], dim=1) + _rand((B, 2, T), 951, 0.2)
    rest = torch.stack([(t * (torch.arange(n) != i).float().view(1, n, 1)).sum(1) for i in range(n)], dim=1)   # fp32, as the loop
    xg = x.cuda().requires_grad_(True)
    loss, idx = ORPIT(NegSDR())(xg, t.cuda())
    loss.backward()
    x64 = x.double().requires_grad_(True)
    loss_b64, idx64, cand = R.orpit_neg_sdr(x64, t.double(), rest.double())
    loss_b64.mean().backward()
    assert torch.equal(idx.cpu(), idx64)
    ar = torch.arange(B)
    b_one = R.sdr_bound(x[:, :1].expand(B, n, T), t)[ar, idx64]
    b_rest = R.sdr_bound(x[:, 1:].expand(B, n, T), rest)[ar, idx64] / (n - 1)
    vbound = (b_one + b_rest + 4 * U * loss_b64.detach().abs()).mean() + 4 * U * loss_b64.detach().abs().mean()
    _assert_within(loss.detach().view(1), loss_b64.detach().mean().view(1), vbound.view(1), "ORPIT loss")
    g = torch.full((B,), -1.0 / B, dtype=torch.float64)
    bound = torch.stack([R.sdr_grad_bound(x[:, 0], t[ar, idx64], g, g_rel=4 * U),
                         R.sdr_grad_bound(x[:, 1], rest[ar, idx64], g / (n - 1), g_rel=4 * U)], dim=1)
    _assert_within(xg.grad, x64.grad, bound, "ORPIT gradient")


def test_sinkpit_neg_sdr_vs_fp64():
    """SinkPIT(NegSDR()) runs the reference's Sinkhorn loop over the S x S row SDRs in fp32 torch; the pair values are held to the
    kernels' bounds, the loss and gradient to the loop's own fp32 rounding (1e-5 of their scale)"""
    B, S, T = 3, 3, 1001
    x, t = _pit_batch(B, S, T, 960)
    xg = x.cuda().requires_grad_(True)
    loss, pattern = SinkPIT(NegSDR(), n_sources=S, coldness=1.0, iteration=10)(xg, t.cuda())
    loss.backward()
    x64 = x.double().requires_grad_(True)
    loss_b64, P64 = R.sinkpit_neg_sdr(x64, t.double())
    loss_b64.mean().backward()
    assert torch.equal(pattern.cpu(), torch.argmax(P64, dim=2))
    scale = float(loss_b64.detach().abs().max())
    assert abs(float(loss.detach()) - float(loss_b64.detach().mean())) <= 1e-5 * scale
    gscale = float(x64.grad.abs().max())
    err = float((xg.grad.cpu().double() - x64.grad).abs().max())
    assert err <= 1e-5 * gscale, (err, gscale)
