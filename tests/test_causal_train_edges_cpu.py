"""The causal training edge rows without a GPU (tests/test_causal_train_edges_gpu.py): the convention-aware cLN its silent-onset
row is referenced against, the rows' frame counts, and that the bounds of causal_train_ref reject plausible bugs of the cLN
backward and causal depthwise kernels.

Each mutant is applied to the fp64 reference at the shapes and inputs of the GPU file's probe rows.  On at least one row it must
land at >= 4 times the bound of an output it changes, while the unmutated reference sits at 0.  A mutant no row can reject means
a row is missing.
"""
import pytest
import torch

import causal_train_ref as R
import convtasnet_oracle as O
from ctn_b200 import _native as N
from test_causal_train_edges_gpu import ENC, ROWS, SILENT_FADE, SILENT_ZERO

REJECT = 4.0


def _silent(B, C, T, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, C, T, generator=g, dtype=torch.float64) + 0.3
    R.silent_onset_(x[0], 5 * T // 8, max(1, T // 32))
    return x, g


@pytest.mark.parametrize("T", [1, 40, 1025])
@pytest.mark.parametrize("Cc", [1, 3, 9])
@pytest.mark.parametrize("silent", [False, True])
def test_convention_aware_cln(Cc, T, silent):
    """forward bit-identical to the oracle's cLN; backward equal to the oracle's autograd wherever that is finite and to the
    closed form causal_train_ref.cln_bwd everywhere, including the frames of exactly zero variance"""
    x, g = _silent(2, Cc, T, Cc * 100 + T)
    if not silent:
        x, g = torch.randn(2, Cc, T, generator=g, dtype=torch.float64) + 0.3, g
    gamma = 1.0 + 0.3 * torch.randn(Cc, generator=g, dtype=torch.float64)
    beta = 0.2 * torch.randn(Cc, generator=g, dtype=torch.float64)
    dy = torch.randn(2, Cc, T, generator=g, dtype=torch.float64)
    eps = 1e-8
    xa, ga, ba = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    xb, gb, bb = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    y_conv, y_orac = R.cln_conv(xa, ga, ba, eps), O.cln(xb, gb, bb, eps)
    assert torch.equal(y_conv, y_orac)
    (y_conv * dy).sum().backward()
    (y_orac * dy).sum().backward()
    assert all(torch.isfinite(t.grad).all() for t in (xa, ga, ba))
    fin = torch.isfinite(xb.grad)
    want = R.cln_bwd(dy, x, gamma, eps)
    tol = dict(rtol=1e-9, atol=1e-9 * float(want["dpre"].abs().sum() + 1))
    torch.testing.assert_close(xa.grad[fin], xb.grad[fin], **tol)
    torch.testing.assert_close(xa.grad, want["dpre"], **tol)
    torch.testing.assert_close(ga.grad, want["dgamma"], **tol)
    torch.testing.assert_close(ba.grad, want["dbeta"], **tol)
    if silent and T > 1:
        assert not fin.all(), "the oracle's autograd is finite on a silent onset: the convention is no longer exercised"


def test_silent_onset_model_gradient():
    """a small causal model on a silent-onset mixture in fp64: the oracle's autograd gives a NaN encoder weight gradient and
    nothing else non-finite; with the convention-aware cLN every gradient is finite and all but the encoder weight's are equal"""
    cfg = O.OracleConfig(n_basis=16, kernel_size=16, sep_hidden_channels=32, sep_bottleneck_channels=16, sep_skip_channels=16,
                         sep_num_blocks=1, sep_num_layers=2, causal=True, n_sources=2)
    sd = O.synth_state_dict(cfg, seed=1, dtype=torch.float64)
    mix, _ = O.synth_batch(2, 2, 1600, seed=2, dtype=torch.float64)
    R.silent_onset_(mix[0], 1000, 50)
    G = torch.randn(2, 2, 1600, generator=torch.Generator().manual_seed(3), dtype=torch.float64)

    def grads(cln):
        sdv = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        with pytest.MonkeyPatch.context() as mp:
            mp.setattr(O, "cln", cln)
            out, _ = O.conv_tasnet_fwd(mix, sdv, cfg)
        out.backward(G)
        return {k: v.grad for k, v in sdv.items()}

    plain, conv = grads(O.cln), grads(R.cln_conv)
    assert [k for k, v in plain.items() if not torch.isfinite(v).all()] == [ENC]
    assert all(torch.isfinite(v).all() for v in conv.values())
    for k in plain:
        if k != ENC:
            torch.testing.assert_close(conv[k], plain[k], rtol=1e-12, atol=1e-12 * float(plain[k].abs().max()))


@pytest.mark.parametrize("case", list(ROWS))
def test_row_frames_equal_the_host_library(case):
    e = ROWS[case]
    L = e.shape["kernel_size"]
    stride = e.shape.get("stride") or L // 2
    assert N.frames_of(e.T, L, stride)[0] == e.frames
    if case == "C11":  # frames whose whole window is silent: exactly zero encoder output, zero cumulative variance in cLN0
        assert (SILENT_ZERO - L) // stride + 1 == 1249


def _worst(ref, mut, bound, keys):
    out = 0.0
    for k in keys:
        err = (mut[k] - ref[k]).abs()
        q = torch.where(torch.isfinite(err), err / bound[k], torch.full_like(err, float("inf")))
        out = max(out, float(q.max()))
    return out


def _cln(frames, C, slope, kind, mut):
    dy, pre, gamma = R.cln_row(frames, C, slope, kind)
    want = R.cln_bwd(dy.double(), pre.double(), gamma.double(), R.EPS_PROBE, slope, mut)
    return want, R.cln_bwd_bounds(want, frames, slope)


def _cln_rows(frames=R.CLN_FRAMES, channels=R.CLN_CHANNELS, kinds=R.CLN_INPUTS):
    return [(f, c, s, k) for f in frames for c in channels for s in (None, 0.25) for k in kinds if c * f <= 9 * 16000]


def _cdw(P, dil, frames, B, C, mut):
    want = R.cdw_expect(*R.cdw_row(P, dil, frames, B, C), dil, mut)
    return {k: v[0] for k, v in want.items()}, {k: v[1] for k, v in want.items()}


MUTANTS = {
    "cdw_drop_tap_P-1": (_cdw, "drop_last", [(8, d, f, b, c) for d in R.CDW_DIL for f in R.CDW_FRAMES for b, c in R.CDW_BC if f < 15999],
                         ["upre", "dhn", "dwd"]),
    "cln_exclusive_suffix": (_cln, "exclusive", _cln_rows(), ["dpre"]),
    "cln_scan_segment_first": (_cln, "seg_first", _cln_rows(frames=(1025, 15999)), ["dpre"]),
    "cln_slices_below_8": (_cln, "slices8", _cln_rows(channels=(9,)), ["dpre"]),
    "cln_unclamped_e": (_cln, "unclamped", _cln_rows(kinds=("silent",)), ["dpre"]),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_mutant(mutant):
    fn, mut, rows, keys = MUTANTS[mutant]
    seen = []
    for row in rows:
        ref, bound = fn(*row, None)
        again, _ = fn(*row, None)
        assert _worst(ref, again, bound, keys) == 0.0
        mutated, _ = fn(*row, mut)
        q = _worst(ref, mutated, bound, keys)
        seen.append(f"{row} {q:.3g}")
        if q >= REJECT:
            print(f"{mutant}: rejected on row {row} at {q:.3g} x the bound")
            return
    pytest.fail(f"{mutant}: no row rejects it ({', '.join(seen)})")
