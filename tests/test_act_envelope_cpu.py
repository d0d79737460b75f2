"""The checks of tests/envelope_ref.py, on the CPU, against an fp32 emulation of the activation envelope (k_fold_batch's row
bounds, k_scale_partials, k_scale_chain in ctn_tcn_simt.cu).

The checks must accept the emulation and reject the regressions a rework of those kernels can introduce: a scale one binade too
high, the PReLU factor max(1, |a2|) lost, the depthwise sum stopped after 3 taps, R = sqrt(H) instead of sqrt(H frames), one
block's vb_out missing from the x chain, and the mask bound without its slope.  Each must fail some row at 4x its bound or more.
"""
import math

import numpy as np
import pytest
import torch

import envelope_ref as E

f32 = np.float32
MUTANTS = ["scale_high", "a2_no_max", "wd_3taps", "R_from_H", "x_chain_skip_one", "mask_no_slope"]


def _pow2_scale(bound):
    """pow2_scale_for (ctn_tcn_simt.cu)"""
    if not (bound > 0.0) or not (bound < 3.0e38):
        return 1.0
    _, e = math.frexp(float(bound))
    return 2.0 ** min(max(15 - e, -100), 100)


def _np(t):
    return t.float().numpy()


def _vb32(W, b, g, beta, R):
    t = np.abs(_np(W)) * (np.abs(_np(g)) * R + np.abs(_np(beta)))[None, :]
    return t.sum(axis=1, dtype=f32) + (np.abs(_np(b)) if b is not None else f32(0))


def emulate(blocks, H, frames, x0, mask_slope, mutant=None):
    """(scales [2n + 1], [(vb_out | None, vb_skip)]) as the library computes them, in fp32"""
    R = f32(np.sqrt(f32(H) * f32(frames))) * f32(1.0001)
    if mutant == "R_from_H":
        R = f32(np.sqrt(f32(H))) * f32(1.0001)
    X, S, scales, vbs = f32(x0), f32(0), [], []
    for i, b in enumerate(blocks):
        vo = _vb32(b["Wo"], b["bo"], b["g2"], b["be2"], R) if b["Wo"] is not None else None
        vs = _vb32(b["Ws"], b["bs"], b["g2"], b["be2"], R)
        vbs.append((vo, vs))
        a2 = abs(f32(b["a2"])) if mutant == "a2_no_max" else max(f32(1), abs(f32(b["a2"])))
        wd = np.abs(_np(b["wd"]))
        wsum = wd[:, :3].sum(1, dtype=f32) if mutant == "wd_3taps" else wd.sum(1, dtype=f32)
        u = (a2 * ((np.abs(_np(b["g1"])) * R + np.abs(_np(b["be1"]))) * wsum + np.abs(_np(b["bd"])))).max()
        scales += [_pow2_scale(X), _pow2_scale(u)]
        if vo is not None and not (mutant == "x_chain_skip_one" and i == 0):
            X = f32(X + vo.max())
        S = f32(S + vs.max())
    am = max(f32(1), abs(f32(mask_slope))) if mask_slope is not None else f32(1)
    scales.append(_pow2_scale(S if mutant == "mask_no_slope" else f32(am * S)))
    if mutant == "scale_high":
        scales = [2.0 * s for s in scales]
    return scales, vbs


def _blocks(seed, n, Bc, H, Sc, P, last_out=False, big_last_tap=False, zero_dw=False, a2=0.25):
    g = torch.Generator().manual_seed(seed)

    def r(*shape, scale=1.0, shift=0.0):
        return (torch.randn(*shape, generator=g) * scale + shift).float().double()
    out = []
    for i in range(n):
        wd = r(H, P, scale=0.5)
        if big_last_tap:
            wd[:, -1] = 4.0 * wd[:, :-1].abs().sum(1) + 0.5
        bd = r(H, scale=0.1)
        if zero_dw:
            wd, bd = torch.zeros_like(wd), torch.zeros_like(bd)
        has_out = last_out or i < n - 1
        out.append(dict(W1=r(H, Bc, scale=Bc ** -0.5), b1=r(H, scale=0.05), a1=0.25, g1=r(H, scale=0.1, shift=1.0),
                        be1=r(H, scale=0.05), wd=wd, bd=bd, a2=a2, g2=r(H, scale=0.1, shift=1.0), be2=r(H, scale=0.05),
                        Wo=r(Bc, H, scale=H ** -0.5) if has_out else None, bo=r(Bc, scale=0.05) if has_out else None,
                        Ws=r(Sc, H, scale=H ** -0.5), bs=r(Sc, scale=0.05)))
    return out


ROWS = {
    # x0 far below the first vb_out: the x chain without block 0's vb_out is many binades short
    "p4_h40_small_x0": dict(n=3, Bc=16, H=40, Sc=12, P=4, frames=1000, x0=1e-3, mask_slope=-3.0, big_last_tap=True),
    "p3_h300_f16000": dict(n=4, Bc=64, H=300, Sc=48, P=3, frames=16000, x0=3.0, mask_slope=0.25, last_out=True, a2=-3.0),
    "p8_h520_nomask": dict(n=2, Bc=32, H=520, Sc=250, P=8, frames=1, x0=0.5, mask_slope=None),
    "zero_dw_p3": dict(n=2, Bc=16, H=33, Sc=16, P=3, frames=129, x0=0.0, mask_slope=0.1, zero_dw=True),
}


def _scores(name, scales, vbs):
    r = ROWS[name]
    blocks = _blocks(sum(map(ord, name)), r["n"], r["Bc"], r["H"], r["Sc"], r["P"], r.get("last_out", False),
                     r.get("big_last_tap", False), r.get("zero_dw", False), r.get("a2", 0.25))
    bounds, vbs64 = E.envelope(blocks, r["H"], r["frames"], f32(r["x0"]), r["mask_slope"])
    sl = E.slack(r["H"], r["n"])
    sc = [E.scale_score(s, b, sl)[0] for s, b in zip(scales, bounds)]
    vs = [E.vb_score(torch.from_numpy(np.asarray(g)), w, r["H"]) for gv, wv in zip(vbs, vbs64) for g, w in zip(gv, wv)
          if w is not None]
    return sc, vs


def _emulated(name, mutant=None):
    r = ROWS[name]
    blocks = _blocks(sum(map(ord, name)), r["n"], r["Bc"], r["H"], r["Sc"], r["P"], r.get("last_out", False),
                     r.get("big_last_tap", False), r.get("zero_dw", False), r.get("a2", 0.25))
    return emulate(blocks, r["H"], r["frames"], r["x0"], r["mask_slope"], mutant)


@pytest.mark.parametrize("name", list(ROWS))
def test_checks_accept_the_emulation(name):
    scales, vbs = _emulated(name)
    sc, vs = _scores(name, scales, vbs)
    print(f"{name}: scale scores {max(sc):.3f}, vb scores {max(vs):.3f}")
    assert max(sc) <= 1.0 and max(vs) <= 1.0, (sc, vs)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_checks_reject_mutant(mutant):
    worst = {}
    for name in ROWS:
        scales, vbs = _emulated(name, mutant)
        sc, _ = _scores(name, scales, vbs)
        worst[name] = max(sc)
    print(f"{mutant}: worst scale score per row " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert max(worst.values()) >= 4.0, worst


def test_zero_bound_gives_scale_one():
    scales, _ = _emulated("zero_dw_p3")
    assert scales[1] == 1.0 and scales[3] == 1.0 and scales[0] == 1.0  # U_i = 0 and X_0 = 0
    assert E.scale_score(2.0, 0.0, 1e-4)[0] == math.inf and E.scale_score(1.0, math.inf, 1e-4)[0] == 0.0


def test_scale_checks_at_powers_of_two():
    sl = E.slack(512, 24)
    assert E.best_scale(2.0 ** 15) == 1.0 and E.best_scale(2.0 ** 15 + 1) == 0.5 and E.best_scale(3.0) == 2.0 ** 13
    assert E.scale_score(1.0, 2.0 ** 15, sl)[0] == 0.0              # s bound == 2^15 exactly: legal and the largest
    assert E.scale_score(0.5, 2.0 ** 15, sl)[0] <= 1.0              # one binade lower: bound64 is a power of two
    assert E.scale_score(0.5, 2.0 ** 15 * (1 - sl / 2), sl)[0] <= 1.0
    assert E.scale_score(0.5, 2.0 ** 15 * (1 - 4 * sl), sl)[0] > 1.0  # not within the fp32 error of 2^15
    assert E.scale_score(2.0, 2.0 ** 14 * (1 + 1e-9), sl)[0] > 1.0    # saturation possible, however slightly
    assert E.scale_score(3.0, 1.0, sl)[0] == math.inf                 # not a power of two


def test_dwp_pack_layout():
    b = _blocks(5, 1, 4, 20, 4, 3)[0]
    d = E.dwp_pack(b, 20)
    assert d.shape == (32, 8) and bool((d[20:] == 0).all()) and bool((d[:, 6:] == 0).all())
    assert torch.equal(d[:20, 2:5], b["wd"].float()) and torch.equal(d[:20, 0], b["g1"].float())
