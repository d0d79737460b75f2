"""The bounds of tests/train_kernel_ref.py reject plausible bugs of the training path's streaming kernels (no GPU).

Each mutant below is applied to the fp64 reference at the shapes and inputs of its kernel's rows.  On at least one row it
must land at >= 4 times the bound of an output it changes, while the unmutated reference sits at 0.  A mutant no row can
reject means a row is missing.
"""
import pytest
import torch

import train_kernel_ref as R

REJECT = 4.0


def _worst(ref, mut, keys):
    out = 0.0
    for k in keys:
        v, b = ref[k]
        m = mut[k][0]
        err = (m - v).abs()
        inf = torch.where(err > 0, torch.full_like(err, float("inf")), err)  # a zero bound admits no error at all
        out = max(out, float(torch.where(b > 0, err / b.clamp_min(1e-300), inf).max()))
    return out


def _dw(name, r, mut):
    _, h, g1, b1, wd, _, dU, stats1 = R.dw_inputs(name, r)
    P, d = r["P"], r["d"]
    return R.dw_bwd(dU, h, R.A1, g1, b1, stats1, r["C"] * r["F"], R.EPS, wd, P, d, R.pad_left_of(P, d), mut)


def _gln(name, r, mut):
    _, sl, pre, dy, gm, stats = R.gln_inputs(name, r)
    return R.gln_bwd(dy, pre, sl, gm, stats, r["C"] * r["F"], R.EPS, mut)


def _prelu(name, r, mut):
    g = R.gen("prelu" + name)
    x = R.activation(g, r)
    return R.prelu_bwd(R.rnd(g, r["B"], r["C"], r["F"]), x, R.A1, mut)


def _mask(name, r, mut):
    g = R.gen("mask" + name)
    B, S, N, F = r["B"], r["S"], r["N"], r["F"]
    dwhat = R.f32(R.rnd(g, B, S, N, F) * R.sample_scale(B)[:, :, :, None])
    w = R.rnd(g, B, N, F).abs()
    m = R.f32(torch.sigmoid(R.rnd(g, B, S, N, F, scale=3.0)))
    return R.mask_bwd(dwhat, w, m, mut)


def _encdec(name, r, mut):
    g = R.gen("encdec" + name)
    F, pl = R.encdec_geometry(r)
    act_ = R.rnd(g, r["R"], r["N"], F)
    sig = R.f32(R.rnd(g, r["R"], r["T"]) * R.sample_scale(r["R"])[:, :, 0])
    return R.encdec_wgrad(act_, sig, r["L"], r["stride"], pl, mut)


SMALL = lambda rows: {k: v for k, v in rows.items() if v["C"] * v["F"] * v["B"] <= 3 * 1025 * 33}  # keep the CPU run short

MUTANTS = {
    "dw_fwd_tap": (_dw, "fwd_tap", SMALL(R.ROWS["dw"]), ["dhn"]),
    "dw_pad_left_up": (_dw, "pl_up", SMALL(R.ROWS["dw"]), ["dhn", "dwd"]),
    "dw_drop_last_quad": (_dw, "drop_quad", SMALL(R.ROWS["dw"]), ["dwd"]),
    "gln_no_xh_mgx": (_gln, "no_mgx", SMALL(R.ROWS["gln_bwd"]), ["dpre"]),
    "gln_n_pitch": (_gln, "n_pitch", SMALL(R.ROWS["gln_bwd"]), ["dpre", "dgamma", "sums"]),
    "gln_sample0_stats": (_gln, "sample0", SMALL(R.ROWS["gln_bwd"]), ["dpre", "dgamma", "sums"]),
    "prelu_identity_at_0": (_prelu, "ident0", SMALL(R.ROWS["prelu"]), ["dpre"]),
    "mask_m_not_m1m": (_mask, "m_only", R.ROWS["mask_bwd"], ["dmpre"]),
    "mask_drop_source": (_mask, "drop_src", R.ROWS["mask_bwd"], ["dwprod"]),
    "encdec_skip_partial": (_encdec, "skip_partial", R.ROWS["encdec"], ["dW"]),
    "encdec_no_pad_left": (_encdec, "no_pl", R.ROWS["encdec"], ["dW"]),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_mutant(mutant):
    fn, mut, rows, keys = MUTANTS[mutant]
    seen = []
    for name, r in rows.items():
        ref = fn(name, r, None)
        assert _worst(ref, fn(name, r, None), keys) == 0.0
        q = _worst(ref, fn(name, r, mut), keys)
        seen.append(f"{name} {q:.3g}")
        if q >= REJECT:
            print(f"{mutant}: rejected on {name} [{r['reaches']}] at {q:.3g} x the bound")
            return
    pytest.fail(f"{mutant}: no row rejects it ({', '.join(seen)})")


WGRAD_ROWS = {  # the shapes of test_pw_contraction_gpu.py::test_wgrad_vs_fp64 (fp32 mode)
    "m33_k144_f31_b5": dict(M=33, K=144, B=5, frames=31, split=None),
    "m144_k33_f32_split": dict(M=144, K=33, B=1, frames=32, split=96),
    "m144_k144_f33_b5_stride": dict(M=144, K=144, B=5, frames=33, split=96),
    "m33_k1_f1000": dict(M=33, K=1, B=1, frames=1000, split=None),
    "m144_k144_f800_b5": dict(M=144, K=144, B=5, frames=800, split=96),
}


@pytest.mark.parametrize("mutant", ["drop_chunk", "split_off"])
def test_wgrad_fp32_bound_rejects_mutant(mutant):
    """the FFMA k_wgrad losing its last 32-frame chunk, or split_row misplaced by one"""
    for name, r in WGRAD_ROWS.items():
        if mutant == "split_off" and not r["split"]:
            continue
        g = torch.Generator().manual_seed(sum(map(ord, name)))
        M, K, B, T = r["M"], r["K"], r["B"], r["frames"]
        dy = R.f32(torch.randn(B, M, T, generator=g, dtype=torch.float64))
        x = R.f32(torch.randn(B, K, T, generator=g, dtype=torch.float64) + 0.2)
        den = torch.einsum("bmt,bkt->mk", dy.abs(), x.abs())
        bound = R.wgrad_fp32_chain(M, K, B, T, r["split"]) * R.U * den
        ref = R.wgrad_fp32(dy, x, r["split"])
        assert float((R.wgrad_fp32(dy, x, r["split"], None) - ref).abs().max()) == 0.0
        q = float(((R.wgrad_fp32(dy, x, r["split"], mutant) - ref).abs() / bound).max())
        if q >= REJECT:
            print(f"wgrad {mutant}: rejected on {name} at {q:.3g} x the bound")
            return
    pytest.fail(f"wgrad {mutant}: no row rejects it")
