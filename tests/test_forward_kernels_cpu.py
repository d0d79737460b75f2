"""The bounds of tests/forward_kernel_ref.py reject plausible bugs of the inference forward's streaming kernels (no GPU).

Each mutant below is applied to the fp64 reference at the shapes and inputs of its kernel's rows.  On at least one row it
must land at >= 4 times the bound of an output it changes, while the unmutated reference sits at 0.  A mutant no row can
reject means a row is missing.
"""
import pytest
import torch

import forward_kernel_ref as R
from test_train_kernels_cpu import REJECT, _worst


def _fold(name, r, mut):
    inputs, Rv = R.fold_inputs(name, r)
    out = {}
    for W, bias, gamma, beta in R.shared_norm(inputs, r):
        for k, v in R.fold(W, bias, gamma, beta, Rv, mut).items():
            out.setdefault(k, []).append(v)
    return {k: (torch.cat([a for a, _ in v]), torch.cat([b for _, b in v])) for k, v in out.items()}


def _dw(name, r, mut):
    h, g1, b1, wd, bd, stats1 = R.dw_inputs(name, r)
    return R.dw_fwd(h, g1, b1, wd, bd, R.A2, stats1, r["C"] * r["F"], R.EPS, r["P"], r["d"], mut)


def _skip(name, r, mut):
    jobs, n2 = R.skip_inputs(name, r)
    return R.skip_reduce(jobs, r["Sc"], n2, R.EPS, mut)


def _finish(name, r, mut):
    x0, rr, v1, v2, stats, n2 = R.finish_inputs(name, r)
    return R.finish(x0, rr, v1, v2, stats, n2, R.EPS, r["Bc"], mut)


def _stats(name, r, mut):
    return R.stats_pitch(R.stats_inputs(name, r), mut)


def _enc_stats(name, r, mut):
    x, W, pl, pr, F = R.enc_inputs(name, r)
    w = R.encoder(x, W, r["S"], pl, pr, r.get("relu", False))["w"][0]
    v4 = r["L"] <= 20 and r["S"] * 2 == r["L"] and not r.get("wpad") and not r.get("woff")
    return R.encoder_stats(w, v4, -(-R.pitch_of(F) // 128), mut)


def _dec(name, r, mut):
    what, Wd, T_out = R.dec_inputs(name, r)
    return R.decoder(what, Wd, r["S"], r["crop"], T_out, mut)


def _plain(name, r, mut):
    h, wd, bd = R.plain_inputs(name, r)
    return R.dw_plain(h, wd, bd, R.A2, r["P"], r["d"], mut)


def _res(name, r, mut):
    rr, xin, skip0, bo, bs = R.res_inputs(name, r)
    return R.res_skip(rr, xin, skip0, bo, bs, r["Bc"], r["has_out"], r["init"], mut)


SMALL = lambda rows: {k: v for k, v in rows.items() if v["B"] * v.get("C", 1) * v.get("F", 1) <= 3 * 5 * 1025}

MUTANTS = {
    "fold_v1_from_gamma": (_fold, "v1_gamma", R.FOLD, ["v1"]),
    "fold_v2_from_W": (_fold, "v2_w", R.FOLD, ["v2"]),
    "fold_missing_bias": (_fold, "no_bias", R.FOLD, ["v1"]),
    "skip_offset_0": (_skip, "off0", R.SKIP, ["skip"]),
    "skip_previous_block_stats": (_skip, "prev_stats", R.SKIP, ["skip"]),
    "skip_sample0_stats": (_skip, "sample0", R.SKIP, ["skip"]),
    "finish_sample0_stats": (_finish, "sample0", SMALL(R.FINISH), ["x"]),
    "dw_sample0_stats": (_dw, "sample0", SMALL(R.DW), ["u"]),
    "dw_pad_left_off_by_one": (_dw, "pl_off", SMALL(R.DW), ["u"]),
    "dw_dilation_halved": (_dw, "dil_half", SMALL(R.DW), ["u"]),
    "dw_stats_count_pad_columns": (_dw, "n_pitch", SMALL(R.DW), ["u"]),
    "dw_plain_symmetric_padding": (_plain, "causal_sym", R.PLAIN, ["u"]),
    "dw_plain_dilation_halved": (_plain, "dil_half", R.PLAIN, ["u"]),
    "stats_pitch_fp32_partials": (_stats, "fp32_partials", R.STATS, ["stats"]),
    "decoder_missing_split_partial": (_dec, "drop_part", R.DEC, ["y"]),
    "decoder_crop_off_by_one": (_dec, "crop_off", R.DEC, ["y"]),
    "res_skip_ignores_skip_init": (_res, "no_skip_init", R.RES, ["skip"]),
    "encoder_spill_loses_partial": (_enc_stats, "spill_lost", {k: v for k, v in R.ENC.items() if v["N"] == 512}, ["stats"]),
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
