"""The rows, references and bounds of tests/mc_filterbank_ref.py without a GPU: the fp64 references agree with torch, every row
reaches the kernel its `reaches` text names under a restatement of the C selection rules, every template instantiation in
ctn_encdec.cu and every fallback reason has a row, and each bound rejects the defects of MUTANTS by at least 10x on some row of its
family.  Also the two launch-shape refusals, which return before any launch."""
import os
import re

import pytest
import torch
import torch.nn.functional as F_

import mc_filterbank_ref as R
from ctn_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENCDEC_CU = os.path.join(ROOT, "dnn-based_source_separation_b200", "csrc", "ctn_encdec.cu")
REJECT = 10.0
FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced


def _encoder(name, r, mut=None):
    x, W = R.enc_inputs(name, r)
    w, mag = R.encoder(x, W, r.S, r.pl, r.pr, r.relu, mut)
    return w, R.encoder_bound(r, mag)


def _decoder(name, r, mut=None):
    what, Wd = R.dec_inputs(name, r)
    crop, T_out = R.dec_geometry(r)
    y, mag = R.decoder(what, Wd, r.S, crop, T_out, mut)
    return y, R.decoder_bound(r, R.decoder_kernel(r)[0], mag)


def _wgrad(name, r, mut=None):
    act, sig, base = R.wg_inputs(name, r)
    dW, mag = R.wgrad(act, sig, r.L, r.S, r.pl, mut)
    return dW, R.wgrad_bound(r, mag, base)


FAMILIES = {"encoder": (R.ENC, _encoder), "decoder": (R.DEC, _decoder), "wgrad": (R.WG, _wgrad)}


# ---- the references against torch ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(R.ENC))
def test_encoder_reference_is_conv1d(name):
    r = R.ENC[name]
    x, W = R.enc_inputs(name, r)
    w, mag = R.encoder(x, W, r.S, r.pl, r.pr, r.relu)
    ref = F_.conv1d(F_.pad(x, (r.pl, r.pr)), W, stride=r.S)
    ref = torch.relu(ref) if r.relu else ref
    assert w.shape == (r.B, r.N, r.frames)
    torch.testing.assert_close(w, ref, rtol=1e-12, atol=1e-12 * float(mag.max()))
    torch.testing.assert_close(mag, F_.conv1d(F_.pad(x, (r.pl, r.pr)).abs(), W.abs(), stride=r.S), rtol=1e-12, atol=0)


@pytest.mark.parametrize("name", list(R.DEC))
def test_decoder_reference_is_conv_transpose1d(name):
    r = R.DEC[name]
    what, Wd = R.dec_inputs(name, r)
    crop, T_out = R.dec_geometry(r)
    y, mag = R.decoder(what, Wd, r.S, crop, T_out)
    ref = F_.conv_transpose1d(what, Wd, stride=r.S)[..., crop:crop + T_out]
    assert y.shape == (r.BS, r.C, T_out) and T_out > 0
    torch.testing.assert_close(y, ref, rtol=1e-12, atol=1e-12 * float(mag.max()))


@pytest.mark.parametrize("name", list(R.WG))
def test_wgrad_reference_is_the_conv1d_weight_gradient(name):
    r = R.WG[name]
    if r.N * r.C * r.L * r.frames * r.R > 5e7:
        pytest.skip("the autograd form of this row takes too long on a CPU; its einsum form is checked by the mutants")
    act, sig, _ = R.wg_inputs(name, r)
    dW, mag = R.wgrad(act, sig, r.L, r.S, r.pl)
    sp = F_.pad(sig, (r.pl, r.pr))
    ref = torch.nn.grad.conv1d_weight(sp, (r.N, r.C, r.L), act, stride=r.S)
    torch.testing.assert_close(dW, ref, rtol=1e-12, atol=1e-12 * float(mag.max()))


# ---- selection rules ---------------------------------------------------------------------------------------------------------
RULES = {"encoder": (R.ENC, R.encoder_kernel), "decoder": (R.DEC, R.decoder_kernel), "wgrad": (R.WG, R.wgrad_kernel)}


@pytest.mark.parametrize("family", list(RULES))
def test_reaches_names_the_selected_kernel(family):
    rows, rule = RULES[family]
    for name, r in rows.items():
        head = R.label(*rule(r))
        assert r.reaches.startswith(head), "{} {}: the rule selects '{}', the row says '{}'".format(family, name, head, r.reaches)


def _source():
    with open(ENCDEC_CU) as f:
        return f.read()


def test_every_encoder_instantiation_has_a_row():
    """the ENC_MC_CASE switch of ctn_encoder_mc_fwd, and each of its lengths reached (plain and, where one exists, opt-in)"""
    src = _source()
    body = src[src.index("extern \"C\" int ctn_encoder_mc_fwd"):]
    switch = re.search(r"switch \(L\) \{([^}]*)\}", body).group(1)
    assert tuple(int(v) for v in re.findall(r"ENC_MC_CASE\((\d+)\)", switch)) == R.ENC_FAST_L
    reached = {R.encoder_kernel(r)[0] for r in R.ENC.values()}
    for L in R.ENC_FAST_L:
        assert "k_encoder_v4_mc<{},{}>".format(L, L // 2) in reached, L


def test_every_decoder_instantiation_has_a_row():
    src = _source()
    body = src[src.index("extern \"C\" int ctn_decoder_mc_fwd"):]
    body = body[:body.index("k_decoder_mc<<<")]
    found = re.findall(r"if \(stride == (\d+) && R == (\d+)\) rc = launch_decoder_mc_v<(\d+), (\d+)>", body)
    assert all(a == c and b == d for a, b, c, d in found)
    assert tuple(int(a) for a, b, _, _ in found) == R.DEC_FAST_S and {b for _, b, _, _ in found} == {"2"}
    reached = {R.decoder_kernel(r)[0] for r in R.DEC.values()}
    for S in R.DEC_FAST_S:
        assert "k_decoder_mc_v<{},2>".format(S) in reached, S


def test_the_limits_restated_here_are_the_sources():
    src = _source()
    assert src.count("if (smem > 200 * 1024) return NO_FAST_PATH;") == 1
    assert src.count("if (smem > 200 * 1024 || nblk > 0x7fffffffLL) return NO_FAST_PATH;") == 1
    assert src.count("if (smem + ENC_STATIC_SMEM > 48 * 1024) {") == 3 and src.count("if (smem > 48 * 1024) {") == 2
    assert "constexpr size_t ENC_STATIC_SMEM = sizeof(double) * 64;" in src and src.count("__shared__ double red[64];") == 4
    assert "constexpr int DEC_SPLIT = 4;" in src
    assert "return sizeof(float) * ((size_t)C * L * ((N + 3) & ~3) + (size_t)C * 32 * XWP);" in src
    assert "const size_t smem = sizeof(float) * ((size_t)N * STRIDE * R + (size_t)(DEC_SPLIT - 1) * STRIDE * 128);" in src


def _tags(rows, rule):
    out = set()
    for r in rows.values():
        kernel, tags = rule(r)
        out |= {(kernel, t) for t in tags} | {(kernel, None)}
    return out


def test_every_fallback_reason_and_edge_has_a_row():
    enc = _tags(R.ENC, R.encoder_kernel)
    for reason in ("L != 2 stride", "L outside the switch", "w_pitch % 128", "w misaligned", "shared memory > 200 KB"):
        assert ("k_encoder_mc", reason) in enc, reason
    assert any(t == "opt-in" for _, t in enc)
    smem = {R.encoder_smem(r.C, r.N, r.L) for r in R.ENC.values() if r.L == 2 * r.S and r.L in R.ENC_FAST_L}
    static = R.ENC_STATIC_SMEM
    assert {R.SMEM_OPT_IN - static, R.SMEM_MAX} <= smem  # the largest sizes without the opt-in and with the fast path
    assert any(R.SMEM_OPT_IN - static < s <= R.SMEM_OPT_IN for s in smem)  # opt-in only because of the static red[64]
    assert any(R.SMEM_MAX < s <= R.SMEM_MAX + 4096 for s in smem)
    dec = _tags(R.DEC, R.decoder_kernel)
    for reason in ("R != 2", "stride outside the list", "shared memory > 200 KB"):
        assert ("k_decoder_mc", reason) in dec, reason
    assert any(t == "opt-in" for _, t in dec)
    assert R.SMEM_MAX in {R.decoder_smem(r.N, r.S, r.R) for r in R.DEC.values()}
    wg = {t for _, t in _tags(R.WG, R.wgrad_kernel)}
    for tag in ("vector", "boundary", "gy = R", "gy = 1", "scalar: L % 4", "scalar: stride % 4", "scalar: pad_left % 4",
                "scalar: T % 4", "scalar: sig misaligned"):
        assert tag in wg, tag
    assert {r.L for r in R.WG.values() if r.L > R.ENCDEC_MAX_L} >= {33, 40, 64}
    assert any(r.N * r.C > 65535 and r.L > R.ENCDEC_MAX_L for r in R.WG.values())


def test_rows_cover_the_listed_sizes():
    enc = R.ENC.values()
    assert {1, 3, 4, 13, 42, 256} <= {r.N for r in enc}
    assert {1, 2, 3, 8, 64} <= {r.C for r in enc}
    assert {1, 3, 4, 5, 127, 128, 129} <= {r.frames for r in enc} and max(r.frames for r in enc) >= 1000
    assert any(r.pl and r.pr for r in enc) and any(r.pl != r.pr for r in enc)
    assert {True, False} == {r.relu for r in enc} == {r.stats for r in enc}
    assert any(r.stats and r.B == 3 for r in enc)
    dec = R.DEC.values()
    assert {1, 3, 5, 512} <= {r.N for r in dec}
    assert {127, 128, 129} <= {r.frames + r.R - 1 for r in dec}
    assert {2, 3, 64} <= {r.C for r in dec} and {1, 12} <= {r.BS for r in dec}
    assert any(r.crop > 0 and r.tail > 0 for r in dec)
    assert {2, 3, 64} <= {r.C for r in R.WG.values()}


# ---- the bounds reject plausible bugs ----------------------------------------------------------------------------------------
def _share(v, ref, bound):
    err = (v - ref).abs()
    inf = torch.where(err > 0, torch.full_like(err, float("inf")), err)
    return float(torch.where(bound > 0, err / bound.clamp_min(1e-300), inf).max())


@pytest.mark.parametrize("mut", R.MUTANTS)
@pytest.mark.parametrize("family", list(FAMILIES))
def test_bounds_reject_mutants(family, mut):
    """the mutant's output against the unmutated reference's bound: at least 10x on some row of the family"""
    rows, fn = FAMILIES[family]
    worst, where = 0.0, None
    for name, r in rows.items():
        if family == "wgrad" and r.N * r.C * r.L * r.frames * r.R > 5e7:
            continue
        ref, bound = fn(name, r)
        share = _share(fn(name, r, mut)[0], ref, bound)
        if share > worst:
            worst, where = share, name
    assert worst >= REJECT, "{} {}: at most {:.2f}x the bound ({})".format(family, mut, worst, where)


# ---- refusals that come before any launch ------------------------------------------------------------------------------------
def test_encoder_refuses_more_than_65535_rows():
    """the encoder's samples ride on gridDim.y; the decoder's adjoint passes B*S rows"""
    assert N.ctn_encoder_mc_fwd(FAKE, FAKE, FAKE, 65536, 2, 32, 0, 0, 4, 16, 8, 0, 128, None, None) == N.CTN_EUNSUPPORTED


def test_generic_wgrad_refuses_more_than_2_31_ctas():
    probe = N._sig("ctn_probe_encdec_wgrad_mc", N._i, N._fp, N._fp, N._fp, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._i, N._fp)
    assert probe(FAKE, FAKE, FAKE, 1, 1 << 20, 64, 1, 128, 64, 64, 32, 0, None) == N.CTN_EUNSUPPORTED
