"""The rows of tests/test_gln_forward_edges_gpu.py without a GPU: each reaches the branch its `reaches` text names by the restated
dispatch predicates (gln_forward_edges_ref.py), every branch is reached by some row, the fp64 references agree with the oracle, and
the GPU file's bound rejects six plausible defects of the forward, each on a named row.

A mutant is applied to the fp64 reference (gln_forward_edges_ref.model64 / chain) and must land at more than REJECT times the
fp32-parity bound (rtol 1e-4 / atol 2e-5) away from the unmutated fp64 answer.
"""
import ctypes as C

import pytest
import torch

import convtasnet_oracle as O
import gln_forward_edges_ref as R
from ctn_b200 import _native as N

REJECT = 4.0


def _sd64(row):
    return {k: v.double() for k, v in R.state_dict(row).items()}


@pytest.mark.parametrize("row", R.all_expected(), ids=[r[0] for r in R.all_expected()])
def test_row_reaches_its_branches(row):
    name, expect, got = row
    assert expect <= got, "{}: declares {} but reaches only {}".format(name, sorted(expect - got), sorted(got))


def test_every_branch_is_reached():
    reached = set().union(*(got & expect for _, expect, got in R.all_expected()))
    assert reached == set(R.BRANCHES), sorted(set(R.BRANCHES) - reached)


@pytest.mark.parametrize("name", list(R.ROWS))
def test_row_frames_match_the_library(name):
    """the restated frame count, pads and pitch equal the library's own (ctn_frames / ctn_pitch)"""
    r = R.ROWS[name]
    for T in r.Ts:
        f, pl, pr = R.frames_of(T, r.cfg.kernel_size, r.cfg.stride)
        assert N.frames_of(T, r.cfg.kernel_size, r.cfg.stride) == (f, pl, pr)
        assert N.ctn_pitch(f) == R.pitch(f)


def test_launch_counts_follow_the_branches():
    """a stand-alone depthwise block costs one launch more than a fused one in the tensor-core modes; fp32 adds a k_finish per
    block with an out head; k_maskdec replaces EPI_MASK + the decoder"""
    base = dict(Bc=32, H=64, Sc=32, mode="tf32x3")
    assert R.tcn_launches(P=3, dils=[1, 3], **base) == R.tcn_launches(P=3, dils=[1, 2], **base) + 1
    assert R.tcn_launches(P=3, dils=[1, 2, 4], Bc=32, H=64, Sc=32, mode="fp32") == 1 + 3 * 3 + 2 + 1
    cfg = R.ROWS["paper"].cfg
    # extract_latent: no k_maskdec, so the decoder runs, then the latent copy
    assert R.model_launches(cfg, 2, "f16x3", latent=False) + 2 == R.model_launches(cfg, 2, "f16x3", latent=True)
    # cfg2 in f16x3: encoder; head fold, 2 images, head; 47 fold jobs and 48 image jobs (one launch each), 2 scale launches,
    # 24 x (pw1 + PRO_DW pw2), skip reduction; k_maskdec
    assert R.model_launches(cfg, 2, "f16x3", latent=False) == 1 + 4 + 1 + 1 + 2 + 48 + 1 + 1


def test_blocks_fwd_refuses_x_out_without_the_last_out_head():
    """ctn_tcn_blocks_fwd returns CTN_EINVAL when x_out is asked for and the last block has no output head"""
    fake = 1 << 20
    blocks = (N.BlockParams * 3)()
    for b in blocks:
        for name in N.BLOCK_FIELDS:
            setattr(b, name, fake)
    blocks[2].out_w = blocks[2].out_b = None
    cfg = N.Config()
    cfg.bottleneck, cfg.hidden, cfg.skip, cfg.sep_kernel, cfg.num_blocks, cfg.num_layers = 8, 16, 8, 3, 1, 3
    cfg.math, cfg.eps, cfg.eps_tcn = N.MATH_FP32, R.EPS, R.EPS
    dil = (C.c_int * 3)(1, 2, 4)
    assert N.ctn_tcn_blocks_fwd(C.byref(cfg), blocks, 3, dil, fake, fake, fake, 1, 32, fake, 1 << 40, None) == N.CTN_EINVAL


def test_chain_equals_tdcn_at_powers_of_two():
    """chain() (O.residual_block per block, explicit dilations) equals O.tdcn_fwd at dilations 2^l (up to the order of the skip
    sum: tdcn_fwd adds per stage first)"""
    cfg = R.cfg_of(R=2, X=4)
    sd = {k: v.double() for k, v in O.synth_state_dict(cfg, seed=31).items()}
    x = torch.randn(2, cfg.sep_bottleneck_channels, 300, generator=torch.Generator().manual_seed(32), dtype=torch.float64)
    ref = O.tdcn_fwd(x, sd, "separator.tdcn.", kernel_size=3, num_blocks=2, num_layers=4, dilated=True, causal=False,
                     nonlinear=True, norm=True, eps=R.EPS)
    prefixes = [f"separator.tdcn.net.{r}.net.{l}." for r in range(2) for l in range(4)]
    _, skip = R.chain(x, sd, prefixes, R.default_dils(cfg), 3, last_out=False)
    torch.testing.assert_close(skip, ref, rtol=1e-13, atol=1e-13)


@pytest.mark.parametrize("name", ["p2", "paper-short", "silence", "rx1"])
def test_model64_equals_the_oracle(name):
    """model64 unmutated (its own block restatement with the pad given) equals O.conv_tasnet_fwd"""
    r = R.ROWS[name]
    sd = _sd64(r)
    x = R.mixture(r, r.Ts[0], R.state_dict(r)).double()
    out, lat = R.model64(x, sd, r.cfg)
    ref, ref_lat = O.conv_tasnet_fwd(x, sd, r.cfg)
    torch.testing.assert_close(out, ref, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(lat, ref_lat, rtol=1e-12, atol=1e-14)


def _model_mutant(name, mut, **kw):
    r = R.ROWS[name]
    sd = _sd64(r)
    x = R.mixture(r, r.Ts[0], R.state_dict(r)).double()
    ref, _ = O.conv_tasnet_fwd(x, sd, r.cfg)
    bad, _ = R.model64(x, sd, r.cfg, mut=mut, **kw)
    return ref, bad


def _blocks_mutant(name, mut, **kw):
    b = R.BLOCKS[name]
    sd, prefixes = R.blocks_state_dict(len(b.dils), b.Bc, b.H, b.Sc, b.P, b.last_out, b.seed)
    sd = {k: v.double() for k, v in sd.items()}
    x = torch.randn(b.B, b.Bc, b.frames, generator=torch.Generator().manual_seed(b.seed + 1)).double()
    good = R.chain(x, sd, prefixes, b.dils, b.P, b.last_out)
    bad = R.chain(x, sd, prefixes, b.dils, b.P, b.last_out, mut=mut, **kw)
    return good, bad


def _silence_eps():
    r = R.ROWS["silence"]
    ref, bad = _model_mutant("silence", "eps_outside")
    # the near-silent sample (3), judged with atol scaled to its amplitude, as the GPU file judges every sample of this row
    scale = float(ref[3].abs().max()) / float(ref[0].abs().max())
    assert r.B == 5 and scale < 1e-3
    return ref[3], bad[3], R.OUT_ATOL * scale


def _mutant(case):
    if case == "pad_up":
        ref, bad = _model_mutant("p2", "pad_up")
        return ref, bad, R.OUT_ATOL
    if case == "drop_last_update":
        (x, _), (xb, _) = _blocks_mutant("mixed-xout", "drop_last_update")
        return x, xb, R.OUT_ATOL
    if case == "pow2":
        (_, s), (_, sb) = _blocks_mutant("mixed", "pow2")
        return s, sb, R.OUT_ATOL
    if case == "crop_off":
        ref, bad = _model_mutant("paper-short", "crop_off")
        return ref, bad, R.OUT_ATOL
    if case == "drop_skip":
        ref, bad = _model_mutant("rx64", "drop_skip", mut_block=40)
        return ref, bad, R.OUT_ATOL
    return _silence_eps()


MUTANTS = {
    "pad_up": "p2: pad_left rounded up for even P",
    "drop_last_update": "blocks mixed-xout: the last block's deferred residual update dropped from x_out",
    "pow2": "blocks mixed: 2^l in place of the explicit dilations",
    "crop_off": "paper-short (T = 17): the decoder crop one sample off",
    "drop_skip": "rx64: block 40's skip head dropped from the 64-term skip sum",
    "eps_outside": "silence, near-silent sample: gLN0's eps outside the sqrt",
}


@pytest.mark.parametrize("case", list(MUTANTS))
def test_mutant_is_rejected(case):
    ref, bad, atol = _mutant(case)
    s = R.share(bad, ref, R.OUT_RTOL, atol)
    print("[mutant {}] {:.1f}x the fp32-parity bound -- {}".format(case, s, MUTANTS[case]))
    assert s > REJECT, (case, s)
