"""The edge tests of DPTNet, SepFormer and LSTM-TasNet without a GPU: the envelope gates of the three attention paths
(``ctn_mha_supported``, ``ctn_sfm_attn_supported``, ``ctn_galr_supported``) against a Python statement of each envelope, and
every planted defect of tests/dual_path_edges_ref.py rejected by the per-unit bound at the shapes the GPU tests use."""
import itertools

import pytest
import torch

import dual_path_edges_ref as R
from ctn_b200 import _native as N

HEAD_DIMS = (8, 16, 32, 64)


def mha_envelope(F, heads):
    return F > 0 and heads > 0 and F % heads == 0 and F <= 128 and F % 4 == 0 and F // heads in HEAD_DIMS


def sfm_attn_envelope(F, heads):
    return F > 0 and heads > 0 and F % heads == 0 and F // heads in HEAD_DIMS


def galr_envelope(F, K, Q, heads):
    return F in (32, 64, 128) and 1 <= Q <= K and mha_envelope(F, heads)


FS = (-32, 0, 4, 8, 12, 16, 24, 32, 33, 48, 64, 96, 100, 128, 132, 136, 192, 256, 512, 1024)
HEADS = (-1, 0, 1, 2, 3, 4, 5, 8, 12, 16, 32, 64, 128)


def test_mha_supported_matches_envelope():
    for F, h in itertools.product(FS, HEADS):
        assert N.ctn_mha_supported(F, h) == int(mha_envelope(F, h)), (F, h)
    assert N.ctn_mha_supported(128, 2) == 1 and N.ctn_mha_supported(128, 1) == 0 and N.ctn_mha_supported(132, 2) == 0


def test_sfm_attn_supported_matches_envelope():
    for F, h in itertools.product(FS, HEADS):
        assert N.ctn_sfm_attn_supported(F, h) == int(sfm_attn_envelope(F, h)), (F, h)
    assert N.ctn_sfm_attn_supported(1024, 16) == 1 and N.ctn_sfm_attn_supported(1024, 8) == 0


def test_galr_supported_matches_envelope():
    for F, h in itertools.product((0, 16, 32, 48, 64, 96, 128, 256), (0, 1, 2, 4, 8, 16)):
        for K in (-1, 0, 1, 16, 100, 250):
            for Q in (-1, 0, 1, 4, 32, K - 1, K, K + 1):
                assert N.ctn_galr_supported(F, K, Q, h) == int(galr_envelope(F, K, Q, h)), (F, K, Q, h)


# the shapes of the GPU tests the defects are shown at
HEAD = dict(B=3, N=64, Bc=32, K=16, P=8, frames=19)   # padding 5: pad_left 2, pad_right 3


def head_case(defect):
    c = HEAD
    w = torch.randn(c["B"], c["N"], c["frames"], generator=torch.Generator().manual_seed(1))
    p = R.dpt_head_params(c["N"], c["Bc"], 2)
    pl, pr, _ = R.segment_geometry(c["frames"], c["K"], c["P"])
    assert pl != pr
    run = lambda d: R.dpt_head(w, p["bn_w"], p["bn_b"], p["g"], p["b"], c["K"], c["P"], pl, pr, 1e-12, d)  # noqa: E731
    return run(None), run(defect), 2


def segment_case(defect):
    K, P, frames, zp = 16, 8, 19, 128
    x = torch.randn(3, 32, frames, generator=torch.Generator().manual_seed(3))
    pl, pr, _ = R.segment_geometry(frames, K, P)
    return R.sfm_segment(x, K, P, pl, pr, zp), R.sfm_segment(x, K, P, pl, pr, zp, defect), 1


def ola_case(defect):
    K, P, frames = 16, 8, 19
    pl, _, S = R.segment_geometry(frames, K, P)
    Z = torch.randn(3, 32, 128, generator=torch.Generator().manual_seed(4))
    return R.sfm_overlap_add(Z, S, K, P, pl, frames, 128, None), R.sfm_overlap_add(Z, S, K, P, pl, frames, 128, defect), 1


def pos_enc_case(defect, intra):
    S, C = 3, 16
    X = R.pitched(2, 32, S * C, 128, 5)
    pe = R.sepformer_ref.positional_encoding(32)
    return R.sfm_pos_enc(X, pe, S, C, intra), R.sfm_pos_enc(X, pe, S, C, intra, defect), 1


def transformer_case(defect):
    F, heads, d_ff, layers, S, C = 32, 4, 48, 65, 2, 3
    sd = R.transformer_sd(F, d_ff, layers, 7)
    X = R.pitched(1, F, S * C, 128, 8)
    run = lambda d: R.sequences(R.sfm_transformer(X, sd, S, C, layers, heads, 1e-12, 1, d), S, C, 1)  # noqa: E731
    return run(None), run(defect), 2


def tail_case(defect, which):
    B, Nb, Bc, n_src, frames, pitch, L, stride = 2, 32, 32, 2, 37, 128, 4, 2
    w = R.pitched(B, Nb, frames, pitch, 9, pad="random")
    T = (frames - 1) * stride + L - 3
    if which == "dpt":
        y = R.pitched(B, Bc, frames, pitch, 10)
        p = R.dpt_tail_params(Nb, Bc, n_src, L, 11)
        run = lambda d: R.dpt_tail(y, w, p, n_src, 1, stride, 1, T, frames, d)  # noqa: E731
    else:
        skip = R.pitched(B, Bc, frames, pitch, 12)
        p = R.tas_tail_params(Nb, Bc, n_src, L, 13, logit_scale=30.0)
        run = lambda d: R.tas_tail(skip, w, p["fc_w"], p["fc_b"], p["dec_w"], n_src, 1, stride, 1, T, frames, d)  # noqa: E731
    (out, what), (bad_out, bad_what) = run(None), run(defect)
    return torch.cat([out.flatten(2), what.flatten(2)], 2), torch.cat([bad_out.flatten(2), bad_what.flatten(2)], 2), 2


CASES = [("pad_split_swapped", head_case), ("pad_split_swapped", segment_case), ("ola_drop_last_chunk", ola_case),
         ("pe_row_shifted", lambda d: pos_enc_case(d, 1)), ("pe_row_shifted", lambda d: pos_enc_case(d, 0)),
         ("head_gln_without_padding", head_case), ("layers_past_64_from_layer_0", transformer_case),
         ("softmax_without_max", lambda d: tail_case(d, "tas")), ("mask_on_pad_columns", lambda d: tail_case(d, "dpt")),
         ("mask_on_pad_columns", lambda d: tail_case(d, "tas"))]


def test_every_defect_has_a_case():
    assert sorted({d for d, _ in CASES}) == sorted(R.DEFECTS)


@pytest.mark.parametrize("i", range(len(CASES)))
def test_bound_rejects_planted_defect(i):
    defect, case = CASES[i]
    ref, bad, lead = case(defect)
    assert R.excess(bad, ref, lead) > 10, defect
    assert R.excess(ref, ref, lead) == 0


def test_large_logits_need_the_max_subtraction():
    """the tail test's logits: large enough that exp overflows fp32, while the fp64 softmax is exact"""
    B, Nb, Bc, frames = 2, 32, 32, 37
    skip = R.pitched(B, Bc, frames, 128, 12)
    p = R.tas_tail_params(Nb, Bc, 2, 4, 13, logit_scale=30.0)
    y = p["fc_w"] @ skip[..., :frames]
    assert 88.8 < float(y.abs().max()) < 200
