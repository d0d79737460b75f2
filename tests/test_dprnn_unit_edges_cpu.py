"""The DPRNN-TasNet edge tests without a GPU (tests/dprnn_unit_edges_ref.py): the restatements still match the reference's goldens,
the geometry the rows are chosen from matches the rows, and every planted mistake is rejected by its section's per-unit bound at
the exact shape of the GPU row meant to catch it."""
import math
import os

import pytest
import torch

import convtasnet_oracle as O
import dprnn_oracle as DO
import dprnn_unit_edges_ref as E
from ctn_b200.models.dprnn_tasnet import DPRNNTasNet, Separator

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- the restatements against the goldens ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["dprnn_tiny", "dprnn_cfg4_short"])
def test_model_restatement_matches_goldens(name):
    rec = torch.load(os.path.join(GOLDEN, name + ".pt"), weights_only=False)
    cfg = {k: v for k, v in rec["cfg"].items() if k in ("n_basis", "kernel_size", "sep_bottleneck_channels", "sep_hidden_channels",
                                                         "sep_chunk_size", "sep_hop_size", "sep_num_blocks", "n_sources", "eps")}
    sd = DO.synth_state_dict(DO.DPRNNConfig(**rec["cfg"]), seed=rec["wseed"])
    mixture, _ = O.synth_batch(rec["batch"], rec["cfg"]["n_sources"], rec["T"], seed=rec["xseed"])
    out = E.model_answer(mixture, sd, cfg)
    so = rec.get("out_stride")
    ref = rec["out"].double()
    got = out if so is None else out[..., ::so]
    assert float((got - ref).abs().max()) < 2e-5 * float(ref.abs().max()), name


def test_step_loop_equals_torch_lstm():
    """the step loop that carries the recurrence mistakes equals torch.lstm when none is planted"""
    r = dict(E.lstm_rows()["proj:F32H64-T3"], NSEQ=5, T=17)
    sd, z = E.lstm_case(r)
    sdd = {k: v.double() for k, v in sd.items()}
    w = [sdd["rnn." + n] for n in E.NAMES]
    loop = torch.cat([E.lstm_loop(z.double(), w[0], w[1], w[2] + w[3], False), E.lstm_loop(z.double(), w[4], w[5], w[6] + w[7], True)], 2)
    assert float((loop - DO._bilstm(z.double(), sdd, "rnn.")).abs().max()) < 1e-13


def test_norm_restatement_equals_the_plain_gln():
    """norm_answer without a mistake is test_dprnn_edges_gpu's GroupNorm(1, F) + R"""
    r = E.norm_rows()["swap1"]
    P, bias, R, gamma, beta = E.norm_case(r)
    out, _ = E.norm_answer([P[0], P[1], bias], R, gamma, beta, r["eps"], 1)
    Y = P[0].double() + P[1].double() + bias.double()
    mean = Y.reshape(r["B"], -1).mean(1).view(-1, 1, 1, 1)
    var = Y.reshape(r["B"], -1).var(1, unbiased=False).view(-1, 1, 1, 1)
    ref = ((Y - mean) / torch.sqrt(var + r["eps"]) * gamma.double() + beta.double() + R.double()).transpose(1, 2)
    assert float((out - ref).abs().max()) < 1e-12


def test_overlap_add_restatement_is_the_oracle_in_fp32():
    Z = torch.randn(2, 33, 7, 12, generator=torch.Generator().manual_seed(1))
    y = E.overlap_add(Z, 12, 5, 2, 40, 48, False)
    assert torch.equal(y[..., :40], DO.overlap_add1d(Z, 12, 5)[..., 2:42]) and not y[..., 40:].any()


# ---- the geometry ---------------------------------------------------------------------------------------------------------------------
def test_ring_geometry_and_its_rows():
    """ring depth and slabs per step of every instantiation (lstm_fixed_smem, SMEM_LIMIT = 232448, MAX_NST = 4 of ctn_lstm.cu), and
    the rows reach every residue of T per_step that the ring depth allows, T = 1 and T = 2"""
    want = {(32, 32): (4, 3), (32, 64): (4, 8), (32, 128): (3, 24), (64, 32): (4, 4), (64, 64): (4, 10), (64, 128): (3, 28),
            (128, 32): (4, 6), (128, 64): (3, 14), (128, 128): (2, 36)}
    assert {fh: E.ring(*fh) for fh in E.INSTANTIATIONS} == want
    assert E.ring(64, 128, proj=False) == (3, 24)
    rows = E.lstm_rows()
    for entry in ("proj", "relu"):
        for F, H in E.INSTANTIATIONS:
            nst, per_step = E.ring(F, H)
            Ts = {r["T"] for r in rows.values() if r["entry"] == entry and (r["F"], r["H"], r["Fo"]) == (F, H, F)}
            assert {1, 2} <= Ts
            reach = {E.residue(F, H, T) for T in Ts}
            assert reach == set(range(0, nst, math.gcd(per_step, nst))), (entry, F, H, reach)


def test_cta_geometry_of_the_rows():
    assert [E.ctas(n) for n in (1, 63, 64, 65, 129, 68)] == [(1, 1), (1, 63), (1, 64), (2, 1), (3, 1), (2, 4)]
    rows = E.lstm_rows()
    for entry in ("proj", "relu"):
        ns = {r["NSEQ"] for r in rows.values() if r["entry"] == entry}
        assert {1, 63, 64, 65, 129} <= ns
        assert {r["Fo"] for r in rows.values() if r["entry"] == entry and r["Fo"] != r["F"]} == {32, 96, 128}
        assert max(r["T"] for r in rows.values() if r["entry"] == entry) >= 3839      # the inter path of 60 s
        assert {r["outs"] for r in rows.values() if r["entry"] == entry} == ({"both", "P", "h"} if entry == "proj" else {"both", "P"})


def test_segment_geometry_is_the_models():
    for K, P in ((12, 5), (250, 125), (20, 30), (25, 25), (40, 15), (100, 50)):
        sep = Separator(16, bottleneck_channels=8, hidden_channels=8, chunk_size=K, hop_size=P, num_blocks=1, causal=False)
        for frames in range(max(1, K - P), K + 3 * P):
            try:
                want = sep.segment_geometry(frames)
            except ValueError:
                continue
            assert E.segment_geometry(frames, K, P) == want, (K, P, frames)
    rows = E.seg_rows()
    for K, P in ((12, 5), (250, 125)):
        assert {(r[2] - K) % P for r in rows.values() if (r[3], r[4]) == (K, P)} == set(range(P))
    assert E.segment_geometry(479999, 250, 125)[2] == 3839 and E.segment_geometry(79999, 250, 125)[2] == 639


def test_forward_refusal_before_cuda():
    """frozen weights and a CPU input that requires grad, under grad mode: the forward would record no graph, so it is refused"""
    m = DPRNNTasNet(16, 4, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=32,
                    sep_bottleneck_channels=32, sep_chunk_size=8, sep_hop_size=4, sep_num_blocks=1, causal=False).requires_grad_(False)
    with pytest.raises(NotImplementedError, match="forward-only"):
        m(torch.randn(1, 1, 64, requires_grad=True))


def test_model_rows_cover_every_padding_remainder():
    rows = E.model_rows()
    small = [r for n, r in rows.items() if n.startswith("small-r")]
    assert {(T - 1 - 12) % 5 for _, _, T, _, _ in small} == set(range(5))
    assert E.model_launches(E.RECIPE, "fp32") == 55 and E.model_launches(E.SMALL, "tf32x3") == 25


# ---- the planted mistakes at their rows' shapes --------------------------------------------------------------------------------------
def lstm_defect(defect, name):
    r = E.lstm_rows()[name]
    sd, z = E.lstm_case(r)
    relu = r["entry"] == "relu"
    h, P = E.lstm_answer(z, sd, relu)
    hb, Pb = E.lstm_answer(z, sd, relu, defect=defect)
    return E.lstm_excess(hb, Pb, h, P), E.lstm_excess(h, P, h, P)


def norm_defect(defect, name):
    r = E.norm_rows()[name]
    P, bias, R, gamma, beta = E.norm_case(r)
    parts = [P[0], P[1], bias]
    ref, scale = E.norm_answer(parts, R, gamma, beta, r["eps"], r["swap"])
    bad, _ = E.norm_answer(parts, R, gamma, beta, r["eps"], r["swap"], defect)
    return E.norm_excess(bad, ref, scale), E.norm_excess(ref, ref, scale)


def seg_defect(defect, name):
    B, F, frames, K, P, _ = E.seg_rows()[name]
    x = torch.randn(B, F, frames, generator=torch.Generator().manual_seed(frames))
    pl, pr, _ = E.segment_geometry(frames, K, P)
    assert pl != pr
    ref, bad = E.segment(x, K, P, pl, pr, 1), E.segment(x, K, P, pl, pr, 1, defect)
    return E.D.excess(bad, ref, 1), E.D.excess(ref, ref, 1)


SECTIONS = {"A": lstm_defect, "B": norm_defect, "C": seg_defect}


def test_every_defect_has_a_row():
    assert sorted(E.DEFECT_ROWS) == sorted(E.DEFECTS)
    rows = {"A": E.lstm_rows(), "B": E.norm_rows(), "C": E.seg_rows()}
    for sec, name in E.DEFECT_ROWS.values():
        assert name in rows[sec], name


@pytest.mark.parametrize("defect", E.DEFECTS)
def test_bound_rejects_planted_defect(defect):
    sec, name = E.DEFECT_ROWS[defect]
    ratio, clean = SECTIONS[sec](defect, name)
    print("[dprnn defect] {:28s} at {:22s} worst unit error / bound {:.3g}".format(defect, name, ratio))
    assert ratio > 4, defect
    assert clean == 0


def test_fp32_partial_statistics_pass_without_the_offset():
    """the same emulation at the DC-free row stays inside the bound: it is the offset that breaks fp32 partials"""
    ratio, _ = norm_defect("fp32_partial_stats", "dc0-bias")
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("entry", ["proj", "relu"])
def test_loudness_row_is_well_conditioned_where_it_holds_the_floors(entry):
    """the bi-LSTM loudness row saturates its gates through W_ih alone: its quiet sequences (x0, x1e-3, x1) are well conditioned, so
    the fp32 CPU recurrence holds the floors there; only the x1e3 sequences take the fp32 rule.  A zero answer or the negated
    answer fails the row by far, on the quiet sequences as on the whole."""
    r = E.lstm_rows()[entry + ":loudness-wih8"]
    sd, z = E.lstm_case(r)
    relu = entry == "relu"
    h64, P64 = E.lstm_answer(z, sd, relu)
    h32, P32 = E.lstm_answer(z, sd, relu, dtype=torch.float32)
    idx = torch.arange(r["NSEQ"])
    m = E.fp32_mask(r, idx)
    assert int(m.sum()) == r["NSEQ"] // 4 and bool((idx[m] % 4 == 3).all())
    quiet = E.lstm_excess(h32[~m].double(), P32[:, ~m].double(), h64[~m], P64[:, ~m])
    assert quiet <= 0.25, quiet
    assert E.lstm_excess(h32.double(), P32.double(), h64, P64, (m, h32, P32)) <= 0.25
    for bad in (torch.zeros_like, torch.neg):
        assert E.lstm_excess(bad(h64)[~m], bad(P64)[:, ~m], h64[~m], P64[:, ~m]) > 1e3
        assert E.lstm_excess(bad(h64), bad(P64), h64, P64, (m, h32, P32)) > 1e3
