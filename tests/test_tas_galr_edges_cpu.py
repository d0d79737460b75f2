"""The edge tests of LSTM-TasNet and GALRNet without a GPU (tests/tas_galr_edges_ref.py): the restatements still match the
reference's goldens, the recurrence geometry restated in Python gives the numbers DESIGN sections 16 and 18 state for an H100 SXM,
and every planted mistake is rejected by the per-unit bound at the exact shape of the GPU row meant to catch it."""
import os

import pytest
import torch

import galrnet_ref as GR
import lstm_tasnet_ref as LR
import tas_galr_edges_ref as E

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SMS, OPTIN = E.H100_SMS, E.H100_SMEM_OPTIN


def gold(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


# ---- the restatements against the goldens ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tasnet.pt", "tasnet_causal_plain.pt"])
def test_tasnet_restatement_matches_goldens(name):
    for case, g in gold(name).items():
        sd = LR.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
        ref = g["out"].double()
        assert float((LR.tasnet_fwd(g["x"], sd, g["cfg"]) - ref).abs().max()) < 2e-5 * float(ref.abs().max()), case


def test_galrnet_restatement_matches_goldens():
    """galrnet_fwd runs inter_block with the gLN eps equal to the LayerNorm's and the attention in slices of sequences"""
    for case, g in gold("galrnet.pt").items():
        sd = GR.synth_state_dict(g["keys_shapes"], g["cfg"]["seed"])
        ref = g["out"].double()
        assert float((GR.galrnet_fwd(g["x"], sd, g["cfg"]) - ref).abs().max()) < 2e-5 * float(ref.abs().max()), case


def test_sliced_attention_equals_the_whole():
    sd = E.inter_weights(32, 40, 8, 1)
    x = torch.randn(2, 9, 40, 32, generator=torch.Generator().manual_seed(2))
    whole = E.inter_answer(x, sd, 4, 8, 1e-3, 1e-1)
    old = GR.MHA_ELEMS
    try:
        GR.MHA_ELEMS = 4 * 9 * 9          # one sequence per slice
        sliced = E.inter_answer(x, sd, 4, 8, 1e-3, 1e-1)
    finally:
        GR.MHA_ELEMS = old
    assert float((whole - sliced).abs().max()) < 1e-12


def test_mistake_restatements_equal_the_plain_ones_without_a_mistake():
    """recurrence() and gated_encoder(), which carry the planted mistakes, equal lstm_ref and enc_norm_ref when none is planted"""
    for dirs in (1, 2):
        ws = E.lstm_weights(7, 19, dirs, 3)
        x = torch.randn(5, 7, 37, generator=torch.Generator().manual_seed(4))
        geo = dict(U=3, cpd=7, group=2)
        assert float((E.recurrence(x, ws, dirs, geo) - LR.lstm_ref(x, ws, dirs)).abs().max()) < 1e-12
    for name, r in list(E.enc_rows().items())[::7]:
        p = E.enc_params(r["N"], r["L"], 5)
        x = E.enc_input(r, 6)
        for a, b in zip(E.gated_encoder(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12),
                        E.enc_answer(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12)):
            assert float((a - b).abs().max()) <= 1e-12 * float(b.abs().max()), name


# ---- the geometry ---------------------------------------------------------------------------------------------------------------------
def test_geometry_gives_designs_numbers():
    g = E.lstm_geo(500, 2, SMS, OPTIN)
    assert (g["U"], g["cpd"], g["group"]) == (8, 63, 16)
    g = E.lstm_geo(500, 1, SMS, OPTIN)
    assert (g["U"], g["cpd"]) == (4, 125) and g["smem"] == 97792          # DESIGN 18: 97,792 bytes
    assert E.lstm_max_hidden(1, SMS, OPTIN) == 1320
    assert E.lstm_geo(E.lstm_max_hidden(2, SMS, OPTIN), 2, SMS, OPTIN)["group"] == 2
    assert E.lstm_geo(E.lstm_max_hidden(1, SMS, OPTIN) + 1, 1, SMS, OPTIN) is None


@pytest.mark.parametrize("nsm", [132, 114])
@pytest.mark.parametrize("dirs", [1, 2])
def test_hidden_rows_reach_every_edge(nsm, dirs):
    """U steps between P and P + 1 and between 2P and 2P + 1, the last CTA of those rows owns a single unit, and H is not always a
    multiple of 4; the rows end at the largest H"""
    rows = dict(E.hidden_rows(dirs, nsm, OPTIN))
    geo = {k: E.lstm_geo(H, dirs, nsm, OPTIN) for k, H in rows.items()}
    assert geo["P"]["U"] == 1 and geo["P+1"]["U"] == 2 and geo["2P"]["U"] == 2 and geo["2P+1"]["U"] == 3
    assert geo["P+1"]["nu"] == 1 and geo["2P+1"]["nu"] == 1
    assert any(H % 4 for H in rows.values())
    assert rows["max"] == E.lstm_max_hidden(dirs, nsm, OPTIN) and E.lstm_geo(rows["max"] + 1, dirs, nsm, OPTIN) is None
    steps = E.u_steps(dirs, nsm, OPTIN)
    assert steps[:3] == [1, nsm // dirs + 1, 2 * (nsm // dirs) + 1]


def test_rows_cover_the_batch_and_step_edges():
    rows = E.lstm_rows(SMS, OPTIN)
    for dirs in (1, 2):
        hmax = E.lstm_max_hidden(dirs, SMS, OPTIN)
        g = E.lstm_geo(hmax, dirs, SMS, OPTIN)["group"]
        assert any(r["H"] == hmax and r["dirs"] == dirs and r["B"] == 2 * g + 1 for r in rows.values())
    assert {r["T"] for r in rows.values()} >= {1, 15, 16, 17, 47, 48, 49}
    assert {r["F"] for r in rows.values()} >= {1, 7, 1001} and {r["mode"] for r in rows.values()} == set(E.MODES)
    assert {1, 2, 3, 5}.issubset({r["B"] for r in rows.values()})


# ---- the planted mistakes at their rows' shapes --------------------------------------------------------------------------------------
def lstm_case(defect):
    name = E.lstm_defect_row(defect, SMS, OPTIN)
    r = E.lstm_rows(SMS, OPTIN)[name]
    ws = E.lstm_weights(r["F"], r["H"], r["dirs"], 1)
    x = E.lstm_input(r, 2)
    geo = E.lstm_geo(r["H"], r["dirs"], SMS, OPTIN)
    u = lambda y: E.lstm_units(y, r["B"], r["dirs"], r["H"])  # noqa: E731
    return u(E.lstm_answer(x, ws, r["dirs"], geo)), u(E.lstm_answer(x, ws, r["dirs"], geo, defect)), 2


def enc_case(defect):
    r = E.enc_rows()[E.ENC_DEFECT_ROWS[defect]]
    p = E.enc_params(r["N"], r["L"], 1)
    x = E.enc_input(r, 2)
    w, _ = E.enc_answer(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12)
    bad, _ = E.enc_answer(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12, defect)
    return w, bad, 1


def galr_case(defect):
    r = E.galr_rows()[E.GALR_DEFECT_ROWS[defect]]
    sd = E.inter_weights(r["F"], r["K"], r["Q"], 1)
    x = E.inter_input(r, 2)
    run = lambda d: E.inter_answer(x, sd, r["heads"], r["Q"], r["ln_eps"], r["gn_eps"], d)  # noqa: E731
    return run(None), run(defect), 2


CASES = {d: lstm_case for d in E.LSTM_DEFECT_ROWS}
CASES.update({d: enc_case for d in E.ENC_DEFECT_ROWS})
CASES.update({d: galr_case for d in E.GALR_DEFECT_ROWS})


def test_every_defect_has_a_row():
    assert sorted(CASES) == sorted(E.DEFECTS)


@pytest.mark.parametrize("defect", E.DEFECTS)
def test_bound_rejects_planted_defect(defect):
    ref, bad, lead = CASES[defect](defect)
    ratio = E.excess(bad, ref, lead)
    print("[tas/galr defect] {:28s} worst unit error / bound {:.3g}".format(defect, ratio))
    assert ratio > 10, defect
    assert E.excess(ref, ref, lead) == 0


def test_whole_tensor_bound_misses_a_batch_coupled_norm():
    """The gated encoder's w does not scale with the input (it divides by the signal norm), so a norm taken over the whole batch
    shows in any batch of ordinary recordings even to the old bound over the whole tensor.  It hides from that bound next to a
    click when the other recording is so quiet that its norm is far below the eps: its w is then about 1e-4 of the click's, and
    all of it is lost.  The per-sample bound sees it."""
    w, bad, lead = enc_case("batch_norm_instead_of_sample")
    whole = float((bad - w).abs().max()) / LR.bound(w)
    assert whole <= 1.0, whole
    assert E.excess(bad, w, lead) > 10
    assert E.excess(bad[:1], w[:1], lead) <= 1.0             # the click itself is right


def test_amplitude_row_catches_the_batch_coupled_norm():
    """the encoder's loudness batch (0, 1e-13, 1e-6, 1, 1e4) rejects it too, under either bound"""
    r = E.enc_rows()["16/8 amplitudes 0 1e-13 1e-6 1 1e4"]
    p = E.enc_params(r["N"], r["L"], 1)
    x = E.enc_input(r, 2)
    w, _ = E.enc_answer(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12)
    bad, _ = E.enc_answer(x, p, r["L"], r["stride"], r["pl"], r["pr"], 1e-12, "batch_norm_instead_of_sample")
    assert E.excess(bad, w, 1) > 10
