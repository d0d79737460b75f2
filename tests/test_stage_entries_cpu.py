"""The rows of tests/test_stage_entries_gpu.py without a GPU: each reaches the branch its `reaches` text names by the restated
dispatch predicates (stage_entries_ref.py), every branch is reached by some row, the fp64 restatements agree with the oracle and
with F.conv1d in float64, and each bound rejects planted defects, each on a named row, by more than REJECT times in every mode.
"""
import pytest
import torch
import torch.nn.functional as F

import convtasnet_oracle as O
import stage_entries_ref as R


@pytest.mark.parametrize("row", R.all_rows(), ids=["{}-{}".format(g, n) for g, n, _, _, _ in R.all_rows()])
def test_row_reaches_its_branches(row):
    grp, name, r, expect, got = row
    assert expect and r.reaches, "{} {}: names no branch".format(grp, name)
    assert expect <= got, "{} {}: names {} but reaches only {}".format(grp, name, sorted(expect - got), sorted(got))


def test_every_branch_is_reached():
    reached = set().union(*(expect & got for _, _, _, expect, got in R.all_rows()))
    assert reached == set(R.BRANCHES), sorted(set(R.BRANCHES) ^ reached)


def test_decoder_predicate_and_launch_counts():
    """the restated dispatch: every k_decoder<S, 2> instantiation and the generic decoder are named; a latent adds one copy per
    65535 rows; fp32 builds no weight image"""
    assert [R.decoder_kernel(L, s) for L, s in ((16, 8), (2, 1), (20, 10), (4, 2), (16, 4), (40, 20), (8, 8))] == [
        "k_decoder<8,2>", "k_decoder<1,2>", "k_decoder<10,2>", "k_decoder<2,2>", "k_decoder_generic", "k_decoder_generic",
        "k_decoder_generic"]
    assert R.head_launches("fp32") == 2 and R.head_launches("f16x3") == 3
    assert R.tail_launches("tf32x3", 2, 2, 128, True) == R.tail_launches("tf32x3", 2, 2, 128, False) + 1
    assert R.tail_launches("fp32", 300, 4, 128, True) == 2 + 3  # 153 600 latent rows: three copies
    assert R.pw_launches("fp32", 37, 129) == 2 and R.pw_launches("tf32", 1000, 129) == 4


def test_frames_of_matches_the_oracle_padding():
    for T, L, s in ((4003, 16, 8), (300, 2, 1), (2001, 20, 10), (513, 16, 4), (16, 16, 8), (1001, 16, 8)):
        f, pl, pr = R.frames_of(T, L, s)
        padding = (s - (T - L) % s) % s
        assert (pl, pr) == (padding // 2, padding - padding // 2)
        assert f == (T + padding - L) // s + 1


# ---- restatements against the oracle / F.conv1d ----------------------------------------------------------------------------
# GroupNorm refuses a group of one element (the 1 x 1 x 1 row); the encoder row's w comes from the GPU
@pytest.mark.parametrize("name", [n for n, r in R.HEAD.items() if not r.enc and r.N * r.frames > 1])
def test_head64_equals_oracle(name):
    r = R.HEAD[name]
    i = R.head_inputs(name, r)
    w = i["w"]
    st = R.stats_frames(w)
    got = R.head64(w, st, i["gamma"], i["beta"], i["W"], i["bias"], r.eps)
    want = F.conv1d(O.gln(w, i["gamma"], i["beta"], r.eps), i["W"][:, :, None], i["bias"])
    torch.testing.assert_close(got, want, rtol=1e-9, atol=1e-9 * float(want.abs().max()))
    ref, _ = R.head_reference(w, st, i["gamma"], i["beta"], i["W"], i["bias"], r.eps)
    torch.testing.assert_close(ref.out["D"][0], want, rtol=1e-9, atol=1e-9 * float(want.abs().max()))


@pytest.mark.parametrize("name", list(R.TAIL))
def test_tail64_equals_oracle(name):
    r = R.TAIL[name]
    i = R.tail_inputs(name, r)
    frames, pl, pr = R.frames_of(r.T, r.L, r.stride)
    out, lat = R.tail64(i["y"], i["w"], i["a"], i["Wm"], i["bm"], i["Wd"], r.S, r.stride, pl, r.T)
    B = r.B
    mask = torch.sigmoid(F.conv1d(O.prelu(i["y"], torch.tensor([i["a"]], dtype=torch.float64)), i["Wm"][:, :, None], i["bm"]))
    what = i["w"][:, None] * mask.view(B, r.S, r.N, frames)
    full = O.decoder_fwd(what.reshape(B * r.S, r.N, frames), i["Wd"][:, None], r.stride).view(B, r.S, -1)
    want = F.pad(full, (-pl, -pr))
    torch.testing.assert_close(out, want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(lat, what, rtol=1e-12, atol=1e-12)
    ref, _ = R.tail_reference(i["y"], i["w"], i["a"], i["Wm"], i["bm"], i["Wd"], r.S, r.stride, pl, r.T)
    torch.testing.assert_close(ref.out["D"][0].reshape(lat.shape), what, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", list(R.DW))
def test_depthwise64_equals_conv1d(name):
    r = R.DW[name]
    i = R.dw_inputs(name, r)
    got, _ = R.depthwise64(i["x"], i["w"], i["bias"], r.stride, r.padding, r.dilation)
    want = F.conv1d(i["x"], i["w"][:, None], i["bias"], stride=r.stride, padding=r.padding, dilation=r.dilation, groups=r.C)
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", list(R.PW))
def test_pointwise64_equals_conv1d(name):
    r = R.PW[name]
    i = R.pw_inputs(name, r)
    want = F.conv1d(i["x"], i["W"][:, :, None], i["bias"])
    torch.testing.assert_close(R.pointwise64(i["x"], i["W"], i["bias"]), want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(R.pointwise_reference(i["x"], i["W"], i["bias"]).out["D"][0], want, rtol=1e-12, atol=1e-12)


# ---- the bounds reject planted defects -------------------------------------------------------------------------------------
HEAD_MUTANTS = {"eps_outside": "eps_var", "n_pitch": "bc129_n513_f129_b37"}
TAIL_MUTANTS = {"no_bias": "s2_l16s8_n128_lat", "prelu_pos": "s1_l2s1_n5", "crop_off": "s4_l20s10_n129",
                "latent_pitch": "s2_l16s4_n7"}
DW_MUTANTS = {"dil_off": "c1_nobias", "one_side": "stride_gt_k", "stride_ignored": "stride_default"}


@pytest.mark.parametrize("mut", list(HEAD_MUTANTS))
def test_head_bound_rejects(mut):
    name = HEAD_MUTANTS[mut]
    r = R.HEAD[name]
    i = R.head_inputs(name, r)
    st = R.stats_frames(i["w"])
    args = (i["w"], st, i["gamma"], i["beta"], i["W"], i["bias"], r.eps)
    bad = R.head64(*args, mut=mut)
    ref, fold = R.head_reference(*args)
    for mode in R.MODES:
        s = R.share(bad, ref.out["D"][0], R.gate_allowance(ref, mode) + fold)
        assert s > R.REJECT, "{} on {} ({}): only {:.2f}x the bound".format(mut, name, mode, s)


@pytest.mark.parametrize("mut", list(TAIL_MUTANTS))
def test_tail_bound_rejects(mut):
    name = TAIL_MUTANTS[mut]
    r = R.TAIL[name]
    i = R.tail_inputs(name, r)
    _, pl, _ = R.frames_of(r.T, r.L, r.stride)
    args = (i["y"], i["w"], i["a"], i["Wm"], i["bm"], i["Wd"], r.S, r.stride, pl, r.T)
    out, lat = R.tail64(*args)
    bout, blat = R.tail64(*args, mut=mut)
    _, allowance = R.tail_reference(*args)
    for mode in R.MODES:
        alat, aout = allowance(mode)
        s = max(R.share(bout, out, aout), R.share(blat, lat, alat) if r.latent else 0.0)
        assert s > R.REJECT, "{} on {} ({}): only {:.2f}x the bound".format(mut, name, mode, s)


@pytest.mark.parametrize("mut", list(DW_MUTANTS))
def test_depthwise_bound_rejects(mut):
    name = DW_MUTANTS[mut]
    r = R.DW[name]
    i = R.dw_inputs(name, r)
    y, m = R.depthwise64(i["x"], i["w"], i["bias"], r.stride, r.padding, r.dilation)
    bad, _ = R.depthwise64(i["x"], i["w"], i["bias"], r.stride, r.padding, r.dilation, mut=mut)
    s = R.share(bad, y, R.depthwise_bound(m, r.K))
    assert s > R.REJECT, "{} on {}: only {:.2f}x the bound".format(mut, name, s)


def test_bounds_accept_float32_rounding():
    """the fp32 evaluation of each restatement (fp32 inputs, fp32 arithmetic) passes its bound in the fp32 mode"""
    name = "bc129_n64_f127_b37"
    r = R.HEAD[name]
    i = R.head_inputs(name, r)
    st = R.stats_frames(i["w"])
    args = (i["w"], st, i["gamma"], i["beta"], i["W"], i["bias"], r.eps)
    ref, fold = R.head_reference(*args)
    x32 = F.conv1d(F.group_norm(i["w"].float(), 1, i["gamma"].float(), i["beta"].float(), r.eps), i["W"].float()[:, :, None],
                   i["bias"].float())
    assert R.share(x32, ref.out["D"][0], R.gate_allowance(ref, "fp32") + fold) <= 1.0
    name = "stride_gt_k"
    r = R.DW[name]
    i = R.dw_inputs(name, r)
    y, m = R.depthwise64(i["x"], i["w"], i["bias"], r.stride, r.padding, r.dilation)
    y32 = F.conv1d(i["x"].float(), i["w"].float()[:, None], i["bias"].float(), stride=r.stride, padding=r.padding, groups=r.C)
    assert R.share(y32, y, R.depthwise_bound(m, r.K)) <= 1.0
