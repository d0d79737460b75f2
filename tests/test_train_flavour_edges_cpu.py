"""The softmax-mask / multichannel edge rows and the silent batches of tests/test_train_flavour_edges_gpu.py without a GPU: every
row's frame count and training workspace query, which rows run the un-fused f16x3 step, the fp64 oracle's autograd on the
silent batches (finite, and the silent sample's share of every gradient exactly 0), the near-silent sample's amplitude, and
that the GPU file's bounds reject plausible defects of the tail of the backward.

Each mutant is applied to an fp64 restatement of that tail (flavour_edges_ref.mixture_grad: mask backward -> encoder adjoint ->
crop) or of the oracle's forward (flavour_edges_ref.forward_kept), on a named row, with the bound the GPU file holds the kernels
to.  It must land at >= REJECT times that bound while the unmutated restatement equals the oracle's own autograd.
"""
import ctypes as C

import pytest
import torch

import convtasnet_oracle as O
import flavour_edges_ref as R
from ctn_b200 import _native as N
from ctn_b200.models import _train
from ctn_b200.models.conv_tasnet import ConvTasNet
from test_train_edges_gpu import GRAD_ATOL, GRAD_PER, OUT_ATOL, OUT_RTOL, _role_scales
from test_train_gpu import _role

REJECT = 4.0
MATHS = {"fp32": N.MATH_FP32, "tf32x3": N.MATH_TF32X3, "f16x3": N.MATH_F16X3}


def _model(cfg):
    """the CPU ConvTasNet of an oracle config, with the training switch of its flavour on"""
    m = ConvTasNet(cfg.n_basis, cfg.kernel_size, stride=cfg.stride, enc_basis="trainable", dec_basis="trainable",
                   enc_nonlinear=cfg.enc_nonlinear, sep_hidden_channels=cfg.sep_hidden_channels,
                   sep_bottleneck_channels=cfg.sep_bottleneck_channels, sep_skip_channels=cfg.sep_skip_channels,
                   sep_kernel_size=cfg.sep_kernel_size, sep_num_blocks=cfg.sep_num_blocks, sep_num_layers=cfg.sep_num_layers,
                   mask_nonlinear=cfg.mask_nonlinear, causal=cfg.causal, n_sources=cfg.n_sources, eps=cfg.eps, in_channels=cfg.in_channels)
    m.softmax_training = m.multichannel_training = True
    return m


def _rows():
    """(id, cfg, batch, T, frames, reaches) of every row of the GPU file"""
    rows = []
    for k, e in R.SOFTMAX.items():
        rows.append(("softmax-" + k, O.OracleConfig(causal=False, mask_nonlinear="softmax", **e.shape), e.batch, e.T, e.frames, e.reaches))
    for k, e in R.MULTICHANNEL.items():
        rows.append(("mc-" + k, O.OracleConfig(causal=False, in_channels=e.C, **e.shape), e.batch, e.T, e.frames, e.reaches))
    for fl in R.FLAVOURS:
        for relu in (False, True):
            cfg = R.silent_batch(fl, relu)[0]
            rows.append(("silent-{}-relu{}".format(fl, int(relu)), cfg, 4, R.SILENT_T, R.SILENT_FRAMES, R.SILENT_REACHES))
    return rows


ROWS = _rows()
WANT_ENTRY = {"softmax": _train.SOFTMAX, "mc": _train.MULTICHANNEL, "silent-gln": _train.GLN, "silent-softmax": _train.SOFTMAX,
              "silent-mc": _train.MULTICHANNEL}


def _ws(cfg, B, T, entry, math, sep_kernel=None):
    c = _model(cfg)
    c.math = math
    nc = c.native_config()
    if sep_kernel is not None:
        nc.sep_kernel = sep_kernel
    n = C.c_size_t(0)
    status = getattr(N, entry.WORKSPACE_BYTES)(C.byref(nc), B, T, C.byref(n))
    return status, n.value


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_row_frames_and_workspace(row):
    """the frame count the host library gives the row, and the training step the model takes: its workspace query returns
    CTN_OK with a non-empty workspace in every math mode"""
    name, cfg, B, T, frames, _ = row
    assert N.frames_of(T, cfg.kernel_size, cfg.stride)[0] == frames
    entry = _train.train_entry(_model(cfg))
    assert entry is WANT_ENTRY[name.rsplit("-", 1)[0] if name.startswith("silent") else name.split("-")[0]]
    for mode in MATHS:
        status, nbytes = _ws(cfg, B, T, entry, mode)
        assert status == N.CTN_OK and nbytes > 0, (mode, status)


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_which_rows_run_the_unfused_f16x3_step(row):
    """fused_tcn = !causal && f16x3 && P == 3, seen through the workspace: the fused TCN's state is carved only when it runs, so
    in f16x3 the row's workspace exceeds that of the same config at P = 1 exactly when P == 3; in fp32 and tf32x3 P changes
    nothing.  Every multichannel row has P != 3, and every row's `reaches` says which step it takes"""
    name, cfg, B, T, _, reaches = row
    entry = _train.train_entry(_model(cfg))
    P = cfg.sep_kernel_size
    f16 = _ws(cfg, B, T, entry, "f16x3")[1]
    assert (f16 > _ws(cfg, B, T, entry, "f16x3", sep_kernel=1)[1]) == (P == 3)
    for mode in ("fp32", "tf32x3"):
        assert _ws(cfg, B, T, entry, mode)[1] == _ws(cfg, B, T, entry, mode, sep_kernel=1)[1]
    if name.startswith("mc-"):
        assert P != 3
    if not name.startswith("silent"):
        assert ("un-fused" in reaches) == (P != 3) and ("fused" in reaches)


EDGE_ROWS = [("softmax", k) for k in R.SOFTMAX] + [("mc", k) for k in R.MULTICHANNEL]


@pytest.mark.parametrize("flavour,case", EDGE_ROWS, ids=["{}-{}".format(*r) for r in EDGE_ROWS])
def test_prelu_inputs_clear_of_the_kink(flavour, case):
    """every PReLU input of an edge row sits at least PRELU_MARGIN of its tensor's largest |entry| from 0, so no kernel rounding
    puts it on the other slope; the fp32-oracle guard of the GPU file cannot see a kink that fp32 and fp64 round to the same
    side.  The silent batches are not held to it: at 16000 samples x 4 they carry ~3.5M PReLU inputs, so some always sit
    closer than that, and no input seed from 712 to 799 clears it"""
    cfg, sd, mixture, _, _ = (R.softmax_setup if flavour == "softmax" else R.mc_setup)(case)
    margin, call = min(R.prelu_margins(cfg, sd, mixture))
    print("[{} {}] smallest |PReLU input| / max {:.2e} (call {})".format(flavour, case, margin, call))
    assert margin >= R.PRELU_MARGIN, (margin, call)


# ---- the silent batches -------------------------------------------------------------------------------------------------------
SILENT = [(fl, relu) for fl in R.FLAVOURS for relu in (False, True)]


@pytest.mark.parametrize("flavour,relu", SILENT)
def test_near_silent_amplitude(flavour, relu):
    """gLN0 sees variance exactly 0 for the zero sample, 1 .. 100 x eps for the near-silent one, and far above eps otherwise"""
    cfg, sd, mixture, _, _ = R.silent_batch(flavour, relu)
    v = R.gln0_var_over_eps(cfg, sd, mixture)
    assert float(v[R.ZERO]) == 0.0
    assert 1.0 <= float(v[R.NEAR]) <= 100.0, float(v[R.NEAR])
    assert float(v[R.ORDINARY]) > 1e6 and float(v[R.ONSET]) > 1e6
    print("[{} relu={}] var(w) / eps of the near-silent sample {:.1f}".format(flavour, relu, float(v[R.NEAR])))


@pytest.mark.parametrize("flavour,relu", SILENT)
def test_oracle_autograd_on_silent_batches(flavour, relu):
    """GroupNorm keeps eps inside the sqrt, so the fp64 oracle needs no convention-aware stand-in here: with the GPU file's
    drivers every gradient (and softmax's d_x) is finite and the zero sample's estimate is exactly 0; with a fixed cotangent the
    gradients equal those of the batch without the zero sample to fp64 rounding (d_mask = d_what w = 0, G x w_hat = 0 and
    d_w x x = 0), and with the encoder ReLU the zero sample's d_x is exactly 0"""
    cfg, sd, mixture, sources, G = R.silent_batch(flavour, relu)
    drives = [((sources,), False), (G, flavour == "softmax")]
    for drive, x_grad in drives:
        out, _, g, dx, _, _ = R.oracle(cfg, sd, mixture, drive, torch.float64, x_grad=x_grad)
        assert torch.equal(out[R.ZERO], torch.zeros_like(out[R.ZERO]))
        assert all(torch.isfinite(v).all() for v in g.values()), [k for k, v in g.items() if not torch.isfinite(v).all()]
        if x_grad:
            assert bool(torch.isfinite(dx).all())
            if relu:
                assert torch.equal(dx[R.ZERO], torch.zeros_like(dx[R.ZERO]))
    keep = [b for b in range(mixture.shape[0]) if b != R.ZERO]
    g_all = R.oracle(cfg, sd, mixture, G, torch.float64)[2]
    g_keep = R.oracle(cfg, sd, mixture[keep], G[keep], torch.float64)[2]
    for k in g_all:
        torch.testing.assert_close(g_all[k], g_keep[k], rtol=1e-9, atol=1e-12 * float(g_all[k].abs().max()) + 1e-300)


# ---- mutants -----------------------------------------------------------------------------------------------------------------
def _tail(cfg, sd, mixture, G):
    """fp64 oracle with d_x, and the restated d_x from its kept d_w: they must agree before a mutant means anything"""
    out, _, g, dx, _, kept = R.oracle(cfg, sd, mixture, G, torch.float64, x_grad=True)
    args = (kept["w"].grad, kept["w_pre"].detach(), sd["encoder.conv1d.weight"].double(), cfg.stride, kept["pl"], mixture.shape[-1],
            cfg.enc_nonlinear == "relu")
    restated = R.mixture_grad(*args)
    torch.testing.assert_close(restated, dx, rtol=1e-10, atol=1e-12 * float(dx.abs().max()))
    return dx, args


def _dx_shares(got, dx64, per_sample):
    """error of each sample's d_x over the GPU file's bound (GRAD_PER of the batch's, or of the sample's, largest |d_x|)"""
    err = (got - dx64).abs().flatten(1).max(dim=1).values
    mag = dx64.abs().flatten(1).max(dim=1).values
    scale = mag if per_sample else mag.max().expand_as(mag)
    return err / (GRAD_PER * scale + GRAD_ATOL)


def mutant_relu_at_zero():
    """k_dw_combine passing d_w where w_pre = 0 (relu'(0) = 1): d_x on the silent-onset sample's frames of exact zeros"""
    cfg, sd, mixture, _, G = R.silent_batch("softmax", True)
    dx64, args = _tail(cfg, sd, mixture, G)
    q = _dx_shares(R.mixture_grad(*args, mut="relu_at_zero"), dx64, per_sample=True)
    return "silent-softmax-relu sample {} (silent onset)".format(R.ONSET), float(q[R.ONSET])


def mutant_no_crop():
    """d_x = conv_transpose1d(d_w, W_enc) without the crop of the encoder's left pad, at E2 (k_decoder_generic, pads 4 / 4)"""
    cfg, sd, mixture, _, G = R.softmax_setup("E2")
    assert R.encoder_pre(cfg, sd, mixture)[1] == 4
    dx64, args = _tail(cfg, sd, mixture, G)
    q = _dx_shares(R.mixture_grad(*args, mut="no_crop"), dx64, per_sample=False)
    return "softmax-E2", float(q.max())


def mutant_gln0_eps_outside():
    """gLN0 as (w - mean) / (sqrt(var) + eps): the near-silent sample's estimate, at its own scale as the GPU file checks it"""
    cfg, sd, mixture, sources, _ = R.silent_batch("gln", False)
    sdv = {k: v.double() for k, v in sd.items()}
    out64, _ = R.forward_kept(mixture.double(), sdv, cfg)
    plain = O._norm

    def norm(x, sd_, prefix, causal, eps):  # gLN0 only; the blocks' gLNs keep eps inside the sqrt
        if prefix == "separator.norm1d.":
            return R.gln_eps_outside(x, sd_[prefix + "norm.weight"], sd_[prefix + "norm.bias"], eps)
        return plain(x, sd_, prefix, causal, eps)

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(O, "_norm", norm)
        bad, _ = R.forward_kept(mixture.double(), sdv, cfg)
    ref, mut = out64[R.NEAR].detach(), bad[R.NEAR].detach()
    bound = OUT_RTOL * ref.abs() + OUT_ATOL * float(ref.abs().max())
    return "silent-gln-relu0 sample {} (near-silent)".format(R.NEAR), float(((mut - ref).abs() / bound).max())


def mutant_silent_mask_grad():
    """the zero sample contributing d_mask = d_what (w taken as 1) instead of d_what w = 0: every gradient upstream of the mask
    against the GPU file's role-scaled bound"""
    cfg, sd, mixture, _, G = R.silent_batch("softmax", False)
    g64 = R.oracle(cfg, sd, mixture, G, torch.float64)[2]
    bad = R.oracle(cfg, sd, mixture, G, torch.float64, mask_grad_from=R.ZERO)[2]
    group = _role_scales(g64)
    q = max(float((bad[k] - g64[k]).abs().max()) / (GRAD_PER * group[_role(k)] + GRAD_ATOL) for k in g64)
    return "silent-softmax-relu0, cotangent", q


MUTANTS = {"relu_backward_at_zero": mutant_relu_at_zero, "d_x_without_crop": mutant_no_crop,
           "gln0_eps_outside_sqrt": mutant_gln0_eps_outside, "silent_sample_mask_gradient": mutant_silent_mask_grad}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_reject_mutant(mutant):
    row, q = MUTANTS[mutant]()
    print("{}: rejected on row {} at {:.3g} x the bound".format(mutant, row, q))
    assert q >= REJECT, "{}: only {:.3g} x the bound on {}".format(mutant, q, row)
