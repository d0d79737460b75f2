"""Softmax-mask training without a GPU: the status codes of the three ctn_softmax_* entry points under single faults and null
pointers, their workspace against the sigmoid step's, the header / EXPORTED / probe, the fp64 closed form of the softmax backward
against autograd (and the kernel bounds against two defects), the oracle against the reference golden tiny_softmax_grad.pt, and the
Python switch."""
import ctypes as C
import os
import re

import pytest
import torch

import convtasnet_oracle as O
import pit_variants_oracle as PV
import softmax_train_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tiny_softmax_grad.pt")
FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced
OK, EINVAL, EUNSUP, EALIGN, EWS = N.CTN_OK, N.CTN_EINVAL, N.CTN_EUNSUPPORTED, N.CTN_EALIGN, N.CTN_EWORKSPACE

TINY = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2, num_layers=4, n_sources=2)
PAPER = dict(n_basis=512, kernel_size=16, stride=8, bottleneck=128, hidden=512, skip=128, sep_kernel=3, num_blocks=3, num_layers=8, n_sources=2)
# egs/wsj0-mix/orpit_conv-tasnet/train.sh: N 512, L 16, H 512, B 128, Sc 128, P 3, X 8, R 3, two outputs (one and rest), softmax
ORPIT = dict(PAPER)


def _cfg(base=TINY, **kw):
    c = N.Config()
    fields = dict(base, causal=0, enc_relu=0, mask_softmax=1, math=N.MATH_FP32, eps=1e-8, eps_tcn=1e-8, in_channels=1)
    fields.update(kw)
    for k, v in fields.items():
        setattr(c, k, v)
    return c


def _params():
    blocks = (N.BlockParams * 8)()
    for b in blocks:
        for name in N.BLOCK_FIELDS:
            setattr(b, name, FAKE)
    p = N.Params()
    for name in N.TOP_FIELDS:
        setattr(p, name, FAKE)
    p.blocks = blocks
    return p, blocks


def _statuses(c, ws=FAKE, nbytes=0, d_x=FAKE):
    n = C.c_size_t(0)
    p, keep = _params()
    return (N.ctn_softmax_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)),
            N.ctn_softmax_fwd_train(C.byref(c), C.byref(p), FAKE, 2, 4000, FAKE, ws, nbytes, None),
            N.ctn_softmax_bwd(C.byref(c), C.byref(p), C.byref(p), FAKE, FAKE, d_x, 2, 4000, ws, nbytes, None))


# the training column of the single-fault table of test_host_plumbing_cpu.py on a softmax base: the config verdict comes first at
# all three entry points; a valid config then meets the empty workspace
FAULTS = [
    (dict(), OK), (dict(in_channels=0), OK), (dict(math=N.MATH_F16X3), OK), (dict(math=N.MATH_TF32X3), OK), (dict(enc_relu=1), OK),
    (dict(n_sources=5), OK), (dict(sep_kernel=8), OK),
    (dict(n_basis=0), EINVAL), (dict(kernel_size=0), EINVAL), (dict(stride=0), EINVAL), (dict(n_sources=0), EINVAL),
    (dict(bottleneck=0), EINVAL), (dict(hidden=0), EINVAL), (dict(skip=0), EINVAL), (dict(sep_kernel=0), EINVAL),
    (dict(num_blocks=0), EINVAL), (dict(num_layers=0), EINVAL), (dict(kernel_size=12), EINVAL), (dict(math=7), EINVAL),
    (dict(mask_softmax=2), EINVAL), (dict(in_channels=-1), EINVAL), (dict(in_channels=65), EINVAL),
    (dict(mask_softmax=0), EUNSUP), (dict(causal=1), EUNSUP), (dict(in_channels=2), EUNSUP), (dict(in_channels=64), EUNSUP),
    (dict(sep_kernel=9), EUNSUP), (dict(num_layers=21), EUNSUP), (dict(num_blocks=9, num_layers=8), EUNSUP),
]


@pytest.mark.parametrize("kw,status", FAULTS, ids=[",".join(f"{k}={v}" for k, v in kw.items()) or "valid" for kw, _ in FAULTS])
def test_single_fault_status(kw, status):
    want = (status, status, status) if status != OK else (OK, EWS, EWS)
    assert _statuses(_cfg(**kw)) == want


def test_call_checks():
    c = _cfg()
    n = C.c_size_t(0)
    assert N.ctn_softmax_train_workspace_bytes(C.byref(c), 0, 4000, C.byref(n)) == EINVAL
    assert N.ctn_softmax_train_workspace_bytes(C.byref(c), 2, 4000, None) == EINVAL
    assert N.ctn_softmax_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)) == OK and n.value > 0
    assert _statuses(c, ws=FAKE + 8, nbytes=n.value)[1:] == (EALIGN, EALIGN)
    assert _statuses(c, ws=None, nbytes=n.value)[1:] == (EINVAL, EINVAL)
    assert _statuses(c, ws=FAKE, nbytes=n.value - 1)[1:] == (EWS, EWS)


def test_null_pointers_are_refused_before_any_cuda_call():
    """every pointer but d_x: CTN_EINVAL with a workspace that passes the size check (a call that got further would launch on FAKE
    addresses); a null d_x is accepted and reaches the workspace check"""
    c = _cfg()
    need = C.c_size_t(0)
    assert N.ctn_softmax_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(need)) == OK
    nb = need.value
    p, keep = _params()
    g, keep2 = _params()
    P, Cb = C.byref(p), C.byref(c)
    fwd = [(P, FAKE, FAKE, FAKE), (None, FAKE, FAKE, FAKE), (P, None, FAKE, FAKE), (P, FAKE, None, FAKE), (P, FAKE, FAKE, None)]
    for i, (pp, x, out, ws) in enumerate(fwd[1:]):
        assert N.ctn_softmax_fwd_train(Cb, pp, x, 2, 4000, out, ws, nb, None) == EINVAL, i
    bwd = [(None, C.byref(g), FAKE, FAKE, FAKE), (P, None, FAKE, FAKE, FAKE), (P, C.byref(g), None, FAKE, FAKE),
           (P, C.byref(g), FAKE, None, FAKE), (P, C.byref(g), FAKE, FAKE, None)]
    for i, (pp, gg, x, d_out, ws) in enumerate(bwd):
        for d_x in (FAKE, None):
            assert N.ctn_softmax_bwd(Cb, pp, gg, x, d_out, d_x, 2, 4000, ws, nb, None) == EINVAL, (i, d_x)
    p.blocks = None
    assert N.ctn_softmax_fwd_train(Cb, P, FAKE, 2, 4000, FAKE, FAKE, nb, None) == EINVAL
    assert N.ctn_softmax_bwd(Cb, P, C.byref(g), FAKE, FAKE, None, 2, 4000, FAKE, nb, None) == EINVAL
    g.blocks = None
    q, keep3 = _params()
    assert N.ctn_softmax_bwd(Cb, C.byref(q), C.byref(g), FAKE, FAKE, FAKE, 2, 4000, FAKE, nb, None) == EINVAL
    for B, T in ((0, 4000), (2, 0), (-1, 4000)):
        assert N.ctn_softmax_fwd_train(Cb, C.byref(q), FAKE, B, T, FAKE, FAKE, nb, None) == EINVAL
    # a null d_x is not an error: the call reaches the workspace check
    assert _statuses(c, d_x=None)[2] == EWS


@pytest.mark.parametrize("base,T,S", [(TINY, 4000, 2), (PAPER, 32000, 2), (ORPIT, 32000, 2), (dict(TINY, n_sources=5), 16000, 5)],
                         ids=["tiny", "paper", "orpit-recipe", "sinkpit-5"])
@pytest.mark.parametrize("math", [N.MATH_FP32, N.MATH_TF32X3, N.MATH_F16X3])
def test_workspace_equals_the_sigmoid_step(base, T, S, math):
    """ws.mask holds the softmax and d_z goes in place over d_what: the same bytes as the sigmoid step of the same separator"""
    sig, soft = C.c_size_t(0), C.c_size_t(0)
    for B in (1, 4):
        assert N.ctn_train_workspace_bytes(C.byref(_cfg(base, mask_softmax=0, math=math)), B, T, C.byref(sig)) == OK
        assert N.ctn_softmax_train_workspace_bytes(C.byref(_cfg(base, math=math)), B, T, C.byref(soft)) == OK
        assert soft.value == sig.value


def test_old_entry_points_still_refuse_softmax():
    n = C.c_size_t(0)
    p, keep = _params()
    c = _cfg()
    for ws_fn, fwd, bwd in ((N.ctn_train_workspace_bytes, N.ctn_convtasnet_fwd_train, N.ctn_convtasnet_bwd),
                            (N.ctn_causal_train_workspace_bytes, N.ctn_causal_fwd_train, N.ctn_causal_bwd)):
        cc = _cfg(causal=1) if ws_fn is N.ctn_causal_train_workspace_bytes else c
        assert ws_fn(C.byref(cc), 2, 4000, C.byref(n)) == EUNSUP
        assert fwd(C.byref(cc), C.byref(p), FAKE, 2, 4000, FAKE, FAKE, 0, None) == EUNSUP
        assert bwd(C.byref(cc), C.byref(p), C.byref(p), FAKE, FAKE, 2, 4000, FAKE, 0, None) == EUNSUP
    mc = _cfg(in_channels=2)
    assert N.ctn_multichannel_train_workspace_bytes(C.byref(mc), 2, 4000, C.byref(n)) == EUNSUP


def test_header_exported_and_probe():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ctn_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ctn_[a-z0-9_]+)\s*\(", hdr))
    new = {"ctn_softmax_train_workspace_bytes", "ctn_softmax_fwd_train", "ctn_softmax_bwd"}
    assert new <= declared and new <= set(N.EXPORTED) and declared == set(N.EXPORTED)
    assert re.search(r"int ctn_softmax_bwd\([^;]*const float\* d_out, float\* d_x, int B, int T", hdr)
    probe = open(os.path.join(ROOT, "include", "ctn_b200_probe.h")).read()
    assert "ctn_probe_softmax_mask_bwd" in probe and hasattr(N.lib, "ctn_probe_softmax_mask_bwd")
    # the probe checks its geometry before any launch
    f = N._sig("ctn_probe_softmax_mask_bwd", N._i, N._fp, N._fp, N._fp, N._fp, N._i, N._i, N._i, N._i, N._i, N._fp)
    for args in ((1, 2, 7, 5, 100), (1, 2, 7, 129, 128), (0, 2, 7, 5, 128), (1, 0, 7, 5, 128), (1, 2, 0, 5, 128)):
        assert f(FAKE, FAKE, FAKE, FAKE, *args, None) == EINVAL, args


# ---- the closed form -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,N_,F", [(1, 7, 5), (2, 16, 9), (5, 8, 3)])
def test_closed_form_equals_autograd(S, N_, F):
    """d_z = m (g - sum_c m_c g_c) and d_w = sum_s d_what m of softmax over all S*N channels equal torch autograd in fp64"""
    g = torch.Generator().manual_seed(7 + S)
    dwhat = torch.randn(3, S, N_, F, generator=g, dtype=torch.float64)
    w = torch.randn(3, N_, F, generator=g, dtype=torch.float64)
    z = 2 * torch.randn(3, S * N_, F, generator=g, dtype=torch.float64)
    dz_ag, dw_ag = R.autograd_softmax_mask(dwhat, w, z)
    ref = R.softmax_mask_bwd(dwhat, w, torch.softmax(z, dim=1).view(3, S, N_, F))
    torch.testing.assert_close(ref["dz"][0], dz_ag, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(ref["dwprod"][0], dw_ag, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("name", [k for k in R.ROWS if k != "2x512-F4000"])
@pytest.mark.parametrize("mut", ["no_dot", "dot_src0"])
def test_bounds_reject_the_defects(name, mut):
    """each kernel row's d_z bound is at least 10x too tight for a kernel that drops dot, or sums it over source 0 only (S = 1
    has no other source: dot_src0 is the right answer there)"""
    dwhat, w, m = R.inputs(name)
    ref, bound = R.softmax_mask_bwd(dwhat, w, m)["dz"]
    bad = R.softmax_mask_bwd(dwhat, w, m, mut=mut)["dz"][0]
    r = float(((bad - ref).abs() / bound.clamp_min(1e-300)).max())
    if mut == "dot_src0" and R.ROWS[name][1] == 1:
        assert r == 0.0
    else:
        assert r >= 10, (name, mut, r)


# ---- reference golden ----------------------------------------------------------------------------------------------------
def _golden():
    return torch.load(GOLDEN, weights_only=False)


def _orpit(est, tgt):
    return PV.orpit(est, tgt, batch_mean=True)


def _check_vs_golden(r, sdv, out, loss, dtype):
    if dtype == torch.float64:
        torch.testing.assert_close(out.detach(), r["out64"], rtol=1e-10, atol=1e-12)
        assert abs(float(loss.detach()) - r["loss64"]) <= 1e-12 * abs(r["loss64"])
        for k, v in sdv.items():
            torch.testing.assert_close(v.grad, r["grads64"][k], rtol=1e-9, atol=1e-12 * float(r["grads64"][k].abs().max() + 1))
    else:
        torch.testing.assert_close(out.detach(), r["out"], rtol=1e-5, atol=1e-6)
        for k, v in sdv.items():
            bound = 4 * r["fp32_vs_fp64_maxabs"][k] + 1e-5 * float(r["grads64"][k].abs().max()) + 1e-12
            assert float((v.grad.double() - r["grads64"][k]).abs().max()) <= bound, k


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32])
@pytest.mark.parametrize("case", ["orpit", "finetune", "sinkpit"])
def test_oracle_autograd_vs_reference_golden(case, dtype):
    """the oracle (the GPU tests' fp64 answer) and the test criteria differentiate the softmax model as the reference does:
    ORPIT over 2- and 3-speaker targets, the two-stage fine-tune step through the mixture gradient, and SinkPIT at 5 outputs"""
    r = _golden()[case]
    cfg = O.OracleConfig(**r["cfg"])
    assert cfg.mask_nonlinear == "softmax"
    sd = O.synth_state_dict(cfg, seed=r["wseed"])
    sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}

    def model(x):
        return O.conv_tasnet_fwd(x, sdv, cfg)[0]

    if case == "orpit":
        lens = [t.shape[0] for t in r["targets"]]
        tgt = torch.zeros(len(lens), max(lens), r["targets"][0].shape[-1], dtype=dtype)
        for b, t in enumerate(r["targets"]):
            tgt[b, :t.shape[0]] = t.to(dtype)
        out = model(r["mixture"].to(dtype))
        loss, idx = PV.orpit(out, tgt, lengths=lens)
        assert torch.equal(idx, r["extra64"])
    elif case == "finetune":
        loss, ests = R.finetune_loss(model, r["mixture"].to(dtype), r["sources"].to(dtype), _orpit)
        out = ests[0]
        assert len(ests) == 2
    else:
        out = model(r["mixture"].to(dtype))
        loss, P = PV.sinkpit(out, r["sources"].to(dtype))
        assert torch.equal(torch.argmax(P, dim=2), r["extra64"])
    loss.backward()
    _check_vs_golden(r, sdv, out, loss, dtype)


# ---- Python switch -------------------------------------------------------------------------------------------------------
def _tiny_model(**kw):
    args = dict(enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=16, sep_bottleneck_channels=8,
                sep_skip_channels=8, sep_num_blocks=1, sep_num_layers=2, causal=False, n_sources=2, mask_nonlinear="softmax")
    args.update(kw)
    return ConvTasNet(16, 4, **args)


def test_switch_defaults_and_refusals_before_any_cuda_requirement():
    m = _tiny_model()
    assert m.softmax_training is False
    assert "softmax_training" not in m.get_config() and not any("softmax_training" in k for k in m.state_dict())
    x = torch.zeros(1, 1, 64)  # a CPU tensor: the refusals come before the CUDA check
    with pytest.raises(RuntimeError, match="CUDA"):  # switch off: the sigmoid node as before, which refuses on the GPU
        m(x)
    m.softmax_training = True
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x.clone().requires_grad_(True))
    causal = _tiny_model(causal=True)
    causal.softmax_training = True
    with pytest.raises(NotImplementedError, match="non-causal monaural"):
        causal(x)
    causal.causal_training = True
    with pytest.raises(NotImplementedError, match="non-causal monaural"):
        causal(x)
    stereo = _tiny_model(in_channels=2)
    stereo.softmax_training = True
    x4 = torch.zeros(1, 1, 2, 64)
    with pytest.raises(NotImplementedError, match="multichannel_training"):  # the multichannel checks still come first
        stereo(x4)
    stereo.multichannel_training = True
    with pytest.raises(NotImplementedError, match="non-causal models with a sigmoid mask"):
        stereo(x4)
