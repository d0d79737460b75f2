"""Causal (cLN) training without a GPU: the closed form of the cLN backward (tests/causal_train_ref.py, the formulas the kernels
implement) against torch autograd over the oracle's cLN in fp64, the status codes of the three causal training entry points, and
the Python switch."""
import ctypes as C
import os
import re

import pytest
import torch

import causal_train_ref as R
import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced
OK, EINVAL, EUNSUP, EALIGN, EWS = N.CTN_OK, N.CTN_EINVAL, N.CTN_EUNSUPPORTED, N.CTN_EALIGN, N.CTN_EWORKSPACE


@pytest.mark.parametrize("eps", [1e-12, 1e-3])
@pytest.mark.parametrize("T", [1, 2, 129])
@pytest.mark.parametrize("Cc", [1, 3, 20])
@pytest.mark.parametrize("slope", [None, 0.25, -0.4])
def test_closed_form_equals_autograd(Cc, T, eps, slope):
    g = torch.Generator().manual_seed(Cc * 1000 + T)
    pre = (torch.randn(2, Cc, T, generator=g, dtype=torch.float64) + 0.3).requires_grad_(True)
    gamma = (1.0 + 0.3 * torch.randn(Cc, generator=g, dtype=torch.float64)).requires_grad_(True)
    beta = (0.2 * torch.randn(Cc, generator=g, dtype=torch.float64)).requires_grad_(True)
    a = None if slope is None else torch.tensor([slope], dtype=torch.float64, requires_grad=True)
    dy = torch.randn(2, Cc, T, generator=g, dtype=torch.float64)
    x = pre if a is None else O.prelu(pre, a)
    y = O.cln(x, gamma, beta, eps)
    torch.testing.assert_close(R.cln_fwd(x.detach(), gamma.detach(), beta.detach(), eps), y.detach(), rtol=1e-12, atol=1e-12)
    if Cc == 1:  # frame 0 of a one-channel tensor has zero variance: autograd differentiates sqrt at 0 there and returns NaN for x[0]
        dy[:, :, 0] = 0
    (y * dy).sum().backward()
    got = R.cln_bwd(dy, pre.detach(), gamma.detach(), eps, slope)
    lo = 1 if Cc == 1 else 0  # the convention for such a frame: its clamped variance is a constant
    assert torch.isfinite(got["dpre"]).all() and torch.isfinite(pre.grad[:, :, lo:]).all()
    tol = dict(rtol=1e-9, atol=1e-9 * float(pre.grad[:, :, lo:].abs().sum() + 1))
    torch.testing.assert_close(got["dpre"][:, :, lo:], pre.grad[:, :, lo:], **tol)
    torch.testing.assert_close(got["dgamma"], gamma.grad, **tol)
    torch.testing.assert_close(got["dbeta"], beta.grad, **tol)
    if slope is not None and Cc > 1:  # one channel: autograd's slope gradient goes through x[0] and is NaN too
        torch.testing.assert_close(got["dslope"], a.grad, **tol)


def test_constant_input_has_finite_gradients():
    pre = torch.full((2, 4, 9), 0.5, dtype=torch.float64)
    got = R.cln_bwd(torch.ones_like(pre), pre, torch.ones(4, dtype=torch.float64), 1e-12)
    assert all(torch.isfinite(got[k]).all() for k in ("dpre", "dgamma", "dbeta"))


def test_causal_depthwise_closed_form_equals_autograd():
    g = torch.Generator().manual_seed(3)
    for P, dil, T in [(1, 1, 7), (2, 1, 7), (3, 8, 40), (5, 128, 50), (3, 4, 1)]:
        hn = torch.randn(2, 3, T, generator=g, dtype=torch.float64, requires_grad=True)
        wd = torch.randn(3, P, generator=g, dtype=torch.float64, requires_grad=True)
        bd = torch.randn(3, generator=g, dtype=torch.float64)
        du = torch.randn(2, 3, T, generator=g, dtype=torch.float64)
        ref = torch.nn.functional.conv1d(torch.nn.functional.pad(hn, ((P - 1) * dil, 0)), wd.unsqueeze(1), bd, dilation=dil, groups=3)
        torch.testing.assert_close(R.cdw_fwd(hn.detach(), wd.detach(), bd, dil), ref.detach(), rtol=1e-12, atol=1e-12)
        (ref * du).sum().backward()
        dhn, dwd, _, _ = R.cdw_bwd(du, hn.detach(), wd.detach(), dil)
        torch.testing.assert_close(dhn, hn.grad, rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(dwd, wd.grad, rtol=1e-12, atol=1e-12)


# ---- status codes ------------------------------------------------------------------------------------------------
TINY = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2, num_layers=4, n_sources=2)


def _cfg(**kw):
    c = N.Config()
    fields = dict(TINY, causal=1, enc_relu=0, mask_softmax=0, math=N.MATH_FP32, eps=1e-8, eps_tcn=1e-8, in_channels=1)
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


def _statuses(c, ws=FAKE, nbytes=0):
    n = C.c_size_t(0)
    p, keep = _params()
    return (N.ctn_causal_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)),
            N.ctn_causal_fwd_train(C.byref(c), C.byref(p), FAKE, 2, 4000, FAKE, ws, nbytes, None),
            N.ctn_causal_bwd(C.byref(c), C.byref(p), C.byref(p), FAKE, FAKE, 2, 4000, ws, nbytes, None))


# the training column of the single-fault table of test_host_plumbing_cpu.py on a causal base: the config verdict comes first
# at all three entry points; a valid config then meets the empty workspace
FAULTS = [
    (dict(), OK), (dict(n_basis=0), EINVAL), (dict(kernel_size=0), EINVAL), (dict(stride=0), EINVAL), (dict(n_sources=0), EINVAL),
    (dict(bottleneck=0), EINVAL), (dict(hidden=0), EINVAL), (dict(skip=0), EINVAL), (dict(sep_kernel=0), EINVAL),
    (dict(num_blocks=0), EINVAL), (dict(num_layers=0), EINVAL), (dict(kernel_size=12), EINVAL), (dict(math=7), EINVAL),
    (dict(mask_softmax=1), EUNSUP), (dict(mask_softmax=2), EINVAL), (dict(in_channels=-1), EINVAL), (dict(in_channels=2), EUNSUP),
    (dict(in_channels=100), EINVAL), (dict(causal=0), EUNSUP), (dict(sep_kernel=9), EUNSUP), (dict(num_layers=21), EUNSUP),
    (dict(num_blocks=9, num_layers=8), EUNSUP),
]


@pytest.mark.parametrize("kw,status", FAULTS, ids=[",".join(f"{k}={v}" for k, v in kw.items()) or "valid" for kw, _ in FAULTS])
def test_single_fault_status(kw, status):
    want = (status, status, status) if status != OK else (OK, EWS, EWS)
    assert _statuses(_cfg(**kw)) == want


def test_call_checks():
    c = _cfg()
    n = C.c_size_t(0)
    assert N.ctn_causal_train_workspace_bytes(C.byref(c), 0, 4000, C.byref(n)) == EINVAL
    assert N.ctn_causal_train_workspace_bytes(C.byref(c), 2, 4000, None) == EINVAL
    assert N.ctn_causal_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)) == OK and n.value > 0
    assert _statuses(c, ws=FAKE + 8, nbytes=n.value)[1:] == (EALIGN, EALIGN)
    assert _statuses(c, ws=None, nbytes=n.value)[1:] == (EINVAL, EINVAL)
    assert _statuses(c, ws=FAKE, nbytes=n.value - 1)[1:] == (EWS, EWS)
    # what the causal path keeps on top of the non-causal workspace: 40 bytes per frame and block, 16 per frame for cLN0, and
    # the backward's scratch (144 bytes per frame)
    g = C.c_size_t(0)
    assert N.ctn_train_workspace_bytes(C.byref(_cfg(causal=0)), 2, 4000, C.byref(g)) == OK
    frames = N.frames_of(4000, 16, 8)[0]
    extra = n.value - g.value
    assert 0 <= extra - 2 * frames * (40 * 8 + 16 + 144) < 256 * (3 * 8 + 3)
    assert N.ctn_cln_bwd(None, None, None, None, None, None, None, 1, 1, 1, 1e-8, None) == EINVAL
    assert N.ctn_cln_bwd(FAKE, FAKE, FAKE, FAKE + 8, FAKE, FAKE, FAKE, 1, 1, 1, 1e-8, None) == EALIGN


def test_old_entry_points_still_refuse_causal():
    n = C.c_size_t(0)
    p, keep = _params()
    c = _cfg()
    assert N.ctn_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)) == EUNSUP
    assert N.ctn_convtasnet_fwd_train(C.byref(c), C.byref(p), FAKE, 2, 4000, FAKE, FAKE, 0, None) == EUNSUP
    assert N.ctn_convtasnet_bwd(C.byref(c), C.byref(p), C.byref(p), FAKE, FAKE, 2, 4000, FAKE, 0, None) == EUNSUP


def _tiny_model():
    return ConvTasNet(16, 4, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=16,
                      sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=1, sep_num_layers=2, causal=True, n_sources=2)


def test_switch_off_refuses_before_any_cuda_requirement():
    m = _tiny_model()
    assert m.causal_training is False
    assert "causal_training" not in m.get_config() and not any("causal_training" in k for k in m.state_dict())
    with pytest.raises(NotImplementedError, match="causal_training"):
        m(torch.zeros(1, 1, 64))  # a CPU tensor: the refusal comes before the CUDA check
    m.causal_training = True
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 1, 64))


def test_header_declares_the_new_entry_points():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ctn_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ctn_[a-z0-9_]+)\s*\(", hdr))
    new = {"ctn_cln_bwd", "ctn_causal_train_workspace_bytes", "ctn_causal_fwd_train", "ctn_causal_bwd"}
    assert new <= declared and new <= set(N.EXPORTED) and declared == set(N.EXPORTED)
    probe = open(os.path.join(ROOT, "include", "ctn_b200_probe.h")).read()
    for name in ("ctn_probe_cln_stats", "ctn_probe_cln_bwd", "ctn_probe_cdw_train_fwd", "ctn_probe_cdw_bwd"):
        assert name in probe and hasattr(N.lib, name)
