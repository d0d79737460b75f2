"""Multichannel (in_channels > 1) training without a GPU: the status codes of the three ctn_multichannel_* entry points, their
workspace against the monaural step's, the oracle's autograd against the reference golden tiny_stereo_grad.pt, the distance
criteria against the reference's values, and the Python switch."""
import ctypes as C
import os
import re

import pytest
import torch

import convtasnet_oracle as O
from ctn_b200 import _native as N
from ctn_b200.criterion.distance import MeanAbsoluteError, MeanSquaredError
from ctn_b200.models.conv_tasnet import ConvTasNet

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tiny_stereo_grad.pt")
FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced
OK, EINVAL, EUNSUP, EALIGN, EWS = N.CTN_OK, N.CTN_EINVAL, N.CTN_EUNSUPPORTED, N.CTN_EALIGN, N.CTN_EWORKSPACE

TINY = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2, num_layers=4, n_sources=2)
PAPER = dict(n_basis=512, kernel_size=16, stride=8, bottleneck=128, hidden=512, skip=128, sep_kernel=3, num_blocks=3, num_layers=8, n_sources=2)
RECIPE = dict(n_basis=256, kernel_size=20, stride=10, bottleneck=256, hidden=512, skip=128, sep_kernel=3, num_blocks=4, num_layers=10,
              n_sources=4)


def _cfg(base=TINY, **kw):
    c = N.Config()
    fields = dict(base, causal=0, enc_relu=0, mask_softmax=0, math=N.MATH_FP32, eps=1e-8, eps_tcn=1e-8, in_channels=2)
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
    return (N.ctn_multichannel_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)),
            N.ctn_multichannel_fwd_train(C.byref(c), C.byref(p), FAKE, 2, 4000, FAKE, ws, nbytes, None),
            N.ctn_multichannel_bwd(C.byref(c), C.byref(p), C.byref(p), FAKE, FAKE, 2, 4000, ws, nbytes, None))


# the training column of the single-fault table of test_host_plumbing_cpu.py on a stereo base: the config verdict comes first at
# all three entry points; a valid config then meets the empty workspace
FAULTS = [
    (dict(), OK), (dict(in_channels=64), OK), (dict(in_channels=3, math=N.MATH_F16X3), OK),
    (dict(n_basis=0), EINVAL), (dict(kernel_size=0), EINVAL), (dict(stride=0), EINVAL), (dict(n_sources=0), EINVAL),
    (dict(bottleneck=0), EINVAL), (dict(hidden=0), EINVAL), (dict(skip=0), EINVAL), (dict(sep_kernel=0), EINVAL),
    (dict(num_blocks=0), EINVAL), (dict(num_layers=0), EINVAL), (dict(kernel_size=12), EINVAL), (dict(math=7), EINVAL),
    (dict(mask_softmax=2), EINVAL), (dict(in_channels=-1), EINVAL), (dict(in_channels=65), EINVAL), (dict(in_channels=100), EINVAL),
    (dict(mask_softmax=1), EUNSUP), (dict(causal=1), EUNSUP), (dict(in_channels=1), EUNSUP), (dict(in_channels=0), EUNSUP),
    (dict(sep_kernel=9), EUNSUP), (dict(num_layers=21), EUNSUP), (dict(num_blocks=9, num_layers=8), EUNSUP),
]


@pytest.mark.parametrize("kw,status", FAULTS, ids=[",".join(f"{k}={v}" for k, v in kw.items()) or "valid" for kw, _ in FAULTS])
def test_single_fault_status(kw, status):
    want = (status, status, status) if status != OK else (OK, EWS, EWS)
    assert _statuses(_cfg(**kw)) == want


def test_call_checks():
    c = _cfg()
    n = C.c_size_t(0)
    assert N.ctn_multichannel_train_workspace_bytes(C.byref(c), 0, 4000, C.byref(n)) == EINVAL
    assert N.ctn_multichannel_train_workspace_bytes(C.byref(c), 2, 4000, None) == EINVAL
    assert N.ctn_multichannel_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)) == OK and n.value > 0
    assert _statuses(c, ws=FAKE + 8, nbytes=n.value)[1:] == (EALIGN, EALIGN)
    assert _statuses(c, ws=None, nbytes=n.value)[1:] == (EINVAL, EINVAL)
    assert _statuses(c, ws=FAKE, nbytes=n.value - 1)[1:] == (EWS, EWS)


@pytest.mark.parametrize("base,T", [(TINY, 4000), (PAPER, 32000), (RECIPE, 352800)], ids=["tiny", "paper", "recipe"])
@pytest.mark.parametrize("math", [N.MATH_FP32, N.MATH_F16X3])
def test_workspace_equals_the_monaural_step(base, T, math):
    """no activation of the step depends on the input channel count: the same bytes as the monaural step of the same separator"""
    mono, multi = C.c_size_t(0), C.c_size_t(0)
    assert N.ctn_train_workspace_bytes(C.byref(_cfg(base, in_channels=1, math=math)), 4, T, C.byref(mono)) == OK
    for cin in (2, 64):
        assert N.ctn_multichannel_train_workspace_bytes(C.byref(_cfg(base, in_channels=cin, math=math)), 4, T, C.byref(multi)) == OK
        assert multi.value == mono.value


def test_old_entry_points_still_refuse_multichannel():
    n = C.c_size_t(0)
    p, keep = _params()
    c = _cfg()
    assert N.ctn_train_workspace_bytes(C.byref(c), 2, 4000, C.byref(n)) == EUNSUP
    assert N.ctn_convtasnet_fwd_train(C.byref(c), C.byref(p), FAKE, 2, 4000, FAKE, FAKE, 0, None) == EUNSUP
    assert N.ctn_convtasnet_bwd(C.byref(c), C.byref(p), C.byref(p), FAKE, FAKE, 2, 4000, FAKE, 0, None) == EUNSUP


# ---- reference golden ------------------------------------------------------------------------------------------------
def _golden():
    return torch.load(GOLDEN, weights_only=False)


def test_oracle_autograd_vs_reference_golden():
    """the oracle (the GPU tests' fp64 answer) differentiates the stereo model as the reference does: fp64 output, loss and every
    gradient equal the reference's fp64 values, and the fp32 ones sit within the reference's own fp32 noise"""
    r = _golden()
    cfg = O.OracleConfig(**r["cfg"])
    sd = O.synth_state_dict(cfg, seed=r["wseed"])
    for dtype in (torch.float64, torch.float32):
        sdv = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
        out, _ = O.conv_tasnet_fwd(r["mixture"].to(dtype), sdv, cfg)
        loss = MeanSquaredError(dim=-1, reduction="mean")(out, r["sources"].to(dtype))
        loss.backward()
        if dtype == torch.float64:
            torch.testing.assert_close(out.detach(), r["out64"], rtol=1e-10, atol=1e-12)
            assert abs(float(loss.detach()) - r["loss64"]) <= 1e-12 * abs(r["loss64"])
            for k, v in sdv.items():
                torch.testing.assert_close(v.grad, r["grads64"][k], rtol=1e-9, atol=1e-12 * float(r["grads64"][k].abs().max() + 1))
        else:
            torch.testing.assert_close(out.detach(), r["out"], rtol=1e-5, atol=1e-6)
            for k, v in sdv.items():
                bound = 4 * r["fp32_vs_fp64_maxabs"][k] + 1e-6 * float(r["grads64"][k].abs().max()) + 1e-12
                assert float((v.grad.double() - r["grads"][k].double()).abs().max()) <= bound, k


def test_distance_criteria_vs_reference_golden():
    c = _golden()["criteria"]
    x, t = c["input"], c["target"]
    n = 0
    for key, want in c.items():
        if not isinstance(key, tuple):
            continue
        name, dim, red, bm = key
        cls = MeanSquaredError if name == "mse" else MeanAbsoluteError
        got = cls(dim=dim, reduction=red)(x, t, batch_mean=bm)
        assert got.shape == want.shape, key
        torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-7)
        n += 1
    assert n == 72
    assert MeanSquaredError().maximize is False and MeanAbsoluteError().maximize is False
    with pytest.raises(NotImplementedError):
        MeanSquaredError(reduction="max")(x, t)


def test_distance_criteria_carry_gradients():
    x = torch.randn(2, 4, 2, 11, dtype=torch.float64, requires_grad=True)
    t = torch.randn(2, 4, 2, 11, dtype=torch.float64)
    MeanSquaredError(dim=-1, reduction="mean")(x, t).backward()
    torch.testing.assert_close(x.grad, 2 * (x - t).detach() / (2 * 11 * 4 * 2))


# ---- Python switch ----------------------------------------------------------------------------------------------------
def _tiny_model(**kw):
    return ConvTasNet(16, 4, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=16,
                      sep_bottleneck_channels=8, sep_skip_channels=8, sep_num_blocks=1, sep_num_layers=2, causal=False, n_sources=2,
                      in_channels=2, **kw)


def test_switch_off_refuses_before_any_cuda_requirement():
    m = _tiny_model()
    assert m.multichannel_training is False
    assert "multichannel_training" not in m.get_config() and not any("multichannel_training" in k for k in m.state_dict())
    x = torch.zeros(1, 1, 2, 64)  # a CPU tensor: the refusals come before the CUDA check
    with pytest.raises(NotImplementedError, match="multichannel_training"):
        m(x)
    m.multichannel_training = True
    with pytest.raises(RuntimeError, match="CUDA"):
        m(x)
    for bad in (_tiny_model(mask_nonlinear="softmax"), ConvTasNet(16, 4, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None,
                                                                  sep_hidden_channels=16, sep_bottleneck_channels=8, sep_skip_channels=8,
                                                                  sep_num_blocks=1, sep_num_layers=2, causal=True, n_sources=2,
                                                                  in_channels=2)):
        bad.multichannel_training = True
        bad.causal_training = True
        with pytest.raises(NotImplementedError, match="non-causal models with a sigmoid mask"):
            bad(x)


def test_header_declares_the_new_entry_points():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "ctn_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(ctn_[a-z0-9_]+)\s*\(", hdr))
    new = {"ctn_multichannel_train_workspace_bytes", "ctn_multichannel_fwd_train", "ctn_multichannel_bwd"}
    assert new <= declared and new <= set(N.EXPORTED) and declared == set(N.EXPORTED)
    probe = open(os.path.join(ROOT, "include", "ctn_b200_probe.h")).read()
    assert "ctn_probe_encdec_wgrad_mc" in probe and hasattr(N.lib, "ctn_probe_encdec_wgrad_mc")
