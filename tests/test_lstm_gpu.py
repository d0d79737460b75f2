"""GPU parity of the native bi-LSTM + projection kernel (``ctn_bilstm_proj_fwd``, csrc/ctn_lstm.cu; ``-m gpu``).

Oracle: the reference's recurrence is torch.nn.LSTM on the CPU (src/models/dprnn.py:60, 85 / 114-120, 138), restated in
oracle/dprnn_oracle.py::_bilstm; here it is evaluated in fp64 as ground truth and in fp32 (the reference's own precision) to
size the tolerance: the kernel must be as close to fp64 as the fp32 CPU recurrence is, up to a small factor.
Tolerance: |h - h64| <= 2e-5 (h in (-1, 1)), projection rtol 1e-4 / atol 2e-5 x max|ref|."""
import ctypes as C

import pytest
import torch

import dprnn_oracle as DO
from ctn_b200 import _native as N
from ctn_b200.models import dprnn as dprnn_mod
from ctn_b200.models.dprnn import DPRNN

pytestmark = pytest.mark.gpu

NAMES = ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0", "weight_ih_l0_reverse", "weight_hh_l0_reverse",
         "bias_ih_l0_reverse", "bias_hh_l0_reverse")


def _weights(Fi, H, Fo, seed, wscale=1.0):
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / H ** 0.5
    sd = {}
    for n in NAMES:
        shape = (4 * H, Fi) if "weight_ih" in n else ((4 * H, H) if "weight_hh" in n else (4 * H,))
        sd["rnn." + n] = (torch.rand(shape, generator=g) * 2 - 1) * k * wscale
    sd["fc.weight"] = (torch.rand(Fo, 2 * H, generator=g) * 2 - 1) / (2 * H) ** 0.5
    sd["fc.bias"] = (torch.rand(Fo, generator=g) * 2 - 1) / (2 * H) ** 0.5
    return sd


def _run(z, sd, H, Fo, want_h=True, want_p=True):
    NSEQ, T, Fi = z.shape
    dev = torch.device("cuda")
    zc = z.to(dev).contiguous()
    w = [sd["rnn." + n].to(dev).contiguous() for n in NAMES]
    ptrs = (N._fp * 8)(*[t.data_ptr() for t in w])
    fc = sd["fc.weight"].to(dev).contiguous()
    nws = N.ctn_bilstm_workspace_bytes(Fi, H, Fo)
    assert nws > 0
    ws = torch.empty(nws, dtype=torch.uint8, device=dev)
    P = torch.full((2, NSEQ, T, Fo), float("nan"), device=dev) if want_p else None
    hout = torch.full((NSEQ, T, 2 * H), float("nan"), device=dev) if want_h else None
    N.check(N.ctn_bilstm_proj_fwd(zc.data_ptr(), NSEQ, T, Fi, H, ptrs, fc.data_ptr() if want_p else None, Fo,
                                  P.data_ptr() if want_p else None, hout.data_ptr() if want_h else None, None, ws.data_ptr(), nws,
                                  N.stream_ptr(dev)), "ctn_bilstm_proj_fwd")
    torch.cuda.synchronize()
    return (hout.cpu() if want_h else None), (P.cpu() if want_p else None)


def _ref(z, sd, dtype):
    sdd = {k: v.to(dtype) for k, v in sd.items()}
    h = DO._bilstm(z.to(dtype), sdd, "rnn.")
    y = torch.nn.functional.linear(h, sdd["fc.weight"], sdd["fc.bias"])
    return h, y


# (64,128,64,5000,3): 79 groups of 64 sequences x 2 directions = 158 CTAs, more than the 132 SMs of an H100 SXM
@pytest.mark.parametrize("Fi,H,Fo,NSEQ,T", [(64, 128, 64, 200, 37), (32, 64, 32, 130, 20), (64, 128, 64, 5, 3), (128, 128, 128, 129, 9),
                                            (32, 32, 32, 64, 11), (64, 64, 64, 300, 1), (64, 128, 64, 5000, 3), (64, 128, 128, 140, 6),
                                            (32, 64, 64, 260, 5)])
def test_bilstm_vs_fp64_oracle(Fi, H, Fo, NSEQ, T):
    if not N.ctn_bilstm_supported(Fi, H, Fo):
        pytest.skip("shape outside the native LSTM envelope")
    sd = _weights(Fi, H, Fo, seed=NSEQ + T)
    z = torch.randn(NSEQ, T, Fi, generator=torch.Generator().manual_seed(T)) * 1.5
    h, P = _run(z, sd, H, Fo)
    h64, y64 = _ref(z, sd, torch.float64)
    h32, y32 = _ref(z, sd, torch.float32)
    assert torch.isfinite(h).all() and torch.isfinite(P).all()
    err, err32 = float((h.double() - h64).abs().max()), float((h32.double() - h64).abs().max())
    assert err <= 2e-5, (err, err32)
    y = P[0] + P[1] + sd["fc.bias"]
    torch.testing.assert_close(y.double(), y64, rtol=1e-4, atol=2e-5 * float(y64.abs().max()))


def test_bilstm_support_matrix():
    """every (F, H, Fo) of the envelope: same tolerance as above"""
    NSEQ, T = 150, 4
    for Fi in (32, 64, 128):
        for H in (32, 64, 128):
            for Fo in (32, 64, 96, 128):
                if not N.ctn_bilstm_supported(Fi, H, Fo):
                    continue
                sd = _weights(Fi, H, Fo, seed=Fi + H + Fo)
                z = torch.randn(NSEQ, T, Fi, generator=torch.Generator().manual_seed(Fo)) * 1.2
                h, P = _run(z, sd, H, Fo)
                h64, y64 = _ref(z, sd, torch.float64)
                assert float((h.double() - h64).abs().max()) <= 2e-5, (Fi, H, Fo)
                y = P[0] + P[1] + sd["fc.bias"]
                torch.testing.assert_close(y.double(), y64, rtol=1e-4, atol=2e-5 * float(y64.abs().max()), msg=lambda m: f"{(Fi, H, Fo)}: {m}")


@pytest.mark.parametrize("xscale,wscale,atol", [(1e3, 1.0, 1e-3), (1e-3, 1.0, 2e-5), (1.0, 8.0, 2e-5), (30.0, 0.05, 2e-5), (0.0, 1.0, 2e-5)])
def test_bilstm_operand_scales(xscale, wscale, atol):
    """the fp16 pieces are rescaled by powers of two measured on the data (x) and the weights: any magnitude is fine.  (x ~ 1e3:
    pre-activations of magnitude ~1e3 carry an absolute error of 2^-22 x 1e3 ~ 2e-4 in ANY 22-24-bit arithmetic; the few gates
    that are not saturated see it)"""
    Fi, H, Fo, NSEQ, T = 64, 128, 64, 140, 12
    if not N.ctn_bilstm_supported(Fi, H, Fo):
        pytest.skip("shape outside the native LSTM envelope")
    sd = _weights(Fi, H, Fo, seed=3, wscale=wscale)
    z = torch.randn(NSEQ, T, Fi, generator=torch.Generator().manual_seed(4)) * xscale
    h, P = _run(z, sd, H, Fo)
    h64, y64 = _ref(z, sd, torch.float64)
    assert float((h.double() - h64).abs().max()) <= atol
    y = P[0] + P[1] + sd["fc.bias"]
    torch.testing.assert_close(y.double(), y64, rtol=1e-4, atol=max(atol, 2e-5 * float(y64.abs().max())))


def test_bilstm_outputs_optional_and_errors():
    Fi, H, Fo = 64, 128, 64
    if not N.ctn_bilstm_supported(Fi, H, Fo):
        pytest.skip("shape outside the native LSTM envelope")
    sd = _weights(Fi, H, Fo, seed=9)
    z = torch.randn(33, 7, Fi, generator=torch.Generator().manual_seed(1))
    h_only, _ = _run(z, sd, H, Fo, want_p=False)
    _, p_only = _run(z, sd, H, Fo, want_h=False)
    h, P = _run(z, sd, H, Fo)
    assert torch.equal(h_only, h) and torch.equal(p_only, P)       # deterministic, outputs independent of each other
    assert N.ctn_bilstm_supported(8, 12, 8) == 0 and N.ctn_bilstm_workspace_bytes(8, 12, 8) == 0
    zc = z.cuda()
    ws = torch.empty(1024, dtype=torch.uint8, device="cuda")
    w = [sd["rnn." + n].cuda() for n in NAMES]
    ptrs = (N._fp * 8)(*[t.data_ptr() for t in w])
    out = torch.empty(33, 7, 2 * H, device="cuda")
    assert N.ctn_bilstm_proj_fwd(zc.data_ptr(), 33, 7, Fi, H, ptrs, None, Fo, None, out.data_ptr(), None, ws.data_ptr(), 1024,
                                 N.stream_ptr(zc.device)) == N.CTN_EWORKSPACE
    assert N.ctn_bilstm_proj_fwd(zc.data_ptr(), 33, 7, 8, 12, ptrs, None, Fo, None, out.data_ptr(), None, ws.data_ptr(), 1024,
                                 N.stream_ptr(zc.device)) == N.CTN_EUNSUPPORTED


def test_dprnn_stack_native_vs_cudnn_and_oracle():
    """DPRNN.forward at the cfg4 feature sizes (F = 64, H = 128): native recurrence vs the cuDNN recurrence vs the CPU oracle"""
    cfg = DO.DPRNNConfig(n_basis=16, kernel_size=4, sep_hidden_channels=128, sep_bottleneck_channels=64, sep_chunk_size=50, sep_hop_size=25,
                         sep_num_blocks=2)
    sd = DO.synth_state_dict(cfg, seed=7)
    sub = {k[len("separator.dprnn."):]: v for k, v in sd.items() if k.startswith("separator.dprnn.")}
    net = DPRNN(64, 128, num_blocks=2, causal=False)
    net.load_state_dict(sub, strict=True)
    net = net.cuda().eval()
    x = torch.randn(3, 64, 11, 50, generator=torch.Generator().manual_seed(8))
    with torch.no_grad():
        assert dprnn_mod.NATIVE_LSTM
        y = net(x.cuda())
        launches = N.ctn_last_launch_count()
        dprnn_mod.NATIVE_LSTM = False
        try:
            y_lib = net(x.cuda())
        finally:
            dprnn_mod.NATIVE_LSTM = True
        ref = DO.dprnn_fwd(x, sd, "separator.dprnn.", 2, cfg.eps)
    assert launches == 2                                           # the last native call: statistics + normalise/residual
    tol = 2e-5 * float(ref.abs().max())
    torch.testing.assert_close(y.cpu(), ref, rtol=1e-4, atol=tol)
    torch.testing.assert_close(y.cpu(), y_lib.cpu(), rtol=1e-4, atol=tol)
