"""ConvTasNet.separate_long without a GPU: the exported symbols, the chunk plan (ctn_chunk_plan) against its restatement, the
C ABI's refusals (each returns before any CUDA call), the workspace formula, and the Python envelope."""
import ctypes as C

import pytest
import torch

import separate_long_ref as R
from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet

FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced: every call below is refused before it would be


def _cfg(**kw):
    c = N.Config()
    base = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2,
                num_layers=4, n_sources=2, causal=0, enc_relu=0, mask_softmax=0, math=0, eps=1e-12, eps_tcn=1e-12, in_channels=1)
    base.update(kw)
    for k, v in base.items():
        setattr(c, k, v)
    return c


def _params():
    blocks = (N.BlockParams * 64)()
    for b in blocks:
        for name in N.BLOCK_FIELDS:
            setattr(b, name, FAKE)
    p = N.Params()
    for name, _ in N.Params._fields_:
        if name != "blocks":
            setattr(p, name, FAKE)
    p.blocks = blocks
    return p, blocks


def _plan(T, chunk, hop):
    K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
    if K < 0:
        return K, None
    starts = (C.c_int * K)()
    assert N.ctn_chunk_plan(T, chunk, hop, starts, K) == K
    return K, list(starts)


def test_symbols_exported():
    for name in ("ctn_chunk_plan", "ctn_chunk_gather", "ctn_chunk_align_scratch_bytes", "ctn_chunk_align", "ctn_chunk_overlap_add",
                 "ctn_separate_long_workspace_bytes", "ctn_convtasnet_separate_long"):
        assert hasattr(N.lib, name) and name in N.EXPORTED


PLANS = [(50, 100, 50), (100, 100, 50), (101, 100, 50), (101, 100, 100), (149, 100, 50), (150, 100, 50), (151, 100, 50),
         (1000, 100, 100), (1001, 100, 100), (1000, 100, 50), (977, 101, 50), (977, 101, 77), (12345, 333, 166), (7, 3, 1),
         (5, 2, 1), (4800000, 32000, 16000), (28800001, 32000, 20000)]


@pytest.mark.parametrize("T,chunk,hop", PLANS)
def test_plan_matches_restatement(T, chunk, hop):
    K, starts = _plan(T, chunk, hop)
    ref, Lc = R.plan(T, chunk, hop)
    assert K == len(ref) and starts == ref
    assert Lc == min(chunk, T)
    assert starts[0] == 0 and all(s >= 0 for s in starts)
    assert starts[-1] + Lc == T                                     # the last chunk ends at T
    assert all(a < b for a, b in zip(starts, starts[1:]))           # no chunk repeats
    assert all(b - a <= Lc for a, b in zip(starts, starts[1:]))     # every sample is covered
    if T <= chunk:
        assert K == 1


@pytest.mark.parametrize("T,chunk,hop", [(1000, 100, 49), (1000, 100, 101), (1000, 101, 49), (1000, 0, 0), (1000, -4, -2),
                                         (0, 100, 50), (-5, 100, 50), (1000, 1, 0)])
def test_plan_rejects(T, chunk, hop):
    assert N.ctn_chunk_plan(T, chunk, hop, None, 0) == N.CTN_EINVAL


def test_plan_capacity():
    starts = (C.c_int * 2)()
    assert N.ctn_chunk_plan(1000, 100, 50, starts, 2) == N.CTN_EINVAL


def _call(c, p, x=FAKE, B=1, T=100000, chunk=4000, hop=2000, cb=16, align=1, out=FAKE, perms=None, ws=FAKE, ws_bytes=1 << 40):
    return N.ctn_convtasnet_separate_long(C.byref(c) if c is not None else None, C.byref(p) if p is not None else None, x, B, T, chunk,
                                          hop, cb, align, out, perms, ws, ws_bytes, None)


def test_argument_errors():
    c = _cfg()
    p, _keep = _params()
    need = C.c_size_t(0)
    assert N.ctn_separate_long_workspace_bytes(C.byref(c), 1, 100000, 4000, 2000, 16, C.byref(need)) == N.CTN_OK
    for kw in (dict(hop=1999), dict(hop=4001), dict(chunk=0, hop=0), dict(chunk=-8, hop=-4), dict(B=0), dict(T=0), dict(cb=0)):
        assert _call(c, p, **kw) == N.CTN_EINVAL, kw
    assert _call(None, p) == N.CTN_EINVAL
    assert _call(c, None) == N.CTN_EINVAL
    for kw in (dict(x=None), dict(out=None), dict(ws=None)):
        assert _call(c, p, **kw) == N.CTN_EINVAL, kw
    assert _call(c, p, ws=FAKE + 4) == N.CTN_EALIGN
    assert _call(c, p, ws_bytes=need.value - 1) == N.CTN_EWORKSPACE
    assert _call(c, p, ws_bytes=16) == N.CTN_EWORKSPACE
    assert _call(c, p, hop=4000) == N.CTN_EINVAL                      # alignment needs chunks that share samples
    assert _call(_cfg(in_channels=2), p) == N.CTN_EUNSUPPORTED
    assert _call(_cfg(n_sources=7), p) == N.CTN_EUNSUPPORTED
    assert _call(c, p, chunk=8, hop=4) == N.CTN_EINVAL                # a chunk shorter than the encoder kernel
    assert N.ctn_separate_long_workspace_bytes(C.byref(c), 1, 100000, 4000, 2000, 16, None) == N.CTN_EINVAL
    assert N.ctn_separate_long_workspace_bytes(C.byref(c), 1, 100000, 4000, 1000, 16, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_separate_long_workspace_bytes(C.byref(_cfg(in_channels=2)), 1, 100000, 4000, 2000, 16, C.byref(need)) == N.CTN_EUNSUPPORTED


def test_step_entry_errors():
    assert N.ctn_chunk_gather(None, 1, 1000, 100, 50, 0, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_chunk_gather(FAKE, 1, 1000, 100, 50, 0, 1, None, None) == N.CTN_EINVAL
    assert N.ctn_chunk_gather(FAKE, 1, 1000, 100, 50, 18, 2, FAKE, None) == N.CTN_EINVAL   # K = 19: chunks 18, 19
    assert N.ctn_chunk_gather(FAKE, 1, 1000, 100, 49, 0, 1, FAKE, None) == N.CTN_EINVAL
    big = 1 << 30
    assert N.ctn_chunk_align(None, 1, 2, 1000, 100, 50, FAKE, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_chunk_align(FAKE, 1, 2, 1000, 100, 50, None, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_chunk_align(FAKE, 1, 2, 1000, 100, 50, FAKE, None, big, None) == N.CTN_EINVAL
    assert N.ctn_chunk_align(FAKE, 1, 2, 1000, 100, 100, FAKE, FAKE, big, None) == N.CTN_EINVAL
    assert N.ctn_chunk_align(FAKE, 1, 7, 1000, 100, 50, FAKE, FAKE, big, None) == N.CTN_EUNSUPPORTED
    assert N.ctn_chunk_align(FAKE, 1, 2, 1000, 100, 50, FAKE, FAKE + 4, big, None) == N.CTN_EALIGN
    need = N.ctn_chunk_align_scratch_bytes(1, 2, 1000, 100, 50)
    assert need == 8 * 18 * 1 * 4                                       # pairs x one CTA per pair (chunk <= 4096) x S*S doubles
    assert N.ctn_chunk_align(FAKE, 1, 2, 1000, 100, 50, FAKE, FAKE, need - 1, None) == N.CTN_EWORKSPACE
    assert N.ctn_chunk_overlap_add(None, None, 1, 2, 1000, 100, 50, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_chunk_overlap_add(FAKE, None, 1, 2, 1000, 100, 50, None, None) == N.CTN_EINVAL
    assert N.ctn_chunk_overlap_add(FAKE, None, 1, 0, 1000, 100, 50, FAKE, None) == N.CTN_EINVAL


def _r256(n):
    return (n + 255) // 256 * 256


def _ws(c, B, T, chunk, hop, cb):
    need = C.c_size_t(0)
    assert N.ctn_separate_long_workspace_bytes(C.byref(c), B, T, chunk, hop, cb, C.byref(need)) == N.CTN_OK
    return need.value


@pytest.mark.parametrize("B,S,chunk,hop", [(1, 2, 32000, 16000), (4, 2, 32000, 16000), (2, 3, 4000, 2500), (1, 1, 4096, 2048)])
def test_workspace_grows_with_T_by_the_chunk_buffers_only(B, S, chunk, hop):
    """beyond chunk_batch chunks, bytes(T) = const + [permutations] + [alignment scratch] + [chunk estimates], each rounded up to 256"""
    c = _cfg(n_basis=512, bottleneck=128, hidden=512, skip=128, num_blocks=3, num_layers=8, n_sources=S)
    split = min(16, (chunk + 4095) // 4096)

    def grows(T):
        K = N.ctn_chunk_plan(T, chunk, hop, None, 0)
        return _r256(4 * B * K * S) + (_r256(8 * B * (K - 1) * split * S * S) if S > 1 else 0) + _r256(4 * B * K * S * chunk)

    T1, T2 = 40 * chunk, 40 * chunk + 1234567
    b1, b2 = _ws(c, B, T1, chunk, hop, 16), _ws(c, B, T2, chunk, hop, 16)
    assert b2 - b1 == grows(T2) - grows(T1)
    # the rest is one chunk batch of the plain forward's workspace and one gathered batch
    fwd = C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(c), 16, chunk, C.byref(fwd)) == N.CTN_OK
    rest = b1 - grows(T1)
    assert fwd.value <= rest <= fwd.value + _r256(4 * 16 * chunk) + 1024
    # and the plain forward on the whole recording needs far more
    whole = C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(c), B, T2, C.byref(whole)) == N.CTN_OK
    assert b2 < whole.value


def test_short_input_needs_the_forward_workspace():
    c = _cfg()
    fwd = C.c_size_t(0)
    assert N.ctn_workspace_bytes(C.byref(c), 3, 3000, C.byref(fwd)) == N.CTN_OK
    assert fwd.value <= _ws(c, 3, 3000, 4000, 2000, 16) <= fwd.value + 1024


def _model(**kw):
    return ConvTasNet(64, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=32,
                      sep_bottleneck_channels=16, sep_skip_channels=16, sep_num_blocks=1, sep_num_layers=2, causal=False, **kw)


def test_python_envelope():
    m = _model()
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            m.separate_long(torch.zeros(1, 1, 1000), 400)
        with pytest.raises(NotImplementedError):
            m.separate_long(torch.zeros(1, 1, 2, 1000), 400)
        with pytest.raises(ValueError):
            m.separate_long(torch.zeros(1, 2, 1000), 400)
    with pytest.raises(NotImplementedError):
        m.separate_long(torch.zeros(1, 1, 1000), 400)      # autograd on, parameters require grad


def test_shim_model_has_separate_long():
    from models.conv_tasnet import ConvTasNet as Shim
    assert Shim.separate_long is ConvTasNet.separate_long
