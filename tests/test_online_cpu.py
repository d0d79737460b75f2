"""Online inference (ctn_online_*, ConvTasNet.online) without a GPU: the C ABI's rejections, which return before any CUDA
call, the state size query, and the Python envelope."""
import ctypes as C

import pytest

from ctn_b200 import _native as N
from ctn_b200.models.conv_tasnet import ConvTasNet

FAKE = 1 << 20  # a 256-byte-aligned address that is never dereferenced: every call below is refused before it would be


def _cfg(**kw):
    c = N.Config()
    base = dict(n_basis=64, kernel_size=16, stride=8, bottleneck=32, hidden=64, skip=32, sep_kernel=3, num_blocks=2,
                num_layers=4, n_sources=2, causal=1, enc_relu=0, mask_softmax=0, math=0, eps=1e-12, eps_tcn=1e-12, in_channels=1)
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


def _bytes(cfg, B=1, frames=32):
    need = C.c_size_t(0)
    st = N.ctn_online_state_bytes(C.byref(cfg), B, frames, C.byref(need))
    return st, need.value


@pytest.mark.parametrize("kw", [dict(causal=0), dict(in_channels=2), dict(in_channels=64)])
def test_envelope_is_unsupported(kw):
    c = _cfg(**kw)
    p, _keep = _params()
    y = C.c_size_t(0)
    assert N.ctn_online_state_bytes(C.byref(c), 1, 32, C.byref(y)) == N.CTN_EUNSUPPORTED
    assert N.ctn_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, 1 << 30, None) == N.CTN_EUNSUPPORTED
    assert N.ctn_online_reset(C.byref(c), FAKE, 1, None) == N.CTN_EUNSUPPORTED
    assert N.ctn_online_push(C.byref(c), C.byref(p), FAKE, FAKE, 1, 32, 8, FAKE, None) == N.CTN_EUNSUPPORTED
    assert N.ctn_online_flush(C.byref(c), FAKE, 1, FAKE, None) == N.CTN_EUNSUPPORTED


@pytest.mark.parametrize("B,n", [(1, 12), (1, 0), (1, -8), (1, 264), (0, 8), (-1, 8)])
def test_push_rejects_bad_sizes(B, n):
    """n % stride != 0, n = 0, n > max_chunk (32 frames = 256 samples), B <= 0"""
    c = _cfg()
    p, _keep = _params()
    assert N.ctn_online_push(C.byref(c), C.byref(p), FAKE, FAKE, B, 32, n, FAKE, None) == N.CTN_EINVAL


def test_null_pointers_and_sizes_are_invalid():
    c = _cfg()
    p, _keep = _params()
    need = C.c_size_t(0)
    assert N.ctn_online_state_bytes(None, 1, 32, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_online_state_bytes(C.byref(c), 1, 32, None) == N.CTN_EINVAL
    assert N.ctn_online_state_bytes(C.byref(c), 0, 32, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_online_state_bytes(C.byref(c), 1, 0, C.byref(need)) == N.CTN_EINVAL
    assert N.ctn_online_init(C.byref(c), None, 1, 32, FAKE, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_online_init(C.byref(c), C.byref(p), 1, 32, None, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_online_init(C.byref(c), C.byref(p), 0, 32, FAKE, 1 << 30, None) == N.CTN_EINVAL
    assert N.ctn_online_init(C.byref(c), C.byref(p), 1, 32, FAKE, 16, None) == N.CTN_EWORKSPACE
    assert N.ctn_online_init(C.byref(c), C.byref(p), 1, 32, FAKE + 4, 1 << 30, None) == N.CTN_EALIGN
    assert N.ctn_online_reset(C.byref(c), None, 1, None) == N.CTN_EINVAL
    assert N.ctn_online_reset(C.byref(c), FAKE, 0, None) == N.CTN_EINVAL
    for args in ((None, FAKE, 1, 32, 8, FAKE), (FAKE, None, 1, 32, 8, FAKE), (FAKE, FAKE, 1, 32, 8, None), (FAKE, FAKE, 1, 0, 8, FAKE)):
        assert N.ctn_online_push(C.byref(c), C.byref(p), *args, None) == N.CTN_EINVAL
    assert N.ctn_online_push(C.byref(c), None, FAKE, FAKE, 1, 32, 8, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), None, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE, 1, None, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE, 0, FAKE, None) == N.CTN_EINVAL


@pytest.mark.parametrize("B,H", [(1, 64), (3, 64), (2, 128)])
@pytest.mark.parametrize("X", [1, 4, 8, 13])
def test_state_bytes_grow_by_the_ring(B, H, X):
    """bytes(P) - bytes(P = 1) = 4 B H (P - 1) sum_i d_i, d_i = 2^(i mod X) over the R X blocks: the depthwise history"""
    R = 2
    sum_d = R * (2 ** X - 1)
    st, base = _bytes(_cfg(sep_kernel=1, hidden=H, num_blocks=R, num_layers=X), B)
    assert st == N.CTN_OK
    for P in (2, 3, 5, 8):
        st, got = _bytes(_cfg(sep_kernel=P, hidden=H, num_blocks=R, num_layers=X), B)
        assert st == N.CTN_OK
        assert got - base == 4 * B * H * (P - 1) * sum_d, (P, X)


def test_state_bytes_at_the_paper_size():
    """H = 512, P = 3, X = 8, R = 3: 3.1 MB of depthwise history per stream"""
    st, b1 = _bytes(_cfg(n_basis=512, bottleneck=128, hidden=512, skip=128, num_blocks=3, num_layers=8), 1)
    st1, b0 = _bytes(_cfg(n_basis=512, bottleneck=128, hidden=512, skip=128, num_blocks=3, num_layers=8, sep_kernel=1), 1)
    assert st == st1 == N.CTN_OK
    assert b1 - b0 == 4 * 512 * 2 * 3 * 255 == 3133440


def _model(causal, **kw):
    return ConvTasNet(64, 16, enc_basis="trainable", dec_basis="trainable", enc_nonlinear=None, sep_hidden_channels=32,
                      sep_bottleneck_channels=16, sep_skip_channels=16, sep_num_blocks=1, sep_num_layers=2, causal=causal, **kw)


def test_online_refuses_gln_models():
    with pytest.raises(NotImplementedError):
        _model(False).online(batch_size=1, max_chunk=256)


def test_online_refuses_multichannel_models():
    with pytest.raises(NotImplementedError):
        _model(True, in_channels=2).online(batch_size=1, max_chunk=256)


def test_online_has_no_cpu_fallback():
    with pytest.raises(RuntimeError):
        _model(True).online(batch_size=1, max_chunk=256)


@pytest.mark.parametrize("B,chunk", [(0, 256), (1, 0), (1, 12)])
def test_online_rejects_bad_geometry(B, chunk):
    with pytest.raises(ValueError):
        _model(True).online(batch_size=B, max_chunk=chunk)


def test_shim_model_has_online():
    from models.conv_tasnet import ConvTasNet as Shim
    assert Shim.online is ConvTasNet.online
