"""The loss and optimizer C ABI without a GPU: ``ctn_clip_adam_chunks`` (a host-only function) and the argument rejections of the
SI-SDR / SDR / PIT entry points, which return before any CUDA call."""
import ctypes as C

import pytest

from ctn_b200 import _native as N

CHUNK = 2048
NUMELS = [1, 3, 2047, 2048, 2049, 6144, 6145, 100003]


def _chunks(numel, capacity=None):
    n = len(numel)
    arr = (C.c_int * n)(*numel)
    count = N.ctn_clip_adam_chunks(arr, n, None, None, 0)
    cap = count if capacity is None else capacity
    ct, co = (C.c_int * max(cap, 1))(), (C.c_int * max(cap, 1))()
    assert N.ctn_clip_adam_chunks(arr, n, ct, co, cap) == count
    return count, [(ct[i], co[i]) for i in range(min(cap, count))]


def test_clip_adam_chunk_table():
    """One entry per started CHUNK of every tensor, in tensor order: a tensor of n elements has ceil(n / 2048) entries at offsets
    0, 2048, ...; the last one may be partial (2049 -> 2 entries, 6144 -> exactly 3, 6145 -> 4)."""
    count, table = _chunks(NUMELS)
    want = [(i, e) for i, n in enumerate(NUMELS) for e in range(0, n, CHUNK)]
    assert count == len(want) == sum(-(-n // CHUNK) for n in NUMELS) == 1 + 1 + 1 + 1 + 2 + 3 + 4 + 49
    assert table == want
    for n in NUMELS:
        assert _chunks([n])[0] == -(-n // CHUNK), n


def test_clip_adam_chunk_table_sizing():
    """Null outputs only count; a short capacity fills the first `capacity` entries and still returns the full count."""
    arr = (C.c_int * len(NUMELS))(*NUMELS)
    assert N.ctn_clip_adam_chunks(arr, len(NUMELS), None, None, 0) == 62
    assert N.ctn_clip_adam_chunks(arr, len(NUMELS), None, None, 1000) == 62
    count, table = _chunks(NUMELS, capacity=5)
    assert count == 62 and table == [(0, 0), (1, 0), (2, 0), (3, 0), (4, 0)]
    assert N.ctn_clip_adam_chunks(None, 3, None, None, 0) == N.CTN_EINVAL
    assert N.ctn_clip_adam_chunks(arr, 0, None, None, 0) == N.CTN_EINVAL


FAKE = 1 << 20  # a non-null pointer that is never dereferenced: every call below is rejected before any CUDA call


def test_sisdr_pit_fwd_rejections():
    fwd = lambda **kw: N.ctn_sisdr_pit_fwd(*{**dict(est=FAKE, tgt=FAKE, B=2, S=2, T=100, eps=1e-12, loss_b=FAKE, perm=FAKE,
                                                    mean=None, pair=None, scratch=FAKE, stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(loss_b=None), dict(perm=None), dict(scratch=None), dict(B=0), dict(B=-1),
                dict(T=0), dict(T=-4)):
        assert fwd(**bad) == N.CTN_EINVAL, bad
    for S in (0, -1, 7, 16):
        assert fwd(S=S) == N.CTN_EUNSUPPORTED, S


def test_sisdr_pit_bwd_rejections():
    bwd = lambda **kw: N.ctn_sisdr_pit_bwd(*{**dict(est=FAKE, tgt=FAKE, perm=FAKE, B=2, S=2, T=100, eps=1e-12, scratch=FAKE,
                                                    g=None, coef=-0.5, d=FAKE, stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(perm=None), dict(scratch=None), dict(d=None), dict(B=0), dict(T=0)):
        assert bwd(**bad) == N.CTN_EINVAL, bad
    for S in (0, 7):
        assert bwd(S=S) == N.CTN_EUNSUPPORTED, S


@pytest.mark.parametrize("fn", ["ctn_sisdr_fwd", "ctn_sdr_fwd"])
def test_row_metric_rejections(fn):
    call = lambda **kw: getattr(N, fn)(*{**dict(est=FAKE, tgt=FAKE, rows=3, T=100, eps=1e-12, out=FAKE, scratch=FAKE,
                                                stream=None), **kw}.values())
    for bad in (dict(est=None), dict(tgt=None), dict(out=None), dict(scratch=None), dict(rows=0), dict(T=0), dict(T=-1)):
        assert call(**bad) == N.CTN_EINVAL, bad


def test_pit_scratch_bytes():
    assert N.ctn_sisdr_pit_scratch_bytes(3, 1) == 8 * 3 * 3
    assert N.ctn_sisdr_pit_scratch_bytes(40000, 2) == 8 * 40000 * 10
    assert N.ctn_sisdr_pit_scratch_bytes(2, 6) == 8 * 2 * (2 * 36 + 6)
