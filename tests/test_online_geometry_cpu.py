"""Online inference (ctn_online_*) at its filter-bank limits, without a GPU: host-only state-size queries and argument
rejections, each returning before any CUDA call.

  - the encoder reads [carry | chunk] into dynamic shared memory, (L - S + n) * 4 bytes, at most 200 KiB;
  - the decoder keeps the history of L/S - 1 frames in shared memory, n_basis * (L/S - 1) * 4 bytes, at most 48 KiB;
  - flush needs a non-null y_tail only when there is a tail, D = L - S > 0.
A flush of a zero-delay model with a null y_tail gets past the argument checks and reads the device, so that case is run
by test_online_geometry_gpu.py."""
import ctypes as C

import pytest

from ctn_b200 import _native as N
from test_online_cpu import FAKE, _bytes, _cfg

ENC_SMEM = 200 * 1024
HIST_SMEM = 48 * 1024


def _max_frames(L, S):
    """largest chunk (frames) whose [carry | chunk] fits the encoder's shared memory"""
    return (ENC_SMEM // 4 - (L - S)) // S


def test_encoder_bound_at_the_paper_filter_bank():
    """L = 16, S = 8: (8 + 8 n) * 4 <= 200 KiB up to n = 6399 frames"""
    assert _max_frames(16, 8) == 6399
    st, need = _bytes(_cfg(kernel_size=16, stride=8), 1, 6399)
    assert st == N.CTN_OK and need > 0
    assert _bytes(_cfg(kernel_size=16, stride=8), 1, 6400)[0] == N.CTN_EUNSUPPORTED


@pytest.mark.parametrize("L,S", [(2, 1), (4, 2), (8, 2), (16, 4), (16, 16), (20, 10), (32, 8), (40, 20), (64, 2)])
def test_encoder_bound_at_every_filter_bank(L, S):
    """the last accepted chunk puts (L - S + n S) * 4 at or just under 200 KiB; one more frame is refused"""
    F = _max_frames(L, S)
    assert (L - S + F * S) * 4 <= ENC_SMEM < (L - S + (F + 1) * S) * 4
    for B in (1, 3):
        assert _bytes(_cfg(kernel_size=L, stride=S), B, F)[0] == N.CTN_OK
        assert _bytes(_cfg(kernel_size=L, stride=S), B, F + 1)[0] == N.CTN_EUNSUPPORTED


@pytest.mark.parametrize("L,S,n_ok", [(64, 16, 4096), (64, 2, 396), (32, 8, 4096), (16, 8, 12288), (40, 20, 12288)])
def test_decoder_history_bound(L, S, n_ok):
    """n_basis * (L/S - 1) * 4 <= 48 KiB: n_ok channels are accepted, n_ok + 1 refused"""
    R = L // S
    assert n_ok * (R - 1) * 4 <= HIST_SMEM < (n_ok + 1) * (R - 1) * 4
    st, need = _bytes(_cfg(n_basis=n_ok, kernel_size=L, stride=S))
    assert st == N.CTN_OK and need > 0
    assert _bytes(_cfg(n_basis=n_ok + 1, kernel_size=L, stride=S))[0] == N.CTN_EUNSUPPORTED


def test_decoder_history_bound_leaves_zero_delay_models_unbounded():
    """L == S keeps no history: any n_basis passes the history check"""
    assert _bytes(_cfg(n_basis=1 << 16, kernel_size=16, stride=16))[0] == N.CTN_OK


def test_history_sizes_are_accepted_by_the_model_check():
    """the sizes above are refused by the online history bound, not by the model's own check: the offline state query of the
    same config accepts them"""
    for L, S, n in ((64, 16, 4097), (64, 2, 397), (16, 8, 12289)):
        need = C.c_size_t(0)
        assert N.ctn_workspace_bytes(C.byref(_cfg(n_basis=n, kernel_size=L, stride=S)), 1, 4 * L, C.byref(need)) == N.CTN_OK


@pytest.mark.parametrize("L,S", [(16, 8), (16, 4), (2, 1), (64, 2), (40, 20)])
def test_flush_needs_y_tail_when_there_is_a_delay(L, S):
    c = _cfg(kernel_size=L, stride=S)
    assert N.ctn_online_flush(C.byref(c), FAKE, 1, None, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), None, 1, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE, 0, FAKE, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE + 4, 1, FAKE, None) == N.CTN_EALIGN


@pytest.mark.parametrize("L", [8, 16])
def test_zero_delay_flush_keeps_the_other_checks(L):
    """L == S, null y_tail: the state, B and alignment are still checked before anything reads the device"""
    c = _cfg(kernel_size=L, stride=L)
    assert N.ctn_online_flush(C.byref(c), None, 1, None, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE, 0, None, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE, -1, None, None) == N.CTN_EINVAL
    assert N.ctn_online_flush(C.byref(c), FAKE + 4, 1, None, None) == N.CTN_EALIGN
    assert N.ctn_online_flush(C.byref(_cfg(kernel_size=L, stride=L, causal=0)), FAKE, 1, None, None) == N.CTN_EUNSUPPORTED
