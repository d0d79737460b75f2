"""The gate of tests/pw_criterion.py, checked on the CPU against an emulation of the 3xTF32 tensor-core arithmetic.

The gate must accept a correct 3-pass contraction even under the pessimistic reading of the accumulator (fp32 with truncation
after every k8 step) and reject the regressions a rework of k_pw_wgmma can introduce: a dropped W_lo or A_lo piece, a last
partial k-slab computed single-pass, and a 128-column tile written one frame off.
"""
import numpy as np
import pytest
import torch

import pw_criterion as PC

M, T = 128, 256


def _data(K, seed, last_scale=1.0):
    rng = np.random.default_rng(seed)
    W = (rng.standard_normal((M, K)) / np.sqrt(K)).astype(np.float32)
    A = rng.standard_normal((K, T)).astype(np.float32)
    A[-1] *= np.float32(last_scale)
    return W, A


def _gate(W, A):
    W64, A64 = torch.from_numpy(W).double(), torch.from_numpy(A).double()[None]
    return PC.Reference(W64, *PC.pro_none(A64), PC.epi_raw())


def _e(ref, D):
    return PC.gate_e(torch.from_numpy(D)[None], ref.out["D"])


@pytest.mark.parametrize("K", [1, 8, 32, 33, 128, 1056])
def test_gate_accepts_correct_3pass(K):
    W, A = _data(K, seed=K)
    ref = _gate(W, A)
    e = _e(ref, PC.emulate_3xtf32(W, A))
    print(f"K={K}: e={e:.3e} E_drop={ref.e_drop['D']:.3e} e/E_drop={e / ref.e_drop['D']:.4f}")
    assert e <= ref.bound("tf32x3"), (K, e, ref.e_drop["D"])
    # the fp32 accumulator also stays inside the tf32 one-pass and the FFMA bounds
    assert e <= ref.bound("tf32") and e <= ref.bound("fp32")


@pytest.mark.parametrize("K", [8, 33, 128, 1056])
@pytest.mark.parametrize("mutant", ["drop_w_lo", "drop_a_lo"])
def test_gate_rejects_dropped_piece(K, mutant):
    W, A = _data(K, seed=100 + K)
    ref = _gate(W, A)
    e = _e(ref, PC.emulate_3xtf32(W, A, **{mutant: True}))
    print(f"{mutant} K={K}: e/bound={e / ref.bound('tf32x3'):.2f}")
    assert e > ref.bound("tf32x3")


def test_gate_rejects_single_pass_last_slab():
    # K = 33: the second k-slab holds one channel.  Its activation row is made the largest so that the lost pieces of that
    # one term are not hidden among the other 32.
    W, A = _data(33, seed=7, last_scale=8.0)
    ref = _gate(W, A)
    e = _e(ref, PC.emulate_3xtf32(W, A, single_pass_from=32))
    print(f"single-pass last slab: e/bound={e / ref.bound('tf32x3'):.2f}")
    assert e > ref.bound("tf32x3")


def test_gate_rejects_tile_shifted_one_frame():
    W, A = _data(128, seed=9)
    ref = _gate(W, A)
    D = PC.emulate_3xtf32(W, A)
    D[:, 128:256] = D[:, 127:255].copy()
    assert _e(ref, D) > ref.bound("tf32x3")
    assert _e(ref, D) > ref.bound("fp32")


def test_gate_rejects_non_finite_output():
    W, A = _data(32, seed=11)
    ref = _gate(W, A)
    D = PC.emulate_3xtf32(W, A)
    D[5, 17] = np.nan
    assert _e(ref, D) == float("inf")


def test_round_sig_and_pieces():
    x = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -12), 3.0], dtype=torch.float64)
    assert PC.round_sig(x).tolist() == [1.0, 1.0 + 2 * 2.0 ** -10, -1.0, 3.0]
    v = np.array([1.0 + 2.0 ** -11, 1.0 + 2.0 ** -12], np.float32)
    assert PC.tf32_rna(v).tolist() == [1.0 + 2.0 ** -10, 1.0]
    assert PC.tf32_trunc(v).tolist() == [1.0, 1.0]
    assert PC.f32_rz(np.array([1.0 + 2.0 ** -30, -(1.0 + 2.0 ** -30)])).tolist() == [1.0, -1.0]
